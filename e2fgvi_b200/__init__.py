"""e2fgvi_b200 — H100-native (sm_90a) implementation of E2FGVI's InpaintGenerator.forward hot path.

Package map (only what the path needs):
  csrc/      hand-written CUDA kernels + the C ABI (include/e2fgvi_b200.h)
  _lib.py    ctypes binding of libe2fgvi_b200.so          build.py  in-tree nvcc build
  ops.py     operator mirror of the reference boundaries (flow_warp, modulated_deform_conv2d, focal attention)
  model/     drop-in ``model.e2fgvi`` / ``model.e2fgvi_hq`` InpaintGenerator (reference state-dict layout)
  synth.py   deterministic synthetic weights / frames (no checkpoints or datasets are available offline)
  clips.py   clip sharding across ranks + the single all-gather output stitch
"""
__version__ = "0.1.0"
