"""TEST INFRASTRUCTURE — runs the reference's UNMODIFIED ``test.py`` (its ``main_worker``; the reference checkout is
found through ``oracle.reference_loader``, ``E2FGVI_REFERENCE_ROOT``) on synthetic videos whose
frames and masks are NOT at model size, so that its front end runs: ``resize_frames`` (PIL bicubic, test.py:98-103)
and ``read_mask`` (NEAREST resize, ``> 0``, 4x cross dilation, test.py:56-70).  Stores what it wrote, as the golden
for ``e2fgvi_b200.video.prepare_inputs`` and the ``e2fgvi_b200.inpaint`` command.

    python -m oracle.gen_golden_frontend       # only where the reference checkout exists

Same offline setup as ``oracle/gen_golden_video.py`` (matplotlib stubbed, mmcv from ``oracle/mmcv_shim``, inputs as
PNGs, synthetic ``state_dict``, ``cv2.VideoWriter`` replaced by a recorder).  In addition the child wraps the
script's own ``resize_frames`` / ``read_mask`` and records the SHA-256 of what they returned, so that the front end
can be checked bit for bit on a machine without Pillow / OpenCV.  The composited frames equal the resized frames
outside the dilated holes (asserted here), so a golden keeps only their hole pixels (``comp_holes``, in C order of
the (N,H,W) hole map) plus the SHA-256 of the whole output: the resized frames with those pixels written back must
hash to it.  Inputs are NOT stored: ``synth_video`` regenerates
them from seeds (frames from one call, masks from a second call at the mask size).
"""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")

# name -> (model, n_frames, (H, W) of the frames, (H, W) of the masks, family, weight seed, frame seed, mask seed,
#          extra test.py argv)
CASES = {
    "video_base_resize": ("e2fgvi", 8, (360, 640), (180, 320), "stress", 2, 31, 32, []),
    "video_hq_set_size": ("e2fgvi_hq", 9, (90, 170), (75, 130), "stress", 3, 33, 34,
                          ["--set_size", "--width", "200", "--height", "100"]),
}

CHILD = r'''
import hashlib, os, runpy, sys
from unittest import mock
import numpy as np
shim, ref, tmp, out = sys.argv[1:5]
argv = sys.argv[5:]
sys.path[:] = [shim, ref] + [p for p in sys.path if p not in ("", os.getcwd())]
for name in ("matplotlib", "matplotlib.pyplot", "matplotlib.animation", "matplotlib.patches", "matplotlib.path"):
    sys.modules[name] = mock.MagicMock(name=name)
import cv2
written = []
class Recorder:
    def __init__(self, *a, **k): pass
    def write(self, bgr): written.append(cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB).copy())   # undo the script's swap
    def release(self): pass
cv2.VideoWriter = Recorder
os.chdir(tmp)                       # the script writes ./results/
sys.argv = [os.path.join(ref, "test.py")] + argv
# run the module body (argument parsing, definitions) without its __main__ block, then main_worker itself with the
# front-end functions wrapped in the namespace main_worker reads them from
g = runpy.run_path(os.path.join(ref, "test.py"), run_name="test_py")["main_worker"].__globals__
seen = {}
resize_frames, read_mask = g["resize_frames"], g["read_mask"]
def rec_resize_frames(frames, size=None):
    res = resize_frames(frames, size)
    seen["frames"] = np.stack([np.asarray(f) for f in res[0]])
    return res
def rec_read_mask(mpath, size):
    res = read_mask(mpath, size)
    seen["masks"] = np.stack([(np.array(m) != 0).astype(np.uint8) for m in res])
    return res
g["resize_frames"], g["read_mask"] = rec_resize_frames, rec_read_mask
g["main_worker"]()
sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
comp, hole = np.stack(written), seen["masks"].astype(bool)
# outside the holes the script's output is its resized frame (test.py:172-179), so only the hole pixels are stored
assert np.array_equal(comp[~hole], seen["frames"][~hole])
np.savez_compressed(out, comp_sha256=np.array(sha(comp)), comp_holes=comp[hole],
                    frames_sha256=np.array(sha(seen["frames"])), frames_shape=np.array(seen["frames"].shape),
                    masks_sha256=np.array(sha(seen["masks"])), masks_shape=np.array(seen["masks"].shape))
print("captured", len(written), "frames", written[0].shape, "masks", seen["masks"].shape)
'''


def main(names=None):
    import cv2
    import torch
    sys.path.insert(0, ROOT)
    import importlib
    from e2fgvi_b200.synth import synth_state_dict, synth_video
    from oracle.reference_loader import REFERENCE_ROOT, SHIM
    os.makedirs(OUT, exist_ok=True)
    for name, (model, n, (h, w), (hm, wm), family, wseed, fseed, mseed, extra) in CASES.items():
        if names and name not in names:
            continue
        frames, _ = synth_video(n, h, w, fseed)
        _, masks = synth_video(n, hm, wm, mseed)
        with tempfile.TemporaryDirectory() as tmp:
            os.makedirs(os.path.join(tmp, "frames"))
            os.makedirs(os.path.join(tmp, "masks"))
            for i in range(n):
                cv2.imwrite(os.path.join(tmp, "frames", f"{i:05d}.png"), cv2.cvtColor(frames[i], cv2.COLOR_RGB2BGR))
                cv2.imwrite(os.path.join(tmp, "masks", f"{i:05d}.png"), masks[i] * 255)
            mine = importlib.import_module("e2fgvi_b200.model." + model).InpaintGenerator()
            torch.save(synth_state_dict(mine, family, wseed), os.path.join(tmp, "ckpt.pth"))
            child = os.path.join(tmp, "child.py")
            with open(child, "w") as f:
                f.write(CHILD)
            argv = ["-v", os.path.join(tmp, "frames"), "-c", os.path.join(tmp, "ckpt.pth"), "-m",
                    os.path.join(tmp, "masks"), "--model", model] + extra
            subprocess.check_call([sys.executable, child, SHIM, REFERENCE_ROOT, tmp, os.path.join(OUT, name + ".npz")]
                                  + argv, cwd=tmp)
        print(name, "done")


if __name__ == "__main__":
    main(sys.argv[1:])
