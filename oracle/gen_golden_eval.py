"""TEST INFRASTRUCTURE — runs the reference's UNMODIFIED ``evaluate.py`` (its ``main_worker``, through ``runpy``; the
reference checkout is found through ``oracle.reference_loader``, ``E2FGVI_REFERENCE_ROOT``) on synthetic DAVIS-layout
datasets and stores what it computed and wrote, as the goldens of ``python -m e2fgvi_b200.evaluate``.

    python -m oracle.gen_golden_eval       # only where the reference checkout exists

The dataset (``synth.write_eval_dataset``) is built in a temp dir: ``test.json``, ``JPEGImages/<v>.zip`` with PNG
members (lossless, so decoding does not depend on the OpenCV build) and DAVIS-style palette masks
``test_masks/<v>/%05d.png`` at frame size.  Frames are not at 432x240, so the script's resize runs.  The child runs
on the CPU with ``num_workers = 0`` and patches only the script's namespace: ``init_i3d_model`` returns the reference's
``InceptionI3d`` with ``synth_i3d_state_dict`` weights in eval mode; ``calc_psnr_and_ssim`` and
``calculate_i3d_activations`` are wrapped to record their values; ``TestDataset.load_item`` is wrapped to record the
dilated masks.  Import stand-ins: ``oracle/metrics_shim`` (for scikit-image and matplotlib, which are not installed) and
``oracle/mmcv_shim``.  scikit-image 0.16.2 is not installed, so the child gives the stand-in ``skimage.measure`` the
restatement ``oracle.restate_ssim.compare_ssim``; SciPy 1.18 dropped the ``disp`` argument the reference passes to
``sqrtm``, so ``core.metrics.linalg.sqrtm`` ignores it (as in ``gen_golden_i3d``).

Stored per case (``tests/golden/<case>.npz``): the metrics.txt text; per-frame PSNR / SSIM; the real and fake I3D
activations; per video the SHA-256 of the resized frames and of the dilated masks; the saved PNGs' hole pixels (in C
order of each video's (N, H, W) hole map, videos concatenated) plus each video's SHA-256 of the full output, as the
front-end goldens store them.  Under recent PyTorch the DataLoader collates a video's name into a tuple, so the stored
lines read ``('bear',)`` where the reference's pinned PyTorch prints ``['bear']``.  Inputs are regenerated from seeds.  Sizes: eval_base.npz 308 KB, eval_hq.npz 157 KB.
"""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")

# name -> (model, {video: frames}, (H, W) of frames and masks, weight family, weight seed, I3D seed)
CASES = {
    "eval_base": ("e2fgvi", {"bear": 13, "cows": 6, "goat": 16}, (270, 480), "stress", 2, 0),
    "eval_hq": ("e2fgvi_hq", {"fox": 7, "owl": 9}, (180, 320), "stress", 3, 1),
}

CHILD = r'''
import hashlib, os, runpy, sys, types
import numpy as np
metrics_shim, mmcv_shim, ref, restate, tmp, out, model, ckpt, i3d_ckpt = sys.argv[1:10]
# metrics_shim last: it only stands in for what is not installed (scikit-image, matplotlib); torchvision is real
sys.path[:] = [mmcv_shim, ref] + [p for p in sys.path if p not in ("", os.getcwd())] + [metrics_shim]
import importlib.util
import torch
import skimage.measure
spec = importlib.util.spec_from_file_location("restate_ssim", restate)
restate_ssim = importlib.util.module_from_spec(spec)
spec.loader.exec_module(restate_ssim)
skimage.measure.compare_ssim = restate_ssim.compare_ssim
import core.metrics as cm
from scipy import linalg as _linalg
class _Linalg:
    def __getattr__(self, name):
        return getattr(_linalg, name)
    @staticmethod
    def sqrtm(a, disp=True):
        root = _linalg.sqrtm(a)
        return root if disp else (root, None)
cm.linalg = _Linalg()
os.chdir(tmp)                                          # the script writes ./results/
g = runpy.run_path(os.path.join(ref, "evaluate.py"), run_name="evaluate_py")["main_worker"].__globals__
def init_i3d_model():
    net = cm.InceptionI3d(400, in_channels=3)
    net.load_state_dict(torch.load(i3d_ckpt), strict=True)
    return net.eval()
rec = {"psnr": [], "ssim": [], "real": [], "fake": [], "masks": [], "frames": []}
calc, acts, load_item = g["calc_psnr_and_ssim"], g["calculate_i3d_activations"], g["TestDataset"].load_item
def rec_calc(a, b):
    p, s = calc(a, b)
    rec["psnr"].append(p); rec["ssim"].append(s); rec["frames"].append(np.asarray(a, dtype=np.uint8))
    return p, s
def rec_acts(v1, v2, model, device):
    r, f = acts(v1, v2, model, device=device)
    rec["real"].append(r); rec["fake"].append(f)
    return r, f
def rec_load_item(self, index):
    item = load_item(self, index)
    rec["masks"].append((item[1][:, 0].numpy() > 0.5).astype(np.uint8))
    return item
g["init_i3d_model"], g["calc_psnr_and_ssim"], g["calculate_i3d_activations"] = init_i3d_model, rec_calc, rec_acts
g["TestDataset"].load_item = rec_load_item
args = types.SimpleNamespace(dataset="davis", data_root=os.path.join(tmp, "data"), model=model, ckpt=ckpt,
                             save_results=True, num_workers=0)
g["main_worker"](args)
import cv2, json
sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
videos = json.load(open(os.path.join(tmp, "data", "davis", "test.json")))
res = os.path.join("results", f"{model}_davis")
start, holes, comp_sha, frames_sha, masks_sha = 0, [], [], [], []
for k, (name, n) in enumerate(videos.items()):
    frames = np.stack(rec["frames"][start:start + n]); start += n
    masks = rec["masks"][k].astype(bool)
    comp = np.stack([cv2.cvtColor(cv2.imread(os.path.join(res, name, f"{i:05d}.png")), cv2.COLOR_BGR2RGB)
                     for i in range(n)])
    # outside the holes the script's output is its resized frame (evaluate.py:101-104)
    assert np.array_equal(comp[~masks], frames[~masks])
    holes.append(comp[masks]); comp_sha.append(sha(comp)); frames_sha.append(sha(frames)); masks_sha.append(sha(masks.astype(np.uint8)))
np.savez_compressed(out, metrics_txt=np.array(open(os.path.join(res, f"{model}_davis_metrics.txt")).read()),
                    videos=np.array(list(videos)), lengths=np.array(list(videos.values())),
                    psnr=np.array(rec["psnr"], dtype=np.float64), ssim=np.array(rec["ssim"], dtype=np.float64),
                    real=np.stack(rec["real"]), fake=np.stack(rec["fake"]), comp_holes=np.concatenate(holes),
                    comp_sha256=np.array(comp_sha), frames_sha256=np.array(frames_sha), masks_sha256=np.array(masks_sha))
print(open(os.path.join(res, f"{model}_davis_metrics.txt")).read())
'''


def main(names=None):
    import importlib
    import torch
    sys.path.insert(0, ROOT)
    from e2fgvi_b200.synth import synth_i3d_state_dict, synth_state_dict, write_eval_dataset
    from oracle.metrics_loader import SHIM as METRICS_SHIM
    from oracle.reference_loader import REFERENCE_ROOT, SHIM
    os.makedirs(OUT, exist_ok=True)
    for name, (model, videos, size, family, wseed, i3d_seed) in CASES.items():
        if names and name not in names:
            continue
        with tempfile.TemporaryDirectory() as tmp:
            write_eval_dataset(os.path.join(tmp, "data"), videos, size=size)
            mine = importlib.import_module("e2fgvi_b200.model." + model).InpaintGenerator()
            ckpt = os.path.join(tmp, "ckpt.pth")
            torch.save(synth_state_dict(mine, family, wseed), ckpt)
            i3d_ckpt = os.path.join(tmp, "i3d.pth")
            torch.save(synth_i3d_state_dict(i3d_seed), i3d_ckpt)
            child = os.path.join(tmp, "child.py")
            with open(child, "w") as f:
                f.write(CHILD)
            subprocess.check_call([sys.executable, child, METRICS_SHIM, SHIM, REFERENCE_ROOT,
                                   os.path.join(ROOT, "oracle", "restate_ssim.py"), tmp,
                                   os.path.join(OUT, name + ".npz"), model, ckpt, i3d_ckpt], cwd=tmp)
        print(name, "done")


if __name__ == "__main__":
    main(sys.argv[1:])
