"""Goldens for the I3D / VFID path, made by the UNMODIFIED reference on the CPU (``python -m oracle.gen_golden_i3d``).

Runs ``InceptionI3d.extract_features(x, 'Logits')`` (eval mode, ``synth.synth_i3d_state_dict(0)``) on synthetic
videos (``synth.synth_video``, x = frames.float().div(255) as ToTorchFormatTensor computes it) and
``calculate_vfid`` on synthetic activation sets.  Stores outputs only, in ``tests/golden/i3d_vfid.npz``:
  * the state-dict layout (keys, shapes, dtypes);
  * per case: the (1, 1024) features and the per-channel mean of every endpoint;
  * twelve 3-frame clips (six "real", six "fake"), their features and the VFID between the two sets;
  * calculate_vfid over synthetic activation sets, one with fewer samples than dimensions (50 x 1024, evaluate.py's
    DAVIS case: singular covariances).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from e2fgvi_b200 import synth  # noqa: E402
from oracle import metrics_loader  # noqa: E402

# name -> (T, H, W, video seed)
CASES = {"eval": (70, 240, 432, 0), "odd": (11, 90, 170, 1), "short": (3, 60, 108, 2), "t1": (1, 60, 108, 3)}
CLIP = (3, 60, 108)
REAL_SEEDS, FAKE_SEEDS = tuple(range(100, 106)), tuple(range(200, 206))
ACT_SETS = {"n200_d32": (200, 32), "n50_d1024": (50, 1024), "n10_d16": (10, 16)}
OUT = os.path.join(ROOT, "tests", "golden", "i3d_vfid.npz")


def video_input(t, h, w, seed):
    frames, _ = synth.synth_video(t, h, w, seed=seed)
    return frames, torch.from_numpy(frames).permute(3, 0, 1, 2).unsqueeze(0).contiguous().float().div(255)


class _Linalg:
    """scipy.linalg for the reference's calculate_frechet_distance: SciPy 1.18 dropped sqrtm's ``disp`` argument, which
    the reference passes (``disp=False`` returned ``(root, error_estimate)``)."""

    def __getattr__(self, name):
        from scipy import linalg
        return getattr(linalg, name)

    @staticmethod
    def sqrtm(a, disp=True):
        from scipy import linalg
        root = linalg.sqrtm(a)
        return root if disp else (root, None)


def main():
    metrics = metrics_loader.import_metrics()
    metrics.linalg = _Linalg()
    net = metrics.InceptionI3d(400, in_channels=3).eval()
    sd = synth.synth_i3d_state_dict(0)
    net.load_state_dict(sd, strict=True)
    out = {}
    ref_sd = net.state_dict()
    out["layout_keys"] = np.array(list(ref_sd.keys()))
    out["layout_shapes"] = np.array([",".join(map(str, v.shape)) for v in ref_sd.values()])
    out["layout_dtypes"] = np.array([str(v.dtype) for v in ref_sd.values()])
    eps = [e for e in metrics.InceptionI3d.VALID_ENDPOINTS if e in net.end_points]
    out["endpoints"] = np.array(eps)
    with torch.no_grad():
        for name, (t, h, w, seed) in CASES.items():
            _, x = video_input(t, h, w, seed)
            y = x
            for e in eps:                       # extract_features' loop, keeping every endpoint
                y = net._modules[e](y)
                out[f"{name}/mean/{e}"] = y.mean(dim=(2, 3, 4)).numpy()
            feats = net.extract_features(x, "Logits")
            out[f"{name}/features"] = feats.numpy()
            print(name, tuple(x.shape), float(feats.abs().max()))
        for tag, seeds in (("real", REAL_SEEDS), ("fake", FAKE_SEEDS)):
            out[f"clips/{tag}"] = np.stack([
                net.extract_features(video_input(*CLIP, s)[1], "Logits").numpy().flatten() for s in seeds])
    out["clips/vfid"] = np.float64(metrics.calculate_vfid(list(out["clips/real"]), list(out["clips/fake"])))
    for tag, (n, d) in ACT_SETS.items():
        real, fake = synth.synth_activations(n, d, 1), synth.synth_activations(n, d, 2)
        out[f"acts/{tag}"] = np.float64(metrics.calculate_vfid(list(real), list(fake)))
        print(tag, out[f"acts/{tag}"])
    print("clips vfid", out["clips/vfid"])
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
