"""VFID as evaluate.py computes it (reference core/metrics.py:62-151), with I3D on the GPU.

Drop-ins with the reference's signatures: ``init_i3d_model``, ``calculate_i3d_activations``, ``calculate_vfid``; and
``frechet_distance``.  The Fréchet distance between N(mu1, S1) and N(mu2, S2),

    d^2 = |mu1 - mu2|^2 + tr(S1) + tr(S2) - 2 tr((S1 S2)^(1/2)),

runs on the host with numpy and ``scipy.linalg.sqrtm`` (once per evaluation, on a 1024 x 1024 matrix).

``python -m e2fgvi_b200.vfid --data_root R --dataset davis --results DIR`` computes evaluate.py's VFID from the frames
``evaluate.py --save_results`` wrote (``DIR/<video>/%05d.png``) against the dataset's frames.
"""
import argparse
import json
import os
import zipfile

import numpy as np
import torch

I3D_SIZE = (432, 240)     # evaluate.py's (w, h)


def init_i3d_model(path="./release_model/i3d_rgb_imagenet.pt"):
    """``InceptionI3d(400, in_channels=3)`` with the checkpoint at ``path`` loaded (strict), on cuda:0."""
    from .i3d import InceptionI3d
    print(f"[Loading I3D model from {path} for FID score ..]")
    model = InceptionI3d(400, in_channels=3)
    model.load_state_dict(torch.load(path, map_location="cpu"))
    return model.to(torch.device("cuda:0")).eval()


def _frames_u8(video):
    """list of PIL RGB images (or HxWx3 uint8 arrays) -> (T, H, W, 3) uint8 numpy array."""
    return np.stack([np.asarray(f.convert("RGB") if hasattr(f, "convert") else f, dtype=np.uint8) for f in video])


def calculate_i3d_activations(video1, video2, i3d_model, device):
    """Features of two videos (lists of PIL images) as flattened numpy arrays, like the reference.  The two videos run
    as one batch of 2 when their shapes agree."""
    a, b = _frames_u8(video1), _frames_u8(video2)
    dev = torch.device(device)
    if a.shape == b.shape:
        x = torch.from_numpy(np.stack([a, b])).to(dev)
        f = i3d_model.features_u8(x).cpu().numpy()
        return f[0].flatten(), f[1].flatten()
    fa = i3d_model.features_u8(torch.from_numpy(a).to(dev)).cpu().numpy().flatten()
    fb = i3d_model.features_u8(torch.from_numpy(b).to(dev)).cpu().numpy().flatten()
    return fa, fb


def frechet_distance(mu1, s1, mu2, s2, eps=1e-6):
    """Fréchet distance between N(mu1, s1) and N(mu2, s2).  When sqrtm(s1 s2) is not finite, eps is added to both
    diagonals and the root retaken; an imaginary part on the root's diagonal above 1e-3 raises ValueError."""
    from scipy import linalg
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    s1, s2 = np.atleast_2d(s1), np.atleast_2d(s2)
    if mu1.shape != mu2.shape or s1.shape != s2.shape:
        raise ValueError(f"frechet_distance: shapes differ: {mu1.shape} / {mu2.shape}, {s1.shape} / {s2.shape}")
    root = linalg.sqrtm(s1.dot(s2))
    if not np.isfinite(root).all():
        print(f"fid calculation produces singular product; adding {eps} to diagonal of cov estimates")
        eye = np.eye(s1.shape[0]) * eps
        root = linalg.sqrtm((s1 + eye).dot(s2 + eye))
    if np.iscomplexobj(root):
        if not np.allclose(np.diagonal(root).imag, 0, atol=1e-3):
            raise ValueError(f"Imaginary component {np.max(np.abs(root.imag))}")
        root = root.real
    d = mu1 - mu2
    return d.dot(d) + np.trace(s1) + np.trace(s2) - 2 * np.trace(root)


def calculate_vfid(real_activations, fake_activations):
    """VFID between two lists of per-video activations (sample rows), with np.cov(rowvar=False)."""
    m1, m2 = np.mean(real_activations, axis=0), np.mean(fake_activations, axis=0)
    s1, s2 = np.cov(real_activations, rowvar=False), np.cov(fake_activations, rowvar=False)
    return frechet_distance(m1, s1, m2, s2)


# ----------------------------------------------------------------------------------------------------------- command
def read_dataset_video(data_root, dataset, name, count):
    """The first ``count`` frames of ``R/<dataset>/JPEGImages/<name>.zip`` as TestZipReader reads them (sorted member
    names, cv2.imdecode, BGR -> RGB): (count, H, W, 3) uint8."""
    import cv2
    path = os.path.join(data_root, dataset, "JPEGImages", f"{name}.zip")
    if not os.path.isfile(path):
        raise FileNotFoundError(f"vfid: video {name!r}: {path} not found")
    with zipfile.ZipFile(path) as z:
        names = sorted(z.namelist())
        if len(names) < count:
            raise ValueError(f"vfid: video {name!r}: {path} has {len(names)} frames, test.json says {count}")
        out = []
        for n in names[:count]:
            im = cv2.imdecode(np.frombuffer(z.read(n), dtype=np.uint8), cv2.IMREAD_COLOR)
            if im is None:
                raise ValueError(f"vfid: video {name!r}: cannot decode {n}")
            out.append(cv2.cvtColor(im, cv2.COLOR_BGR2RGB))
    return np.stack(out)


def read_results(results, name, count):
    """``DIR/<name>/%05d.png`` for frames 0 .. count-1 as (count, H, W, 3) uint8 RGB."""
    import cv2
    folder = os.path.join(results, name)
    if not os.path.isdir(folder):
        raise FileNotFoundError(f"vfid: video {name!r}: results folder {folder} not found")
    out = []
    for i in range(count):
        p = os.path.join(folder, f"{i:05d}.png")
        if not os.path.isfile(p):
            raise FileNotFoundError(f"vfid: video {name!r}: {p} missing ({count} frames expected)")
        im = cv2.imread(p, cv2.IMREAD_COLOR)
        if im is None:
            raise ValueError(f"vfid: video {name!r}: cannot decode {p}")
        out.append(cv2.cvtColor(im, cv2.COLOR_BGR2RGB))
    return np.stack(out)


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="python -m e2fgvi_b200.vfid",
                                 description="evaluate.py's VFID from saved results (evaluate.py --save_results)")
    ap.add_argument("--data_root", required=True, help="dataset root R (R/<dataset>/test.json, R/<dataset>/JPEGImages)")
    ap.add_argument("--dataset", required=True, choices=["davis", "youtube-vos"])
    ap.add_argument("--results", required=True, help="folder with <video>/%%05d.png per test video")
    ap.add_argument("--i3d", default="./release_model/i3d_rgb_imagenet.pt", help="I3D checkpoint")
    ap.add_argument("--save_activations", default=None, help="folder to write real.npy and fake.npy (videos x 1024)")
    return ap.parse_args(argv)


def main(argv=None, model=None):
    args = parse_args(argv)
    from .video import resize_frames
    with open(os.path.join(args.data_root, args.dataset, "test.json")) as f:
        videos = json.load(f)
    if model is None:
        model = init_i3d_model(args.i3d)
    dev = next(model.parameters()).device
    w, h = I3D_SIZE
    real, fake = [], []
    for k, (name, count) in enumerate(videos.items()):
        gt = read_dataset_video(args.data_root, args.dataset, name, count)
        res = read_results(args.results, name, count)
        gt = resize_frames(torch.from_numpy(gt).to(dev), (w, h))
        res = torch.from_numpy(res).to(dev)
        if tuple(res.shape[1:3]) != (h, w):
            raise ValueError(f"vfid: video {name!r}: results are {res.shape[2]}x{res.shape[1]}, expected {w}x{h}")
        feats = model.features_u8(torch.stack([gt, res])).cpu().numpy()
        real.append(feats[0].flatten())
        fake.append(feats[1].flatten())
        print(f"[{k + 1:3}/{len(videos)}] Name: {name}")
    if args.save_activations:
        os.makedirs(args.save_activations, exist_ok=True)
        np.save(os.path.join(args.save_activations, "real.npy"), np.stack(real))
        np.save(os.path.join(args.save_activations, "fake.npy"), np.stack(fake))
    score = calculate_vfid(real, fake)
    print(f"Finish evaluation... VFID: {score:.3f}")
    return score


if __name__ == "__main__":
    main()
