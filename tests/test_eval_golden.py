"""The evaluate command against the unmodified reference ``evaluate.py`` (goldens from ``oracle/gen_golden_eval.py``).

CPU: the goldens are self-consistent with their regenerated inputs — the numpy restatement of the front end reproduces
the script's resized frames and dilated masks (SHA-256), and those frames with the stored hole pixels written back
reproduce the digest of every PNG the script saved.

H100: ``python -m e2fgvi_b200.evaluate`` on the same dataset and weights.  Its resized frames and masks match the
digests; its PNGs equal the script's outside the holes and are within 1 LSB on all but < 5 % of hole pixels (the
networks differ in the last bits); its per-frame PSNR / SSIM equal the restatement applied to its own composite (PSNR
bit-identical, SSIM within 1e-12) and are within 0.05 dB / 1e-3 of the script's; its I3D activations are within
1e-3 * max(1, max |ref|) of the script's; metrics.txt has the script's lines, names and format, with the numbers
checked against the same bars and the final VFID equal to ``calculate_vfid`` of its own activations."""
import hashlib
import importlib
import os
import re
import types

import numpy as np
import pytest

from e2fgvi_b200 import evaluate as E
from e2fgvi_b200 import synth
from oracle import restate_frontend as RF
from oracle.gen_golden_eval import CASES

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LINE = re.compile(r"^\[(.{3})/(\d+)\] Name: (.{25}) \| PSNR/SSIM: (\d+\.\d{4})/(\d+\.\d{4})$")
FINAL = re.compile(r"^Finish evaluation\.\.\. Average Frame PSNR/SSIM/VFID: (\d+\.\d{2})/(\d+\.\d{4})/(-?\d+\.\d{3})$")


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _dataset(name, root):
    _, videos, size, *_ = CASES[name]
    root, _ = synth.write_eval_dataset(root, videos, size=size)
    return root, videos, np.load(os.path.join(GOLDEN, name + ".npz"))


def _split_holes(g, masks_per_video):
    """The stored hole pixels, per video."""
    out, start = [], 0
    for m in masks_per_video:
        k = int(m.sum())
        out.append(g["comp_holes"][start:start + k])
        start += k
    assert start == len(g["comp_holes"])
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_self_consistent(name, tmp_path):
    root, videos, g = _dataset(name, str(tmp_path))
    args = types.SimpleNamespace(data_root=root, dataset="davis")
    frames, masks = [], []
    for k, (video, n) in enumerate(videos.items()):
        f, planes = E.read_video(args, video, n)
        frames.append(RF.resize_bicubic(f, E.SIZE))
        masks.append(RF.read_mask(np.stack(planes), E.SIZE))
        assert _sha(frames[-1]) == str(g["frames_sha256"][k])
        assert _sha(masks[-1]) == str(g["masks_sha256"][k])
    for k, holes in enumerate(_split_holes(g, masks)):
        comp = frames[k].copy()
        comp[masks[k].astype(bool)] = holes
        assert _sha(comp) == str(g["comp_sha256"][k])
    assert list(g["videos"]) == list(videos) and len(g["psnr"]) == len(g["ssim"]) == sum(videos.values())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_command_matches_evaluate_py(name, cuda, tmp_path, monkeypatch):
    import cv2
    from e2fgvi_b200 import vfid
    from e2fgvi_b200.i3d import InceptionI3d
    from oracle import restate_ssim
    model, videos, size, family, wseed, i3d_seed = CASES[name]
    root, videos, g = _dataset(name, str(tmp_path / "data"))
    gen = importlib.import_module("e2fgvi_b200.model." + model).InpaintGenerator()
    gen.load_state_dict(synth.synth_state_dict(gen, family, wseed))
    i3d = InceptionI3d()
    i3d.load_state_dict(synth.synth_i3d_state_dict(i3d_seed))
    gen, i3d = gen.eval().to(cuda), i3d.to(cuda).eval()

    seen, prepared, acts = [], [], []
    fm, prep, cv = E.frame_metrics, E.prepare_inputs, vfid.calculate_vfid

    def rec_prepare(*a, **k):
        out = prep(*a, **k)
        prepared.append(tuple(t.cpu().numpy() for t in out))
        return out

    def rec_metrics(a, b):
        out = fm(a, b)
        seen.append((a.cpu().numpy(), b.cpu().numpy(), out))
        return out

    def rec_vfid(real, fake):
        acts.append((np.stack(real), np.stack(fake)))
        return cv(real, fake)
    monkeypatch.setattr(E, "prepare_inputs", rec_prepare)
    monkeypatch.setattr(E, "frame_metrics", rec_metrics)
    monkeypatch.setattr(vfid, "calculate_vfid", rec_vfid)
    monkeypatch.chdir(tmp_path)
    argv = ["--dataset", "davis", "--data_root", root, "--model", model, "--ckpt", "unused", "--save_results",
            "--num_workers", "0"]
    avg_psnr, avg_ssim, score = E.main(argv, model=gen, i3d=i3d)
    res = tmp_path / "results" / f"{model}_davis"

    masks = [m for _, m in prepared]
    holes = _split_holes(g, masks)
    ref_psnr, ref_ssim, start = g["psnr"], g["ssim"], 0
    for k, (video, n) in enumerate(videos.items()):
        frames, m = prepared[k]
        assert _sha(frames) == str(g["frames_sha256"][k]) and _sha(m) == str(g["masks_sha256"][k])
        hole = m.astype(bool)
        saved = np.stack([cv2.cvtColor(cv2.imread(str(res / video / f"{i:05d}.png")), cv2.COLOR_BGR2RGB)
                          for i in range(n)])
        assert np.array_equal(saved[~hole], frames[~hole])                    # exact outside the holes
        diff = np.abs(saved[hole].astype(np.int16) - holes[k].astype(np.int16))
        assert diff.max() <= 1 and (diff > 0).mean() < 0.05, (diff.max(), (diff > 0).mean())
        ori, comp, (psnr, ssim) = seen[k]
        assert np.array_equal(ori, frames) and np.array_equal(saved, comp.astype(np.uint8))
        for f in range(n):
            x, y = ori[f].astype(np.float64), comp[f].astype(np.float64)
            mse = np.mean((x - y) ** 2)
            assert psnr[f] == (float("inf") if mse == 0 else 20. * np.log10(255. / np.sqrt(mse)))
            want = restate_ssim.compare_ssim(x, y, data_range=255, multichannel=True, win_size=65)
            assert abs(ssim[f] - want) <= 1e-12
        assert np.abs(psnr - ref_psnr[start:start + n]).max() <= 0.05
        assert np.abs(ssim - ref_ssim[start:start + n]).max() <= 1e-3
        start += n

    real, fake = acts[0]
    for got, want in ((real, g["real"]), (fake, g["fake"])):
        assert np.abs(got - want).max() <= 1e-3 * max(1.0, np.abs(want).max())
    assert score == cv(list(real), list(fake))

    got_lines = (res / f"{model}_davis_metrics.txt").read_text().split("\n")
    ref_lines = str(g["metrics_txt"]).split("\n")
    assert len(got_lines) == len(ref_lines) == len(videos) + 1
    for k, (video, n) in enumerate(videos.items()):
        got, ref = LINE.match(got_lines[k]), LINE.match(ref_lines[k])
        assert got and ref and got.group(1, 2) == ref.group(1, 2)                  # "[  k/N]"
        # DataLoader collates the name into a list under the reference's pinned PyTorch (['bear']) and into a tuple
        # under recent releases (('bear',)); the command prints the list form, padded to 25 as the script pads it
        assert got.group(3) == f"{str([video]):25}" and ref.group(3).strip() in (str([video]), str((video,)))
        psnr, ssim = seen[k][2]
        assert got.group(4, 5) == (f"{sum(psnr) / n:.4f}", f"{sum(ssim) / n:.4f}")
        assert abs(float(got.group(4)) - float(ref.group(4))) <= 0.05 + 1e-4
        assert abs(float(got.group(5)) - float(ref.group(5))) <= 1e-3 + 1e-4
    got, ref = FINAL.match(got_lines[-1]), FINAL.match(ref_lines[-1])
    assert got and ref
    assert got.groups() == (f"{avg_psnr:.2f}", f"{avg_ssim:.4f}", f"{score:.3f}")
    assert abs(float(got.group(1)) - float(ref.group(1))) <= 0.05 + 0.005
    assert abs(float(got.group(2)) - float(ref.group(2))) <= 1e-3 + 1e-4
    with pytest.raises(FileExistsError):
        E.main(argv, model=gen, i3d=i3d)
