"""PSNR / SSIM on the H100: the fused kernel against the skimage 0.16.2 restatement (PSNR bit-identical, SSIM within
1e-12) over frame sizes, channel counts, operand dtypes and batch sizes; determinism; the drop-ins; the float32
composite of ``VideoInpainter``; and the evaluate command end to end on a synthetic dataset."""
import os

import cv2
import numpy as np
import pytest
import torch

from e2fgvi_b200 import evaluate as E
from e2fgvi_b200 import metrics as M
from e2fgvi_b200 import synth
from e2fgvi_b200 import vfid
from e2fgvi_b200.video import VideoInpainter, finalize, prepare_inputs
from oracle import restate_ssim

pytestmark = pytest.mark.gpu


def _want(ori, comp, win):
    x, y = ori.astype(np.float64), comp.astype(np.float64)
    mse = np.mean((x - y) ** 2)
    psnr = float("inf") if mse == 0 else 20. * np.log10(255. / np.sqrt(mse))
    return psnr, restate_ssim.compare_ssim(x, y, data_range=255, multichannel=True, win_size=win)


def _check(oris, comps, win, psnr, ssim):
    for f in range(len(oris)):
        wp, ws = _want(oris[f], comps[f], win)
        assert psnr[f] == wp, (f, psnr[f], wp)
        assert abs(ssim[f] - ws) <= 1e-12, (f, ssim[f], ws)


@pytest.mark.parametrize("h,w,c,win", [(240, 432, 3, 65), (240, 432, 1, 65), (65, 65, 3, 65), (65, 433, 3, 65),
                                       (97, 131, 3, 7), (97, 131, 1, 7), (1080, 1920, 3, 65)])
@pytest.mark.parametrize("kinds", ["u8/u8", "u8/f32", "f32/f32"])
def test_kernel_matches_restatement(cuda, h, w, c, win, kinds):
    oris, comps = zip(*[synth.synth_composite_pair(h, w, c, seed=s) for s in range(2)])
    oris, comps = np.stack(oris), np.stack(comps)
    if kinds == "u8/u8":
        comps = np.floor(comps).astype(np.uint8)
    a = torch.from_numpy(oris if kinds != "f32/f32" else oris.astype(np.float32)).to(cuda)
    b = torch.from_numpy(comps).to(cuda)
    psnr, ssim = M.frame_metrics(a, b, win_size=win)
    _check(oris, comps, win, psnr, ssim)


def test_seventy_distinct_frames_and_identical_frames(cuda):
    oris, comps = zip(*[synth.synth_composite_pair(240, 432, 3, seed=100 + s, holes=s % 7 != 0) for s in range(70)])
    oris, comps = np.stack(oris), np.stack(comps)
    a, b = torch.from_numpy(oris).to(cuda), torch.from_numpy(comps).to(cuda)
    psnr, ssim = M.frame_metrics(a, b)
    _check(oris, comps, 65, psnr, ssim)
    assert np.isinf(psnr[::7]).all() and (ssim[::7] == 1.0).all()
    psnr2, ssim2 = M.frame_metrics(a, b)                          # deterministic: bit-identical on a second run
    assert np.array_equal(psnr, psnr2) and np.array_equal(ssim, ssim2)


def test_arbitrary_fp32_operands(cuda):
    rng = np.random.default_rng(7)
    x = (rng.random((2, 120, 200, 3)) * 255).astype(np.float32)
    y = np.clip(x + rng.normal(0, 9, x.shape), 0, 255).astype(np.float32)
    psnr, ssim = M.frame_metrics(torch.from_numpy(x).to(cuda), torch.from_numpy(y).to(cuda))
    for f in range(2):
        wp, ws = _want(x[f], y[f], 65)
        assert abs(psnr[f] - wp) <= 1e-12 * abs(wp)
        assert abs(ssim[f] - ws) <= 1e-12


def test_frame_metrics_errors(cuda):
    a = torch.zeros((1, 70, 70, 3), dtype=torch.uint8, device=cuda)
    with pytest.raises(ValueError, match="odd"):
        M.frame_metrics(a, a, win_size=64)
    with pytest.raises(ValueError, match="exceeds"):
        M.frame_metrics(a[:, :60], a[:, :60])
    with pytest.raises(TypeError):
        M.frame_metrics(a, a.double())


def test_dropins_equal_restatement(cuda):
    for seed in range(3):
        ori, comp = synth.synth_composite_pair(240, 432, 3, seed=200 + seed)
        psnr, ssim = M.calc_psnr_and_ssim(ori, comp)
        wp, ws = restate_ssim.calc_psnr_and_ssim(ori, comp)
        assert isinstance(psnr, float) and isinstance(ssim, float)
        assert psnr == wp and abs(ssim - ws) <= 1e-12
        assert M.calculate_psnr(ori, comp) == wp
        assert M.calculate_psnr(ori[..., 0], comp[..., 0]) == _want(ori[..., :1], comp[..., :1], 3)[0]
    ori, comp = synth.synth_composite_pair(2, 1, 3, seed=9, holes=False)         # smaller than any SSIM window
    comp[0, 0, 1] += 0.25
    mse = np.mean((ori.astype(np.float64) - comp) ** 2)
    assert M.calculate_psnr(ori, comp) == 20. * np.log10(255. / np.sqrt(mse))
    assert M.calculate_psnr(ori, ori) == float("inf")
    oris, comps = zip(*[synth.synth_composite_pair(240, 432, 3, seed=s) for s in range(5)])
    sse = M.frame_sse(torch.from_numpy(np.stack(oris)).to(cuda), torch.from_numpy(np.stack(comps)).to(cuda))
    assert np.array_equal(sse, [((o.astype(np.float64) - c) ** 2).sum() for o, c in zip(oris, comps)])


class _ToyModel(torch.nn.Module):
    """Per-clip stand-in for InpaintGenerator with outputs in (-1, 1)."""

    def forward(self, x, l_t):
        b, t, c, h, w = x.shape
        y = torch.tanh(x.roll(1, 3) * 0.7 + x.mean(dim=(1, 2), keepdim=True) + 0.1 * l_t)
        return y.reshape(b * t, c, h, w), None


def test_composite_quarters_and_finalize(cuda):
    frames, masks = synth.synth_video(13, 240, 432, seed=3)
    drv = VideoInpainter(_ToyModel(), cuda_graphs=False)
    f, m = torch.from_numpy(frames).to(cuda), torch.from_numpy(masks).to(cuda)
    comp = drv.composite(f, m)
    assert comp.dtype == torch.float32 and comp.shape == f.shape
    c = comp.cpu().numpy()
    assert np.array_equal(c * 4, np.round(c * 4))
    assert (c != np.floor(c)).any()                          # blended frames hold fractions
    assert torch.equal(finalize(comp), drv(f, m))


# ------------------------------------------------------------------------------------------ the evaluate command
@pytest.fixture(scope="module")
def nets(cuda):
    import importlib
    from e2fgvi_b200.i3d import InceptionI3d
    gen = importlib.import_module("e2fgvi_b200.model.e2fgvi").InpaintGenerator()
    gen.load_state_dict(synth.synth_state_dict(gen, "stress", 2))
    i3d = InceptionI3d()
    i3d.load_state_dict(synth.synth_i3d_state_dict(0))
    return gen.eval().to(cuda), i3d.to(cuda).eval()


def test_command_end_to_end(nets, tmp_path, monkeypatch, capsys):
    gen, i3d = nets
    videos = {"bear": 13, "cows": 6, "goat": 16}
    root, data = synth.write_eval_dataset(str(tmp_path / "data"), videos, size=(270, 480))
    monkeypatch.chdir(tmp_path)
    seen, acts = [], []
    fm, cv = E.frame_metrics, vfid.calculate_vfid

    def rec_metrics(a, b):
        out = fm(a, b)
        seen.append((a.cpu().numpy(), b.cpu().numpy(), out))
        return out

    def rec_vfid(real, fake):
        acts.append((np.stack(real), np.stack(fake)))
        return cv(real, fake)
    monkeypatch.setattr(E, "frame_metrics", rec_metrics)
    monkeypatch.setattr(vfid, "calculate_vfid", rec_vfid)
    argv = ["--dataset", "davis", "--data_root", root, "--model", "e2fgvi", "--ckpt", "unused", "--save_results",
            "--num_workers", "0"]
    avg_psnr, avg_ssim, score = E.main(argv, model=gen, i3d=i3d)
    lines = open(tmp_path / "results" / "e2fgvi_davis" / "e2fgvi_davis_metrics.txt").read().split("\n")
    assert len(lines) == 4 and capsys.readouterr().out.count("Name:") == 3
    all_psnr, all_ssim = [], []
    drv = VideoInpainter(gen)
    for k, (name, n) in enumerate(videos.items()):
        ori, comp, (psnr, ssim) = seen[k]
        frames, masks = data[name]
        f, m = prepare_inputs(frames, list(masks * 255), E.SIZE)
        assert np.array_equal(ori, f.cpu().numpy())
        assert np.array_equal(comp, drv.composite(f, m).cpu().numpy())             # the command's own composite
        _check(ori, comp, 65, psnr, ssim)
        all_psnr += psnr.tolist()
        all_ssim += ssim.tolist()
        want = f"[{k + 1:3}/3] Name: {str([name]):25} | PSNR/SSIM: {sum(psnr) / n:.4f}/{sum(ssim) / n:.4f}"
        assert lines[k] == want
        saved = np.stack([cv2.cvtColor(cv2.imread(str(tmp_path / "results" / "e2fgvi_davis" / name / f"{i:05d}.png")),
                                       cv2.COLOR_BGR2RGB) for i in range(n)])
        assert np.array_equal(saved, comp.astype(np.uint8))
    real, fake = acts[0]
    assert real.shape == fake.shape == (3, 1024)
    assert score == cv(list(real), list(fake))
    assert (avg_psnr, avg_ssim) == (sum(all_psnr) / len(all_psnr), sum(all_ssim) / len(all_ssim))
    assert lines[3] == f"Finish evaluation... Average Frame PSNR/SSIM/VFID: {avg_psnr:.2f}/{avg_ssim:.4f}/{score:.3f}"
    with pytest.raises(FileExistsError):
        E.main(argv, model=gen, i3d=i3d)
