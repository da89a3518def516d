"""PSNR / SSIM on the CPU: the skimage 0.16.2 restatement against an independent exact formulation and against the
unmodified reference ``core.metrics.calc_psnr_and_ssim`` (where the reference is present), edge cases, the C-ABI
argument checks of ``e2f_frame_metrics``, and the evaluate command's argument and dataset handling."""
import numpy as np
import pytest

from e2fgvi_b200 import evaluate as E
from e2fgvi_b200 import metrics as M
from e2fgvi_b200 import synth
from oracle import metrics_loader, restate_ssim

needs_reference = pytest.mark.skipif(not metrics_loader.available(), reason="reference not present")


def exact_ssim(x, y, win):
    """compare_ssim from exact integer box sums (cumulative sums of values scaled by 4), for the crop's windows."""
    NP = win * win
    cov_norm = NP / (NP - 1)
    C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
    out = []
    for ch in range(x.shape[-1]):
        a = np.round(x[..., ch].astype(np.float64) * 4).astype(np.int64)
        b = np.round(y[..., ch].astype(np.float64) * 4).astype(np.int64)

        def box(v):                              # sums over every win x win window inside the image
            s = np.pad(v.cumsum(0).cumsum(1), ((1, 0), (1, 0)))
            return s[win:, win:] - s[:-win, win:] - s[win:, :-win] + s[:-win, :-win]
        ux, uy = box(a) / (4 * NP), box(b) / (4 * NP)
        uxx, uyy, uxy = box(a * a) / (16 * NP), box(b * b) / (16 * NP), box(a * b) / (16 * NP)
        vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
        S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
        out.append(S.mean())
    return np.mean(out)


@pytest.mark.parametrize("shape,win,holes", [((240, 432, 3), 65, True), ((240, 432, 3), 65, False),
                                             ((65, 130, 1), 65, True), ((97, 131, 3), 7, True)])
def test_restatement_matches_exact_box_sums(shape, win, holes):
    ori, comp = synth.synth_composite_pair(*shape, seed=sum(shape) + win, holes=holes)
    got = restate_ssim.compare_ssim(ori.astype(np.float64), comp.astype(np.float64), data_range=255,
                                    multichannel=True, win_size=win)
    assert abs(got - exact_ssim(ori, comp, win)) <= 1e-12


@needs_reference
def test_reference_calc_psnr_and_ssim_equals_restatement(monkeypatch):
    ref = metrics_loader.import_metrics()
    # the reference's skimage.measure (an import stand-in here) gets the restatement as its compare_ssim
    monkeypatch.setattr(ref.measure, "compare_ssim", restate_ssim.compare_ssim)
    for seed in range(3):
        ori, comp = synth.synth_composite_pair(120, 160, 3, seed)
        psnr, ssim = ref.calc_psnr_and_ssim(ori, comp)
        want_psnr, want_ssim = restate_ssim.calc_psnr_and_ssim(ori, comp)
        assert psnr == want_psnr
        assert ssim == want_ssim
        assert M.psnr_from_sse(((ori.astype(np.float64) - comp) ** 2).sum(), ori.size) == psnr


def test_edge_cases():
    ori, _ = synth.synth_composite_pair(70, 80, 3, 0)
    x = ori.astype(np.float64)
    assert restate_ssim.compare_ssim(x, x, data_range=255, multichannel=True, win_size=65) == 1.0
    assert restate_ssim.calc_psnr_and_ssim(ori, ori)[0] == float("inf")
    assert M.psnr_from_sse(0.0, ori.size) == float("inf")
    with pytest.raises(ValueError, match="odd"):
        restate_ssim.compare_ssim(x, x, data_range=255, multichannel=True, win_size=64)
    with pytest.raises(ValueError, match="exceeds"):
        restate_ssim.compare_ssim(x[:60], x[:60], data_range=255, multichannel=True, win_size=65)
    with pytest.raises(NotImplementedError):
        restate_ssim.compare_ssim(x, x, data_range=255, multichannel=True, win_size=65, gaussian_weights=True)


def test_dropins_reject_other_dtypes():
    a = np.zeros((70, 70, 3), dtype=np.float64)
    with pytest.raises(TypeError):
        M.calc_psnr_and_ssim(a, a)
    with pytest.raises(TypeError):
        M.calculate_psnr(a.astype(np.int16), a.astype(np.int16))
    with pytest.raises(AssertionError):
        M.calc_psnr_and_ssim(a.astype(np.uint8), a[:69].astype(np.uint8))


def test_abi_argument_checks(lib):
    assert lib.e2f_frame_metrics_work_elems(70, 240, 432, 3, 65) == 70 * 2 * 4     # two 256-column tiles per frame
    assert lib.e2f_frame_metrics_work_elems(1, 65, 65, 1, 65) == 2
    assert lib.e2f_frame_metrics_work_elems(70, 240, 432, 3, 0) == 70 * 76            # SSE only: 4096 values per CTA
    assert lib.e2f_frame_metrics_work_elems(2, 1, 1, 1, 0) == 2
    for bad in [(0, 240, 432, 3, 65), (1, 240, 432, 5, 65), (1, 240, 432, 0, 65), (1, 240, 432, 3, 64),
                (1, 240, 432, 3, 1), (1, 64, 432, 3, 65), (1, 240, 64, 3, 65)]:
        assert lib.e2f_frame_metrics_work_elems(*bad) == -1, bad
    p = 1 << 20

    def call(a=p, a_u8=1, b=p, b_u8=0, sse=p, ssim=p, work=p, n=1, h=240, w=432, c=3, win=65, rng=255.0):
        return lib.e2f_frame_metrics(a, a_u8, b, b_u8, sse, ssim, work, n, h, w, c, win, rng, None)
    assert call(a=None) == -1
    assert call(sse=None) == -1
    assert call(work=None) == -1
    assert call(a_u8=2) == -1
    assert call(n=0) == -1
    assert call(c=5) == -1
    assert call(win=64) == -1
    assert call(h=64) == -1
    assert call(rng=0.0) == -1
    assert call(rng=float("nan")) == -1
    assert call(ssim=None) == -1
    assert call(h=600, w=600, c=4, win=501) == -2                                   # window too wide for shared memory
    assert call(h=800, w=800, c=3, win=711) == -2                                   # 709 is the largest at c = 3
    assert call(h=800, w=800, c=4, win=469) == -2                                   # 467 is the largest at c = 4
    assert call(b=p + 2) == -3                                                      # fp32 operand misaligned
    assert call(ssim=p + 4) == -3
    assert b"e2f_frame_metrics" in lib.e2f_last_error()


# ------------------------------------------------------------------------------------------ the evaluate command
def test_command_arguments():
    a = E.parser().parse_args(["--dataset", "davis", "--data_root", "R", "--model", "e2fgvi", "--ckpt", "c.pth"])
    assert (a.dataset, a.data_root, a.model, a.ckpt, a.save_results, a.num_workers) == \
        ("davis", "R", "e2fgvi", "c.pth", False, 4)
    a = E.parser().parse_args(["--dataset", "youtube-vos", "--data_root", "R", "--model", "e2fgvi_hq", "--ckpt", "c",
                               "--save_results", "--num_workers", "0"])
    assert (a.save_results, a.num_workers) == (True, 0)
    for bad in (["--dataset", "kitti", "--data_root", "R", "--ckpt", "c"], ["--dataset", "davis", "--ckpt", "c"],
                ["--dataset", "davis", "--data_root", "R", "--ckpt", "c", "--model", "sttn"],
                ["--dataset", "davis", "--data_root", "R", "--ckpt", "c", "--set_size"]):
        with pytest.raises(SystemExit):
            E.parser().parse_args(bad)


def test_command_reads_dataset(tmp_path):
    import types
    root, frames = synth.write_eval_dataset(str(tmp_path), {"cows": 3, "bear": 2}, drop_mask=("bear", 1))
    args = types.SimpleNamespace(data_root=root, dataset="davis")
    f, m = E.read_video(args, "cows", 3)
    assert np.array_equal(f, frames["cows"][0])
    assert len(m) == 3 and all(np.array_equal(mi != 0, mw != 0) for mi, mw in zip(m, frames["cows"][1]))
    with pytest.raises(FileNotFoundError, match="bear"):
        E.read_video(args, "bear", 2)                         # mask 00001.png is missing
    with pytest.raises(FileNotFoundError, match="goat"):
        E.read_video(args, "goat", 1)                         # no zip
    with pytest.raises(ValueError, match="cows"):
        E.read_video(args, "cows", 5)                         # test.json asks for more frames than the zip holds
