"""Video front end (test.py:56-70 ``read_mask``, :98-103 ``resize_frames``): the product's Pillow tables and the numpy
restatement against Pillow / OpenCV and against what the unmodified test.py produced (digests in the goldens), the
C-ABI argument checks, the ``inpaint`` command's argument handling, and — on the GPU — the two kernels bit for bit,
``prepare_inputs`` and the whole driver / command against the goldens."""
import hashlib
import itertools
import os

import numpy as np
import pytest
import torch

from e2fgvi_b200 import inpaint as I
from e2fgvi_b200 import video as V
from e2fgvi_b200.synth import synth_state_dict, synth_video
from oracle import restate_frontend as RF
from oracle.gen_golden_frontend import CASES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

SIZES_IN = (3840, 1920, 1280, 853, 432, 200, 5, 1)
SIZES_OUT = (432, 240, 216, 100, 5, 1)
SWEEP = list(itertools.product(SIZES_IN, SIZES_OUT))


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _args(name):
    model, n, _, _, _, _, _, _, extra = CASES[name]
    return I.parser().parse_args(["-v", "frames", "-c", "ckpt.pth", "-m", "masks", "--model", model] + extra)


def _case(name):
    """Inputs of a golden case as the script read them: RGB frames and the masks' 'L' planes (PNG of mask * 255)."""
    model, n, (h, w), (hm, wm), family, wseed, fseed, mseed, _ = CASES[name]
    frames, _ = synth_video(n, h, w, fseed)
    _, masks = synth_video(n, hm, wm, mseed)
    return frames, masks * 255, np.load(os.path.join(GOLDEN, name + ".npz"))


def _golden_comp(g, frames, masks):
    """What the script wrote: its resized frames with the stored hole pixels written back at its dilated holes, checked
    against the digest of the script's whole output."""
    comp = np.array(frames, copy=True)
    comp[masks.astype(bool)] = g["comp_holes"]
    assert _sha(comp) == str(g["comp_sha256"])
    return comp


def _driver_kwargs(args):
    return dict(neighbor_stride=args.neighbor_stride, ref_length=args.step, num_ref=args.num_ref)


# ------------------------------------------------------------------------------------------------------------- CPU
def test_bicubic_tables_match_pillow_sweep():
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(0)
    for a, b in SWEEP:
        # a -> b along the width, then along the height, the other axis 48 -> 40.  Recent Pillow (12.2 among
        # them) resizes an image more than 100x taller than wide vertically first; Pillow 9 and video frames never do.
        for shape, size in (((48, a, 3), (b, 40)), ((a, 48, 3), (40, b))):
            img = rng.integers(0, 256, shape, dtype=np.uint8)
            want = np.asarray(Image.fromarray(img).resize(size))
            assert np.array_equal(RF.resize_bicubic(img, size), want), (shape, size)
    for shape, size in (((1080, 1920, 3), (432, 240)), ((720, 1280, 3), (432, 240)), ((481, 853, 3), (432, 240)),
                        ((100, 200, 3), (432, 240)), ((61, 37, 3), (33, 100)), ((240, 432, 3), (432, 240))):
        img = rng.integers(0, 256, shape, dtype=np.uint8)
        assert np.array_equal(RF.resize_bicubic(img, size), np.asarray(Image.fromarray(img).resize(size))), shape


def test_nearest_tables_match_pillow_sweep():
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(1)
    for a, b in SWEEP:
        for shape, size in (((7, a), (b, 5)), ((a, 7), (5, b))):
            m = rng.integers(0, 256, shape, dtype=np.uint8)
            want = np.asarray(Image.fromarray(m).resize(size, Image.NEAREST))
            assert np.array_equal(RF.nearest(m, size), want), (shape, size)


def test_read_mask_restatement_matches_pillow_and_opencv():
    Image = pytest.importorskip("PIL.Image")
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2)
    for shape, size in (((180, 320), (432, 240)), ((1080, 1920), (432, 240)), ((75, 130), (200, 100)),
                        ((9, 9), (5, 5))):
        planes = (rng.random((2,) + shape) < 0.02).astype(np.uint8) * rng.integers(1, 256, (2,) + shape, dtype=np.uint8)
        planes[1, 0, :] = 7                                                  # a hole along the border
        want = []
        for p in planes:                                                     # test.py:62-68
            m = np.array(Image.fromarray(p).resize(size, Image.NEAREST).convert("L"))
            m = np.array(m > 0).astype(np.uint8)
            want.append(cv2.dilate(m, cv2.getStructuringElement(cv2.MORPH_CROSS, (3, 3)), iterations=4))
        assert np.array_equal(RF.read_mask(planes, size), np.stack(want)), shape


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_reproduces_test_py_front_end(name):
    frames, masks, g = _case(name)
    size = I.target_size(_args(name)) or frames.shape[2:0:-1]
    resized = RF.resize_bicubic(frames, size)
    assert resized.shape == tuple(g["frames_shape"]) and _sha(resized) == str(g["frames_sha256"])
    prepared = RF.read_mask(masks, (resized.shape[2], resized.shape[1]))
    assert prepared.shape == tuple(g["masks_shape"]) and _sha(prepared) == str(g["masks_sha256"])
    _golden_comp(g, resized, prepared)


def test_front_end_abi_rejects_bad_arguments(lib):
    """Validated before any CUDA call."""
    p = 256
    assert lib.e2f_video_resize_bicubic(None, p, p, p, 4, p, 4, 1, 8, 8, 4, 4, None) == -1
    assert b"null" in lib.e2f_last_error()
    assert lib.e2f_video_resize_bicubic(p, None, p, p, 4, p, 4, 1, 8, 8, 4, 4, None) == -1
    assert lib.e2f_video_resize_bicubic(p, p, None, p, 4, p, 4, 1, 8, 8, 4, 4, None) == -1   # both passes need scratch
    assert lib.e2f_video_resize_bicubic(p, p, p, None, 4, p, 4, 1, 8, 8, 4, 4, None) == -1   # width changes, no xtab
    assert lib.e2f_video_resize_bicubic(p, p, p, p, 0, p, 4, 1, 8, 8, 4, 4, None) == -1
    assert lib.e2f_video_resize_bicubic(p, p, p, p, 4, None, 4, 1, 8, 8, 4, 4, None) == -1   # height changes, no ytab
    assert lib.e2f_video_resize_bicubic(p, p, p, p, 4, p, 4, -1, 8, 8, 4, 4, None) == -1
    assert lib.e2f_video_resize_bicubic(p, p, p, p, 4, p, 4, 1, 0, 8, 4, 4, None) == -1
    assert lib.e2f_video_resize_bicubic(p, p, p, p, 4, p, 4, 1, 8, 8, 4, -4, None) == -1
    assert lib.e2f_video_resize_bicubic(p, p, p, p, 4, p, 4, 1, 8, 70000, 4, 4, None) == -1
    assert b"bad shape" in lib.e2f_last_error()
    assert lib.e2f_video_resize_bicubic(p, p, p, p, 4, p, 4, 0, 8, 8, 4, 4, None) == 0        # nothing to do
    assert lib.e2f_video_prepare_masks(None, p, p, p, 1, 8, 8, 4, 4, None) == -1
    assert lib.e2f_video_prepare_masks(p, p, p, None, 1, 8, 8, 4, 4, None) == -1
    assert lib.e2f_video_prepare_masks(p, p, p, p, 1, 0, 8, 4, 4, None) == -1
    assert lib.e2f_video_prepare_masks(p, p, p, p, 1, 8, 8, 4, -1, None) == -1
    assert lib.e2f_video_prepare_masks(p, p, p, p, -1, 8, 8, 4, 4, None) == -1
    assert lib.e2f_video_prepare_masks(p, p, p, p, 0, 8, 8, 4, 4, None) == 0


def test_front_end_wrappers_have_no_cpu_fallback():
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        V.resize_frames(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), (4, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        V.prepare_masks(torch.zeros(1, 8, 8, dtype=torch.uint8), (4, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        V.prepare_inputs(np.zeros((2, 8, 8, 3), np.uint8), np.zeros((2, 8, 8), np.uint8), device="cpu")
    with pytest.raises(IndexError):                 # test.py indexes a mask per frame
        V.prepare_inputs(np.zeros((3, 8, 8, 3), np.uint8), np.zeros((2, 8, 8), np.uint8), device="cpu")
    with pytest.raises(TypeError):
        V.prepare_inputs(np.zeros((2, 8, 8, 3), np.float32), np.zeros((2, 8, 8), np.uint8), device="cpu")


def test_tables_edge_cases():
    assert V.nearest_index(5, 5) == tuple(range(5)) and V.nearest_index(1, 4) == (0, 0, 0, 0)
    assert V.nearest_index(1920, 432)[-1] < 1920
    for a, b in SWEEP:
        tab, taps = V.bicubic_table(a, b)
        assert tab.shape == (b, 2 + taps) and tab.dtype == np.int32
        assert (tab[:, 0] >= 0).all() and (tab[:, 0] + tab[:, 1] <= a).all() and (tab[:, 1] <= taps).all()
    assert V.bicubic_coeffs(1, 7) == ((0, (1 << 22,)),) * 7


def test_command_arguments_size_rule_and_output_name():
    p = I.parser()
    a = p.parse_args(["-v", "data/tennis", "-c", "ck.pth", "-m", "data/tennis_mask", "--model", "e2fgvi"])
    assert (a.step, a.num_ref, a.neighbor_stride, a.savefps, a.set_size) == (10, -1, 5, 24, False)
    assert I.target_size(a) == (432, 240)
    a = p.parse_args(["-v", "x", "-c", "c", "-m", "m", "--model", "e2fgvi", "--set_size", "--width", "9", "--height", "7"])
    assert I.target_size(a) == (432, 240)                          # the base model always runs at 432x240
    a = p.parse_args(["-v", "x", "-c", "c", "-m", "m", "--model", "e2fgvi_hq", "--set_size", "--width", "200",
                      "--height", "100", "--step", "4", "--num_ref", "2", "--neighbor_stride", "3", "--savefps", "10"])
    assert I.target_size(a) == (200, 100) and (a.step, a.num_ref, a.neighbor_stride, a.savefps) == (4, 2, 3, 10)
    a = p.parse_args(["-v", "x", "-c", "c", "-m", "m", "--model", "e2fgvi_hq"])
    assert I.target_size(a) is None
    with pytest.raises(SystemExit):
        p.parse_args(["-v", "x", "-c", "c", "-m", "m", "--model", "e2fgvi_xl"])
    with pytest.raises(SystemExit):
        p.parse_args(["-c", "c", "-m", "m"])
    assert I.output_path("examples/tennis") == os.path.join("results", "tennis_results.mp4")
    assert I.output_path("examples/schoolgirls.mp4") == os.path.join("results", "schoolgirls_results.mp4")
    assert I.output_path("clip") == os.path.join("results", "clip_results.mp4")


# ------------------------------------------------------------------------------------------------------------- GPU
def _close_to_golden(got, g, frames, masks):
    """The bar of test_video_driver_vs_reference_test_py: exact outside the holes, <= 1 LSB, < 5 % of hole pixels off.
    ``frames`` / ``masks`` are the resized frames and dilated masks (equal to the script's, checked by digest)."""
    d = np.abs(got.astype(np.int32) - _golden_comp(g, frames, masks).astype(np.int32))
    hole = np.broadcast_to(masks.astype(bool)[..., None], d.shape)
    assert d[~hole].max() == 0
    assert d.max() <= 1 and (d[hole] > 0).mean() < 0.05, (d.max(), (d[hole] > 0).mean())


@pytest.mark.gpu
def test_resize_kernel_bit_exact_sweep(cuda):
    g = torch.Generator().manual_seed(0)
    for a, b in SWEEP:
        for shape, size in (((2, 7, a, 3), (b, 5)), ((2, a, 7, 3), (5, b)), ((1, 3, a, 3), (b, 3)),
                            ((1, a, 3, 3), (3, b))):
            x = torch.randint(0, 256, shape, dtype=torch.uint8, generator=g)
            got = V.resize_frames(x.to(cuda), size).cpu().numpy()
            assert np.array_equal(got, RF.resize_bicubic(x.numpy(), size)), (shape, size)
    for shape, size in (((3, 1080, 1920, 3), (432, 240)), ((2, 720, 1280, 3), (432, 240)),
                        ((2, 481, 853, 3), (432, 240)), ((2, 100, 200, 3), (432, 240)), ((2, 90, 170, 3), (200, 100)),
                        ((2, 240, 432, 3), (432, 240)), ((1, 2160, 3840, 3), (1920, 1080))):
        x = torch.randint(0, 256, shape, dtype=torch.uint8, generator=g)
        got = V.resize_frames(x.to(cuda), size).cpu().numpy()
        assert np.array_equal(got, RF.resize_bicubic(x.numpy(), size)), (shape, size)
    x = torch.randint(0, 256, (2, 61, 37, 3), dtype=torch.uint8, generator=g)          # rows not 16-byte aligned
    got = V.resize_frames(x.to(cuda)[1:], (33, 100)).cpu().numpy()
    assert np.array_equal(got, RF.resize_bicubic(x[1:].numpy(), (33, 100)))


@pytest.mark.gpu
def test_mask_kernel_bit_exact_sweep(cuda):
    g = torch.Generator().manual_seed(1)
    cases = [((2, 7, a), (b, 5)) for a, b in SWEEP] + [((2, a, 7), (5, b)) for a, b in SWEEP]
    cases += [((3, 1080, 1920), (432, 240)), ((4, 180, 320), (432, 240)), ((2, 75, 130), (200, 100)),
              ((2, 240, 432), (432, 240)), ((1, 1, 1), (1, 1)), ((2, 33, 65), (64, 32))]
    for shape, size in cases:
        m = (torch.rand(shape, generator=g) < 0.01).to(torch.uint8) * torch.randint(1, 256, shape, dtype=torch.uint8,
                                                                                      generator=g)
        m[0, 0, :] = 255                                              # holes touching every border
        m[-1, :, -1] = 1
        m[-1, -1, :1] = 3
        got = V.prepare_masks(m.to(cuda), size).cpu().numpy()
        assert np.array_equal(got, RF.read_mask(m.numpy(), size)), (shape, size)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_prepare_inputs_reproduces_test_py_front_end(cuda, name):
    frames, masks, g = _case(name)
    size = I.target_size(_args(name))
    f, m = V.prepare_inputs(frames, masks, size, device=cuda)
    assert _sha(f.cpu().numpy()) == str(g["frames_sha256"]) and _sha(m.cpu().numpy()) == str(g["masks_sha256"])
    planes = list(masks) + [np.zeros((3, 3), np.uint8)]               # a list of planes; an extra mask is ignored
    f2, m2 = V.prepare_inputs(torch.from_numpy(frames).to(cuda), planes, size)
    assert torch.equal(f2, f) and torch.equal(m2, m)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_driver_fed_by_prepare_inputs_vs_reference_test_py(cuda, name):
    import importlib
    frames, masks, g = _case(name)
    args = _args(name)
    family, wseed = CASES[name][4:6]
    gen = importlib.import_module("e2fgvi_b200.model." + args.model).InpaintGenerator().eval()
    gen.load_state_dict(synth_state_dict(gen, family, wseed), strict=True)
    gen.to(cuda)
    f, m = V.prepare_inputs(frames, masks, I.target_size(args), device=cuda)
    got = V.VideoInpainter(gen, **_driver_kwargs(args))(f, m).cpu().numpy()
    _close_to_golden(got, g, f.cpu().numpy(), m.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_inpaint_command_vs_reference_test_py(cuda, name, tmp_path, monkeypatch):
    """``python -m e2fgvi_b200.inpaint`` on PNG directories, with the video writer captured before the lossy encode."""
    cv2 = pytest.importorskip("cv2")
    pytest.importorskip("PIL.Image")
    import importlib
    frames, masks, g = _case(name)
    model, n = CASES[name][:2]
    family, wseed = CASES[name][4:6]
    (tmp_path / "frames").mkdir()
    (tmp_path / "masks").mkdir()
    for i in range(n):
        cv2.imwrite(str(tmp_path / "frames" / f"{i:05d}.png"), cv2.cvtColor(frames[i], cv2.COLOR_RGB2BGR))
        cv2.imwrite(str(tmp_path / "masks" / f"{i:05d}.png"), masks[i])
    gen = importlib.import_module("e2fgvi_b200.model." + model).InpaintGenerator()
    torch.save(synth_state_dict(gen, family, wseed), str(tmp_path / "ckpt.pth"))
    written = []

    class Recorder:
        def __init__(self, path, fourcc, fps, size):
            written.append((path, fourcc, fps, size))

        def write(self, bgr):
            written.append(cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB))

        def release(self):
            pass
    monkeypatch.setattr(cv2, "VideoWriter", Recorder)
    monkeypatch.chdir(tmp_path)
    extra = CASES[name][8]
    path = I.main(["-v", str(tmp_path / "frames"), "-c", str(tmp_path / "ckpt.pth"), "-m", str(tmp_path / "masks"),
                   "--model", model] + extra)
    assert path == os.path.join("results", "frames_results.mp4") and os.path.isdir(tmp_path / "results")
    (p, fourcc, fps, size), got = written[0], np.stack(written[1:])
    assert (p, fourcc, fps, size) == (path, cv2.VideoWriter_fourcc(*"mp4v"), 24, got.shape[2:0:-1])
    f, m = V.prepare_inputs(frames, masks, I.target_size(_args(name)), device=cuda)
    _close_to_golden(got, g, f.cpu().numpy(), m.cpu().numpy())
