"""I3D / VFID on the CPU: the state-dict layout against the reference's (golden), the Fréchet distance against the
reference's values, the "same" padding arithmetic and the functional restatement against the reference modules (where
the reference is present), the C-ABI argument checks of the new entry points, and the vfid command's argument and
dataset-layout handling."""
import ctypes
import json
import os
import zipfile

import numpy as np
import pytest
import torch

from e2fgvi_b200 import synth
from e2fgvi_b200 import vfid as V
from e2fgvi_b200.i3d import ENDPOINTS, InceptionI3d, compute_pad, same_pad
from oracle import metrics_loader
from oracle.gen_golden_i3d import ACT_SETS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "i3d_vfid.npz"))

needs_reference = pytest.mark.skipif(not metrics_loader.available(), reason="reference not present")


def test_state_dict_layout_matches_reference():
    sd = InceptionI3d(400, in_channels=3).state_dict()
    assert list(sd) == list(GOLDEN["layout_keys"])
    assert [",".join(map(str, v.shape)) for v in sd.values()] == list(GOLDEN["layout_shapes"])
    assert [str(v.dtype) for v in sd.values()] == list(GOLDEN["layout_dtypes"])
    assert len(sd) == 344
    assert list(GOLDEN["endpoints"]) == list(ENDPOINTS)


def test_strict_load_of_synthetic_state_dict():
    model = InceptionI3d()
    sd = synth.synth_i3d_state_dict(0)
    model.load_state_dict(sd, strict=True)
    assert torch.equal(model.Mixed_4b.b1b.bn.running_var, sd["Mixed_4b.b1b.bn.running_var"])
    assert model.Conv3d_1a_7x7.bn.num_batches_tracked.dtype == torch.int64


def test_unsupported_uses_raise():
    with pytest.raises(NotImplementedError):
        InceptionI3d(final_endpoint="Mixed_4b")
    model = InceptionI3d()
    with pytest.raises(NotImplementedError):
        model(torch.zeros(1, 3, 4, 8, 8))
    with pytest.raises(NotImplementedError):
        model.extract_features(torch.zeros(1, 3, 4, 8, 8), "Mixed_5c")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model.extract_features(torch.zeros(1, 3, 4, 8, 8))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model.features_u8(torch.zeros(4, 8, 8, 3, dtype=torch.uint8))


@pytest.mark.parametrize("tag", sorted(ACT_SETS))
def test_vfid_matches_reference_values(tag):
    n, d = ACT_SETS[tag]
    real, fake = synth.synth_activations(n, d, 1), synth.synth_activations(n, d, 2)
    got = V.calculate_vfid(list(real), list(fake))
    want = float(GOLDEN[f"acts/{tag}"])
    assert abs(got - want) <= 1e-6 * abs(want), (got, want)


def test_frechet_distance_branches():
    mu = np.zeros(3)
    s = np.diag([1.0, 2.0, 3.0])
    assert abs(V.frechet_distance(mu, s, mu, s)) < 1e-12
    assert abs(V.frechet_distance(mu + 1, s, mu, s) - 3.0) < 1e-12
    # sqrt of the product of diag(1, 4) and diag(4, 1) is diag(2, 2): d = 0 + 5 + 5 - 8
    assert abs(V.frechet_distance(np.zeros(2), np.diag([1.0, 4.0]), np.zeros(2), np.diag([4.0, 1.0])) - 2.0) < 1e-12
    with pytest.raises(ValueError):
        V.frechet_distance(np.zeros(2), np.eye(2), np.zeros(3), np.eye(3))
    # a product with a negative eigenvalue has a root with a large imaginary diagonal
    with pytest.raises(ValueError, match="Imaginary"):
        V.frechet_distance(np.zeros(2), np.eye(2), np.zeros(2), np.diag([-1.0, -1.0]))


@needs_reference
def test_padding_arithmetic_matches_reference():
    m = metrics_loader.import_metrics()
    for k, s in ((7, 2), (3, 1), (1, 1), (3, 2), (2, 2)):
        unit = m.Unit3D(4, 8, kernel_shape=[k] * 3, stride=(s,) * 3)
        pool = m.MaxPool3dSamePadding(kernel_size=[k] * 3, stride=(s,) * 3, padding=0)
        for n in range(1, 80):
            p = unit.compute_pad(0, n)
            assert pool.compute_pad(0, n) == p
            assert compute_pad(k, s, n) == (p // 2, p - p // 2)
            pads, out = same_pad((k,) * 3, (s,) * 3, (n, n, n))
            assert out[0] == -(-n // s)


@needs_reference
def test_restatement_matches_reference_modules():
    from oracle import restate_i3d
    m = metrics_loader.import_metrics()
    net = m.InceptionI3d(400, in_channels=3).eval()
    sd = synth.synth_i3d_state_dict(3)
    net.load_state_dict(sd)
    frames, _ = synth.synth_video(5, 37, 53, seed=4)
    x = torch.from_numpy(frames).permute(3, 0, 1, 2).unsqueeze(0).float().div(255)
    eps = {}
    with torch.no_grad():
        got = restate_i3d.extract_features(sd, x, eps)
        y = x
        for name in ENDPOINTS:
            y = net._modules[name](y)
            assert torch.equal(eps[name], y), name
        assert torch.equal(got, net.extract_features(x, "Logits"))


def _pads(*v):
    return (ctypes.c_int * 6)(*v)


def test_argument_errors_i3d_entry_points(lib):
    k3 = (ctypes.c_int * 3)
    p1 = _pads(1, 1, 1, 1, 1, 1)
    ok = [16, 16, 64, 16, 16, 16, 16, None, None, 64, 1, 4, 8, 8, 64, 3, p1, 1, None]
    assert lib.e2f_conv3d_bf16x3(*ok[:-2], 2, None) == -1                       # relu flag
    bad = list(ok)
    bad[0] = None
    assert lib.e2f_conv3d_bf16x3(*bad) == -1
    assert b"null" in lib.e2f_last_error()
    bad = list(ok)
    bad[2] = 12                                                                   # cin % 8
    assert lib.e2f_conv3d_bf16x3(*bad) == -2
    bad = list(ok)
    bad[9] = 32                                                                   # out_cs < cout
    assert lib.e2f_conv3d_bf16x3(*bad) == -2
    bad = list(ok)
    bad[15] = 5                                                                   # ksize
    assert lib.e2f_conv3d_bf16x3(*bad) == -2
    bad = list(ok)
    bad[16] = _pads(3, 0, 1, 1, 1, 1)                                             # pad >= ksize
    assert lib.e2f_conv3d_bf16x3(*bad) == -1
    bad = list(ok)
    bad[6] = 8                                                                    # misaligned fp32 output
    assert lib.e2f_conv3d_bf16x3(*bad) == -3
    assert lib.e2f_i3d_stem_elems(1, 0, 8, 8) == -1
    assert lib.e2f_i3d_stem_elems(1, 3, 60, 108) > 0
    assert lib.e2f_i3d_stem_pack(None, 1, 16, 16, 1, 3, 8, 8, None) == -1
    assert lib.e2f_i3d_stem_pack(16, 2, 16, 16, 1, 3, 8, 8, None) == -1
    assert lib.e2f_i3d_stem_pack(16, 1, 8, 16, 1, 3, 8, 8, None) == -3
    assert lib.e2f_i3d_stem_conv(16, 16, 16, 16, None, 16, None, None, 64, 1, 3, 8, 8, 60, None) == -1   # cout % 8
    assert lib.e2f_i3d_stem_conv(16, 16, 16, 16, None, None, 16, None, 64, 1, 3, 8, 8, 64, None) == -1  # lo missing
    pool = [16, 16, None, None, 1, 3, 8, 8, 64, k3(3, 3, 3), k3(2, 2, 2), _pads(0, 1, 0, 1, 0, 1), None]
    bad = list(pool)
    bad[8] = 6
    assert lib.e2f_maxpool3d(*bad) == -1                                          # c % 4
    bad = list(pool)
    bad[9] = k3(5, 3, 3)
    assert lib.e2f_maxpool3d(*bad) == -2
    bad = list(pool)
    bad[11] = _pads(0, 3, 0, 1, 0, 1)
    assert lib.e2f_maxpool3d(*bad) == -2
    bad = list(pool)
    bad[1] = 8
    assert lib.e2f_maxpool3d(*bad) == -3
    assert lib.e2f_mean_thw(None, 16, 1, 1, 1, 1, 8, None) == -1
    assert lib.e2f_mean_thw(16, 16, 1, 0, 1, 1, 8, None) == -1


# ------------------------------------------------------------------------------------------------- the vfid command
def make_tree(root, videos, size=(60, 108), results_size=(240, 432), drop=None):
    """A tiny dataset tree as TestDataset reads it and a results folder as evaluate.py --save_results writes it.
    ``videos``: name -> frame count.  Returns (data_root, results, {name: (gt RGB, result RGB)})."""
    import cv2
    data = os.path.join(root, "data", "davis")
    os.makedirs(os.path.join(data, "JPEGImages"))
    results = os.path.join(root, "results")
    with open(os.path.join(data, "test.json"), "w") as f:
        json.dump(videos, f)
    frames = {}
    for k, (name, n) in enumerate(videos.items()):
        gt, _ = synth.synth_video(n + 1, *size, seed=10 + k)          # one extra member: only the first n are read
        res, _ = synth.synth_video(n, *results_size, seed=20 + k)
        with zipfile.ZipFile(os.path.join(data, "JPEGImages", f"{name}.zip"), "w") as z:
            for i in reversed(range(n + 1)):                             # stored out of order: readers sort names
                ok, buf = cv2.imencode(".png", cv2.cvtColor(gt[i], cv2.COLOR_RGB2BGR))
                z.writestr(f"{i:05d}.png", buf.tobytes())
        os.makedirs(os.path.join(results, name))
        for i in range(n if drop != name else n - 1):
            cv2.imwrite(os.path.join(results, name, f"{i:05d}.png"), cv2.cvtColor(res[i], cv2.COLOR_RGB2BGR))
        frames[name] = (gt[:n], res)
    return os.path.join(root, "data"), results, frames


def test_command_arguments():
    a = V.parse_args(["--data_root", "R", "--dataset", "youtube-vos", "--results", "D"])
    assert (a.data_root, a.dataset, a.results, a.save_activations) == ("R", "youtube-vos", "D", None)
    with pytest.raises(SystemExit):
        V.parse_args(["--data_root", "R", "--dataset", "kitti", "--results", "D"])
    with pytest.raises(SystemExit):
        V.parse_args(["--dataset", "davis", "--results", "D"])


def test_command_reads_dataset_and_results(tmp_path):
    root, results, frames = make_tree(str(tmp_path), {"cows": 3, "bear": 2})
    gt = V.read_dataset_video(root, "davis", "cows", 3)
    assert np.array_equal(gt, frames["cows"][0])                 # sorted member names, BGR -> RGB
    res = V.read_results(results, "bear", 2)
    assert np.array_equal(res, frames["bear"][1])
    with pytest.raises(ValueError, match="cows"):
        V.read_dataset_video(root, "davis", "cows", 9)
    with pytest.raises(FileNotFoundError, match="goat"):
        V.read_dataset_video(root, "davis", "goat", 1)
    with pytest.raises(FileNotFoundError, match="goat"):
        V.read_results(results, "goat", 1)


def test_command_short_results_folder_names_the_video(tmp_path):
    root, results, _ = make_tree(str(tmp_path), {"cows": 3, "bear": 2}, drop="bear")
    with pytest.raises(FileNotFoundError, match="bear"):
        V.read_results(results, "bear", 2)
