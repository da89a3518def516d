"""I3D / VFID on an H100: the conv3d entry point against fp64 F.conv3d for every Unit3D shape of the network
(channel-slice outputs, odd sizes), the max pool bit for bit, the features and per-endpoint channel means against the
reference's goldens, batch / uint8 consistency, VFID from GPU activations and the vfid command end to end.

VFID bound: the golden clip sets have 6 samples of 1024 dimensions, so both covariances have rank <= 5 and sqrtm works
on a singular product, where a relative perturbation d of the activations moves the root by up to O(sqrt(d)).  The
activations agree to ~1e-5 relative, so the VFID is held to 2e-2 relative; the activation checks are the real gate."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import synth
from e2fgvi_b200 import vfid as V
from e2fgvi_b200.i3d import ENDPOINTS, MIXED, POOLS, InceptionI3d, Unit3D, _Act, same_pad
from oracle import restate_i3d
from oracle.gen_golden_i3d import CASES, CLIP, FAKE_SEEDS, REAL_SEEDS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "i3d_vfid.npz"))

# every distinct (cin, cout, k) Unit3D of the network (the stem has its own test)
SHAPES = sorted({(64, 64, 1), (64, 192, 3)} | {
    s for _, cin, c in MIXED for s in ((cin, c[0], 1), (cin, c[1], 1), (c[1], c[2], 3), (cin, c[3], 1), (c[3], c[4], 3),
                                        (cin, c[5], 1))})


@pytest.fixture(scope="module")
def model(cuda):
    m = InceptionI3d()
    m.load_state_dict(synth.synth_i3d_state_dict(0))
    return m.to(cuda).eval()


def _video(t, h, w, seed):
    frames, _ = synth.synth_video(t, h, w, seed=seed)
    return frames, torch.from_numpy(frames).permute(3, 0, 1, 2).unsqueeze(0).contiguous().float().div(255)


def _unit(cin, cout, k, seed):
    u = Unit3D(cin, cout, (k,) * 3)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        u.conv3d.weight.normal_(0, (2.0 / (cin * k ** 3)) ** 0.5, generator=g)
        u.bn.weight.copy_(1 + 0.1 * torch.randn(cout, generator=g))
        u.bn.bias.copy_(0.1 * torch.randn(cout, generator=g))
        u.bn.running_mean.copy_(0.1 * torch.randn(cout, generator=g))
        u.bn.running_var.copy_(1 + 0.3 * torch.rand(cout, generator=g))
    return u


@pytest.mark.parametrize("cin,cout,k", SHAPES)
def test_conv3d_matches_fp64(cuda, cin, cout, k):
    from e2fgvi_b200 import ops
    torch.manual_seed(cin * 7 + cout + k)
    b, size = 2, (5, 11, 19)                                      # odd sizes, partial tiles
    u = _unit(cin, cout, k, cin + cout).to(cuda).eval()
    x = torch.randn((b,) + size + (cin,), device=cuda).relu_()
    hi, lo = ops.split_bf16(x)
    xa = _Act(None, hi, lo, size, cin)
    coff, wide = 8, cout + 24                                     # a channel slice of a wider output
    out = InceptionI3d._alloc(b, size, wide, cuda)
    out.f32.fill_(7.0)
    InceptionI3d()._conv(u, xa, b, out, coff)
    pads, _ = same_pad((k,) * 3, (1, 1, 1), size)
    x64 = F.pad(x.permute(0, 4, 1, 2, 3).double(), [pads[4], pads[5], pads[2], pads[3], pads[0], pads[1]])
    y = F.conv3d(x64, u.conv3d.weight.double())
    y = F.batch_norm(y, u.bn.running_mean.double(), u.bn.running_var.double(), u.bn.weight.double(),
                     u.bn.bias.double(), False, 0.0, 1e-3).relu().permute(0, 2, 3, 4, 1)
    got = out.f32[..., coff:coff + cout].double()
    bound = 1e-4 * y.abs().max().item()
    assert (got - y).abs().max().item() <= bound
    split = out.hi[..., coff:coff + cout].double() + out.lo[..., coff:coff + cout].double()
    assert (split - y).abs().max().item() <= bound
    assert torch.all(out.f32[..., :coff] == 7.0) and torch.all(out.f32[..., coff + cout:] == 7.0)


@pytest.mark.parametrize("name", sorted(POOLS) + ["b3a"])
@pytest.mark.parametrize("size", [(5, 11, 19), (4, 12, 18), (1, 3, 2)])
def test_maxpool_bit_exact(cuda, name, size):
    from e2fgvi_b200 import ops
    from e2fgvi_b200.i3d import _ints
    from e2fgvi_b200 import _lib
    k, s = POOLS[name] if name in POOLS else ((3, 3, 3), (1, 1, 1))
    b, c = 2, 24
    torch.manual_seed(sum(size))
    x = torch.randn((b,) + size + (c,), device=cuda) - 0.5       # mostly negative: the zero padding shows
    pads, osz = same_pad(k, s, size)
    out = torch.empty((b,) + osz + (c,), device=cuda)
    hi = torch.empty_like(out, dtype=torch.bfloat16)
    lo = torch.empty_like(out, dtype=torch.bfloat16)
    st = _lib.load().e2f_maxpool3d(x.data_ptr(), out.data_ptr(), hi.data_ptr(), lo.data_ptr(), b, *size, c, _ints(k),
                                   _ints(s), _ints(pads), ops._stream())
    _lib.check(st, "e2f_maxpool3d")
    want = restate_i3d.max_pool(x.permute(0, 4, 1, 2, 3), k, s).permute(0, 2, 3, 4, 1)
    assert torch.equal(out, want)
    h2, l2 = ops.split_bf16(want.contiguous())
    assert torch.equal(hi, h2) and torch.equal(lo, l2)


@pytest.mark.parametrize("case", sorted(CASES))
def test_features_match_reference_goldens(model, case):
    t, h, w, seed = CASES[case]
    _, x = _video(t, h, w, seed)
    eps = {}
    feats = model._run(x.cuda(), 0, 1, t, h, w, eps)
    want = GOLDEN[f"{case}/features"]
    got = feats.cpu().numpy()
    assert np.abs(got - want).max() <= 1e-3 * max(1.0, np.abs(want).max())
    for name in ENDPOINTS:
        m = eps[name].mean(dim=(1, 2, 3)).cpu().numpy()
        r = GOLDEN[f"{case}/mean/{name}"]
        assert np.abs(m - r).max() <= 1e-3 * max(1.0, np.abs(r).max()), name


def test_stem_and_endpoints_match_restatement(model, cuda):
    """Layer by layer on odd sizes, against the fp64 restatement on the GPU."""
    t, h, w = 9, 47, 83
    _, x = _video(t, h, w, 11)
    eps = {}
    model._run(x.cuda(), 0, 1, t, h, w, eps)
    sd = {k: (v.double() if v.is_floating_point() else v) for k, v in model.state_dict().items()}
    ref = {}
    restate_i3d.extract_features(sd, x.cuda().double(), ref)
    for name in ENDPOINTS:
        r = ref[name].permute(0, 2, 3, 4, 1)
        assert tuple(eps[name].shape) == tuple(r.shape), name
        err = (eps[name].double() - r).abs().max().item()
        assert err <= 1e-3 * max(1.0, r.abs().max().item()), (name, err)


def test_batch_and_uint8_paths_bit_identical(model):
    t, h, w = 6, 60, 108
    fa, xa = _video(t, h, w, 5)
    fb, xb = _video(t, h, w, 6)
    single_a = model.extract_features(xa.cuda())
    single_b = model.extract_features(xb.cuda())
    both = model.extract_features(torch.cat([xa, xb]).cuda())
    assert torch.equal(both[0], single_a[0]) and torch.equal(both[1], single_b[0])
    u8 = model.features_u8(torch.from_numpy(np.stack([fa, fb])).cuda())
    assert torch.equal(u8, both)
    assert torch.equal(model.features_u8(torch.from_numpy(fa).cuda()), single_a)


def test_weight_cache_follows_parameters(cuda):
    m = InceptionI3d()
    m.load_state_dict(synth.synth_i3d_state_dict(0))
    m = m.to(cuda).eval()
    _, x = _video(3, 30, 54, 7)
    f0 = m.extract_features(x.cuda())
    with torch.no_grad():
        m.Mixed_5c.b0.bn.weight.mul_(2.0)                         # bumps the version: the folded operands are rebuilt
    f1 = m.extract_features(x.cuda())
    assert not torch.equal(f0, f1)
    m.load_state_dict(synth.synth_i3d_state_dict(0))
    assert torch.equal(m.extract_features(x.cuda()), f0)


def test_vfid_from_gpu_activations(model):
    acts = {}
    for tag, seeds in (("real", REAL_SEEDS), ("fake", FAKE_SEEDS)):
        frames = np.stack([synth.synth_video(*CLIP, seed=s)[0] for s in seeds])
        acts[tag] = model.features_u8(torch.from_numpy(frames).cuda()).cpu().numpy()
        want = GOLDEN[f"clips/{tag}"]
        assert np.abs(acts[tag] - want).max() <= 1e-3 * max(1.0, np.abs(want).max())
    got = V.calculate_vfid(list(acts["real"]), list(acts["fake"]))
    want = float(GOLDEN["clips/vfid"])
    assert abs(got - want) <= 2e-2 * abs(want), (got, want)


def test_calculate_i3d_activations_dropin(model):
    from PIL import Image
    fa, _ = synth.synth_video(4, 60, 108, seed=8)
    fb, _ = synth.synth_video(4, 60, 108, seed=9)
    a, b = V.calculate_i3d_activations([Image.fromarray(f) for f in fa], [Image.fromarray(f) for f in fb], model, "cuda:0")
    assert a.shape == (1024,) and b.shape == (1024,)
    assert np.array_equal(a, model.features_u8(torch.from_numpy(fa).cuda()).cpu().numpy().flatten())
    c, _ = V.calculate_i3d_activations([Image.fromarray(f) for f in fa], [Image.fromarray(f) for f in fb[:3]], model,
                                       "cuda:0")
    assert np.array_equal(a, c)


def test_command_end_to_end(model, tmp_path, capsys):
    from test_i3d_host import make_tree
    from e2fgvi_b200.video import resize_frames
    root, results, frames = make_tree(str(tmp_path), {"cows": 4, "bear": 3})
    acts = str(tmp_path / "acts")
    score = V.main(["--data_root", root, "--dataset", "davis", "--results", results, "--save_activations", acts],
                   model=model)
    real, fake = [], []
    for name, (gt, res) in frames.items():
        g = resize_frames(torch.from_numpy(gt).cuda(), (432, 240))
        real.append(model.features_u8(g).cpu().numpy().flatten())
        fake.append(model.features_u8(torch.from_numpy(res).cuda()).cpu().numpy().flatten())
    assert np.array_equal(np.load(os.path.join(acts, "real.npy")), np.stack(real))
    assert np.array_equal(np.load(os.path.join(acts, "fake.npy")), np.stack(fake))
    assert score == V.calculate_vfid(real, fake)
    assert f"VFID: {score:.3f}" in capsys.readouterr().out
