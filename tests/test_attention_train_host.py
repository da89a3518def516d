"""CPU: the focal attention backward's host side — argument rejections of its C entry points (all made before any CUDA
call), its gather lists against a pure-torch enumeration of the reference's key list, and its workspace arithmetic."""
from collections import Counter

import pytest
import torch
import torch.nn.functional as F

from e2fgvi_b200 import ops
from e2fgvi_b200.model.modules.tfocal_transformer import rolled_valid_indices

WIN, EXP, FOC = (5, 9), (2, 4), (5, 9)


def _bwd(lib, **kw):
    a = dict(qkv=0x1000, pooled=0x2000, dout=0x3000, dqkv=0x4000, dpooled=0x5000, work=0x6000, b=1, t=2, h=20, w=36,
             heads=4, hd=128, wh=5, ww=9, eh=2, ew=4, fh=5, fw=9, use_pooled=1, scale=128 ** -0.5)
    a.update(kw)
    return lib.e2f_focal_window_attention_backward(a["qkv"], a["pooled"], a["dout"], a["dqkv"], a["dpooled"], a["work"],
                                                   a["b"], a["t"], a["h"], a["w"], a["heads"], a["hd"], a["wh"], a["ww"],
                                                   a["eh"], a["ew"], a["fh"], a["fw"], a["use_pooled"], a["scale"], None)


# every case fails one check, so the fake device addresses are never dereferenced
@pytest.mark.parametrize("kw,status", [
    (dict(qkv=None), -1), (dict(dout=None), -1), (dict(dqkv=None), -1), (dict(work=None), -1),
    (dict(pooled=None), -1), (dict(dpooled=None), -1),
    (dict(hd=64), -2),                                    # heads x 128 must be C
    (dict(h=21), -1), (dict(w=35), -1),                   # grid not a multiple of the window
    (dict(fh=4), -1), (dict(fw=8), -1),                   # even focal sizes
    (dict(use_pooled=2), -1), (dict(t=0), -1), (dict(b=-1), -1), (dict(scale=0.0), -1),
    (dict(qkv=0x1008), -3), (dict(dout=0x3004), -3), (dict(dqkv=0x4008), -3), (dict(work=0x6004), -3),
    (dict(dpooled=0x5008), -3),
])
def test_backward_rejects_bad_arguments(lib, kw, status):
    assert _bwd(lib, **kw) == status, lib.e2f_last_error()


def test_work_elems_rejects_bad_geometry(lib):
    f = lib.e2f_focal_window_attention_backward_work_elems
    assert f(1, 2, 20, 36, 4, 128, 5, 9, 2, 4, 5, 9, 1) > 0
    assert f(1, 2, 20, 36, 4, 64, 5, 9, 2, 4, 5, 9, 1) == -2
    assert f(1, 2, 21, 36, 4, 128, 5, 9, 2, 4, 5, 9, 1) == -1
    assert f(1, 2, 20, 36, 4, 128, 5, 9, 2, 4, 4, 9, 1) == -1
    with pytest.raises(ValueError):
        ops.focal_attention_key_sources(2, (20, 36), WIN, EXP, FOC, True, 2, False, 0, 0)     # frame out of range
    with pytest.raises(ValueError):
        ops.focal_attention_key_sources(2, (20, 36), WIN, EXP, FOC, False, 0, True, 0, 0)     # no pooled keys


def _partition(ids, ws):
    H, W = ids.shape
    return ids.view(H // ws[0], ws[0], W // ws[1], ws[1]).permute(0, 2, 1, 3).reshape(-1, ws[0] * ws[1])


def reference_key_lists(H, W, use_pooled):
    """Per window, the key tokens of one frame as tfocal_transformer.py lists them: own window, the four rolled windows
    filtered by valid_ind_rolled, the unfolded pooled windows (zero padding dropped).  Token ids: y * W + x; pooled
    tokens: ('p', pi, pj)."""
    ids = torch.arange(H * W).view(H, W)
    eh, ew = EXP
    parts = [_partition(torch.roll(ids, shifts=s, dims=(0, 1)), WIN) for s in ((-eh, -ew), (-eh, ew), (eh, -ew), (eh, ew))]
    rolled = torch.cat(parts, 1)[:, rolled_valid_indices(WIN, EXP)]
    own = _partition(ids, WIN)
    lists = [[("t", int(i) // W, int(i) % W) for i in torch.cat([own[w], rolled[w]])] for w in range(own.shape[0])]
    if use_pooled:
        nWh, nWw = H // WIN[0], W // WIN[1]
        pid = (torch.arange(nWh * nWw) + 1).double().view(1, 1, nWh, nWw)
        u = F.unfold(pid, FOC, padding=(FOC[0] // 2, FOC[1] // 2)).view(FOC[0] * FOC[1], -1).t().long()
        for w in range(u.shape[0]):
            lists[w] += [("p", (int(i) - 1) // nWw, (int(i) - 1) % nWw) for i in u[w] if i > 0]
    return lists


# the training grid, a one-window grid (rolls wrap onto the window itself), 10x18 and 15x27 (pooled grids smaller than
# the 5x9 neighbourhood), an HQ-style grid
GRIDS = [(20, 36), (5, 9), (10, 18), (15, 27), (40, 72)]


@pytest.mark.parametrize("use_pooled", [True, False])
@pytest.mark.parametrize("H,W", GRIDS)
def test_gather_lists_match_reference_key_lists(lib, H, W, use_pooled):
    """Every (query window, key token) pair appears exactly as often as the reference lists it (as the sum of the
    multiplicities of its gather entries), and every (window, key slot) of two frames belongs to one token only."""
    ref = reference_key_lists(H, W, use_pooled)
    want = Counter((w, tok) for w, keys in enumerate(ref) for tok in keys)
    got = Counter()
    owner = {}
    T = 2
    nWh, nWw = H // WIN[0], W // WIN[1]
    tokens = [("t", y, x) for y in range(H) for x in range(W)]
    if use_pooled:
        tokens += [("p", i, j) for i in range(nWh) for j in range(nWw)]
    for t in range(T):
        for tok in tokens:
            for w, slot, m in ops.focal_attention_key_sources(T, (H, W), WIN, EXP, FOC, use_pooled, t, tok[0] == "p",
                                                              tok[1], tok[2]):
                assert m >= 1
                assert owner.setdefault((w, slot), (t, tok)) == (t, tok), (w, slot)
                if t == 0:
                    got[(w, tok)] += m
    assert got == want
    # each window's slots are exactly 0 .. NK - 1, NK = its listed distinct keys over both frames
    for w in range(nWh * nWw):
        slots = sorted(s for (ww_, s) in owner if ww_ == w)
        assert slots == list(range(len(slots)))


def _ring_positions():
    """n1 + n2: the expanded-window positions the reference lists (distinct tokens of an interior window's ring)."""
    ref = reference_key_lists(20, 36, False)
    return len(set(ref[5]))


@pytest.mark.parametrize("b,t,h,w,heads,use_pooled", [(8, 8, 20, 36, 4, 1), (1, 1, 5, 9, 4, 1), (2, 8, 10, 18, 4, 0),
                                                      (3, 2, 40, 72, 4, 1)])
def test_workspace_arithmetic(lib, b, t, h, w, heads, use_pooled):
    """Row statistics (log2-sum-exp, D) per query row and head, plus per-(window, key slot) dK | dV partials and eight
    per-window dQ partials for as many (clip, head) pairs as fit in 32M floats (at least one)."""
    got = lib.e2f_focal_window_attention_backward_work_elems(b, t, h, w, heads, 128, 5, 9, 2, 4, 5, 9, use_pooled)
    nW = (h // 5) * (w // 9)
    stats = -(-(b * nW * heads * t * 45 * 2) // 4) * 4
    nks = t * (_ring_positions() + (45 if use_pooled else 0))
    unit = nW * (nks * 256 + 8 * t * 45 * 128)
    chunk = max(1, min(b * heads, (32 << 20) // unit))
    assert got == stats + chunk * unit
    if (b, t, h, w) == (8, 8, 20, 36):
        # the training shape: 49 MB of partials per (clip, head), two per chunk; qkv alone is 141 MB
        assert chunk == 2 and got * 4 < 100 << 20
