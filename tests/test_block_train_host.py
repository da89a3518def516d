"""CPU: the transformer block backward's host side — argument rejections of the LayerNorm and LayerNorm + pooling
backward entry points (all made before any CUDA call), their partial-row workspace arithmetic, and the wrappers' shape
checks, which raise before anything is allocated."""
import pytest
import torch

from e2fgvi_b200 import ops


def _ln(lib, **kw):
    a = dict(x=0x1000, dy=0x2000, gamma=0x3000, res=0x4000, dx=0x5000, hi=0x6000, lo=0x7000, dg=0x8000, db=0x9000,
             work=0xa000, rows=46080, c=512, eps=1e-5)
    a.update(kw)
    return lib.e2f_layernorm_backward(a["x"], a["dy"], a["gamma"], a["res"], a["dx"], a["hi"], a["lo"], a["dg"], a["db"],
                                      a["work"], a["rows"], a["c"], a["eps"], None)


# every case fails one check, so the fake device addresses are never dereferenced
@pytest.mark.parametrize("kw,status", [
    (dict(x=None), -1), (dict(dy=None), -1), (dict(gamma=None), -1),
    (dict(dx=None, hi=None, lo=None, dg=None, db=None), -1),    # no output at all
    (dict(lo=None), -1),                                         # half a split pair
    (dict(work=None), -1),                                       # parameter gradients need the workspace
    (dict(rows=-1), -1), (dict(c=0), -1),
    (dict(c=256), -2), (dict(c=768), -2),                       # specialised for 512 channels
    (dict(x=0x1004), -3), (dict(dy=0x2008), -3), (dict(res=0x4004), -3), (dict(dx=0x5004), -3),
    (dict(hi=0x6008), -3), (dict(work=0xa004), -3),
])
def test_layernorm_backward_rejects_bad_arguments(lib, kw, status):
    assert _ln(lib, **kw) == status, lib.e2f_last_error()


def _pool(lib, **kw):
    a = dict(x=0x1000, gamma=0x2000, beta=0x3000, pw=0x4000, drows=0x5000, dx1=0x6000, dx=0x7000, dg=0x8000,
             db=0x9000, dpw=0xa000, dpb=0xb000, work=0xc000, bt=8, h=20, w=36, c=512, wh=5, ww=9, eps=1e-5)
    a.update(kw)
    return lib.e2f_layernorm_pool_backward(a["x"], a["gamma"], a["beta"], a["pw"], a["drows"], a["dx1"], a["dx"], a["dg"],
                                           a["db"], a["dpw"], a["dpb"], a["work"], a["bt"], a["h"], a["w"], a["c"],
                                           a["wh"], a["ww"], a["eps"], None)


@pytest.mark.parametrize("kw,status", [
    (dict(x=None), -1), (dict(gamma=None), -1), (dict(beta=None), -1), (dict(pw=None), -1), (dict(drows=None), -1),
    (dict(dx1=None), -1),                                        # dx needs dx1
    (dict(dx=None, dg=None, db=None, dpw=None, dpb=None), -1),   # no output at all
    (dict(work=None), -1),
    (dict(h=21), -1), (dict(w=35), -1),                          # grid not a multiple of the window
    (dict(bt=-1), -1), (dict(h=0), -1), (dict(wh=0), -1), (dict(c=-512), -1),
    (dict(c=256), -2), (dict(bt=65536), -2),
    (dict(x=0x1004), -3), (dict(drows=0x5008), -3), (dict(dx1=0x6004), -3), (dict(dx=0x7004), -3),
    (dict(work=0xc008), -3),
])
def test_layernorm_pool_backward_rejects_bad_arguments(lib, kw, status):
    assert _pool(lib, **kw) == status, lib.e2f_last_error()


def test_workspace_arithmetic(lib):
    """One partial row of (dgamma | dbeta) per 64 rows; one row of (dgamma | dbeta | d w_pool | d b_pool) per
    (frame, window)."""
    f = lib.e2f_layernorm_backward_work_elems
    for rows in (1, 3, 63, 64, 65, 46080, 46081):
        assert f(rows, 512) == (rows + 63) // 64 * 1024, rows
    assert f(0, 512) == 0
    assert f(-1, 512) == -1 and f(64, 256) == -2
    g = lib.e2f_layernorm_pool_backward_work_elems
    for bt, h, w in ((64, 20, 36), (1, 5, 9), (8, 40, 72), (3, 10, 18)):
        assert g(bt, h, w, 512, 5, 9) == bt * (h // 5) * (w // 9) * (1024 + 45 + 1), (bt, h, w)
    assert g(1, 21, 36, 512, 5, 9) == -1 and g(1, 20, 36, 384, 5, 9) == -2


def test_wrappers_check_shapes_before_allocating():
    x = torch.zeros(2, 512)
    w = torch.ones(512)
    with pytest.raises(ValueError, match="dy"):
        ops.layer_norm_backward(x, torch.zeros(3, 512), w)
    with pytest.raises(ValueError, match="residual"):
        ops.layer_norm_backward(x, x, w, residual=torch.zeros(2, 256))
    with pytest.raises(ValueError, match="512"):
        ops.layer_norm_backward(torch.zeros(2, 256), torch.zeros(2, 256), torch.ones(256))
    with pytest.raises(ValueError, match="nothing"):
        ops.layer_norm_backward(x, x, w, out=None, need_weight=False, need_bias=False)
    xb = torch.zeros(1, 2, 5, 9, 512)
    rows = torch.zeros(2 * 45 + 2, 512)
    pw = torch.zeros(1, 45)
    with pytest.raises(ValueError, match="multiple of the window"):
        ops.layer_norm_pool_backward(torch.zeros(1, 2, 6, 9, 512), rows, xb, w, w, 1e-5, pw, (5, 9))
    with pytest.raises(ValueError, match="drows"):
        ops.layer_norm_pool_backward(xb, rows[:-1], xb, w, w, 1e-5, pw, (5, 9))
    with pytest.raises(ValueError, match="pool weight"):
        ops.layer_norm_pool_backward(xb, rows, xb, w, w, 1e-5, torch.zeros(1, 44), (5, 9))
    with pytest.raises(ValueError, match="dx1"):
        ops.layer_norm_pool_backward(xb, rows, None, w, w, 1e-5, pw, (5, 9))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.layer_norm_pool_backward(xb, rows, xb, w, w, 1e-5, pw, (5, 9))
