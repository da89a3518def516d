"""CPU: the deformable alignment backward's host side — argument rejections of the sampler-adjoint and scatter entry
points (all made before any CUDA call), the scatter workspace arithmetic, and the wrappers' shape checks, which raise
before anything is launched."""
import pytest
import torch

from e2fgvi_b200 import ops


def _sample(lib, **kw):
    a = dict(x=0x1000, head=0x2000, f1=0x3000, f2=0x4000, da=0x5000, dhead=0x6000, dflow=0x7000, hi=0x8000, lo=0x9000,
             work=0xa000, n=8, h=60, w=108, cin=256, dg=16, res=10.0)
    a.update(kw)
    return lib.e2f_deform_align_backward_sample(a["x"], a["head"], a["f1"], a["f2"], a["da"], a["dhead"], a["dflow"],
                                                a["hi"], a["lo"], a["work"], a["n"], a["h"], a["w"], a["cin"], a["dg"],
                                                a["res"], None)


# every case fails one check, so the fake device addresses are never dereferenced
@pytest.mark.parametrize("kw,status", [
    (dict(x=None), -1), (dict(head=None), -1), (dict(f1=None), -1), (dict(f2=None), -1),
    (dict(dhead=None, dflow=None, hi=None, lo=None, work=None), -1),   # nothing to compute
    (dict(lo=None), -1),                                                # half a split pair
    (dict(da=None), -1),                                                # d head needs dA
    (dict(dhead=None), -1),                                             # d flow goes with d head
    (dict(n=-1), -1), (dict(h=0), -1), (dict(w=0), -1),
    (dict(cin=128), -2), (dict(dg=8), -2), (dict(n=4000, h=60, w=108), -2),   # specialised shape; list too long
    (dict(x=0x1010), -3), (dict(head=0x2008), -3), (dict(f1=0x3004), -3), (dict(da=0x5008), -3),
    (dict(dhead=0x6008), -3), (dict(dflow=0x7008), -3), (dict(hi=0x8008), -3), (dict(work=0xa080), -3),
])
def test_sample_backward_rejects_bad_arguments(lib, kw, status):
    assert _sample(lib, **kw) == status, lib.e2f_last_error()


def _scatter(lib, **kw):
    a = dict(da=0x1000, work=0x2000, dx=0x3000, n=8, h=60, w=108, cin=256, dg=16)
    a.update(kw)
    return lib.e2f_deform_align_backward_scatter(a["da"], a["work"], a["dx"], a["n"], a["h"], a["w"], a["cin"], a["dg"],
                                                 None)


@pytest.mark.parametrize("kw,status", [
    (dict(da=None), -1), (dict(work=None), -1), (dict(dx=None), -1),
    (dict(n=-1), -1), (dict(h=0), -1),
    (dict(cin=512), -2), (dict(dg=1), -2),
    (dict(da=0x1008), -3), (dict(dx=0x3004), -3), (dict(work=0x2010), -3),
])
def test_scatter_backward_rejects_bad_arguments(lib, kw, status):
    assert _scatter(lib, **kw) == status, lib.e2f_last_error()


def test_workspace_arithmetic(lib):
    """L = 576 entries per pixel (144 sample points x 4 corners): keys and source indices twice (the sort's double
    buffers) and one coefficient each, rounded up to 64 words, then L bytes + 64 KB of sort scratch rounded up to 256
    bytes."""
    f = lib.e2f_deform_align_backward_work_elems

    def want(m):
        L = 576 * m
        return (5 * L + 63) // 64 * 64 + (L + 65536 + 255) // 256 * 64
    for n, h, w in [(8, 60, 108), (1, 5, 7), (3, 11, 13), (0, 4, 4)]:
        assert f(n, h, w, 256, 16) == want(n * h * w)
    assert f(8, 60, 108, 256, 16) * 4 < 700 * 2 ** 20        # about 0.6 GB at the training shape
    assert f(-1, 4, 4, 256, 16) == -1
    assert f(1, 4, 4, 128, 16) == -2
    assert f(4000, 60, 108, 256, 16) == -2
    assert ops.deform_align_backward_work_elems(1, 5, 7) == want(35)


def test_wrapper_shape_checks():
    """The wrapper needs CUDA tensors and matching shapes; both are checked before any launch."""
    x = torch.zeros(1, 256, 5, 7)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.deform_align_backward(x, torch.zeros(1, 432, 5, 7), torch.zeros(1, 2, 5, 7), torch.zeros(1, 2, 5, 7),
                                  torch.zeros(128, 2304, dtype=torch.float16), torch.zeros(1, 128, 5, 7))


def test_wrapper_rejects_mismatched_shapes(monkeypatch):
    monkeypatch.setattr(ops, "_need_cuda", lambda *ts: None)
    x = torch.zeros(1, 256, 5, 7)
    good = dict(head=torch.zeros(1, 432, 5, 7), flow_1=torch.zeros(1, 2, 5, 7), flow_2=torch.zeros(1, 2, 5, 7),
                w_packed=torch.zeros(128, 2304, dtype=torch.float16), dy=torch.zeros(1, 128, 5, 7))
    for key, bad in [("head", torch.zeros(1, 431, 5, 7)), ("flow_1", torch.zeros(1, 2, 5, 6)),
                     ("flow_2", torch.zeros(2, 2, 5, 7)), ("dy", torch.zeros(1, 64, 5, 7)),
                     ("w_packed", torch.zeros(128, 2300, dtype=torch.float16))]:
        with pytest.raises(ValueError, match="do not match"):
            ops.deform_align_backward(x, **{**good, key: bad})
    with pytest.raises(ValueError, match="goes with"):
        ops.deform_align_backward(x, **good, need_head=False, need_flow=True)
