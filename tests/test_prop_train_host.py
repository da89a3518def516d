"""CPU: the flow-warp backward's host side — argument rejections of the NHWC and NCHW entry points (all made before any
CUDA call), the scatter workspace arithmetic, the wrapper's shape checks, which raise before anything is launched, and
the tracked propagation's parameter order."""
import pytest
import torch

from e2fgvi_b200 import ops
from e2fgvi_b200.model.modules.feat_prop import BidirectionalPropagation


def _nhwc(lib, **kw):
    a = dict(x=0x1000, flow=0x2000, dout=0x3000, fres=0x4000, dflow=0x5000, res=0x6000, dx=0x7000, work=0x8000, n=8,
             h=60, w=108, c=128)
    a.update(kw)
    return lib.e2f_flow_warp_backward_nhwc(a["x"], a["flow"], a["dout"], a["fres"], a["dflow"], a["res"], a["dx"],
                                           a["work"], a["n"], a["h"], a["w"], a["c"], None)


def _nchw(lib, **kw):
    a = dict(x=0x1000, xbs=8 * 60 * 108, flow=0x2000, dout=0x3000, fres=0x4000, dflow=0x5000, res=0x6000, dx=0x7000,
             work=0x8000, n=8, c=2, h=60, w=108)
    a.update(kw)
    return lib.e2f_flow_warp_backward_nchw(a["x"], a["xbs"], a["flow"], a["dout"], a["fres"], a["dflow"], a["res"],
                                           a["dx"], a["work"], a["n"], a["c"], a["h"], a["w"], None)


# every case fails one check, so the fake device addresses are never dereferenced
_COMMON = [
    (dict(flow=None), -1), (dict(dout=None), -1),
    (dict(dflow=None, fres=None, dx=None, res=None), -1),              # nothing to compute
    (dict(x=None), -1),                                                # d flow reads x
    (dict(work=None), -1),                                             # dx needs the scatter list
    (dict(dflow=None), -1), (dict(dx=None), -1),                       # a residual without its output
    (dict(n=-1), -1), (dict(h=0), -1), (dict(w=0), -1), (dict(c=0), -1),
    (dict(n=200000, h=60, w=108), -2),                                 # N*H*W*4 past int
    (dict(flow=0x2004), -3), (dict(dflow=0x5004), -3), (dict(fres=0x4004), -3), (dict(work=0x8080), -3),
]


@pytest.mark.parametrize("kw,status", _COMMON + [
    (dict(c=130), -2),                                                 # the NHWC kernel takes 4-channel vectors
    (dict(x=0x1008), -3), (dict(dout=0x3008), -3), (dict(dx=0x7008), -3), (dict(res=0x6008), -3),
])
def test_nhwc_backward_rejects_bad_arguments(lib, kw, status):
    assert _nhwc(lib, **kw) == status, lib.e2f_last_error()


@pytest.mark.parametrize("kw,status", _COMMON + [
    (dict(xbs=2 * 60 * 108 - 1), -1),                                  # planes of one image overlap the next
])
def test_nchw_backward_rejects_bad_arguments(lib, kw, status):
    assert _nchw(lib, **kw) == status, lib.e2f_last_error()


def test_workspace_arithmetic(lib):
    """L = 4 entries per pixel (one per corner): keys and source indices twice (the sort's double buffers) and one
    coefficient each, rounded up to 64 words, then L bytes + 64 KB of sort scratch rounded up to 256 bytes — the
    layout the deformable conv's backward uses."""
    f = lib.e2f_flow_warp_backward_work_elems

    def want(m):
        L = 4 * m
        return (5 * L + 63) // 64 * 64 + (L + 65536 + 255) // 256 * 64
    for n, h, w in [(8, 60, 108), (1, 13, 19), (3, 5, 7), (0, 4, 4)]:
        assert f(n, h, w) == want(n * h * w)
    assert f(8, 60, 108) * 4 < 5 * 2 ** 20                # about 4.3 MB at the training shape
    assert f(-1, 4, 4) == -1
    assert f(1, 0, 4) == -1
    assert f(200000, 60, 108) == -2
    assert ops.flow_warp_backward_work_elems(1, 13, 19) == want(13 * 19)


def test_wrapper_needs_cuda():
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.flow_warp_backward(torch.zeros(1, 128, 5, 7), torch.zeros(1, 5, 7, 2), torch.zeros(1, 128, 5, 7))


def test_wrapper_rejects_mismatched_shapes(monkeypatch):
    monkeypatch.setattr(ops, "_need_cuda", lambda *ts: None)
    x, flow, dout = torch.zeros(2, 128, 5, 7), torch.zeros(2, 5, 7, 2), torch.zeros(2, 128, 5, 7)
    for bad in (torch.zeros(2, 5, 7), torch.zeros(1, 5, 7, 2), torch.zeros(2, 5, 6, 2), torch.zeros(2, 2, 5, 7)):
        with pytest.raises(ValueError, match="flow"):
            ops.flow_warp_backward(x, bad, dout)
    with pytest.raises(ValueError, match="dout"):
        ops.flow_warp_backward(x, flow, torch.zeros(2, 64, 5, 7))
    with pytest.raises(ValueError, match="residual"):
        ops.flow_warp_backward(x, flow, dout, residual=torch.zeros(2, 128, 5, 6))
    with pytest.raises(ValueError, match="flow_residual"):
        ops.flow_warp_backward(x, flow, dout, flow_residual=torch.zeros(2, 2, 5, 7))
    with pytest.raises(ValueError, match="nothing"):
        ops.flow_warp_backward(x, flow, dout, need_x=False, need_flow=False)


def test_tracked_parameter_order():
    """The tracked call hands autograd all 30 parameters: per direction the alignment's 10 and the backbone's 4, then
    the fusion's 2."""
    m = BidirectionalPropagation(16)
    ps = m._params()
    assert len(ps) == 30 == len(list(m.parameters()))
    assert {id(p) for p in ps} == {id(p) for p in m.parameters()}
    named = {id(p): k for k, p in m.named_parameters()}
    assert [named[id(p)] for p in ps[10:14]] == [f"backbone.backward_.{k}" for k in ("0.weight", "0.bias", "2.weight",
                                                                                    "2.bias")]
    assert named[id(ps[14])] == "deform_align.forward_.weight"
    assert [named[id(p)] for p in ps[28:]] == ["fusion.weight", "fusion.bias"]

