"""Operator-level mirror of the three reference boundaries the CUDA kernels sit behind (SURVEY §8(b)):

* ``flow_warp``                   — model/modules/flow_comp.py:345-383
* ``modulated_deform_conv2d``     — mmcv.ops.modulated_deform_conv2d as called at model/modules/feat_prop.py:55-58
* ``deform_align_fused``          — the tail of SecondOrderDeformableAlignment.forward, feat_prop.py:41-58
* ``focal_window_attention``      — WindowAttention.forward between qkv and proj, tfocal_transformer.py:226-396

Same names / argument meaning / error behaviour as the reference operators; every call goes through the C ABI of
``libe2fgvi_b200.so`` on the current CUDA stream.  There is no CPU path: CPU tensors raise.
"""
import ctypes
import weakref

import torch

from . import _lib

_PAD = {"zeros": 0, "border": 1}
_DT = {torch.float32: 0, torch.float16: 1}


def _stream():
    return torch.cuda.current_stream().cuda_stream


# Optional live kernel timing for bench.py's roofline block: name -> [(start_event, end_event, work)], recorded on
# the launching stream around the C-ABI call (the call is one kernel launch).
_PROFILE = None


def profile_kernels(enable=True):
    """Start (returns the live dict) or stop (enable=False) recording CUDA events around kernel launches."""
    global _PROFILE
    _PROFILE = {} if enable else None
    return _PROFILE


class _timed:
    def __init__(self, name, work=0.0):
        self.name, self.work = name, work

    def __enter__(self):
        if _PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if _PROFILE is not None:
            self.e1.record()
            _PROFILE.setdefault(self.name, []).append((self.e0, self.e1, self.work))
        return False


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("e2fgvi_b200 kernels need CUDA tensors on an H100 (sm_90a); there is no CPU fallback")


def _is_cl(x):
    """True if the 4-D tensor is dense NHWC in memory (channels_last or a permuted NHWC view)."""
    n, c, h, w = x.shape
    return x.stride() == (h * w * c, 1, w * c, c)


def flow_warp(x, flow, interpolation="bilinear", padding_mode="zeros", align_corners=True):
    """Warp ``x`` (n,c,h,w) with ``flow`` (n,h,w,2; pixel units, [...,0] = x-displacement).

    Mirrors flow_comp.py:345-383, including the ValueError on a spatial mismatch (:364-366).  Output keeps the
    memory format of ``x`` (NCHW-contiguous or channels_last) and its dtype (fp32 / fp16).
    """
    if x.size()[-2:] != flow.size()[1:3]:
        raise ValueError(f"The spatial sizes of input ({x.size()[-2:]}) and "
                         f"flow ({flow.size()[1:3]}) are not the same.")
    if interpolation != "bilinear" or not align_corners:
        raise NotImplementedError("only bilinear / align_corners=True is on the E2FGVI path")
    if padding_mode not in _PAD:
        raise NotImplementedError(f"padding_mode={padding_mode!r} is not on the E2FGVI path")
    _need_cuda(x, flow)
    lib = _lib.load()
    n, c, h, w = x.shape
    flow = flow.contiguous().float()
    vec = 8 if x.dtype == torch.float16 else 4
    if x.dtype in _DT and _is_cl(x) and c % vec == 0:
        out = torch.empty_like(x)  # preserves strides (dense)
        st = lib.e2f_flow_warp(x.data_ptr(), flow.data_ptr(), out.data_ptr(), n, h, w, c, _DT[x.dtype],
                               _PAD[padding_mode], _stream())
        _lib.check(st, "e2f_flow_warp")
        return out
    xc = x.contiguous()
    if xc.dtype != torch.float32:
        xc = xc.float()
    out = torch.empty_like(xc)
    st = lib.e2f_flow_warp_nchw(xc.data_ptr(), flow.data_ptr(), out.data_ptr(), n, c, h, w, _PAD[padding_mode],
                                _stream())
    _lib.check(st, "e2f_flow_warp_nchw")
    return out if out.dtype == x.dtype else out.to(x.dtype)


def pack_dcn_weight(weight, deform_groups):
    """fp32 [Cout,Cin,3,3] -> fp16 [Cout, 9*Cin] GEMM operand in sampler K-order (k = (g*9+tap)*cpg + c).

    Not cached here; ``SecondOrderDeformableAlignment.packed_weight`` caches it per parameter (``_derived_one``)."""
    _need_cuda(weight)
    cout, cin, kh, kw = weight.shape
    if (kh, kw) != (3, 3):
        raise ValueError("only 3x3 deformable kernels are on the E2FGVI path")
    w32 = weight.detach().contiguous().float()
    packed = torch.empty(cout, 9 * cin, dtype=torch.float16, device=weight.device)
    st = _lib.load().e2f_dcn_pack_weight(w32.data_ptr(), packed.data_ptr(), cout, cin, deform_groups, _stream())
    _lib.check(st, "e2f_dcn_pack_weight")
    return packed


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def _square(kernel_size, stride, padding):
    """(k, s, p) of a square kernel / stride / padding given as ints or pairs."""
    (k, k2), (s, s2), (p, p2) = _pair(kernel_size), _pair(stride), _pair(padding)
    if k != k2 or s != s2 or p != p2:
        raise NotImplementedError("square kernel / stride / padding only (E2FGVI uses 7 / 3 / 3)")
    return k, s, p


def _outputs(out, modes, shape, device, into=None):
    """Check ``out`` against the ``modes`` a wrapper accepts, then return its (fp32, bf16 hi, bf16 lo) output buffers
    of ``shape``: fp32 for "f32" / "both", the split pair for "split" / "both", None for what is not asked for (a
    "rows" pair comes from ``_rows_pair``).  ``into`` = (o32, hi, lo): existing buffers to return instead of new ones."""
    if out not in modes:
        raise ValueError(f"out must be one of {', '.join(map(repr, modes))}, got {out!r}")
    f32, split = out in ("f32", "both"), out in ("split", "both")
    if into is not None:
        o32, hi, lo = into
        if (f32 and o32 is None) or (split and (hi is None or lo is None)):
            raise ValueError("`into` lacks a buffer for the requested output")
        return (o32 if f32 else None), (hi if split else None), (lo if split else None)
    return (torch.empty(shape, dtype=torch.float32, device=device) if f32 else None,
            torch.empty(shape, dtype=torch.bfloat16, device=device) if split else None,
            torch.empty(shape, dtype=torch.bfloat16, device=device) if split else None)


def _result(out, t32, sp):
    """What a wrapper with "f32" / "split" / "both" modes returns: the fp32 tensor, the split operand, or both."""
    return t32 if out == "f32" else sp if out == "split" else (t32, sp)


def modulated_deform_conv2d(x, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                            deform_groups=1, out_dtype=torch.float32):
    """Drop-in for ``mmcv.ops.modulated_deform_conv2d`` (call site feat_prop.py:55-58).

    x (n,cin,h,w), offset (n,2*9*dg,h,w) with channel (g*9+tap)*2+{dy,dx}, mask (n,9*dg,h,w), weight
    (cout,cin,3,3).  Returns (n,cout,h,w) in channels_last memory format.
    """
    if _pair(stride) != (1, 1) or _pair(padding) != (1, 1) or _pair(dilation) != (1, 1) or groups != 1:
        raise NotImplementedError("E2FGVI uses 3x3 / stride 1 / padding 1 / dilation 1 / groups 1 only")
    _need_cuda(x, offset, mask, weight, bias)
    n, cin, h, w = x.shape
    cout = weight.shape[0]
    if offset.shape != (n, 18 * deform_groups, h, w) or mask.shape != (n, 9 * deform_groups, h, w):
        raise ValueError(f"offset/mask shapes {tuple(offset.shape)}/{tuple(mask.shape)} do not match x {tuple(x.shape)}")
    wp = pack_dcn_weight(weight, deform_groups)
    x_cl = x.to(dtype=torch.float16, memory_format=torch.channels_last)
    off_cl = offset.to(dtype=torch.float32, memory_format=torch.channels_last)
    msk_cl = mask.to(dtype=torch.float32, memory_format=torch.channels_last)
    b32 = None if bias is None else bias.detach().float().contiguous()
    out = torch.empty((n, cout, h, w), dtype=out_dtype, device=x.device, memory_format=torch.channels_last)
    st = _lib.load().e2f_modulated_deform_conv2d(
        x_cl.data_ptr(), off_cl.data_ptr(), msk_cl.data_ptr(), wp.data_ptr(),
        None if b32 is None else b32.data_ptr(), out.data_ptr(), n, h, w, cin, cout, deform_groups,
        _DT[out_dtype], 0, _stream())
    _lib.check(st, "e2f_modulated_deform_conv2d")
    return out


class GroupedX:
    """DCN input in the group-major fp16 layout [N][G][H][W][16] (see ``dcn_pack_input``)."""

    __slots__ = ("data", "shape")

    def __init__(self, data, shape):
        self.data, self.shape = data, shape       # shape: logical (N, Cin, H, W)


def dcn_pack_input(a, b):
    """``torch.cat([a, b], 1)`` (feat_prop.py:126) converted to fp16 in the group-major layout the deformable sampler
    reads best (adjacent bilinear corners contiguous).  a, b: (N,C,H,W) fp32, C % 16 == 0 -> ``GroupedX``."""
    _need_cuda(a, b)
    n, ca, h, w = a.shape
    cb = b.shape[1]
    a_cl = a.permute(0, 2, 3, 1).contiguous().float()
    b_cl = b.permute(0, 2, 3, 1).contiguous().float()
    xg = torch.empty((n, (ca + cb) // 16, h, w, 16), dtype=torch.float16, device=a.device)
    st = _lib.load().e2f_dcn_pack_input(a_cl.data_ptr(), b_cl.data_ptr(), xg.data_ptr(), n, h, w, ca, cb, _stream())
    _lib.check(st, "e2f_dcn_pack_input")
    return GroupedX(xg, (n, ca + cb, h, w))


def prop_prologue(prop, feat_n2, flow_n1, flow_prev):
    """Everything one propagation step does before its offset-head conv and its DCN (feat_prop.py:106-126), fused:

        cond_n1 = flow_warp(prop, flow_n1);  flow_n2 = flow_n1 + flow_warp(flow_prev, flow_n1)
        cond_n2 = flow_warp(feat_n2, flow_n2);  cat([flow_n1, flow_n2], 1);  cat([prop, feat_n2], 1)

    prop, feat_n2: (n,c,h,w) fp32 channels_last (feat_n2 / flow_prev None on the second frame of a sweep: zeros);
    flow_n1, flow_prev: (n,2,h,w) fp32 with contiguous (h,w) planes (slices ``flows[:, i]`` of the (b,t-1,2,h,w) tensor).
    Returns ``(x, cond_n1, cond_n2, flows, flow_n1, flow_n2)``: x a ``GroupedX`` (DCN input), cond_* / flows ``SplitNHWC``
    conv operands, flow_n1 / flow_n2 (n,2,h,w) views of NHWC buffers (what ``deform_align_fused`` reads without a copy).
    Bit-identical to the unfused sequence of ``flow_warp`` / add / ``split_nhwc`` / ``dcn_pack_input``."""
    _need_cuda(prop, feat_n2, flow_n1, flow_prev)
    n, c, h, w = prop.shape
    if (feat_n2 is None) != (flow_prev is None):
        raise ValueError("prop_prologue: feat_n2 and flow_prev go together")
    if c % 16:
        raise ValueError("prop_prologue: the channel count must be a multiple of 16")

    def nhwc(t):
        return t if (t.dtype == torch.float32 and _is_cl(t)) else t.float().contiguous(memory_format=torch.channels_last)

    def planes(f):
        if f.dtype != torch.float32 or f.stride()[1:] != (h * w, w, 1):
            f = f.float().contiguous()
        return f

    prop, flow_n1 = nhwc(prop), planes(flow_n1)
    if feat_n2 is not None:
        feat_n2, flow_prev = nhwc(feat_n2), planes(flow_prev)
    dev = prop.device
    bf = torch.bfloat16
    c1h, c1l = torch.empty((n, h, w, c), dtype=bf, device=dev), torch.empty((n, h, w, c), dtype=bf, device=dev)
    c2h, c2l = torch.empty((n, h, w, c), dtype=bf, device=dev), torch.empty((n, h, w, c), dtype=bf, device=dev)
    f1 = torch.empty((n, h, w, 2), dtype=torch.float32, device=dev)
    f2 = torch.empty((n, h, w, 2), dtype=torch.float32, device=dev)
    flh, fll = torch.empty((n, h, w, 8), dtype=bf, device=dev), torch.empty((n, h, w, 8), dtype=bf, device=dev)
    xg = torch.empty((n, 2 * c // 16, h, w, 16), dtype=torch.float16, device=dev)
    st = _lib.load().e2f_prop_prologue(
        prop.data_ptr(), None if feat_n2 is None else feat_n2.data_ptr(), flow_n1.data_ptr(), flow_n1.stride(0),
        None if flow_prev is None else flow_prev.data_ptr(), 0 if flow_prev is None else flow_prev.stride(0),
        c1h.data_ptr(), c1l.data_ptr(), c2h.data_ptr(), c2l.data_ptr(), f1.data_ptr(), f2.data_ptr(), flh.data_ptr(),
        fll.data_ptr(), xg.data_ptr(), n, h, w, c, _stream())
    _lib.check(st, "e2f_prop_prologue")
    return (GroupedX(xg, (n, 2 * c, h, w)), SplitNHWC(c1h, c1l, (n, c, h, w)), SplitNHWC(c2h, c2l, (n, c, h, w)),
            SplitNHWC(flh, fll, (n, 4, h, w)), f1.permute(0, 3, 1, 2), f2.permute(0, 3, 1, 2))


def deform_align_fused(x, head, flow_1, flow_2, w_packed, bias, deform_groups, max_residue_magnitude=10.0,
                       out_dtype=torch.float32, out_split=False):
    """feat_prop.py:41-58 in one kernel: 10*tanh + flow.flip(1) add, sigmoid, deformable sampling, GEMM, bias.

    x (n,cin,h,w) fp16 channels_last; head (n,27*dg,h,w) fp32 channels_last (raw conv_offset output);
    flow_k (n,2,h,w) any layout (converted to (n,h,w,2) fp32).  Returns (n,cout,h,w) channels_last; with
    ``out_split=True`` (fp32 output only) ``(tensor, SplitNHWC)`` — the bf16 operand pair of the backbone conv that
    consumes the aligned features, written by the same epilogue.
    """
    grouped = isinstance(x, GroupedX)
    _need_cuda(None if grouped else x, head, flow_1, flow_2, w_packed, bias)
    n, cin, h, w = x.shape
    cout = w_packed.shape[0]
    if grouped:
        x = x.data
    elif x.dtype != torch.float16 or not _is_cl(x):
        x = x.to(dtype=torch.float16, memory_format=torch.channels_last)
    if head.dtype != torch.float32 or not _is_cl(head):
        head = head.to(dtype=torch.float32, memory_format=torch.channels_last)
    f1 = flow_1.permute(0, 2, 3, 1).contiguous().float()
    f2 = flow_2.permute(0, 2, 3, 1).contiguous().float()
    b32 = None if bias is None else bias.detach().float().contiguous()
    out = torch.empty((n, cout, h, w), dtype=out_dtype, device=head.device, memory_format=torch.channels_last)
    if out_split:
        if out_dtype != torch.float32:
            raise ValueError("deform_align_fused: out_split goes with the fp32 output")
        ohi = torch.empty((n, h, w, cout), dtype=torch.bfloat16, device=head.device)
        olo = torch.empty((n, h, w, cout), dtype=torch.bfloat16, device=head.device)
        with _timed("deform_align_fused", 2.0 * cout * cin * 9 * n * h * w):
            st = _lib.load().e2f_deform_align_fused_split(
                x.data_ptr(), head.data_ptr(), f1.data_ptr(), f2.data_ptr(), w_packed.data_ptr(),
                None if b32 is None else b32.data_ptr(), out.data_ptr(), ohi.data_ptr(), olo.data_ptr(), n, h, w, cin,
                cout, deform_groups, float(max_residue_magnitude), 1 if grouped else 0, _stream())
        _lib.check(st, "e2f_deform_align_fused_split")
        return out, SplitNHWC(ohi, olo, (n, cout, h, w))
    with _timed("deform_align_fused", 2.0 * cout * cin * 9 * n * h * w):
        st = _lib.load().e2f_deform_align_fused(
            x.data_ptr(), head.data_ptr(), f1.data_ptr(), f2.data_ptr(), w_packed.data_ptr(),
            None if b32 is None else b32.data_ptr(), out.data_ptr(), n, h, w, cin, cout, deform_groups,
            float(max_residue_magnitude), _DT[out_dtype], 1 if grouped else 0, _stream())
    _lib.check(st, "e2f_deform_align_fused")
    return out


def dcn_transposed_split(weight, deform_groups):
    """bf16 (hi, lo) split of W16^T, the packed fp16 DCN weight transposed to (9*Cin, Cout): the weight operand of
    dA = dY . W16 on ``e2f_linear_bf16x3``.  fp16 is exact as two bf16 terms.  ``weight``: the fp32 (Cout, Cin, 3, 3)
    parameter or an already packed fp16 (Cout, 9*Cin) operand."""
    w16 = weight if weight.dtype == torch.float16 and weight.dim() == 2 else pack_dcn_weight(weight, deform_groups)
    return split_bf16(w16.float().t().contiguous())


def deform_align_backward_work_elems(n, h, w, cin=256, deform_groups=16):
    """32-bit words of the dx scatter workspace of ``deform_align_backward`` (``e2f_deform_align_backward_work_elems``)."""
    elems = int(_lib.load().e2f_deform_align_backward_work_elems(n, h, w, cin, deform_groups))
    if elems < 0:
        _lib.check(elems, "e2f_deform_align_backward_work_elems")
    return elems


def deform_align_backward(x, head, flow_1, flow_2, w_packed, dy, deform_groups=16, max_residue_magnitude=10.0,
                          need_x=True, need_head=True, need_flow=True, need_weight=True, need_bias=True, wt_split=None):
    """Gradients of ``deform_align_fused`` (NHWC x) from dy = d loss / d out (n, Cout, h, w):

    1. dA = dY . W16 (fp32 (M, 9*Cin)) on ``e2f_linear_bf16x3`` with ``wt_split`` = ``dcn_transposed_split`` (built from
       ``w_packed`` when None); dY is split to bf16 once and serves steps 1 and 3.
    2. the sampler's adjoint (``e2f_deform_align_backward_sample``): d head, the offsets' share of d flow, the split
       sample rows A and the dx scatter list, each only when asked for.
    3. dW = dY^T . A and db on ``e2f_linear_wgrad_bf16x3``, unpacked from the sampler's K order to (Cout, Cin, 3, 3).
    4. dx by sorting the scatter list and gathering each destination in source order
       (``e2f_deform_align_backward_scatter``).

    x: (n, Cin, h, w) (the forward's fp16 input; converted like the forward does), head: the raw (n, 27*dg, h, w) fp32
    head, flow_k (n, 2, h, w).  Returns (dx (n, Cin, h, w) fp32 channels_last, d head (n, 27*dg, h, w) fp32
    channels_last, d flow (n, h, w, 8) fp32 = [d flow_1 (u, v), d flow_2 (u, v), 0 x 4], dW, db), None where not asked
    for; d flow needs ``need_head``."""
    _need_cuda(x, head, flow_1, flow_2, w_packed, dy)
    n, cin, h, w = x.shape
    cout = w_packed.shape[0]
    kt = w_packed.shape[1]
    if tuple(head.shape) != (n, 27 * deform_groups, h, w) or tuple(flow_1.shape) != (n, 2, h, w) or \
            tuple(flow_2.shape) != (n, 2, h, w) or tuple(dy.shape) != (n, cout, h, w) or kt != 9 * cin:
        raise ValueError(f"deform_align_backward: shapes x {tuple(x.shape)}, head {tuple(head.shape)}, flows "
                         f"{tuple(flow_1.shape)} / {tuple(flow_2.shape)}, w_packed {tuple(w_packed.shape)}, dy "
                         f"{tuple(dy.shape)} do not match")
    if need_flow and not need_head:
        raise ValueError("deform_align_backward: the flows' gradient goes with the head's")
    lib = _lib.load()
    m = n * h * w
    if x.dtype != torch.float16 or not _is_cl(x):
        x = x.to(dtype=torch.float16, memory_format=torch.channels_last)
    if head.dtype != torch.float32 or not _is_cl(head):
        head = head.to(dtype=torch.float32, memory_format=torch.channels_last)
    f1 = flow_1.permute(0, 2, 3, 1).contiguous().float()
    f2 = flow_2.permute(0, 2, 3, 1).contiguous().float()
    dy_hi, dy_lo = split_bf16(dy.permute(0, 2, 3, 1).reshape(m, cout))
    dev = head.device
    da = None
    if need_x or need_head:
        wt_hi, wt_lo = wt_split if wt_split is not None else dcn_transposed_split(w_packed, deform_groups)
        da = torch.empty((m, kt), dtype=torch.float32, device=dev)
        with _timed("linear_bf16x3", 2.0 * m * kt * cout):
            st = lib.e2f_linear_bf16x3(dy_hi.data_ptr(), dy_lo.data_ptr(), wt_hi.data_ptr(), wt_lo.data_ptr(), None, None,
                                       da.data_ptr(), m, kt, cout, _DT[torch.float32], 0, _stream())
        _lib.check(st, "e2f_linear_bf16x3")
    dhead = torch.empty((n, h, w, 27 * deform_groups), dtype=torch.float32, device=dev) if need_head else None
    dflow = torch.empty((n, h, w, 8), dtype=torch.float32, device=dev) if need_flow else None
    need_a = need_weight or need_bias
    a_hi = torch.empty((m, kt), dtype=torch.bfloat16, device=dev) if need_a else None
    a_lo = torch.empty((m, kt), dtype=torch.bfloat16, device=dev) if need_a else None
    work = None
    if need_x:
        work = torch.empty(deform_align_backward_work_elems(n, h, w, cin, deform_groups), dtype=torch.int32, device=dev)
    if need_head or need_a or need_x:
        with _timed("deform_align_backward_sample", float(m * kt * 2 * (need_head * 2 + need_a * 2) + m * 576 * 12 * need_x)):
            st = lib.e2f_deform_align_backward_sample(
                x.data_ptr(), head.data_ptr(), f1.data_ptr(), f2.data_ptr(), None if da is None else da.data_ptr(),
                None if dhead is None else dhead.data_ptr(), None if dflow is None else dflow.data_ptr(),
                None if a_hi is None else a_hi.data_ptr(), None if a_lo is None else a_lo.data_ptr(),
                None if work is None else work.data_ptr(), n, h, w, cin, deform_groups, float(max_residue_magnitude),
                _stream())
        _lib.check(st, "e2f_deform_align_backward_sample")
    dw = db = None
    if need_a:
        dw, db = linear_wgrad(SplitMat(dy_hi, dy_lo), SplitMat(a_hi, a_lo), with_bias=need_bias, shape=(cout, kt))
        # packed K order k = (g*9 + tap)*cpg + c  ->  (Cout, Cin, 3, 3)
        cpg = cin // deform_groups
        dw = dw.view(cout, deform_groups, 9, cpg).transpose(2, 3).reshape(cout, cin, 3, 3) if need_weight else None
    dx = None
    if need_x:
        dx = torch.empty((n, h, w, cin), dtype=torch.float32, device=dev)
        with _timed("deform_align_backward_scatter", float(m * 576 * 40)):
            st = lib.e2f_deform_align_backward_scatter(da.data_ptr(), work.data_ptr(), dx.data_ptr(), n, h, w, cin,
                                                       deform_groups, _stream())
        _lib.check(st, "e2f_deform_align_backward_scatter")
        dx = dx.permute(0, 3, 1, 2)
    return dx, None if dhead is None else dhead.permute(0, 3, 1, 2), dflow, dw, db


def focal_window_attention(qkv, qkv_pooled, num_heads, window_size, expand_size, focal_window, scale,
                           out_dtype=torch.float16):
    """softmax(q k_all^T) v_all of tfocal_transformer.py:226-396, un-partitioned output.

    qkv (B,T,H,W,3C) fp16, qkv_pooled (B,T,nWh,nWw,3C) fp16 or None (focal_level 1) -> (B,T,H,W,C) in
    ``out_dtype`` (torch.float32 / torch.float16), or — ``out_dtype="split"`` — a ``SplitMat``, the bf16 (hi, lo)
    operand pair of the following ``linear`` (attn.proj) written by the epilogue.
    """
    _need_cuda(qkv, qkv_pooled)
    B, T, H, W, C3 = qkv.shape
    C = C3 // 3
    wh, ww = window_size
    if H % wh or W % ww:
        raise ValueError(f"token grid {H}x{W} is not a multiple of the window {wh}x{ww}")
    if qkv.dtype != torch.float16 or not qkv.is_contiguous():
        qkv = qkv.contiguous().half()
    use_pooled = qkv_pooled is not None
    if use_pooled:
        if qkv_pooled.shape != (B, T, H // wh, W // ww, C3):
            raise ValueError(f"qkv_pooled shape {tuple(qkv_pooled.shape)} != {(B, T, H // wh, W // ww, C3)}")
        if qkv_pooled.dtype != torch.float16 or not qkv_pooled.is_contiguous():
            qkv_pooled = qkv_pooled.contiguous().half()
    split = isinstance(out_dtype, str) and out_dtype == "split"
    if split:
        out = torch.empty((2, B, T, H, W, C), dtype=torch.bfloat16, device=qkv.device)
    else:
        out = torch.empty((B, T, H, W, C), dtype=out_dtype, device=qkv.device)
    with _timed("focal_window_attention", attention_flops(B, T, H, W, C, window_size, expand_size, focal_window,
                                                            use_pooled)):
        st = _lib.load().e2f_focal_window_attention(
            qkv.data_ptr(), qkv_pooled.data_ptr() if use_pooled else None, out.data_ptr(), B, T, H, W, num_heads,
            C // num_heads, wh, ww, expand_size[0], expand_size[1], focal_window[0], focal_window[1],
            1 if use_pooled else 0, float(scale), 2 if split else _DT[out_dtype], _stream())
    _lib.check(st, "e2f_focal_window_attention")
    return SplitMat(out[0], out[1]) if split else out


def focal_window_attention_backward(qkv, qkv_pooled, dout, num_heads, window_size, expand_size, focal_window, scale):
    """Gradients of ``focal_window_attention`` (``e2f_focal_window_attention_backward``): qkv / qkv_pooled the fp16
    operands the forward read, dout (B,T,H,W,C) fp32 -> one fp32 buffer (B*T*H*W + B*T*nWh*nWw, 3C): the token rows'
    dq | dk | dv, then the pooled rows' 0 | dk | dv (none without qkv_pooled) — the qkv Linear's output gradient for
    the token rows and pooled rows together."""
    _need_cuda(qkv, qkv_pooled, dout)
    B, T, H, W, C3 = qkv.shape
    C = C3 // 3
    wh, ww = window_size
    use_pooled = qkv_pooled is not None
    if qkv.dtype != torch.float16 or not qkv.is_contiguous():
        raise ValueError("focal_window_attention_backward: qkv must be the contiguous fp16 tensor the forward read")
    if use_pooled and (qkv_pooled.dtype != torch.float16 or not qkv_pooled.is_contiguous()
                       or qkv_pooled.shape != (B, T, H // wh, W // ww, C3)):
        raise ValueError("focal_window_attention_backward: qkv_pooled must be the contiguous fp16 tensor the forward read")
    if dout.shape != (B, T, H, W, C):
        raise ValueError(f"focal_window_attention_backward: dout shape {tuple(dout.shape)} != {(B, T, H, W, C)}")
    dout = dout.contiguous().float()
    geo = (B, T, H, W, num_heads, C // num_heads, wh, ww, expand_size[0], expand_size[1], focal_window[0],
           focal_window[1], 1 if use_pooled else 0)
    lib = _lib.load()
    elems = int(lib.e2f_focal_window_attention_backward_work_elems(*geo))
    if elems < 0:
        _lib.check(elems, "e2f_focal_window_attention_backward_work_elems")
    n_tok, n_pool = B * T * H * W, (B * T * (H // wh) * (W // ww) if use_pooled else 0)
    d = torch.empty((n_tok + n_pool, C3), dtype=torch.float32, device=qkv.device)
    work = torch.empty(max(elems, 4), dtype=torch.float32, device=qkv.device)
    # the backward's algorithmic products: S, dP, dV, dQ, dK
    with _timed("focal_window_attention_backward",
                2.5 * attention_flops(B, T, H, W, C, window_size, expand_size, focal_window, use_pooled)):
        st = lib.e2f_focal_window_attention_backward(
            qkv.data_ptr(), qkv_pooled.data_ptr() if use_pooled else None, dout.data_ptr(), d.data_ptr(),
            d[n_tok:].data_ptr() if use_pooled else None, work.data_ptr(), *geo[:12], geo[12], float(scale), _stream())
    _lib.check(st, "e2f_focal_window_attention_backward")
    return d


def focal_attention_key_sources(t_count, grid, window_size, expand_size, focal_window, use_pooled, t, pooled, y, x):
    """The backward's gather list of one key token: [(window index, key slot, multiplicity), ...] in the order the
    backward adds them (``e2f_focal_window_attention_key_sources``; host only)."""
    cap = 256
    win, slot, mult = (ctypes.c_int * cap)(), (ctypes.c_int * cap)(), (ctypes.c_int * cap)()
    n = _lib.load().e2f_focal_window_attention_key_sources(
        t_count, grid[0], grid[1], window_size[0], window_size[1], expand_size[0], expand_size[1], focal_window[0],
        focal_window[1], 1 if use_pooled else 0, t, 1 if pooled else 0, y, x, win, slot, mult, cap)
    if n < 0:
        _lib.check(n, "e2f_focal_window_attention_key_sources")
    return [(win[i], slot[i], mult[i]) for i in range(n)]


class SplitMat:
    """A (..., K) activation as two bf16 terms (hi + lo): the A operand of ``linear`` produced directly by a fused
    producer (LayerNorm, unfold+GELU), so no fp32 round trip and no standalone split launch."""

    __slots__ = ("hi", "lo")

    def __init__(self, hi, lo):
        self.hi, self.lo = hi, lo

    @property
    def shape(self):
        return self.hi.shape

    def view(self, *shape):
        return SplitMat(self.hi.view(*shape), self.lo.view(*shape))


def t2t_unfold(img, kernel_size, stride, padding, gelu=False, out="f32"):
    """``F.unfold(img, k, padding=p, stride=s).permute(0, 2, 1)`` (tfocal_transformer.py:39-43, :94-96) in one
    gather kernel, optionally followed by the exact GELU.  img (BT,C,H,W) fp32 -> tokens (BT, L, C*k*k): fp32
    tensor (out="f32") or a ``SplitMat`` (out="split")."""
    _need_cuda(img)
    k, s, p = _square(kernel_size, stride, padding)
    bt, c, h, w = img.shape
    fh, fw = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    shape = (bt, fh * fw, c * k * k)
    tok, hi, lo = _outputs(out, ("f32", "split"), shape, img.device)
    # channels_last storage (conv / linear epilogues write it) is read in place by the staged 7/3/3 kernel
    nhwc = ((k, s, p) == (7, 3, 3) and c % 8 == 0 and img.dtype == torch.float32 and not img.is_contiguous()
            and img.permute(0, 2, 3, 1).is_contiguous() and bt <= 65535
            and 8 * 7 * (w + 6) * 4 <= 200 * 1024)      # the staged kernel's shared-memory row buffer (t2t.cu: U2_CC rows)
    if not nhwc:
        img = img.contiguous().float()
    numel = shape[0] * shape[1] * shape[2]
    with _timed("t2t_unfold", float(numel * 4 + img.numel() * 4)):
        fn = _lib.load().e2f_t2t_unfold_nhwc if nhwc else _lib.load().e2f_t2t_unfold
        st = fn(img.data_ptr(), None if tok is None else tok.data_ptr(),
                                        None if hi is None else hi.data_ptr(), None if lo is None else lo.data_ptr(),
                                        bt, c, h, w, k, s, p, 1 if gelu else 0, _stream())
    _lib.check(st, "e2f_t2t_unfold")
    return tok if out == "f32" else SplitMat(hi, lo)


def t2t_fold_unfold(tokens, output_size, kernel_size, stride, padding, gelu=False, out="f32", pitch=None):
    """``unfold(fold(tokens) / fold(ones))`` (+ exact GELU): the middle of FusionFeedForward.forward
    (tfocal_transformer.py:89-96) as ONE kernel for the 7/3/3 geometry — the folded image lives in shared memory only.
    Other geometries compose ``t2t_fold(normalize=True)`` and ``t2t_unfold``.  tokens (BT, L, C*k*k) fp32 -> same
    shape, fp32 (out="f32") or ``SplitMat`` (out="split").  ``pitch`` (multiple of 4 >= C*k*k) pads every output row
    with zero columns — ``linear`` zero-pads its weight to match — so that GEMM rows start on 128-byte lines."""
    _need_cuda(tokens)
    k, s, p = _square(kernel_size, stride, padding)
    h, w = output_size
    tokens = tokens.contiguous().float()
    bt, n_tok, ck = tokens.shape
    c = ck // (k * k)
    fh, fw = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    if n_tok != fh * fw or c * k * k != ck:
        raise ValueError(f"t2t_fold_unfold: tokens {tuple(tokens.shape)} do not match output_size {output_size}")
    fused = (k, s, p) == (7, 3, 3) and c % 4 == 0 and bt <= 65535      # any width: the kernel tiles wide images in x
    if not fused:
        img = t2t_fold(tokens, output_size, kernel_size, stride, padding, normalize=True)
        return t2t_unfold(img, kernel_size, stride, padding, gelu=gelu, out=out)
    pitch = ck if pitch is None else int(pitch)
    if pitch < ck or pitch % 4:
        raise ValueError(f"t2t_fold_unfold: pitch {pitch} must be a multiple of 4 >= {ck}")
    tok, hi, lo = _outputs(out, ("f32", "split"), (bt, n_tok, pitch), tokens.device)
    with _timed("t2t_fold_unfold", float(tokens.numel() * 8)):
        st = _lib.load().e2f_t2t_fold_unfold(tokens.data_ptr(), None if tok is None else tok.data_ptr(),
                                             None if hi is None else hi.data_ptr(),
                                             None if lo is None else lo.data_ptr(), bt, c, h, w, k, s, p,
                                             1 if gelu else 0, pitch, _stream())
    _lib.check(st, "e2f_t2t_fold_unfold")
    return tok if out == "f32" else SplitMat(hi, lo)


def t2t_fold_unfold_train(tokens, output_size, kernel_size, stride, padding, u=None, out="split", pitch=None):
    """The training modes of ``t2t_fold_unfold`` with GELU (``e2f_t2t_fold_unfold_train``), 7/3/3 only.

    ``u=None``: the forward, returns ``(GELU(u), u)`` with u = unfold(fold(tokens) / fold(ones)) fp32 (BT, L, C*k*k) —
    the first the same bits as ``t2t_fold_unfold(gelu=True)``.  ``u`` given (the forward's): the input gradient of that
    forward at dz = ``tokens``, unfold(fold(dz * GELU'(u)) / fold(ones)).  Outputs as ``t2t_fold_unfold``."""
    k, s, p = _square(kernel_size, stride, padding)
    if (k, s, p) != (7, 3, 3):
        raise NotImplementedError("t2t_fold_unfold_train: the 7/3/3 geometry only (the fused kernel)")
    _need_cuda(tokens, u)
    h, w = output_size
    tokens = tokens.contiguous().float()
    bt, n_tok, ck = tokens.shape
    c = ck // 49
    fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
    if n_tok != fh * fw or c * 49 != ck:
        raise ValueError(f"t2t_fold_unfold_train: tokens {tuple(tokens.shape)} do not match output_size {output_size}")
    backward = u is not None
    if backward and tuple(u.shape) != tuple(tokens.shape):
        raise ValueError(f"t2t_fold_unfold_train: u {tuple(u.shape)} != tokens {tuple(tokens.shape)}")
    u = torch.empty_like(tokens) if u is None else u.contiguous()
    pitch = ck if pitch is None else int(pitch)
    tok, hi, lo = _outputs(out, ("f32", "split"), (bt, n_tok, pitch), tokens.device)
    name = "t2t_fold_unfold_adjoint" if backward else "t2t_fold_unfold"
    with _timed(name, float(tokens.numel() * (12 if backward else 8))):
        st = _lib.load().e2f_t2t_fold_unfold_train(tokens.data_ptr(), u.data_ptr(), None if tok is None else tok.data_ptr(),
                                                   None if hi is None else hi.data_ptr(),
                                                   None if lo is None else lo.data_ptr(), bt, c, h, w, k, s, p,
                                                   1 if backward else 0, pitch, _stream())
    _lib.check(st, "e2f_t2t_fold_unfold_train")
    res = tok if out == "f32" else SplitMat(hi, lo)
    return res if backward else (res, u)


def window_pool(x, weight, bias, window_size, out="split"):
    """pool_layers[0] (``nn.Linear(wh*ww, 1)`` across the tokens of each window, per channel; tfocal_transformer.py:
    508-516) in one kernel.  x: the split LayerNorm output as a ``SplitMat`` of shape (B,T,H,W,C); weight (1, wh*ww);
    bias (1,).  Returns the pooled tokens ordered (B,T,nWh,nWw,C) — the reference's (B,nWh,nWw,T,C) after its
    ``permute(0,3,1,2,4)`` — as fp32 (out="f32") or ``SplitMat`` (out="split")."""
    if not isinstance(x, SplitMat):
        raise TypeError("window_pool takes the SplitMat written by layer_norm(out='split')")
    _need_cuda(x.hi, weight, bias)
    B, T, H, W, C = x.shape
    wh, ww = window_size
    if H % wh or W % ww:
        raise ValueError(f"token grid {H}x{W} must be a multiple of the window {wh}x{ww}")
    o32, ohi, olo = _outputs(out, ("f32", "split"), (B, T, H // wh, W // ww, C), x.hi.device)
    w32 = weight.detach().float().contiguous()
    b32 = None if bias is None else bias.detach().float().contiguous()
    with _timed("window_pool", float(x.hi.numel() * 4)):
        st = _lib.load().e2f_window_pool(x.hi.data_ptr(), x.lo.data_ptr(), w32.data_ptr(),
                                         None if b32 is None else b32.data_ptr(),
                                         None if o32 is None else o32.data_ptr(),
                                         None if ohi is None else ohi.data_ptr(),
                                         None if olo is None else olo.data_ptr(), B * T, H, W, C, wh, ww, _stream())
    _lib.check(st, "e2f_window_pool")
    return o32 if out == "f32" else SplitMat(ohi, olo)


def upsample2x_split(x):
    """``F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=True)`` (deconv.forward, e2fgvi.py:125-129)
    fused with the bf16 split: (N,C,H,W) fp32 -> ``SplitNHWC`` of (N,C,2H,2W); the upsampled fp32 tensor never exists."""
    _need_cuda(x)
    n, c, h, w = x.shape
    if c % 8:
        raise ValueError("upsample2x_split needs C % 8 == 0")
    xcl = x.permute(0, 2, 3, 1).contiguous().float()      # no-op for channels_last inputs
    hi = torch.empty((n, 2 * h, 2 * w, c), dtype=torch.bfloat16, device=x.device)
    lo = torch.empty((n, 2 * h, 2 * w, c), dtype=torch.bfloat16, device=x.device)
    with _timed("upsample2x_split", float(xcl.numel() * 4 + hi.numel() * 4)):
        st = _lib.load().e2f_upsample2x_split(xcl.data_ptr(), hi.data_ptr(), lo.data_ptr(), n, h, w, c, _stream())
    _lib.check(st, "e2f_upsample2x_split")
    return SplitNHWC(hi, lo, (n, c, 2 * h, 2 * w))


def layer_norm(x, weight, bias, eps=1e-5, out="f32"):
    """``F.layer_norm(x, (C,), weight, bias, eps)`` over the last dim (C = 512).  out = "f32": tensor; "split": a
    ``SplitMat`` (operand of the following ``linear``); "both": (tensor, SplitMat)."""
    _need_cuda(x, weight, bias)
    c = x.shape[-1]
    o32, hi, lo = _outputs(out, ("f32", "split", "both"), x.shape, x.device)
    xc = x.contiguous().float()
    rows = xc.numel() // c
    g32, b32 = weight.detach().float().contiguous(), bias.detach().float().contiguous()
    with _timed("layernorm_split", float(xc.numel() * 4 * (1 + (o32 is not None) + (hi is not None)))):
        st = _lib.load().e2f_layernorm_split(xc.data_ptr(), g32.data_ptr(), b32.data_ptr(),
                                             None if o32 is None else o32.data_ptr(),
                                             None if hi is None else hi.data_ptr(),
                                             None if lo is None else lo.data_ptr(), rows, c, float(eps), _stream())
    _lib.check(st, "e2f_layernorm_split")
    return _result(out, o32, None if hi is None else SplitMat(hi, lo))


def layer_norm_pool(x, weight, bias, eps, pool_weight, pool_bias, window_size):
    """norm1 + pool_layers[0] of a TemporalFocalTransformerBlock in one kernel (tfocal_transformer.py:470, :508-516):
    LayerNorm every token and — from the normalised values still in registers — pool every (frame, window) with the
    ``nn.Linear(wh*ww, 1)`` weights.  x (B,T,H,W,C) fp32, C = 512.

    Returns ``(all_rows, n_tok)``: ``all_rows`` a ``SplitMat`` of shape (B*T*H*W + B*T*nWh*nWw, C) — the normalised
    tokens followed by the pooled tokens ordered (B,T,nWh,nWw) — so ONE qkv ``linear`` over it yields qkv and qkv_pooled
    back to back; ``n_tok`` = B*T*H*W."""
    _need_cuda(x, weight, bias, pool_weight, pool_bias)
    B, T, H, W, C = x.shape
    wh, ww = window_size
    if H % wh or W % ww:
        raise ValueError(f"token grid {H}x{W} must be a multiple of the window {wh}x{ww}")
    xc = x.contiguous().float()
    n_tok, n_pool = B * T * H * W, B * T * (H // wh) * (W // ww)
    hi = torch.empty((n_tok + n_pool, C), dtype=torch.bfloat16, device=x.device)
    lo = torch.empty((n_tok + n_pool, C), dtype=torch.bfloat16, device=x.device)
    g32, b32 = weight.detach().float().contiguous(), bias.detach().float().contiguous()
    pw = pool_weight.detach().float().contiguous()
    pb = None if pool_bias is None else pool_bias.detach().float().contiguous()
    with _timed("layernorm_split", float(xc.numel() * 8 + n_pool * C * 4)):
        st = _lib.load().e2f_layernorm_pool_split(xc.data_ptr(), g32.data_ptr(), b32.data_ptr(), pw.data_ptr(),
                                                  None if pb is None else pb.data_ptr(), hi.data_ptr(), lo.data_ptr(),
                                                  B * T, H, W, C, wh, ww, float(eps), _stream())
    _lib.check(st, "e2f_layernorm_pool_split")
    return SplitMat(hi, lo), n_tok


def layer_norm_backward(x, dy, weight, eps=1e-5, residual=None, out="f32", need_weight=True, need_bias=True):
    """Gradients of ``layer_norm`` (``e2f_layernorm_backward``, C = 512): x the forward's fp32 input, dy the output's
    gradient, both (..., C) -> ``(dx, dweight, dbias)``.  dx = residual + LN'(x; dy) (``residual`` of x's shape or
    None) as an fp32 tensor (out="f32"), a ``SplitMat`` ("split"), both ("both") or None (out=None; then a parameter
    gradient must be asked for).  dweight / dbias (C,) fp32, or None when not asked for — neither: no partial sums."""
    c = x.shape[-1]
    if tuple(dy.shape) != tuple(x.shape):
        raise ValueError(f"layer_norm_backward: dy {tuple(dy.shape)} != x {tuple(x.shape)}")
    if residual is not None and tuple(residual.shape) != tuple(x.shape):
        raise ValueError(f"layer_norm_backward: residual {tuple(residual.shape)} != x {tuple(x.shape)}")
    if c != 512 or tuple(weight.shape) != (c,):
        raise ValueError(f"layer_norm_backward: 512 channels and a (512,) weight only (x {tuple(x.shape)}, weight "
                         f"{tuple(weight.shape)})")
    if out is None and not (need_weight or need_bias):
        raise ValueError("layer_norm_backward: nothing to compute")
    _need_cuda(x, dy, weight, residual)
    o32, hi, lo = _outputs(out, ("f32", "split", "both"), x.shape, x.device) if out is not None else (None, None, None)
    xc, dyc = x.contiguous().float(), dy.contiguous().float()
    res = None if residual is None else residual.contiguous().float()
    rows = xc.numel() // c
    g32 = weight.detach().float().contiguous()
    lib = _lib.load()
    dw = torch.empty(c, dtype=torch.float32, device=x.device) if need_weight else None
    db = torch.empty(c, dtype=torch.float32, device=x.device) if need_bias else None
    work = None
    if need_weight or need_bias:
        elems = int(lib.e2f_layernorm_backward_work_elems(rows, c))
        if elems < 0:
            _lib.check(elems, "e2f_layernorm_backward_work_elems")
        work = torch.empty(max(elems, 4), dtype=torch.float32, device=x.device)
    n_out = (o32 is not None) + (hi is not None)
    with _timed("layernorm_backward", float(xc.numel() * 4 * (2 + (res is not None) + n_out))):
        st = lib.e2f_layernorm_backward(xc.data_ptr(), dyc.data_ptr(), g32.data_ptr(),
                                        None if res is None else res.data_ptr(),
                                        None if o32 is None else o32.data_ptr(), None if hi is None else hi.data_ptr(),
                                        None if lo is None else lo.data_ptr(), None if dw is None else dw.data_ptr(),
                                        None if db is None else db.data_ptr(),
                                        None if work is None else work.data_ptr(), rows, c, float(eps), _stream())
    _lib.check(st, "e2f_layernorm_backward")
    dx = None if out is None else _result(out, o32, None if hi is None else SplitMat(hi, lo))
    return dx, dw, db


def layer_norm_pool_backward(x, drows, dx1, weight, bias, eps, pool_weight, window_size, need_x=True, need_norm=True,
                             need_pool=True):
    """Gradients of ``layer_norm_pool`` (``e2f_layernorm_pool_backward``): x (B,T,H,W,C) the forward's fp32 input, drows
    (B*T*H*W + B*T*nWh*nWw, C) fp32 the gradient of its joint output (token rows, then pooled rows ordered
    (B,T,nWh,nWw)), dx1 (B,T,H,W,C) the gradient x already receives past the LayerNorm (the block's residual).
    Returns ``(dx, dweight, dbias, dpool_weight (1, wh*ww), dpool_bias (1,))``: dx = dx1 + LN'(x; dxn + w_pool *
    dpooled) when ``need_x``, the norm's gradients when ``need_norm``, the pooling's when ``need_pool``; None otherwise."""
    B, T, H, W, C = x.shape
    wh, ww = window_size
    if H % wh or W % ww:
        raise ValueError(f"token grid {H}x{W} must be a multiple of the window {wh}x{ww}")
    n_tok, n_pool = B * T * H * W, B * T * (H // wh) * (W // ww)
    if C != 512 or tuple(weight.shape) != (C,) or tuple(bias.shape) != (C,):
        raise ValueError(f"layer_norm_pool_backward: 512 channels only (x {tuple(x.shape)})")
    if tuple(drows.shape) != (n_tok + n_pool, C):
        raise ValueError(f"layer_norm_pool_backward: drows {tuple(drows.shape)} != {(n_tok + n_pool, C)}")
    if pool_weight.numel() != wh * ww:
        raise ValueError(f"layer_norm_pool_backward: pool weight has {pool_weight.numel()} entries, the window {wh * ww}")
    if need_x and (dx1 is None or tuple(dx1.shape) != tuple(x.shape)):
        raise ValueError(f"layer_norm_pool_backward: dx needs dx1 of x's shape {tuple(x.shape)}")
    if not (need_x or need_norm or need_pool):
        raise ValueError("layer_norm_pool_backward: nothing to compute")
    _need_cuda(x, drows, dx1, weight, bias, pool_weight)
    xc, dr = x.contiguous().float(), drows.contiguous().float()
    d1 = dx1.contiguous().float() if need_x else None
    g32, b32 = weight.detach().float().contiguous(), bias.detach().float().contiguous()
    pw = pool_weight.detach().float().contiguous()
    dev = x.device
    dx = torch.empty((B, T, H, W, C), dtype=torch.float32, device=dev) if need_x else None
    dw = torch.empty(C, dtype=torch.float32, device=dev) if need_norm else None
    db = torch.empty(C, dtype=torch.float32, device=dev) if need_norm else None
    dpw = torch.empty((1, wh * ww), dtype=torch.float32, device=dev) if need_pool else None
    dpb = torch.empty(1, dtype=torch.float32, device=dev) if need_pool else None
    lib = _lib.load()
    work = None
    if need_norm or need_pool:
        elems = int(lib.e2f_layernorm_pool_backward_work_elems(B * T, H, W, C, wh, ww))
        if elems < 0:
            _lib.check(elems, "e2f_layernorm_pool_backward_work_elems")
        work = torch.empty(max(elems, 4), dtype=torch.float32, device=dev)
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    with _timed("layernorm_pool_backward", float(xc.numel() * 4 * (2 + 2 * need_x) + n_pool * C * 4)):
        st = lib.e2f_layernorm_pool_backward(xc.data_ptr(), g32.data_ptr(), b32.data_ptr(), pw.data_ptr(), dr.data_ptr(),
                                             ptr(d1), ptr(dx), ptr(dw), ptr(db), ptr(dpw), ptr(dpb), ptr(work), B * T, H,
                                             W, C, wh, ww, float(eps), _stream())
    _lib.check(st, "e2f_layernorm_pool_backward")
    return dx, dw, db, dpw, dpb


def t2t_fold(tokens, output_size, kernel_size, stride, padding, normalize=False, bias=None, residual=None,
             channels_last=False):
    """``F.fold(tokens.permute(0, 2, 1), output_size, k, padding=p, stride=s)`` (tfocal_transformer.py:65-72,
    :89-96), optionally divided by fold(ones) and/or with a (C,H,W) bias map added.
    tokens (BT, L, C*k*k) fp32 -> img (BT, C, H, W) fp32.  ``channels_last=True`` returns the image in channels_last
    storage (what the decoder's convs read) and lets ``residual`` (BT,C,H,W) be added by the same kernel."""
    _need_cuda(tokens, bias, residual)
    k, s, p = _square(kernel_size, stride, padding)
    tokens = tokens.contiguous().float()
    bt, L, ck = tokens.shape
    h, w = output_size
    fh, fw = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    if L != fh * fw or ck % (k * k):
        raise ValueError(f"tokens {tuple(tokens.shape)} do not match output_size {output_size} with k={k}, s={s}, p={p}")
    c = ck // (k * k)
    if bias is not None:
        if tuple(bias.shape) != (c, h, w):
            raise ValueError(f"bias {tuple(bias.shape)} != {(c, h, w)}")
        bias = bias.detach().contiguous().float()
    if residual is not None and tuple(residual.shape) != (bt, c, h, w):
        raise ValueError(f"residual {tuple(residual.shape)} != {(bt, c, h, w)}")
    # the shared-memory fold needs a band of >= 3 image rows x 8 channels (+ two count tables) in 200 KB (t2t.cu)
    band_fits = (8 * 3 * 4 + 8) * (w + 6) <= 200 * 1024
    if channels_last and (k, s, p) == (7, 3, 3) and c % 8 == 0 and bt <= 65535 and band_fits:
        res = None if residual is None else residual.permute(0, 2, 3, 1).contiguous().float()   # no-op if channels_last
        img = torch.empty((bt, h, w, c), dtype=torch.float32, device=tokens.device)
        with _timed("t2t_fold", float(tokens.numel() * 4 + img.numel() * (8 if res is not None else 4))):
            st = _lib.load().e2f_t2t_fold_nhwc(tokens.data_ptr(), None if bias is None else bias.data_ptr(),
                                               None if res is None else res.data_ptr(), img.data_ptr(), bt, c, h, w,
                                               k, s, p, 1 if normalize else 0, _stream())
        _lib.check(st, "e2f_t2t_fold_nhwc")
        return img.permute(0, 3, 1, 2)
    img = torch.empty((bt, c, h, w), dtype=torch.float32, device=tokens.device)
    with _timed("t2t_fold", float(tokens.numel() * 4 + img.numel() * 4)):
        st = _lib.load().e2f_t2t_fold(tokens.data_ptr(), None if bias is None else bias.data_ptr(), img.data_ptr(), bt,
                                      c, h, w, k, s, p, 1 if normalize else 0, _stream())
    _lib.check(st, "e2f_t2t_fold")
    if residual is not None:
        img = img + residual
    return img.contiguous(memory_format=torch.channels_last) if channels_last else img


def split_bf16(x):
    """fp32 tensor -> (hi, lo) bf16 tensors with x ~= hi + lo to 2^-17 relative (numel % 8 == 0)."""
    _need_cuda(x)
    x = x.contiguous().float()
    hi = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    lo = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    st = _lib.load().e2f_split_bf16(x.data_ptr(), hi.data_ptr(), lo.data_ptr(), x.numel(), _stream())
    _lib.check(st, "e2f_split_bf16")
    return hi, lo


# The one cache of operands derived from parameters (bf16 splits, packed weights, folded bias maps):
#   (id(param), tag)         -> (weakref, version, data_ptr, operand)                            (_derived_one)
#   (tuple of ids, tag)      -> (weakrefs, ((version, data_ptr) per parameter), operand)          (_derived)
_DERIVED = {}


def _derived_one(param, tag, build, *args):
    """The operand ``build(param, *args)`` makes from the parameter ``param``, cached under ``tag``: rebuilt when the
    parameter changes version or address, dropped when it dies.  ``linear`` and the convs look their weights up on
    every call and a one-clip step is bound by host launch time, so a hit builds no closure, list or generator."""
    key = (id(param), tag)
    hit = _DERIVED.get(key)
    if hit is not None and hit[1] == param._version and hit[2] == param.data_ptr() and hit[0]() is param:
        return hit[3]
    val = build(param, *args)
    if hit is None or hit[0]() is not param:
        weakref.finalize(param, _DERIVED.pop, key, None)
    _DERIVED[key] = (weakref.ref(param), param._version, param.data_ptr(), val)
    return val


def _derived(params, tag, build):
    """The operand ``build()`` makes from a list of parameters, cached under ``tag``: rebuilt when any of them
    changes version or address, dropped when the first one dies."""
    key = (tuple(id(p) for p in params), tag)
    stamp = tuple((p._version, p.data_ptr()) for p in params)
    hit = _DERIVED.get(key)
    if hit is None or hit[1] != stamp or any(r() is not p for r, p in zip(hit[0], params)):
        val = build()
        if hit is None or hit[0][0]() is not params[0]:
            weakref.finalize(params[0], _DERIVED.pop, key, None)
        hit = _DERIVED[key] = (tuple(weakref.ref(p) for p in params), stamp, val)
    return hit[2]


def transposed_linear_weight(weight, k):
    """fp32 W^T of an (N, K) Linear weight as (K, k), k >= N: zero columns appended to match an operand whose rows are
    padded to k — the weight operand of the input gradient dY . W."""
    wt = weight.detach().reshape(weight.shape[0], -1).float().t()
    return torch.nn.functional.pad(wt, (0, k - wt.shape[1])) if k > wt.shape[1] else wt.contiguous()


def _padded_split(weight, k, transpose=False):
    """bf16 (hi, lo) split of an (N, K) or (N, K, 1, 1) weight as (N, k), k >= K: zero columns appended to match an
    operand whose rows are padded to k.  ``transpose``: of ``transposed_linear_weight(weight, k)`` instead."""
    if transpose:
        return split_bf16(transposed_linear_weight(weight, k))
    w2 = weight.detach().reshape(weight.shape[0], -1)
    if k > w2.shape[1]:
        w2 = torch.nn.functional.pad(w2.float(), (0, k - w2.shape[1]))
    return split_bf16(w2)


def linear(x, weight, bias=None, residual=None, out_dtype=torch.float32, tile_hint=0, transpose=False):
    """``F.linear(x, weight, bias) (+ residual)`` on the bf16 tensor pipe with a 3-term split (fp32-level accuracy).

    x (..., K) fp32, weight (N, K) fp32 nn.Parameter (its bf16 split is cached per parameter object and refreshed
    when the parameter changes), bias (N,), residual (..., N) fp32 -> (..., N) ``out_dtype``.
    ``transpose=True``: ``x . weight`` instead, x (..., N) -> (..., K) (the input gradient of the Linear; W^T's split is
    cached under its own tag)."""
    n, k = weight.shape[:2]            # (N, K) Linear weight or (N, K, 1, 1) 1x1-conv weight
    if transpose:
        n, k = k, n
    lead = x.shape[:-1]
    k_pad = 0
    if isinstance(x, SplitMat):         # operand pair written by a fused producer
        _need_cuda(weight, bias, residual)
        if x.shape[-1] != k:            # rows padded with zero columns (t2t_fold_unfold pitch): pad the weight alike
            if x.shape[-1] < k:
                raise ValueError(f"linear: operand has {x.shape[-1]} columns, weight expects {k}")
            k_pad = k = x.shape[-1]
        a_hi, a_lo = x.hi.reshape(-1, k), x.lo.reshape(-1, k)
        m = a_hi.shape[0]
    else:
        _need_cuda(x, weight, bias, residual)
        x2 = x.reshape(-1, k)
        m = x2.shape[0]
        a_hi, a_lo = split_bf16(x2)
    w_hi, w_lo = _derived_one(weight, ("split_t" if transpose else "split", k_pad), _padded_split, k, transpose)
    b32 = None if bias is None else bias.detach().float().contiguous()
    res = None
    if residual is not None:
        res = residual.reshape(m, n).contiguous().float()
    out = torch.empty((m, n), dtype=out_dtype, device=weight.device)
    with _timed("linear_bf16x3", 2.0 * m * n * k):
        st = _lib.load().e2f_linear_bf16x3(a_hi.data_ptr(), a_lo.data_ptr(), w_hi.data_ptr(), w_lo.data_ptr(),
                                           None if b32 is None else b32.data_ptr(),
                                           None if res is None else res.data_ptr(), out.data_ptr(), m, n, k,
                                           _DT[out_dtype], tile_hint, _stream())
    _lib.check(st, "e2f_linear_bf16x3")
    return out.view(*lead, n)


def linear_wgrad(dy, x, with_bias=True, shape=None):
    """(dW fp32 (N, K), db fp32 (N,) or None) of a Linear: dW = dY^T . X, db = the sum of dY over rows
    (``e2f_linear_wgrad_bf16x3``).  dy (..., N) and x (..., K): fp32 tensors or ``SplitMat`` operands (rows may be padded
    with zero columns, e.g. ``t2t_fold_unfold``'s pitch); ``shape`` = the parameter's (N, K) when they are padded."""
    ops_ = []
    for t in (dy, x):
        if isinstance(t, SplitMat):
            _need_cuda(t.hi)
            w = t.shape[-1]
            ops_.append((t.hi.reshape(-1, w), t.lo.reshape(-1, w)))
        else:
            _need_cuda(t)
            w = t.shape[-1]
            if w % 8:
                t = torch.nn.functional.pad(t.float(), (0, 8 - w % 8))
            ops_.append(split_bf16(t.reshape(-1, t.shape[-1])))
    (dy_hi, dy_lo), (x_hi, x_lo) = ops_
    m, ldy, ldx = dy_hi.shape[0], dy_hi.shape[1], x_hi.shape[1]
    if x_hi.shape[0] != m:
        raise ValueError(f"linear_wgrad: dy has {m} rows, x {x_hi.shape[0]}")
    n, k = shape if shape is not None else (dy.shape[-1], x.shape[-1])
    if n > ldy or k > ldx:
        raise ValueError(f"linear_wgrad: shape {(n, k)} exceeds the operands' widths {(ldy, ldx)}")
    lib = _lib.load()
    elems = int(lib.e2f_linear_wgrad_work_elems(m, n, k))
    if elems < 0:
        _lib.check(elems, "e2f_linear_wgrad_work_elems")
    work = torch.empty(elems, dtype=torch.float32, device=dy_hi.device) if elems else None
    dw = torch.empty((n, k), dtype=torch.float32, device=dy_hi.device)
    db = torch.empty(n, dtype=torch.float32, device=dy_hi.device) if with_bias else None
    with _timed("linear_wgrad_bf16x3", 2.0 * m * n * k):
        st = lib.e2f_linear_wgrad_bf16x3(dy_hi.data_ptr(), dy_lo.data_ptr(), ldy, x_hi.data_ptr(), x_lo.data_ptr(), ldx,
                                         dw.data_ptr(), None if db is None else db.data_ptr(),
                                         None if work is None else work.data_ptr(), m, n, k, _stream())
    _lib.check(st, "e2f_linear_wgrad_bf16x3")
    return dw, db


class SplitNHWC:
    """An NHWC activation as two bf16 terms (hi + lo) — the operand format of ``conv3x3``. Reusable across convs."""

    __slots__ = ("hi", "lo", "shape")

    def __init__(self, hi, lo, shape):
        self.hi, self.lo, self.shape = hi, lo, shape   # hi/lo: (N,H,W,Cpad) bf16; shape: logical (N,C,H,W)


def split_nhwc(x):
    """(N,C,H,W) fp32 (any memory format) -> SplitNHWC with channels zero-padded to a multiple of 8."""
    if isinstance(x, SplitNHWC):
        return x
    _need_cuda(x)
    n, c, h, w = x.shape
    nhwc = x.permute(0, 2, 3, 1)
    if c % 8:
        nhwc = torch.nn.functional.pad(nhwc, (0, 8 - c % 8))
    hi, lo = split_bf16(nhwc)            # .contiguous() inside is a no-op for channels_last inputs
    return SplitNHWC(hi, lo, (n, c, h, w))


class RowsNHWC:
    """A small-channel activation in the row-gapped layout of the window-packed conv (include/e2fgvi_b200.h,
    ``e2f_conv2d_rows_bf16x3``): bf16 (hi, lo), flat [N][H][pitch][cin] + tail with pitch = lead + W (+1 rounding
    pixel for odd rows of 4 channels), zeros in gaps / tail / pad channels."""

    __slots__ = ("hi", "lo", "shape", "lead", "cin", "pitch")

    def __init__(self, hi, lo, shape, lead, cin):
        self.hi, self.lo, self.shape, self.lead, self.cin = hi, lo, shape, lead, cin   # shape: logical (N,C,H,W)
        self.pitch = int(_lib.load().e2f_conv_rows_pitch(shape[3], lead, cin))

    def dense(self):
        """fp32 (N,C,H,W) view of the content (tests / debugging)."""
        n, c, h, w = self.shape
        body = (self.hi.float() + self.lo.float())[: n * h * self.pitch * self.cin]
        return body.view(n, h, self.pitch, self.cin)[:, :, self.lead: self.lead + w, :c].permute(0, 3, 1, 2)


def rows_channels(c):
    """Channel count of the row-gapped layout that holds c channels (4, 8, 16 or 32), or None if c > 32."""
    for cin in (4, 8, 16, 32):
        if c <= cin:
            return cin
    return None


def _rows_pair(n, h, w, lead, cin, device):
    """Flat bf16 (hi, lo) buffers of a ``RowsNHWC`` operand: n x h rows of ``lead`` + w pixels x ``cin`` channels."""
    lib = _lib.load()
    numel = (n * h * int(lib.e2f_conv_rows_pitch(w, lead, cin)) + int(lib.e2f_conv_rows_tail(lead, cin))) * cin
    return (torch.empty(numel, dtype=torch.bfloat16, device=device),
            torch.empty(numel, dtype=torch.bfloat16, device=device))


def pack_rows(x, lead, cin=None):
    """(N,C,H,W) fp32 -> ``RowsNHWC`` with ``lead`` zero pixels in front of every row (= the padding of the conv
    that consumes it) and channels zero-padded to ``cin`` (default: the smallest of 4/8/16/32 that holds C)."""
    if isinstance(x, RowsNHWC):
        return x
    _need_cuda(x)
    n, c, h, w = x.shape
    cin = cin or rows_channels(c)
    if cin is None or c > cin:
        raise ValueError(f"pack_rows: {c} channels do not fit a row-gapped layout (<= 32)")
    x = x.contiguous().float()
    hi, lo = _rows_pair(n, h, w, lead, cin, x.device)
    with _timed("pack_rows", float(x.numel() * 4 + hi.numel() * 4)):
        st = _lib.load().e2f_pack_rows_bf16(x.data_ptr(), hi.data_ptr(), lo.data_ptr(), n, c, h, w, cin, lead, _stream())
    _lib.check(st, "e2f_pack_rows_bf16")
    return RowsNHWC(hi, lo, (n, c, h, w), lead, cin)


def pack_conv_rows_weight(weight, cin):
    """fp32 (Cout, C, k, k), C <= cin -> (hi, lo) bf16 (Cout, k*G*64) in the window-packed K order of
    ``e2f_conv2d_rows_bf16x3``: chunk (ky, g) holds taps kx = g*PX .. g*PX+PX-1 (PX = 64/cin) x cin channels, zeros
    for kx >= k and for channels >= C."""
    cout, c, kh, kw = weight.shape
    assert kh == kw and c <= cin
    px = 64 // cin
    g = (kw + px - 1) // px
    w = weight.detach().float()
    packed = torch.zeros((cout, kh, g * px, cin), dtype=torch.float32, device=weight.device)
    packed[:, :, :kw, :c] = w.permute(0, 2, 3, 1)          # [co][ky][kx][c]
    return split_bf16(packed.view(cout, kh * g * 64))


def pack_conv3x3_weight(weight, src_channels, groups=1):
    """fp32 (Cout, Cin/G, 3, 3) -> (hi, lo) bf16 (Cout, 9*T*64) in the K order of ``e2f_conv3x3_bf16x3``:
    tap-major, then source, then 64-channel chunk; the group-local input channel axis is the concatenation of the
    sources' per-group slices (exactly the channel order of the torch.cat the reference performs)."""
    cout, cin_g, kh, kw = weight.shape
    assert kh == kw
    taps = kh * kw
    cig = [c // groups for c in src_channels]
    assert sum(cig) == cin_g, (src_channels, groups, cin_g)
    chunks = [(c + 63) // 64 for c in cig]
    T = sum(chunks)
    w = weight.detach().float()
    packed = torch.zeros((cout, taps, T, 64), dtype=torch.float32, device=weight.device)
    off, base = 0, 0
    for c, nch in zip(cig, chunks):
        for j in range(nch):
            cc = min(64, c - 64 * j)
            packed[:, :, base + j, :cc] = w[:, off + 64 * j: off + 64 * j + cc].reshape(cout, cc, taps).transpose(1, 2)
        off += c
        base += nch
    return split_bf16(packed.view(cout, taps * T * 64))


def merge_conv_groups(weight, src_channels, groups):
    """Rewrite a grouped conv whose groups have few output channels as one with fewer, wider groups and
    block-diagonal weights: m = largest power of two with m * Cout/G <= 64 and G % m == 0 groups are merged, so a
    64-wide N tile and the 64-channel K chunks of every source are filled instead of padded (encoder conv 7,
    e2fgvi.py:97: G=8 with 32 outputs and 32 + 48 inputs per group).  Returns (weight', groups')."""
    cout, cin_g = weight.shape[0], weight.shape[1]
    cog = cout // groups
    m = 1
    while groups % (2 * m) == 0 and 2 * m * cog <= 64:
        m *= 2
    if m == 1:
        return weight, groups
    cig = [c // groups for c in src_channels]
    w = weight.detach().float()
    merged = torch.zeros((cout, m * cin_g) + tuple(weight.shape[2:]), dtype=torch.float32, device=weight.device)
    sub = (torch.arange(cout, device=weight.device) % (m * cog)) // cog      # position of o's group in its merge
    off = 0
    for c in cig:
        for j in range(m):
            rows = (sub == j).nonzero().flatten()
            merged[rows, m * off + j * c: m * off + (j + 1) * c] = w[rows, off: off + c]
        off += c
    return merged, groups // m


def _conv3x3_operand(weight, src_channels, groups, rows_cin):
    """(hi, lo, effective groups) of a conv3x3-path weight: the value of its ("conv3x3", src_channels, groups,
    rows_cin) ``_derived`` entry.  rows_cin > 0: window-packed K for a ``RowsNHWC`` source of that many channels."""
    if rows_cin:
        return (*pack_conv_rows_weight(weight, rows_cin), 1)
    w_eff, g_eff = merge_conv_groups(weight, src_channels, groups)
    return (*pack_conv3x3_weight(w_eff, src_channels, g_eff), g_eff)


def _source_arrays(sources):
    """ctypes arrays (hi pointers, lo pointers, stored channel counts) of a conv's ``SplitNHWC`` / ``RowsNHWC``
    operands."""
    k = len(sources)
    return ((_lib._vp * k)(*[s.hi.data_ptr() for s in sources]), (_lib._vp * k)(*[s.lo.data_ptr() for s in sources]),
            (_lib._i * k)(*[s.cin if isinstance(s, RowsNHWC) else s.hi.shape[-1] for s in sources]))


def conv3x3(sources, weight, bias=None, groups=1, negative_slope=1.0, residual=None, out="f32", stride=1,
            padding=None, out_lead=0):
    """``leaky_relu(F.conv2d(torch.cat(sources, 1) [group-wise for groups > 1], weight, bias, 1, 1, 1, groups),
    negative_slope) (+ residual)`` as one wgmma implicit-GEMM launch; the cat is never built.

    Also serves square k x k kernels (k = 3, 7) with stride 1 / 2 (``padding`` defaults to k // 2): the stride-2
    encoder convs and SPyNet's 7x7 convs (negative_slope = 0 is ReLU).

    sources: list of (N,C_i,H,W) fp32 tensors or ``SplitNHWC``, or ONE ``RowsNHWC`` (small-channel input, window-packed
    K; its lead must equal the padding); weight: the nn.Conv2d parameter (Cout, sum C_i / G, k, k).
    out = "f32": (N,Cout,H,W) fp32 channels_last tensor; "split": a ``SplitNHWC`` (the bf16 operand pair of a
    following conv3x3, written by the epilogue, no fp32 round trip); "both": (tensor, SplitNHWC); "rows": a
    ``RowsNHWC`` with ``out_lead`` zero pixels per row (operand of a following small-channel conv with that padding)."""
    cout, ks = weight.shape[0], weight.shape[2]
    pad = ks // 2 if padding is None else padding
    rows_in = sources if isinstance(sources, RowsNHWC) else (
        sources[0] if isinstance(sources, (list, tuple)) and len(sources) == 1 and isinstance(sources[0], RowsNHWC) else None)
    _need_cuda(weight, bias, residual)
    if rows_in is not None:
        if rows_in.lead != pad or groups != 1:
            raise ValueError(f"conv3x3: RowsNHWC source with lead {rows_in.lead} needs padding {rows_in.lead} and groups 1")
        if rows_in.shape[1] != weight.shape[1]:
            raise ValueError("conv3x3: weight does not match the source's channel count")
        splits = [rows_in]
        true_channels = [rows_in.cin]
    else:
        splits = [split_nhwc(s) for s in (sources if isinstance(sources, (list, tuple)) else [sources])]
        true_channels = [s.shape[1] for s in splits]
        if groups != 1 and any(s.hi.shape[-1] != c for s, c in zip(splits, true_channels)):
            raise NotImplementedError("grouped conv3x3 needs channel counts that are multiples of 8")
    n, _, h_in, w_in = splits[0].shape
    for s in splits:
        if (s.shape[0], s.shape[2], s.shape[3]) != (n, h_in, w_in):
            raise ValueError("conv3x3 sources must share N, H, W")
    if out == "rows" and (out_lead <= 0 or cout not in (8, 16, 32)):
        raise ValueError("conv3x3: out='rows' needs out_lead > 0 and 8, 16 or 32 output channels")
    h, w = (h_in + 2 * pad - ks) // stride + 1, (w_in + 2 * pad - ks) // stride + 1
    o32, ohi, olo = _outputs(out, ("f32", "split", "both", "rows"), (n, h, w, cout), weight.device)
    if out == "rows":
        ohi, olo = _rows_pair(n, h, w, out_lead, cout, weight.device)
    rows_cin = 0 if rows_in is None else rows_in.cin
    w_hi, w_lo, g_eff = _derived_one(weight, ("conv3x3", tuple(true_channels), groups, rows_cin), _conv3x3_operand,
                                     true_channels, groups, rows_cin)
    b32 = None if bias is None else bias.detach().float().contiguous()
    res = None
    if residual is not None:
        res = residual.permute(0, 2, 3, 1).contiguous().float()
    with _timed("conv3x3_bf16x3", 2.0 * n * h * w * cout * weight.shape[1] * ks * ks):
        st = _lib.load().e2f_conv2d_rows_bf16x3(len(splits), *_source_arrays(splits), 1 if rows_in is not None else 0,
                                                w_hi.data_ptr(), w_lo.data_ptr(),
                                                None if b32 is None else b32.data_ptr(),
                                                None if res is None else res.data_ptr(),
                                                None if o32 is None else o32.data_ptr(),
                                                None if ohi is None else ohi.data_ptr(),
                                                None if olo is None else olo.data_ptr(),
                                                out_lead if out == "rows" else 0, n, h_in, w_in, cout,
                                                g_eff, float(negative_slope), ks, stride, pad, _stream())
    _lib.check(st, "e2f_conv2d_rows_bf16x3")
    if out == "rows":
        return RowsNHWC(ohi, olo, (n, cout, h, w), out_lead, cout)
    return _result(out, None if o32 is None else o32.permute(0, 3, 1, 2),
                   None if ohi is None else SplitNHWC(ohi, olo, (n, cout, h, w)))


# ------------------------------------------------------------------------------------------------- SoftSplit / SoftComp
def _best_tile(gh, gw, stride):
    """(tile_w, tile_h) with tile_w * tile_h <= 128 that wastes the fewest accumulator rows on a gh x gw GEMM grid
    (12 x 10 tiles the 20x36 and 60x108 token grids exactly; 18 x 7 the 90x162 one)."""
    best, best_cost = (16, 8), None
    for tw in range(1, min(gw, 128, 256 // stride) + 1):
        th = min(128 // tw, gh, 256 // stride)
        cost = -(-gh // th) * -(-gw // tw)                 # number of 128-row tiles
        key = (cost, abs(tw - th), -tw * th)            # fewest tiles, then the squarest (best TMA box / L2 reuse)
        if best_cost is None or key < best_cost:
            best, best_cost = (tw, th), key
    return best


def _nhwc_stride(t, what):
    """Batch stride in PIXELS of a (n, h, w, c) tensor whose inner three dims are dense (a frame slice of a
    (b, t, h, w, c) buffer is such a view)."""
    n, h, w, c = t.shape
    if t.stride()[1:] != (w * c, c, 1) or (n > 1 and t.stride(0) % c):
        raise ValueError(f"{what}: expected a (n, h, w, c) tensor with dense (h, w, c) dims, got strides {t.stride()}")
    return (t.stride(0) // c) if n > 1 else h * w


def _conv_gather(sources, w_hi, w_lo, bias, bias_map, residual, out, cout, stride, grid, taps, phases, ostep,
                 out_size, flops, slope=1.0, into=None):
    """One launch of e2f_conv_gather_bf16x3.  sources: list of ``SplitNHWC`` (hi / lo may be batch-strided views);
    taps: list of (dy, dx); phases: list of (first tap, oy, ox); residual: logical (n, cout, oh, ow) fp32 with NHWC
    storage; ``into`` = (o32, ohi, olo) optional pre-existing (n, oh, ow, cout) NHWC views to write (batch-strided allowed,
    all with the same batch stride, which the residual must share)."""
    import ctypes
    sources = list(sources)
    n, _, h_in, w_in = sources[0].shape
    gh, gw = grid
    oh, ow = out_size
    tw, th = _best_tile(gh, gw, stride)
    o32, ohi, olo = _outputs(out, ("f32", "split", "both"), (n, oh, ow, cout), sources[0].hi.device, into)
    outs = [t for t in (o32, ohi, olo) if t is not None]
    for t in outs:
        if tuple(t.shape) != (n, oh, ow, cout):
            raise ValueError(f"conv: output buffer {tuple(t.shape)} != {(n, oh, ow, cout)}")
    ostrides = {_nhwc_stride(t, "conv output") for t in outs}
    res = None
    if residual is not None:
        res = residual.permute(0, 2, 3, 1)
        if res.dtype != torch.float32 or res.stride()[1:] != (ow * cout, cout, 1):
            res = res.contiguous().float()
        ostrides.add(_nhwc_stride(res, "conv residual"))
    if len(ostrides) != 1:
        raise ValueError(f"conv: outputs and residual must share one batch stride, got {sorted(ostrides)}")
    out_nstride = ostrides.pop()
    k = len(sources)
    for s_ in sources:
        if (s_.shape[0], s_.shape[2], s_.shape[3]) != (n, h_in, w_in):
            raise ValueError("conv sources must share N, H, W")
    nt, nph = len(taps), len(phases)
    dy = (ctypes.c_int8 * nt)(*[t[0] for t in taps])
    dx = (ctypes.c_int8 * nt)(*[t[1] for t in taps])
    tap0 = (ctypes.c_uint8 * (nph + 1))(*([p[0] for p in phases] + [nt]))
    oy = (ctypes.c_uint8 * nph)(*[p[1] for p in phases])
    ox = (ctypes.c_uint8 * nph)(*[p[2] for p in phases])
    sn = [_nhwc_stride(s_.hi, "conv source") for s_ in sources]
    for s_, v in zip(sources, sn):
        if _nhwc_stride(s_.lo, "conv source") != v:
            raise ValueError("conv: hi / lo of a source must share the batch stride")
    sn_arr = (ctypes.c_int64 * k)(*sn)
    b32 = None if bias is None else bias.detach().float().contiguous()
    with _timed("conv3x3_bf16x3", flops):
        st = _lib.load().e2f_conv_gather_bf16x3(
            k, *_source_arrays(sources), w_hi.data_ptr(), w_lo.data_ptr(), None if b32 is None else b32.data_ptr(),
            None if bias_map is None else bias_map.data_ptr(), None if res is None else res.data_ptr(),
            None if o32 is None else o32.data_ptr(), None if ohi is None else ohi.data_ptr(),
            None if olo is None else olo.data_ptr(), n, h_in, w_in, cout, float(slope), stride, gh, gw, tw, th, nt, dy, dx,
            nph, tap0, oy, ox, ostep, oh, ow, sn_arr, out_nstride, _stream())
    _lib.check(st, "e2f_conv_gather_bf16x3")
    return _result(out, None if o32 is None else o32.permute(0, 3, 1, 2),
                   None if ohi is None else SplitNHWC(ohi, olo, (n, cout, oh, ow)))


def conv_frames(sources, weight, bias=None, negative_slope=1.0, residual=None, out="f32", into=None):
    """``conv3x3`` (k x k, stride 1, pad k//2, groups 1) whose sources, residual and outputs may be FRAME SLICES of
    (b, t, h, w, c) buffers (batch-strided NHWC views): the per-frame tensors of BidirectionalPropagation
    (feat_prop.py:88-149) are read and written in place — no ``x[:, i].contiguous()`` gathers, no stack / cat copies.
    sources: list of ``SplitNHWC`` (or fp32 tensors, split on the fly); ``into`` = (o32, ohi, olo) NHWC views or None."""
    cout, ks = weight.shape[0], weight.shape[2]
    pad = ks // 2
    _need_cuda(weight, bias, residual)
    splits = [split_nhwc(s_) for s_ in (sources if isinstance(sources, (list, tuple)) else [sources])]
    chans = [s_.shape[1] for s_ in splits]         # true channel counts (storage may be zero-padded to a multiple of 8)
    if sum(chans) != weight.shape[1]:
        raise ValueError(f"conv_frames: source channels {chans} do not add up to the weight's {weight.shape[1]} input channels")
    n, _, h, w = splits[0].shape
    w_hi, w_lo, _ = _derived_one(weight, ("conv3x3", tuple(chans), 1, 0), _conv3x3_operand, chans, 1, 0)
    taps = [(ky - pad, kx - pad) for ky in range(ks) for kx in range(ks)]
    return _conv_gather(splits, w_hi, w_lo, bias, None, residual, out, cout, 1, (h, w), taps, [(0, 0, 0)], 1, (h, w),
                        2.0 * n * h * w * cout * weight.shape[1] * ks * ks, slope=negative_slope, into=into)


def soft_split_weight(weight, c, k, transpose=False):
    """The conv weight (hidden, c, k, k) that ``soft_split`` runs: the Linear weight (hidden, c*k*k) viewed as a conv,
    or with ``transpose`` that of W^T for a (c*k*k, hidden) weight — SoftComp's token gradient unfold(dfeat) . W_sc."""
    w = weight.detach().float()
    if transpose:
        w = w.t()
    return w.reshape(w.shape[0], c, k, k)


def soft_split(x, weight, bias, kernel_size, stride, padding, transpose=False):
    """SoftSplit.forward (tfocal_transformer.py:39-46): ``Linear(unfold(x, k, s, p))`` evaluated as the k x k / stride-s
    convolution it is — an implicit GEMM whose A operand is fetched by TMA straight from the NHWC feature map; the
    k*k-times larger unfolded token matrix is never built.

    x (BT,C,H,W) fp32 (any memory format) or ``SplitNHWC``; weight (hidden, C*k*k) = ``ss.embedding.weight``;
    bias (hidden,).  Returns tokens (BT, fh*fw, hidden) fp32 — exactly ``embedding(unfold(x).permute(0, 2, 1))``."""
    k, s, p = _square(kernel_size, stride, padding)
    src = split_nhwc(x)
    n, c, h, w = src.shape
    hidden, ck = (weight.shape[1], weight.shape[0]) if transpose else tuple(weight.shape)
    if ck != c * k * k or k * k > 64 or c % 8:
        raise ValueError(f"soft_split: weight {tuple(weight.shape)} does not match C={c}, k={k}")
    _need_cuda(weight, bias)
    fh, fw = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    w_hi, w_lo = _derived_one(weight, ("soft_split_t" if transpose else "soft_split", c, k),
                              lambda wt: pack_conv3x3_weight(soft_split_weight(wt, c, k, transpose), [c], 1))
    taps = [(ky - p, kx - p) for ky in range(k) for kx in range(k)]
    tok = _conv_gather([src], w_hi, w_lo, bias, None, None, "f32", hidden, s, (fh, fw), taps, [(0, 0, 0)], 1,
                       (fh, fw), 2.0 * n * fh * fw * hidden * c * k * k)
    return tok.permute(0, 2, 3, 1).reshape(n, fh * fw, hidden)       # NHWC storage: a view


def _soft_comp_tables(k, s, p):
    """Phases and taps of the transposed conv that Linear + fold(k, s, p) is, for p == s (E2FGVI: 7 / 3 / 3): output
    pixel (s*a + ry, s*b + rx) sums token (a + 1 - dy, b + 1 - dx) times the (ky, kx) = (s*dy + ry, s*dx + rx) slice
    of the weight over all dy, dx with ky, kx < k.  Returns (taps [(dy_tok, dx_tok)], phases [(tap0, ry, rx)],
    kernel positions [(ky, kx)] in tap order)."""
    if p != s:
        raise NotImplementedError("soft_comp: the phase decomposition is implemented for padding == stride (7 / 3 / 3)")
    taps, phases, kpos = [], [], []
    for ry in range(s):
        for rx in range(s):
            phases.append((len(taps), ry, rx))
            for dy in range((k - 1 - ry) // s + 1):
                for dx in range((k - 1 - rx) // s + 1):
                    taps.append((1 - dy, 1 - dx))
                    kpos.append((s * dy + ry, s * dx + rx))
    return taps, phases, kpos


def soft_comp_weight(weight, k, s, p, transpose=False):
    """fp32 (C, k*k*hidden) operand of ``soft_comp``: the Linear weight (C*k*k, hidden) with its kernel positions in the
    phase tap order of ``_soft_comp_tables``, or with ``transpose`` that of W^T for a (hidden, C*k*k) weight — SoftSplit's
    input gradient fold(dT . W_ss)."""
    w = weight.detach().float()
    if transpose:
        w = w.t()
    hidden = w.shape[1]
    c = w.shape[0] // (k * k)
    _, _, kpos = _soft_comp_tables(k, s, p)
    order = torch.tensor([ky * k + kx for ky, kx in kpos], device=w.device)
    return w.reshape(c, k * k, hidden)[:, order, :].reshape(c, k * k * hidden)


def soft_comp(tokens, weight, bias, output_size, kernel_size, stride, padding, bias_map_extra=None, residual=None,
              out="f32", transpose=False):
    """SoftComp.forward up to (and including) the fold (tfocal_transformer.py:65-72, _hq.py:67-79):
    ``fold(Linear(tokens))`` evaluated as the transposed convolution it is, one implicit-GEMM launch over the nine
    output phases; the (C*k*k)-wide token matrix and the fold pass never exist.

    tokens (BT, fh, fw, hidden) fp32 or ``SplitMat``; weight (C*k*k, hidden) = ``sc.embedding.weight``; bias (C*k*k,);
    ``bias_map_extra``: the base model's ``sc.bias`` (C, H, W) parameter or None; ``residual`` (BT, C, H, W) fp32 added
    in the epilogue (enc_feat + trans_feat, e2fgvi.py:263).  Returns (BT, C, H, W) fp32 channels_last (out="f32"),
    a ``SplitNHWC`` (out="split", operand of the HQ model's bias_conv) or both."""
    k, s, p = _square(kernel_size, stride, padding)
    h, w = output_size
    fh, fw = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    hidden, ck = (weight.shape[0], weight.shape[1]) if transpose else (weight.shape[1], weight.shape[0])
    c = ck // (k * k)
    if isinstance(tokens, SplitMat):
        hi, lo = tokens.hi, tokens.lo
    else:
        _need_cuda(tokens)
        hi, lo = split_bf16(tokens)
    n = hi.numel() // (fh * fw * hidden)
    if hi.numel() != n * fh * fw * hidden or hidden % 64 or c * k * k != ck:
        raise ValueError(f"soft_comp: tokens {tuple(hi.shape)} / weight {tuple(weight.shape)} do not match output_size "
                         f"{output_size}")
    _need_cuda(weight, bias, bias_map_extra, residual)
    if residual is not None and tuple(residual.shape) != (n, c, h, w):
        raise ValueError(f"residual {tuple(residual.shape)} != {(n, c, h, w)}")
    taps, phases, kpos = _soft_comp_tables(k, s, p)
    src = SplitNHWC(hi.view(n, fh, fw, hidden), lo.view(n, fh, fw, hidden), (n, hidden, fh, fw))

    w_hi, w_lo = _derived_one(weight, ("soft_comp_t" if transpose else "soft_comp", k, s),
                              lambda wt: split_bf16(soft_comp_weight(wt, k, s, p, transpose)))

    def fold_bias():
        # fold of the Linear bias: every pixel receives b[c, ky, kx] from each token patch that covers it (border
        # pixels from fewer patches) + the base model's learned (C, H, W) bias map; layout [H][W][C]
        F = torch.nn.functional
        m = torch.zeros((1, c, h, w), dtype=torch.float32, device=weight.device)
        if bias is not None:
            cols = bias.detach().float().view(1, c * k * k, 1).expand(1, c * k * k, fh * fw)
            m = F.fold(cols, (h, w), (k, k), padding=(p, p), stride=(s, s))
        if bias_map_extra is not None:
            m = m + bias_map_extra.detach().float().view(1, c, h, w)
        return m[0].permute(1, 2, 0).contiguous()

    bparams = [q for q in (bias, bias_map_extra) if q is not None]
    bias_map = _derived(bparams, ("soft_comp_bias", h, w, k, s), fold_bias) if bparams else None
    return _conv_gather([src], w_hi, w_lo, None, bias_map, residual, out, c, 1, (fh, fw), taps, phases, s,
                        (h, w), 2.0 * n * fh * fw * hidden * c * k * k)


def pack_conv_kxn_weight(weight, co_pad, src_channels=None, groups=1):
    """fp32 (Cout, Cin/G, k, k) -> (hi, lo) bf16 (G*k*co_pad, k*chunks*64) in the operand order of ``e2f_conv_kxn_bf16x3``:
    row = g*k*co_pad + kx*co_pad + co, column = (ky*chunks + chunk)*64 + channel, the chunks of source 0 first, then source
    1 (the group-local input channel axis is the concatenation of the sources' per-group slices, like
    ``pack_conv3x3_weight``); zeros for co >= Cout/G and for padded channels."""
    cout, cin_g, kh, kw = weight.shape
    assert kh == kw and cout % groups == 0
    cog = cout // groups
    assert cog <= co_pad
    src_channels = [cin_g * groups] if src_channels is None else list(src_channels)
    cig = [c // groups for c in src_channels]
    assert sum(cig) == cin_g, (src_channels, groups, cin_g)
    nch = [(c + 63) // 64 for c in cig]
    chunks = sum(nch)
    w = weight.detach().float().view(groups, cog, cin_g, kh, kw)
    packed = torch.zeros((groups, kw, co_pad, kh, chunks * 64), dtype=torch.float32, device=weight.device)
    off, base = 0, 0
    for c, n_ in zip(cig, nch):
        # [g][co][c][ky][kx] -> [g][kx][co][ky][c]
        packed[:, :, :cog, :, base * 64: base * 64 + c] = w[:, :, off: off + c].permute(0, 4, 1, 3, 2)
        off += c
        base += n_
    return split_bf16(packed.view(groups * kw * co_pad, kh * chunks * 64))


def _kxn_co_pad(cout, ks):
    """Smallest padded channel count (multiple of 8, <= 32) with ks*co_pad % 16 == 0 that holds cout, or None."""
    for cp in (8, 16, 24, 32):
        if cp >= cout and (ks * cp) % 16 == 0:
            return cp
    return None


def conv_kxn(x, weight, bias=None, negative_slope=1.0, residual=None, out="f32", tanh_nchw=False, groups=1):
    """k x k / stride 1 / pad k//2 conv (k = 3 or 7) with FEW output channels per group (<= 32) on the "kx-in-N" kernel:
    SPyNet's 64 -> 32 / 32 -> 16 / 16 -> 2 convs (flow_comp.py:181-215), the decoder's output conv (e2fgvi.py:149-150) and
    the encoder's groups-of-32 conv (e2fgvi.py:97; two sources, group-wise concatenation never built).
    x: (N,C,H,W) fp32 / ``SplitNHWC`` or a list of up to two of them; residual (N,Cout,H,W) logical with NHWC storage;
    out = "f32" | "split" | "both"; ``tanh_nchw``: tanh + contiguous NCHW fp32 result (the prediction, e2fgvi.py:262)."""
    srcs = [split_nhwc(s_) for s_ in (x if isinstance(x, (list, tuple)) else [x])]
    n, _, h, w = srcs[0].shape
    chans = [s_.shape[1] for s_ in srcs]
    cout, cin_g, ks, ks2 = weight.shape
    co_pad = _kxn_co_pad(cout // groups, ks) if cout % groups == 0 else None
    if (ks != ks2 or ks not in (3, 7) or sum(chans) != cin_g * groups or co_pad is None or len(srcs) > 2
            or any(c % groups or s_.hi.shape[-1] != c for c, s_ in zip(chans, srcs))):
        raise ValueError(f"conv_kxn: unsupported weight {tuple(weight.shape)} / groups {groups} for sources {chans}")
    for s_ in srcs:
        if (s_.shape[0], s_.shape[2], s_.shape[3]) != (n, h, w) or not s_.hi.is_contiguous() or not s_.lo.is_contiguous():
            raise ValueError("conv_kxn: sources must be dense and share N, H, W")
    _need_cuda(weight, bias, residual)
    if tanh_nchw and out != "f32":
        raise ValueError("conv_kxn: tanh_nchw returns the fp32 NCHW tensor only")
    if out in ("split", "both") and (cout // groups) % 8:
        raise ValueError("conv_kxn: split output needs Cout / groups % 8 == 0")
    o32, ohi, olo = _outputs(out, ("f32", "split", "both"), (n, cout, h, w) if tanh_nchw else (n, h, w, cout),
                             weight.device)
    w_hi, w_lo = _derived_one(weight, ("kxn", co_pad, tuple(chans), groups), pack_conv_kxn_weight, co_pad, chans, groups)
    b32 = None if bias is None else bias.detach().float().contiguous()
    res = None
    if residual is not None:
        res = residual.permute(0, 2, 3, 1).contiguous().float()          # no-op for NHWC storage
    with _timed("conv3x3_bf16x3", 2.0 * n * h * w * cout * cin_g * ks * ks):
        st = _lib.load().e2f_conv_kxn_bf16x3(len(srcs), *_source_arrays(srcs), w_hi.data_ptr(), w_lo.data_ptr(),
                                             None if b32 is None else b32.data_ptr(),
                                             None if res is None else res.data_ptr(),
                                             None if o32 is None else o32.data_ptr(), None if ohi is None else ohi.data_ptr(),
                                             None if olo is None else olo.data_ptr(), n, h, w, cout, groups, co_pad, ks,
                                             float(negative_slope), 3 if tanh_nchw else 0, _stream())
    _lib.check(st, "e2f_conv_kxn_bf16x3")
    if tanh_nchw:
        return o32
    return _result(out, None if o32 is None else o32.permute(0, 3, 1, 2),
                   None if ohi is None else SplitNHWC(ohi, olo, (n, cout, h, w)))


def conv3x3_tanh_nchw(x, weight, bias):
    """``torch.tanh(F.conv2d(x, weight, bias, 1, 1))`` returned as a CONTIGUOUS (N, Cout, H, W) fp32 tensor: the
    decoder's 64 -> 3 output conv (e2fgvi.py:149-150) with the tanh of :262 and the NHWC -> NCHW layout change of the
    prediction fused into the conv epilogue, on the kx-in-N kernel.  x: (N,C,H,W) fp32 or ``SplitNHWC``."""
    c = x.shape[1]
    if tuple(weight.shape[1:]) != (c, 3, 3) or weight.shape[0] > 32:
        raise ValueError(f"conv3x3_tanh_nchw: weight {tuple(weight.shape)} (needs (Cout, {c}, 3, 3), Cout <= 32)")
    return conv_kxn(x, weight, bias, tanh_nchw=True)


# ------------------------------------------------------------------------------------------------- SPyNet glue
class FlowPyramid:
    """The six normalised pyramid levels of every local frame (``spynet_pyramid``)."""

    __slots__ = ("levels", "b", "l_t", "size", "up")

    def __init__(self, levels, b, l_t, size, up):
        self.levels, self.b, self.l_t, self.size, self.up = levels, b, l_t, size, up


def spynet_pyramid(masked_frames, num_local_frames, mean, std, unit=False):
    """Everything in front of SPyNet's first level, once per LOCAL FRAME (the reference does it per (ref, supp) pair):
    ``(x + 1) / 2`` and the 1/4 bilinear downsample of e2fgvi.py:210-218,247, the resize to multiples of 32, the
    normalisation and the five 2x2 average pools of flow_comp.py:95-115,152-158.  masked_frames (b,t,3,H,W) fp32 in
    [-1, 1], or in [0, 1] with ``unit`` (``e2f_spynet_pyramid_unit``: no ``(x + 1) / 2``); mean / std: the (1,3,1,1)
    buffers.  Returns a ``FlowPyramid``: levels[k] = (b*l_t, 3, h_up >> k, w_up >> k) fp32."""
    _need_cuda(masked_frames, mean, std)
    b, t, c, H, W = masked_frames.shape
    if c != 3:
        raise ValueError("spynet_pyramid: frames must have 3 channels")
    x = masked_frames.contiguous().float()
    l_t = int(num_local_frames)
    h, w = int(H * 0.25), int(W * 0.25)                 # F.interpolate(scale_factor=1/4, recompute_scale_factor=True)
    hu = h if h % 32 == 0 else 32 * (h // 32 + 1)
    wu = w if w % 32 == 0 else 32 * (w // 32 + 1)
    n = b * l_t
    sizes = [n * 3 * (hu >> k) * (wu >> k) for k in range(6)]
    buf = torch.empty(sum(sizes), dtype=torch.float32, device=x.device)
    m32, s32 = mean.detach().float().contiguous(), std.detach().float().contiguous()
    fn = "e2f_spynet_pyramid_unit" if unit else "e2f_spynet_pyramid"
    st = getattr(_lib.load(), fn)(x.data_ptr(), buf.data_ptr(), b, t, l_t, H, W, h, w, hu, wu, m32.data_ptr(),
                                  s32.data_ptr(), _stream())
    _lib.check(st, fn)
    levels, off = [], 0
    for k in range(6):
        levels.append(buf[off: off + sizes[k]].view(n, 3, hu >> k, wu >> k))
        off += sizes[k]
    return FlowPyramid(levels, b, l_t, (h, w), (hu, wu))


def spynet_level_input(pyr, k, prev_flow, lead=3):
    """Input of one SPyNet level for all 2*b*(l_t-1) (ref, supp) pairs (forward pairs, then backward pairs): x2 flow
    upsample * 2, border warp of the support frame, ``cat([ref, warped, flow_up])`` (flow_comp.py:121-133) as the
    row-gapped ``RowsNHWC`` operand of the level's first 7x7 conv, plus ``flow_up`` (P, hk, wk, 2) fp32 — the residual the
    level's last conv adds.  pyr: ``FlowPyramid``; k: pyramid level (5 = coarsest); prev_flow (P, hk/2, wk/2, 2) or None."""
    img = pyr.levels[k]
    _, _, hk, wk = img.shape
    P = 2 * pyr.b * (pyr.l_t - 1)
    if prev_flow is not None:
        if tuple(prev_flow.shape) != (P, hk // 2, wk // 2, 2) or not prev_flow.is_contiguous() or prev_flow.dtype != torch.float32:
            raise ValueError(f"spynet_level_input: prev_flow {tuple(prev_flow.shape)} != {(P, hk // 2, wk // 2, 2)} fp32 contiguous")
    hi, lo = _rows_pair(P, hk, wk, lead, 8, img.device)
    flow_up = torch.empty((P, hk, wk, 2), dtype=torch.float32, device=img.device)
    st =_lib.load().e2f_spynet_level_input(img.data_ptr(), None if prev_flow is None else prev_flow.data_ptr(),
                                            hi.data_ptr(), lo.data_ptr(), flow_up.data_ptr(), pyr.b, pyr.l_t, hk, wk, lead,
                                            _stream())
    _lib.check(st, "e2f_spynet_level_input")
    return RowsNHWC(hi, lo, (P, 8, hk, wk), lead, 8), flow_up


def spynet_final(flow, pyr):
    """flow_comp.py:160-167 for both directions: level-0 flow (P, h_up, w_up, 2) fp32 -> (flows_forward, flows_backward),
    each (b, l_t-1, 2, h, w) fp32 (resize to (h, w), u * w / w_up, v * h / h_up)."""
    _need_cuda(flow)
    h, w = pyr.size
    hu, wu = pyr.up
    P = 2 * pyr.b * (pyr.l_t - 1)
    if tuple(flow.shape) != (P, hu, wu, 2) or not flow.is_contiguous() or flow.dtype != torch.float32:
        raise ValueError(f"spynet_final: flow {tuple(flow.shape)} != {(P, hu, wu, 2)} fp32 contiguous")
    fwd = torch.empty((pyr.b, pyr.l_t - 1, 2, h, w), dtype=torch.float32, device=flow.device)
    bwd = torch.empty((pyr.b, pyr.l_t - 1, 2, h, w), dtype=torch.float32, device=flow.device)
    st = _lib.load().e2f_spynet_final(flow.data_ptr(), fwd.data_ptr(), bwd.data_ptr(), pyr.b, pyr.l_t, h, w, hu, wu, _stream())
    _lib.check(st, "e2f_spynet_final")
    return fwd, bwd


# ---------------------------------------------------------------------------------------------- SPyNet backward
def spynet_final_backward(d_forward, d_backward, pyr):
    """Adjoint of ``spynet_final``: d flows_forward / d flows_backward (b, l_t-1, 2, h, w) -> d level-0 flow
    (P, h_up, w_up, 2) fp32."""
    _need_cuda(d_forward, d_backward)
    h, w = pyr.size
    hu, wu = pyr.up
    P = 2 * pyr.b * (pyr.l_t - 1)
    shape = (pyr.b, pyr.l_t - 1, 2, h, w)
    if tuple(d_forward.shape) != shape or tuple(d_backward.shape) != shape:
        raise ValueError(f"spynet_final_backward: gradients {tuple(d_forward.shape)} / {tuple(d_backward.shape)} != {shape}")
    gf, gb = d_forward.contiguous().float(), d_backward.contiguous().float()
    dflow = torch.empty((P, hu, wu, 2), dtype=torch.float32, device=gf.device)
    st = _lib.load().e2f_spynet_final_backward(gf.data_ptr(), gb.data_ptr(), dflow.data_ptr(), pyr.b, pyr.l_t, h, w, hu, wu,
                                               _stream())
    _lib.check(st, "e2f_spynet_final_backward")
    return dflow


def spynet_level_input_backward(d_in, dflow, pyr, k, flow_up):
    """Adjoint of ``spynet_level_input`` with respect to the coarser level's flow.  d_in (P, hk, wk, 8) fp32: gradient
    of the level's conv input (channels 3..7 are read); dflow (P, hk, wk, 2): gradient of the level's output flow;
    flow_up: what ``spynet_level_input`` returned.  Returns d prev_flow (P, hk/2, wk/2, 2) fp32."""
    img = pyr.levels[k]
    _, _, hk, wk = img.shape
    P = 2 * pyr.b * (pyr.l_t - 1)
    for name, t, c in (("d_in", d_in, 8), ("dflow", dflow, 2), ("flow_up", flow_up, 2)):
        if tuple(t.shape) != (P, hk, wk, c) or not t.is_contiguous() or t.dtype != torch.float32:
            raise ValueError(f"spynet_level_input_backward: {name} {tuple(t.shape)} != {(P, hk, wk, c)} fp32 contiguous")
    dprev = torch.empty((P, hk // 2, wk // 2, 2), dtype=torch.float32, device=img.device)
    st = _lib.load().e2f_spynet_level_input_backward(d_in.data_ptr(), dflow.data_ptr(), img.data_ptr(), flow_up.data_ptr(),
                                                     dprev.data_ptr(), pyr.b, pyr.l_t, hk, wk, _stream())
    _lib.check(st, "e2f_spynet_level_input_backward")
    return dprev


def conv_dgrad_weight(weight):
    """The input gradient's weight: fp32 (Cout, Cin, k, k) -> Wt (Cin, Cout, k, k), Wt[ci][co][ky][kx] =
    W[co][ci][k-1-ky][k-1-kx] (rotated by 180 degrees, in / out swapped)."""
    return weight.detach().float().flip(2, 3).transpose(0, 1).contiguous()


def pack_conv_dgrad_weight(weight, dy_rows_cin=0):
    """``conv_dgrad_weight`` packed as the forward packs a weight for that dY: window-packed K for a row-gapped dY of
    ``dy_rows_cin`` channels (``pack_conv_rows_weight``), tap-major 64-channel chunks for a dense one."""
    wt = conv_dgrad_weight(weight)
    if dy_rows_cin:
        return pack_conv_rows_weight(wt, dy_rows_cin)
    return pack_conv3x3_weight(wt, [weight.shape[0]])


def conv2d_dgrad(dy, weight, act=None, out="f32", out_lead=3):
    """Input gradient of a 7x7 / stride 1 / pad 3 conv (``e2f_conv2d_dgrad_bf16x3``): dy = the gradient of its output
    as a ``RowsNHWC`` (lead 3) or dense ``SplitNHWC``; weight = the forward's nn.Conv2d weight (Cout, Cin, 7, 7).
    ``act`` (``RowsNHWC`` / ``SplitNHWC`` with Cin channels, the ReLU output the conv read, or None) multiplies the result
    by ReLU's derivative.  Returns (dx fp32 (N, H, W, Cin), operand): operand = None (out "f32"), a ``RowsNHWC`` with
    ``out_lead`` (out "rows") or a ``SplitNHWC`` (out "split") of dx: the next input gradient's dy."""
    cout, cin, ks, _ = weight.shape
    if ks != 7 or tuple(weight.shape[2:]) != (7, 7):
        raise ValueError(f"conv2d_dgrad: 7x7 kernels only, got {tuple(weight.shape)}")
    rows = isinstance(dy, RowsNHWC)
    if rows and dy.lead != 3:
        raise ValueError("conv2d_dgrad: a row-gapped dy needs lead 3")
    dy_c = dy.cin if rows else dy.hi.shape[-1]
    if dy.shape[1] != cout:
        raise ValueError(f"conv2d_dgrad: dy has {dy.shape[1]} channels, the weight {cout} outputs")
    n, _, h, w = dy.shape
    _need_cuda(weight, dy.hi)
    act_ptr, act_lead = None, 0
    if act is not None:
        if act.shape != (n, cin, h, w) or (isinstance(act, RowsNHWC) and act.cin != cin) or (
                isinstance(act, SplitNHWC) and act.hi.shape[-1] != cin):
            raise ValueError(f"conv2d_dgrad: act {act.shape} does not match ({n}, {cin}, {h}, {w})")
        act_ptr, act_lead = act.hi.data_ptr(), (act.lead if isinstance(act, RowsNHWC) else 0)
    dx, ohi, olo = _outputs(out, ("f32", "rows", "split"), (n, h, w, cin), weight.device)
    if dx is None:                    # every mode returns dx; "rows" / "split" add an operand
        dx = torch.empty((n, h, w, cin), dtype=torch.float32, device=weight.device)
    if out == "rows":
        ohi, olo = _rows_pair(n, h, w, out_lead, cin, weight.device)
    lead = out_lead if out == "rows" else 0
    w_hi, w_lo = _derived_one(weight, ("dgrad", dy_c if rows else 0), pack_conv_dgrad_weight, dy_c if rows else 0)
    with _timed(f"conv2d_dgrad_c{cin}", 2.0 * n * h * w * cout * cin * 49):
        st = _lib.load().e2f_conv2d_dgrad_bf16x3(dy.hi.data_ptr(), dy.lo.data_ptr(), dy_c, 3 if rows else 0,
                                                 w_hi.data_ptr(), w_lo.data_ptr(), act_ptr, act_lead, dx.data_ptr(),
                                                 None if ohi is None else ohi.data_ptr(),
                                                 None if olo is None else olo.data_ptr(), lead, n, h, w, cin, _stream())
    _lib.check(st, "e2f_conv2d_dgrad_bf16x3")
    if out == "rows":
        return dx, RowsNHWC(ohi, olo, (n, cin, h, w), out_lead, cin)
    if out == "split":
        return dx, SplitNHWC(ohi, olo, (n, cin, h, w))
    return dx, None


def conv2d_wgrad(dy, x, cin, with_bias=True):
    """(dW fp32 (Cout, cin, 7, 7), db fp32 (Cout,) or None) of a 7x7 / stride 1 / pad 3 conv (``e2f_conv2d_wgrad_bf16x3``)
    from dy fp32 (N, H, W, Cout) (Cout padded to a multiple of 8 here) and the forward's operand x (``RowsNHWC`` or dense
    ``SplitNHWC``); the first ``cin`` input channels are returned."""
    n, h, w, cout = dy.shape
    _need_cuda(dy, x.hi)
    dy = dy.contiguous().float()
    cpad = -(-cout // 8) * 8
    if cpad != cout:
        dy = torch.nn.functional.pad(dy, (0, cpad - cout))
    rows = isinstance(x, RowsNHWC)
    xc = x.cin if rows else x.hi.shape[-1]
    if x.shape[0] != n or tuple(x.shape[2:]) != (h, w) or cin > xc:
        raise ValueError(f"conv2d_wgrad: x {x.shape} does not match dy {tuple(dy.shape)} / cin {cin}")
    lib = _lib.load()
    elems = lib.e2f_conv2d_wgrad_work_elems(n, h, w, xc, cpad)
    if elems < 0:
        _lib.check(int(elems), "e2f_conv2d_wgrad_work_elems")
    work = torch.empty(int(elems), dtype=torch.float32, device=dy.device)
    dw = torch.empty(cpad, xc, 7, 7, dtype=torch.float32, device=dy.device)
    db = torch.empty(cpad, dtype=torch.float32, device=dy.device) if with_bias else None
    with _timed(f"conv2d_wgrad_c{cout}", 2.0 * n * h * w * cout * xc * 49):
        st = lib.e2f_conv2d_wgrad_bf16x3(dy.data_ptr(), x.hi.data_ptr(), x.lo.data_ptr(), x.lead if rows else 0,
                                         dw.data_ptr(), None if db is None else db.data_ptr(), work.data_ptr(), n, h, w, xc,
                                         cpad, _stream())
    _lib.check(st, "e2f_conv2d_wgrad_bf16x3")
    if cpad != cout or cin != xc:
        dw = dw[:cout, :cin].contiguous()
    if db is not None and cpad != cout:
        db = db[:cout].contiguous()
    return dw, db


# ------------------------------------------------------------------------------------- encoder / decoder backward
def conv_dgrad_s2_taps():
    """(phase, ky, kx) of the stride-2 / pad-1 3x3 input gradient's taps in the kernel's order: phase ph = 2 (y % 2) +
    (x % 2) of the output pixel (y, x) takes the taps with ky = y + 1 and kx = x + 1 (mod 2), in increasing order; tap
    (ky, kx) of pixel (2 gy + oy, 2 gx + ox) reads dY at (gy + (oy + 1 - ky) / 2, gx + (ox + 1 - kx) / 2)."""
    return [(ph, ky, kx) for ph in range(4) for ky in range(3) for kx in range(3)
            if (ph // 2 + 1 - ky) % 2 == 0 and (ph % 2 + 1 - kx) % 2 == 0]


def source_dgrad_weight(weight, groups=1, src_channels=None, source=0):
    """The stride-1 input gradient's weight for one source of a (grouped, multi-source) conv: fp32 (Cout, Cin/G, k, k)
    -> a conv weight (C_s, Cout/G, k, k), G groups, with Wt[g cig + ci][co][ky][kx] = W[g cog + co][off + ci][k-1-ky]
    [k-1-kx] (cig = C_s / G, off = the source's offset in the group-wise concatenation)."""
    cout, cin_g, k, _ = weight.shape
    src_channels = [cin_g * groups] if src_channels is None else list(src_channels)
    cig = src_channels[source] // groups
    off = sum(c // groups for c in src_channels[:source])
    w = weight.detach().float().view(groups, cout // groups, cin_g, k, k)[:, :, off: off + cig]
    return w.transpose(1, 2).reshape(groups * cig, cout // groups, k, k).flip(2, 3).contiguous()


def pack_conv_dgrad_s2_weight(weight, src_channels=None, source=0):
    """The stride-2 input gradient's weight (groups 1): fp32 (Cout, Cin, 3, 3) -> (hi, lo) bf16 (C_s, 9 *
    ceil(Cout / 64) * 64), taps in ``conv_dgrad_s2_taps`` order, Wt[ci][tap][co] = W[co][off + ci][ky][kx]."""
    cout, cin = weight.shape[:2]
    src_channels = [cin] if src_channels is None else list(src_channels)
    off, cs = sum(src_channels[:source]), src_channels[source]
    idx = torch.tensor([3 * ky + kx for _, ky, kx in conv_dgrad_s2_taps()], device=weight.device)
    p = weight.detach().float()[:, off: off + cs].reshape(cout, cs, 9).index_select(2, idx).permute(1, 2, 0)
    kc = -(-cout // 64) * 64
    p = torch.nn.functional.pad(p, (0, kc - cout))
    return split_bf16(p.reshape(cs, 9 * kc))


def _dgrad_operand(weight, groups, src_channels, source, stride, rows_cin):
    """(hi, lo, effective groups) of an input gradient's weight, the value of its ("dgrad", ...) ``_derived`` entry."""
    if stride == 2:
        return (*pack_conv_dgrad_s2_weight(weight, src_channels, source), 1)
    wt = source_dgrad_weight(weight, groups, src_channels, source)
    if rows_cin:
        return (*pack_conv_rows_weight(wt, rows_cin), 1)
    return _conv3x3_operand(wt, [weight.shape[0]], groups, 0)


def conv_dgrad(dy, weight, groups=1, stride=1, in_size=None, src_channels=None, source=0, act=None, residual=None,
               out="f32"):
    """Input gradient of one source of a k x k conv (``e2f_conv_dgrad_bf16x3``): k = 3 or 7 at stride 1 (pad k // 2),
    k = 3 at stride 2 (pad 1); groups 1 / 2 / 4 / 8; the forward read ``src_channels`` group-wise concatenated and this
    is the gradient of source ``source``.  dy: the gradient of the conv's output as a dense ``SplitNHWC``, or a
    ``RowsNHWC`` with lead k // 2 (stride 1, groups 1).  weight: the forward's nn.Conv2d weight.  in_size: the forward's
    input (h, w) (default: dy's size, stride 1).  The result is (acc + residual) * LeakyReLU(0.2)'(act): ``residual``
    fp32 (N, h, w, C_s) NHWC or None, ``act`` the source's ``SplitNHWC`` (its hi part decides) or None.
    out = "f32": dx fp32 (N, h, w, C_s) NHWC; "split": its ``SplitNHWC``; "both": (dx, SplitNHWC)."""
    cout, cin_g, ks, _ = weight.shape
    src_channels = [cin_g * groups] if src_channels is None else list(src_channels)
    cs = src_channels[source]
    rows = isinstance(dy, RowsNHWC)
    if dy.shape[1] != cout or sum(src_channels) != cin_g * groups:
        raise ValueError(f"conv_dgrad: dy {dy.shape} / sources {src_channels} do not match the weight {tuple(weight.shape)}")
    if rows and dy.lead != ks // 2:
        raise ValueError(f"conv_dgrad: a row-gapped dy needs lead {ks // 2}")
    n, _, h_o, w_o = dy.shape
    h, w = in_size if in_size is not None else (h_o, w_o)
    if ((h - 1) // stride + 1, (w - 1) // stride + 1) != (h_o, w_o):
        raise ValueError(f"conv_dgrad: input size {(h, w)} does not give dy's {(h_o, w_o)} at stride {stride}")
    _need_cuda(weight, dy.hi, residual)
    dy_c = dy.cin if rows else dy.hi.shape[-1]
    act_ptr = None
    if act is not None:
        if act.shape != (n, cs, h, w) or act.hi.shape[-1] != cs:
            raise ValueError(f"conv_dgrad: act {act.shape} does not match ({n}, {cs}, {h}, {w})")
        act_ptr = act.hi.data_ptr()
    res = None
    if residual is not None:
        if tuple(residual.shape) != (n, h, w, cs):
            raise ValueError(f"conv_dgrad: residual {tuple(residual.shape)} != {(n, h, w, cs)}")
        res = residual.contiguous().float()
    dx, ohi, olo = _outputs(out, ("f32", "split", "both"), (n, h, w, cs), weight.device)
    rows_cin = dy_c if rows else 0
    w_hi, w_lo, g_eff = _derived_one(weight, ("dgrad", tuple(src_channels), groups, source, stride, rows_cin),
                                     _dgrad_operand, groups, src_channels, source, stride, rows_cin)
    with _timed(f"conv_dgrad_c{cs}", 2.0 * n * h_o * w_o * cout * (cs // groups) * ks * ks):
        st = _lib.load().e2f_conv_dgrad_bf16x3(dy.hi.data_ptr(), dy.lo.data_ptr(), dy_c, dy.lead if rows else 0,
                                               w_hi.data_ptr(), w_lo.data_ptr(), act_ptr,
                                               None if res is None else res.data_ptr(),
                                               None if dx is None else dx.data_ptr(),
                                               None if ohi is None else ohi.data_ptr(),
                                               None if olo is None else olo.data_ptr(), n, h, w, cs, g_eff, ks, stride,
                                               _stream())
    _lib.check(st, "e2f_conv_dgrad_bf16x3")
    return _result(out, dx, None if ohi is None else SplitNHWC(ohi, olo, (n, cs, h, w)))


def conv3x3_wgrad(dy, sources, groups=1, stride=1, with_bias=True, cin=None):
    """(dW fp32 (Cout, Cin/G, 3, 3), db fp32 (Cout,) or None) of a 3x3 / pad 1 conv (``e2f_conv3x3_wgrad_bf16x3``) from dy
    fp32 (N, h_o, w_o, Cout) NHWC (Cout padded to a multiple of 8 here) and the forward's operands: a list of one or two
    dense ``SplitNHWC`` read group-wise concatenated, or one ``RowsNHWC`` with lead 1.  ``cin``: keep the first cin input
    channels (a row-gapped source's padding channels get their own, zero-valued, gradient)."""
    sources = list(sources) if isinstance(sources, (list, tuple)) else [sources]
    n, h_o, w_o, cout = dy.shape
    _need_cuda(dy, *[s_.hi for s_ in sources])
    rows = isinstance(sources[0], RowsNHWC)
    if rows and (len(sources) != 1 or sources[0].lead != 1):
        raise ValueError("conv3x3_wgrad: a row-gapped operand must be the only source and have lead 1")
    h, w = sources[0].shape[2:]
    for s_ in sources:
        if s_.shape[0] != n or tuple(s_.shape[2:]) != (h, w):
            raise ValueError("conv3x3_wgrad: sources must share N, H, W")
    if ((h - 1) // stride + 1, (w - 1) // stride + 1) != (h_o, w_o):
        raise ValueError(f"conv3x3_wgrad: dy {tuple(dy.shape)} is not the stride-{stride} output of {(h, w)}")
    dy = dy.contiguous().float()
    cpad = -(-cout // 8) * 8
    if cpad != cout:
        dy = torch.nn.functional.pad(dy, (0, cpad - cout))
    lib = _lib.load()
    x_c = [s_.cin if rows else s_.hi.shape[-1] for s_ in sources]
    xc = sum(x_c)
    elems = lib.e2f_conv3x3_wgrad_work_elems(n, h, w, xc, cpad, groups, stride)
    if elems < 0:
        _lib.check(int(elems), "e2f_conv3x3_wgrad_work_elems")
    work = torch.empty(int(elems), dtype=torch.float32, device=dy.device)
    dw = torch.empty(cpad, xc // groups, 3, 3, dtype=torch.float32, device=dy.device)
    db = torch.empty(cpad, dtype=torch.float32, device=dy.device) if with_bias else None
    hi_p, lo_p, c_p = _source_arrays(sources)
    with _timed(f"conv3x3_wgrad_c{cout}", 2.0 * n * h_o * w_o * cout * (xc // groups) * 9):
        st = lib.e2f_conv3x3_wgrad_bf16x3(dy.data_ptr(), len(sources), hi_p, lo_p, c_p, 1 if rows else 0, dw.data_ptr(),
                                          None if db is None else db.data_ptr(), work.data_ptr(), n, h, w, cpad, groups,
                                          stride, _stream())
    _lib.check(st, "e2f_conv3x3_wgrad_bf16x3")
    keep = xc // groups if cin is None else cin
    if cpad != cout or keep != xc // groups:
        dw = dw[:cout, :keep].contiguous()
    if db is not None and cpad != cout:
        db = db[:cout].contiguous()
    return dw, db


def upsample2x_backward(dy, act=None, out="f32"):
    """Adjoint of ``upsample2x_split`` (x2 bilinear, align_corners=True): dy fp32 (N, 2H, 2W, C) NHWC -> dx (N, H, W, C)
    NHWC, times LeakyReLU(0.2)'(act) when ``act`` (fp32 (N, C, H, W), the upsampled LeakyReLU output) is given.
    out = "f32" | "split" | "both" as ``conv_dgrad``."""
    _need_cuda(dy, act)
    n, oh, ow, c = dy.shape
    h, w = oh // 2, ow // 2
    if (oh, ow) != (2 * h, 2 * w) or c % 8:
        raise ValueError(f"upsample2x_backward: dy {tuple(dy.shape)} (even H, W and C % 8 == 0)")
    a = None
    if act is not None:
        if tuple(act.shape) != (n, c, h, w):
            raise ValueError(f"upsample2x_backward: act {tuple(act.shape)} != {(n, c, h, w)}")
        a = act.permute(0, 2, 3, 1).contiguous().float()        # no-op for channels_last
    dy = dy.contiguous().float()
    dx, hi, lo = _outputs(out, ("f32", "split", "both"), (n, h, w, c), dy.device)
    with _timed("upsample2x_backward", float(dy.numel() * 4 + n * h * w * c * 4 * (1 + (a is not None)))):
        st = _lib.load().e2f_upsample2x_backward(dy.data_ptr(), None if a is None else a.data_ptr(),
                                                 None if dx is None else dx.data_ptr(), None if hi is None else hi.data_ptr(),
                                                 None if lo is None else lo.data_ptr(), n, h, w, c, _stream())
    _lib.check(st, "e2f_upsample2x_backward")
    return _result(out, dx, None if hi is None else SplitNHWC(hi, lo, (n, c, h, w)))


def tanh_backward_rows(dout, out, lead=1):
    """dY = dOut * (1 - out^2) of the prediction ``out = tanh(conv)`` (both fp32 (N, C, H, W), C <= 8): returns (dy fp32
    (N, H, W, 8) NHWC, channels >= C zero — the weight gradient's operand; the row-gapped ``RowsNHWC`` of dy with
    ``lead`` — the input gradient's operand)."""
    _need_cuda(dout, out)
    n, c, h, w = out.shape
    if tuple(dout.shape) != (n, c, h, w):
        raise ValueError(f"tanh_backward_rows: dout {tuple(dout.shape)} != out {tuple(out.shape)}")
    dout, out = dout.contiguous().float(), out.contiguous().float()
    dy = torch.empty((n, h, w, 8), dtype=torch.float32, device=out.device)
    hi, lo = _rows_pair(n, h, w, lead, 8, out.device)
    with _timed("tanh_backward_rows", float(out.numel() * 8 + dy.numel() * 4 + hi.numel() * 4)):
        st = _lib.load().e2f_tanh_backward_rows(dout.data_ptr(), out.data_ptr(), dy.data_ptr(), hi.data_ptr(),
                                                lo.data_ptr(), n, c, h, w, lead, _stream())
    _lib.check(st, "e2f_tanh_backward_rows")
    return dy, RowsNHWC(hi, lo, (n, c, h, w), lead, 8)


def leaky_relu_backward(dy, act, slope=0.2, out="both"):
    """dy * LeakyReLU(slope)'(act) for two fp32 NHWC tensors of one shape (N, H, W, C): out = "f32" | "split" | "both"
    as ``conv_dgrad``."""
    _need_cuda(dy, act)
    if dy.shape != act.shape or dy.dim() != 4:
        raise ValueError(f"leaky_relu_backward: dy {tuple(dy.shape)} and act {tuple(act.shape)} must be one (N, H, W, C)")
    dy, act = dy.contiguous().float(), act.contiguous().float()
    n, h, w, c = dy.shape
    dx, hi, lo = _outputs(out, ("f32", "split", "both"), dy.shape, dy.device)
    with _timed("leaky_relu_backward", float(dy.numel() * (8 + 4 * (dx is not None) + 4 * (hi is not None)))):
        st = _lib.load().e2f_leaky_relu_backward(dy.data_ptr(), act.data_ptr(), None if dx is None else dx.data_ptr(),
                                                 None if hi is None else hi.data_ptr(), None if lo is None else lo.data_ptr(),
                                                 dy.numel(), float(slope), _stream())
    _lib.check(st, "e2f_leaky_relu_backward")
    return _result(out, dx, None if hi is None else SplitNHWC(hi, lo, (n, c, h, w)))


def attention_flops(B, T, H, W, C, window_size, expand_size, focal_window, use_pooled=True):
    """Algorithmic FLOPs of one attention launch as the REFERENCE counts keys (SURVEY §8d): QK^T + PV over
    T*(own window + listed ring keys incl. duplicates + fh*fw pooled keys incl. masked ones) keys per query."""
    wh, ww = window_size
    eh, ew = expand_size
    ring = 4 * (wh * ww - (wh - eh) * (ww - ew)) if (eh or ew) else 0
    keys = T * (wh * ww + ring + (focal_window[0] * focal_window[1] if use_pooled else 0))
    return 4.0 * B * T * H * W * keys * C


def invalidate_weight_caches():
    """Drop every operand derived from model parameters (bf16 splits, packed conv / gather-conv / DCN weights, folded
    bias maps).  The cache keys on ``(param._version, data_ptr)``; in-place updates through ``param.data`` (``nn.init``
    on ``.data``, EMA ``p.data.copy_()``, manual surgery) do NOT bump the version, so call this after such updates.
    ``InpaintGenerator.init_weights`` and ``load_state_dict`` do it for you."""
    _DERIVED.clear()


_GRAPH_REPLAY_LAUNCHES = 0


def note_graph_replay(kernel_launches):
    """A CUDA-graph replay relaunches the kernels recorded at capture time without passing through the C ABI's launch
    functions; ``e2fgvi_b200.graph`` reports them here so that ``launch_count`` keeps counting kernels, not host calls."""
    global _GRAPH_REPLAY_LAUNCHES
    _GRAPH_REPLAY_LAUNCHES += int(kernel_launches)


def launch_count():
    """Kernels of this library launched so far: host-side launches (``e2f_launch_count``) + kernels replayed by graphs."""
    return int(_lib.load().e2f_launch_count()) + _GRAPH_REPLAY_LAUNCHES


# ---------------------------------------------------------------------------------------------------------------------
# Temporal PatchGAN discriminator layers (model/e2fgvi.py:271-344): Conv3d, kernel (3, 5, 5), stride (1, 2, 2), zero
# padding (1, pad, pad).  Activations are NDHWC; see include/e2fgvi_b200.h for the operand layouts.
def dis_out_size(s, pad):
    return (s + 2 * pad - 5) // 2 + 1


def dis_dgrad_taps(pad):
    """Tap order of the input-gradient weight: phase by phase (ph = 2 (y % 2) + x % 2), taps 25 kt + 5 ky + kx with
    ky = y + pad and kx = x + pad (mod 2) in increasing order."""
    taps = []
    for ph in range(4):
        oy, ox = ph >> 1, ph & 1
        taps += [25 * kt + 5 * ky + kx for kt in range(3) for ky in range(5) for kx in range(5)
                 if (oy + pad - ky) % 2 == 0 and (ox + pad - kx) % 2 == 0]
    return taps


def dis_pack_weight(weight, cin_s):
    """fp32 [cout, cin, 3, 5, 5] -> bf16 (hi, lo) [cout, 75 * ceil(cin_s / 64) * 64] in tap-major K order."""
    cout, cin = weight.shape[:2]
    kc = -(-cin_s // 64) * 64
    p = weight.detach().float().permute(0, 2, 3, 4, 1).reshape(cout, 75, cin)
    p = torch.nn.functional.pad(p, (0, kc - cin))
    return split_bf16(p.reshape(cout, 75 * kc))


def dis_pack_weight_t(weight, pad, cin_s):
    """fp32 [cout, cin, 3, 5, 5] -> the input gradient's bf16 (hi, lo) [cin_s, 75 * ceil(cout / 64) * 64]: flipped
    roles (rows = input channels, zero rows past cin), taps in dis_dgrad_taps(pad) order."""
    cout, cin = weight.shape[:2]
    kc = -(-cout // 64) * 64
    idx = torch.tensor(dis_dgrad_taps(pad), device=weight.device)
    p = weight.detach().float().permute(1, 2, 3, 4, 0).reshape(cin, 75, cout).index_select(1, idx)
    p = torch.nn.functional.pad(p, (0, kc - cout, 0, 0, 0, cin_s - cin))
    return split_bf16(p.reshape(cin_s, 75 * kc))


def dis_conv3d(x_hi, x_lo, w_hi, w_lo, bias, cout, pad, leaky):
    """One discriminator conv on the split operand x [b, t, h, w, cin]: returns (fp32 out, out_hi, out_lo), each
    [b, t, h_o, w_o, cout], with LeakyReLU(0.2) fused when ``leaky``."""
    _need_cuda(x_hi, x_lo, w_hi, w_lo, bias)
    b, t, h, w, cin = x_hi.shape
    ho, wo = dis_out_size(h, pad), dis_out_size(w, pad)
    out = torch.empty(b, t, ho, wo, cout, dtype=torch.float32, device=x_hi.device)
    hi = torch.empty(out.shape, dtype=torch.bfloat16, device=x_hi.device)
    lo = torch.empty_like(hi)
    with _timed(f"dis_conv3d_c{cout}", 2.0 * b * t * ho * wo * cout * cin * 75):
        st = _lib.load().e2f_dis_conv3d(x_hi.data_ptr(), x_lo.data_ptr(), cin, w_hi.data_ptr(), w_lo.data_ptr(),
                                        None if bias is None else bias.data_ptr(), out.data_ptr(), hi.data_ptr(),
                                        lo.data_ptr(), b, t, h, w, cout, pad, 1 if leaky else 0, _stream())
    _lib.check(st, "e2f_dis_conv3d")
    return out, hi, lo


def dis_conv3d_dgrad(dy_hi, dy_lo, wt_hi, wt_lo, act, h_in, w_in, cin_s, pad, split=False):
    """Input gradient fp32 [b, t, h_in, w_in, cin_s] of a discriminator conv from the split dy [b, t, h_o, w_o, cout];
    times LeakyReLU(0.2)'s derivative at ``act`` (bf16, the hi part of the layer's input) unless ``act`` is None.
    Returns (dx, dx_hi, dx_lo); the bf16 split, the next input gradient's operand, only when ``split``."""
    _need_cuda(dy_hi, dy_lo, wt_hi, wt_lo, act)
    b, t, _, _, cout = dy_hi.shape
    dx = torch.empty(b, t, h_in, w_in, cin_s, dtype=torch.float32, device=dy_hi.device)
    hi = lo = None
    if split:
        hi = torch.empty(dx.shape, dtype=torch.bfloat16, device=dx.device)
        lo = torch.empty_like(hi)
    with _timed(f"dis_dgrad_c{cin_s}", 2.0 * b * t * dy_hi.shape[2] * dy_hi.shape[3] * cout * cin_s * 75):
        st = _lib.load().e2f_dis_conv3d_dgrad(dy_hi.data_ptr(), dy_lo.data_ptr(), cout, wt_hi.data_ptr(), wt_lo.data_ptr(),
                                              dx.data_ptr(), None if hi is None else hi.data_ptr(),
                                              None if lo is None else lo.data_ptr(),
                                              None if act is None else act.data_ptr(), b, t, h_in, w_in, cin_s, pad,
                                              _stream())
    _lib.check(st, "e2f_dis_conv3d_dgrad")
    return dx, hi, lo


def dis_conv3d_wgrad(dy, x_hi, x_lo, cin, pad, with_bias):
    """(dW fp32 [cout, cin, 3, 5, 5], db fp32 [cout] or None) of a discriminator conv from dy fp32 [b, t, h_o, w_o,
    cout] and the forward's split operand x [b, t, h, w, x_cs]: the kernel computes all x_cs channels (the padded
    ones are zero) and the first ``cin`` are returned."""
    _need_cuda(dy, x_hi, x_lo)
    lib = _lib.load()
    dy = dy.contiguous()
    b, t, h, w, cs = x_hi.shape
    cout = dy.shape[-1]
    elems = lib.e2f_dis_conv3d_wgrad_work_elems(b, t, h, w, cs, cout, pad)
    if elems < 0:
        _lib.check(int(elems), "e2f_dis_conv3d_wgrad_work_elems")
    work = torch.empty(int(elems), dtype=torch.float32, device=dy.device)
    dw = torch.empty(cout, cs, 3, 5, 5, dtype=torch.float32, device=dy.device)
    db = torch.empty(cout, dtype=torch.float32, device=dy.device) if with_bias else None
    with _timed(f"dis_wgrad_c{cout}", 2.0 * dy.numel() * cs * 75):
        st = lib.e2f_dis_conv3d_wgrad(dy.data_ptr(), x_hi.data_ptr(), x_lo.data_ptr(), dw.data_ptr(),
                                      None if db is None else db.data_ptr(), work.data_ptr(), b, t, h, w, cs, cout, pad,
                                      _stream())
    _lib.check(st, "e2f_dis_conv3d_wgrad")
    return (dw if cin == cs else dw[:, :cin].contiguous()), db
