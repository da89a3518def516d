"""Temporal focal transformer (reference: model/modules/tfocal_transformer.py:19-536 and _hq.py).

One implementation serves both variants: the base model fixes ``output_size`` at construction
(tfocal_transformer.py:30-37,56-59,83-87), the HQ model threads it through at run time (_hq.py:32-46,92-119).
Parameter / buffer names follow the reference so released ``state_dict``s load strictly.

The attention core (window partition, 4 rolled ring key sets, pooled-window keys with the -100 mask, softmax,
P·V, window reverse) is ONE kernel, ``ops.focal_window_attention``; rolled K/V copies and the logits matrix are
never materialised.
"""
import math
from functools import reduce

import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops


def _token_grid(output_size, kernel_size, stride, padding):
    return tuple((output_size[i] + 2 * padding[i] - (kernel_size[i] - 1) - 1) // stride[i] + 1 for i in range(2))


def _tracked(inputs, params):
    """Grad mode is on and a tensor input or a parameter requires grad: the call gets a ``grad_fn``."""
    return torch.is_grad_enabled() and (any(isinstance(t, torch.Tensor) and t.requires_grad for t in inputs)
                                        or any(p.requires_grad for p in params))


def _second_backward(what):
    return RuntimeError(f"{what}: the backward frees the operands it keeps, so the output cannot be backpropagated a "
                        "second time (retain_graph=True is not supported); run the forward again")


class SoftSplit(nn.Module):
    """unfold(7x7, s3, p3) + Linear(49*C -> hidden) (tfocal_transformer.py:19-46)."""

    def __init__(self, channel, hidden, kernel_size, stride, padding, t2t_param=None):
        super().__init__()
        self.kernel_size, self.stride, self.padding = tuple(kernel_size), tuple(stride), tuple(padding)
        self.embedding = nn.Linear(reduce(lambda a, b: a * b, kernel_size) * channel, hidden)
        self.t2t_param = t2t_param
        self.output_size = None if t2t_param is None else t2t_param.get("output_size")

    def forward(self, x, b, output_size=None):
        """x (BT, C, H, W) fp32 (or the encoder's ``SplitNHWC``) -> tokens (b, T, fh, fw, hidden).  Trainable
        (``_SoftSplitGrad``) when grad mode is on and the tensor x or a parameter requires grad; the tokens are the same
        bits as the untracked call."""
        output_size = output_size or self.output_size
        f_h, f_w = _token_grid(output_size, self.kernel_size, self.stride, self.padding)
        params = (self.embedding.weight, self.embedding.bias)
        if isinstance(x, torch.Tensor) and _tracked([x], params):
            feat = _SoftSplitGrad.apply(self, x, *params)
        else:
            # unfold + Linear == a 7x7 / stride-3 conv: one implicit-GEMM launch, the 49x unfolded operand never exists
            feat = ops.soft_split(x, *params, self.kernel_size, self.stride, self.padding)
        return feat.view(b, -1, f_h, f_w, feat.size(2))


class _SoftSplitGrad(torch.autograd.Function):
    """``SoftSplit``'s launch with a backward into ``embedding`` and x: dW = dT^T . unfold(x) (the unfold materialised as
    a split operand), db = the sum of dT, dx = fold(dT . W) on ``soft_comp``'s transposed-conv launch with W^T."""

    @staticmethod
    def forward(ctx, mod, x, weight, bias):
        ctx.mod, ctx.live = mod, True
        ctx.save_for_backward(x, weight, bias)
        return ops.soft_split(x, weight, bias, mod.kernel_size, mod.stride, mod.padding)

    @staticmethod
    def backward(ctx, grad):
        if not ctx.live:
            raise _second_backward("SoftSplit")
        x, weight, bias = ctx.saved_tensors
        ctx.live = False
        mod = ctx.mod
        n, c, h, w = x.shape
        _, need_x, need_w, need_b = ctx.needs_input_grad
        dx = dw = db = None
        if need_w or need_b:
            cols = ops.t2t_unfold(x, mod.kernel_size, mod.stride, mod.padding, out="split")
            dw, db = ops.linear_wgrad(grad, cols, with_bias=need_b)
            dw = dw if need_w else None
        if need_x:
            fh, fw = _token_grid((h, w), mod.kernel_size, mod.stride, mod.padding)
            dx = ops.soft_comp(grad.reshape(n, fh, fw, -1), weight, None, (h, w), mod.kernel_size, mod.stride,
                               mod.padding, transpose=True)
        return None, dx, dw, db


class SoftComp(nn.Module):
    """Linear(hidden -> 49*C) + fold + bias map (base, tfocal_transformer.py:49-72) or 3x3 conv (HQ, _hq.py:49-79)."""

    def __init__(self, channel, hidden, output_size=None, kernel_size=(7, 7), stride=(3, 3), padding=(3, 3), hq=False):
        super().__init__()
        self.kernel_size, self.stride, self.padding = tuple(kernel_size), tuple(stride), tuple(padding)
        self.embedding = nn.Linear(hidden, reduce(lambda a, b: a * b, kernel_size) * channel)
        self.output_size = output_size
        self.hq = hq
        if hq:
            self.bias_conv = nn.Conv2d(channel, channel, kernel_size=3, stride=1, padding=1)
        else:
            self.bias = nn.Parameter(torch.zeros((channel, output_size[0], output_size[1]), dtype=torch.float32))

    def params(self):
        """The parameters in ``_SoftCompGrad``'s order: embedding weight and bias, then the bias map (base) or
        bias_conv's weight and bias (HQ)."""
        tail = (self.bias_conv.weight, self.bias_conv.bias) if self.hq else (self.bias,)
        return (self.embedding.weight, self.embedding.bias) + tail

    def forward(self, x, t, output_size=None, residual=None):
        """``residual`` (b*t, C, H, W), optional: added to the result by the fold kernel (base model) or the conv
        epilogue (HQ) — the ``enc_feat + trans_feat`` of e2fgvi.py:263; the result is then channels_last.  Trainable
        (``_SoftCompGrad``) when grad mode is on and x, the residual or a parameter requires grad; the result is the
        same bits as the untracked call."""
        output_size = tuple(output_size or self.output_size)
        if isinstance(x, torch.Tensor) and _tracked([x, residual], self.params()):
            return _SoftCompGrad.apply(self, x, residual, output_size, *self.params())
        return self._forward(x, t, output_size, residual)

    def _forward(self, x, t, output_size=None, residual=None, keep=None):
        """The launch sequence of ``forward`` (untracked); ``keep`` (a dict or None) receives the split tokens and, HQ,
        the split operand of bias_conv."""
        output_size = output_size or self.output_size
        b_, t_, f_h, f_w, c_ = x.shape
        # Linear + fold == the transposed 7x7 / stride-3 conv: one implicit-GEMM launch over nine output phases; the
        # 6272-wide token matrix and the fold pass never exist
        tokens = x.view(b_ * t_, f_h, f_w, c_)
        if keep is not None:
            tokens = keep["tokens"] = ops.SplitMat(*ops.split_bf16(tokens))
        if self.hq:
            feat = ops.soft_comp(tokens, self.embedding.weight, self.embedding.bias, output_size, self.kernel_size,
                                 self.stride, self.padding, out="split")
            if keep is not None:
                keep["feat"] = feat
            return ops.conv3x3([feat], self.bias_conv.weight, self.bias_conv.bias, residual=residual)
        return ops.soft_comp(tokens, self.embedding.weight, self.embedding.bias, output_size, self.kernel_size,
                             self.stride, self.padding, bias_map_extra=self.bias, residual=residual)


class _SoftCompGrad(torch.autograd.Function):
    """``SoftComp``'s launches with a backward into its parameters, the tokens and the residual.  With dfeat = the
    gradient of the folded features (HQ: bias_conv's input gradient on ``conv_dgrad``, its weight gradient on
    ``conv3x3_wgrad``): the base bias map gets the sum of dfeat over BT, the embedding dW = unfold(dfeat)^T . tokens
    and db = the sum of unfold(dfeat), the tokens unfold(dfeat) . W on ``soft_split``'s launch with W^T; the residual
    receives the gradient unchanged."""

    @staticmethod
    def forward(ctx, mod, tokens, residual, output_size, *params):
        keep = {}
        out = mod._forward(tokens, tokens.shape[1], output_size, residual, keep)
        ctx.mod, ctx.keep, ctx.output_size, ctx.shape = mod, keep, output_size, tokens.shape
        ctx.save_for_backward(*params)
        return out

    @staticmethod
    def backward(ctx, grad):
        if ctx.keep is None:
            raise _second_backward("SoftComp")
        params = ctx.saved_tensors
        mod, keep = ctx.mod, ctx.keep
        ctx.keep = None
        need_tok, need_res = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        needs = ctx.needs_input_grad[4:]
        grads = [None] * len(params)
        k, s, p = mod.kernel_size, mod.stride, mod.padding
        dfeat = grad
        if mod.hq:
            if needs[2] or needs[3]:
                dw, db = ops.conv3x3_wgrad(grad.permute(0, 2, 3, 1), [keep["feat"]], with_bias=needs[3])
                grads[2], grads[3] = (dw if needs[2] else None), db
            dfeat = None
            if need_tok or needs[0] or needs[1]:
                dfeat = ops.conv_dgrad(ops.split_nhwc(grad), params[2]).permute(0, 3, 1, 2)
        elif needs[2]:
            grads[2] = grad.sum(0)
        if needs[0] or needs[1]:
            cols = ops.t2t_unfold(dfeat, k, s, p, out="split")
            dw, db = ops.linear_wgrad(cols, keep["tokens"], with_bias=needs[1])
            grads[0], grads[1] = (dw if needs[0] else None), db
        dtok = None
        if need_tok:
            dtok = ops.soft_split(dfeat, params[0], None, k, s, p, transpose=True).reshape(ctx.shape)
        return (None, dtok, grad if need_res else None, None) + tuple(grads)


class FusionFeedForward(nn.Module):
    """Linear(512->1960), overlap-average through fold/normalise/unfold, GELU, Linear(1960->512)
    (tfocal_transformer.py:75-98; _hq.py:82-119)."""

    def __init__(self, d_model, n_vecs=None, t2t_params=None):
        super().__init__()
        hd = 1960
        self.conv1 = nn.Sequential(nn.Linear(d_model, hd))
        self.conv2 = nn.Sequential(nn.GELU(), nn.Linear(hd, d_model))
        assert t2t_params is not None
        self.t2t_params = dict(t2t_params)
        self.n_vecs = n_vecs

    def forward(self, x, output_size=None, residual=None):
        """conv1 -> [fold / fold(ones) -> unfold -> GELU] (one fused kernel on the token-major layout) -> conv2
        (+ residual, fused into the GEMM epilogue).  Trainable (``_FusionFeedForwardGrad``) when grad mode is on, x is
        an fp32 tensor (B, N, 512) and x, the residual or a Linear's parameter requires grad; the output is the same
        bits as the untracked call."""
        params = (self.conv1[0].weight, self.conv1[0].bias, self.conv2[1].weight, self.conv2[1].bias)
        if isinstance(x, torch.Tensor) and _tracked([x, residual], params):
            p = self.t2t_params
            return _FusionFeedForwardGrad.apply(self, x, residual, tuple(output_size or p.get("output_size")), *params)
        p = self.t2t_params
        output_size = output_size or p.get("output_size")
        f_h, f_w = _token_grid(output_size, p["kernel_size"], p["stride"], p["padding"])
        n_vecs = f_h * f_w
        x = ops.linear(x, self.conv1[0].weight, self.conv1[0].bias)
        b, n, c = x.size()
        # fold / fold(ones) -> unfold -> conv2[0] (GELU): one kernel, the folded image stays in shared memory
        # rows padded 1960 -> 1984 (zero columns) so that the A operand of conv2 starts every row on a 128-byte line
        x = ops.t2t_fold_unfold(x.view(-1, n_vecs, c), output_size, p["kernel_size"], p["stride"], p["padding"],
                                gelu=True, out="split", pitch=(c + 63) // 64 * 64)
        x = x.view(b, n, x.shape[-1])
        return ops.linear(x, self.conv2[1].weight, self.conv2[1].bias, residual=residual)

    def geometry(self, output_size):
        p = self.t2t_params
        return output_size, p["kernel_size"], p["stride"], p["padding"]


def _ffn_forward(mod, xs, output_size, w1, b1, w2, b2, residual):
    """``FusionFeedForward``'s training launches on the split operand xs (rows, 512): conv1, the fold/normalise/unfold
    kernel in its training mode (which also keeps u, the normalised values before GELU), conv2 (+ residual).  Returns
    (out (rows, 512), the dict ``_ffn_backward`` reads)."""
    geo = mod.geometry(output_size)
    h = ops.linear(xs, w1, b1)
    hd = h.shape[-1]
    f_h, f_w = _token_grid(*geo)
    z, u = ops.t2t_fold_unfold_train(h.view(-1, f_h * f_w, hd), *geo, out="split", pitch=(hd + 63) // 64 * 64)
    out = ops.linear(z.view(-1, z.shape[-1]), w2, b2, residual=residual)
    return out, {"x": xs, "u": u, "z": z, "geo": geo}


def _ffn_backward(keep, grad, w1, w2, need_x, nw1, nb1, nw2, nb2):
    """The backward of ``_ffn_forward`` at g = grad (rows, 512) fp32: (dx (rows, 512) or None, dW1, db1, dW2, db2), each
    None when not asked for.
      dz = g . W2 (``linear`` with W2^T), dW2 = g^T . GELU(u) (the kept split operand), db2 = sum g;
      dh = U D F (dz * GELU'(u)) (the fold/normalise/unfold kernel's adjoint mode, a split operand with the 1984 pitch);
      dx = dh . W1 (``linear`` with W1^T, padded alike), dW1 = dh^T . x, db1 = sum dh."""
    z, u = keep["z"], keep["u"]
    g = ops.SplitMat(*ops.split_bf16(grad.reshape(-1, grad.shape[-1])))
    dw1 = db1 = dw2 = db2 = dx = None
    if nw2 or nb2:
        dw2, db2 = ops.linear_wgrad(g, z.view(-1, z.shape[-1]), with_bias=nb2, shape=tuple(w2.shape))
        dw2 = dw2 if nw2 else None
    if need_x or nw1 or nb1:
        dz = ops.linear(g, w2, transpose=True)
        dh = ops.t2t_fold_unfold_train(dz.view(u.shape), *keep["geo"], u=u, out="split", pitch=z.shape[-1])
        dh = dh.view(-1, dh.shape[-1])
        if nw1 or nb1:
            dw1, db1 = ops.linear_wgrad(dh, keep["x"], with_bias=nb1, shape=tuple(w1.shape))
            dw1 = dw1 if nw1 else None
        if need_x:
            dx = ops.linear(dh, w1, transpose=True)
    return dx, dw1, db1, dw2, db2


class _FusionFeedForwardGrad(torch.autograd.Function):
    """``FusionFeedForward``'s launches with a backward into both Linears, x and the residual: the forward splits x
    once (conv1's operand, kept for its weight gradient) and runs ``_ffn_forward``; the backward is ``_ffn_backward``,
    and the residual receives the output's gradient."""

    @staticmethod
    def forward(ctx, mod, x, residual, output_size, w1, b1, w2, b2):
        b, n, _ = x.shape
        xs = ops.SplitMat(*ops.split_bf16(x.reshape(-1, x.shape[-1])))
        out, ctx.keep = _ffn_forward(mod, xs, output_size, w1, b1, w2, b2, residual)
        ctx.shape = x.shape
        ctx.save_for_backward(w1, w2)
        return out.view(b, n, -1)

    @staticmethod
    def backward(ctx, grad):
        if ctx.keep is None:
            raise _second_backward("FusionFeedForward")
        w1, w2 = ctx.saved_tensors
        keep = ctx.keep
        ctx.keep = None
        need_x, need_res = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        dx, dw1, db1, dw2, db2 = _ffn_backward(keep, grad, w1, w2, need_x, *ctx.needs_input_grad[4:])
        return None, None if dx is None else dx.view(ctx.shape), grad if need_res else None, None, dw1, db1, dw2, db2


def window_partition(x, window_size):
    """(B,T,H,W,C) -> (B*nW, T*wh*ww, C) (tfocal_transformer.py:101-114)."""
    B, T, H, W, C = x.shape
    wh, ww = window_size
    x = x.view(B, T, H // wh, wh, W // ww, ww, C)
    return x.permute(0, 2, 4, 1, 3, 5, 6).reshape(-1, T * wh * ww, C)


def window_partition_noreshape(x, window_size):
    """(B,T,H,W,C) -> (B, nWh, nWw, T, wh, ww, C) (tfocal_transformer.py:117-129)."""
    B, T, H, W, C = x.shape
    wh, ww = window_size
    return x.view(B, T, H // wh, wh, W // ww, ww, C).permute(0, 2, 4, 1, 3, 5, 6).contiguous()


def window_reverse(windows, window_size, T, H, W):
    """(B*nW, T, wh, ww, C) -> (B,T,H,W,C) (tfocal_transformer.py:132-147)."""
    wh, ww = window_size
    B = windows.shape[0] // ((H // wh) * (W // ww))
    x = windows.view(B, H // wh, W // ww, T, wh, ww, -1)
    return x.permute(0, 3, 1, 4, 2, 5, 6).reshape(B, T, H, W, -1)


def rolled_valid_indices(window_size, expand_size):
    """Flat indices kept from the 4 rolled window copies (tfocal_transformer.py:166-179): positions of the
    (tl, tr, bl, br) rolled windows that fall OUTSIDE the query window."""
    wh, ww = window_size
    eh, ew = expand_size
    keep = []
    for quad, (row_from_end, col_from_end) in enumerate(((True, True), (True, False), (False, True), (False, False))):
        for r in range(wh):
            for c in range(ww):
                row_ok = r >= wh - eh if row_from_end else r < eh
                col_ok = c >= ww - ew if col_from_end else c < ew
                if row_ok or col_ok:
                    keep.append(quad * wh * ww + r * ww + c)
    return torch.tensor(keep, dtype=torch.int64)


class WindowAttention(nn.Module):
    """Temporal focal window attention (tfocal_transformer.py:150-399)."""

    def __init__(self, dim, expand_size, window_size, focal_window, focal_level, num_heads, qkv_bias, pool_method):
        super().__init__()
        self.dim, self.num_heads = dim, num_heads
        self.expand_size, self.window_size = tuple(expand_size), tuple(window_size)
        self.focal_window, self.focal_level, self.pool_method = tuple(focal_window), focal_level, pool_method
        self.scale = (dim // num_heads) ** -0.5
        if focal_level > 2:
            raise NotImplementedError("E2FGVI uses focal_level=2 (one pooled level)")
        if any(i > 0 for i in self.expand_size) and focal_level > 0:
            self.register_buffer("valid_ind_rolled", rolled_valid_indices(self.window_size, self.expand_size))
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)

    @property
    def uses_pooled(self):
        return self.pool_method != "none" and self.focal_level > 1

    def pooled_kernel(self):
        """Neighbourhood of pooled windows each query window attends (unfold kernel, tfocal_transformer.py:186-196)."""
        return tuple(2 * (i // 2) + 1 for i in self.focal_window)

    def attend(self, x, pooled, residual=None, joint_shape=None, keep=None):
        """x (B,T,H,W,C) normed tokens (tensor or ops.SplitMat), pooled (B,nWh,nWw,T,C) tensor or the SplitMat of
        ops.window_pool (already (B,T,nWh,nWw,C)) -> (B,T,H,W,C) after proj (+ residual).
        ``joint_shape`` = (B,T,H,W): x is the SplitMat of ``ops.layer_norm_pool`` (token rows followed by pooled rows) and
        ONE qkv GEMM serves both.  Trainable (``_WindowAttentionGrad``) when grad mode is on, x is a tensor, no
        ``joint_shape`` is given and x, pooled, the residual or a parameter of ``qkv`` / ``proj`` requires grad; the result
        is the same bits as the untracked call.  ``keep`` (a dict or None; untracked calls on a SplitMat x without pooled
        only) receives what ``_attention_backward`` reads: x, the fp16 qkv / qkv_pooled and the split attention output."""
        params = self.params()
        if (keep is None and joint_shape is None and isinstance(x, torch.Tensor) and not isinstance(pooled, ops.SplitMat)
                and _tracked([x, pooled if self.uses_pooled else None, residual], [p for p in params if p is not None])):
            return _WindowAttentionGrad.apply(self, x, pooled if self.uses_pooled else None, residual, *params)
        if joint_shape is not None:
            B, T, H, W = joint_shape
            wh, ww = self.window_size
            n_tok = B * T * H * W
            both = ops.linear(x, self.qkv.weight, self.qkv.bias, out_dtype=torch.float16)
            qkv = both[:n_tok].view(B, T, H, W, -1)
            qkv_pooled = both[n_tok:].view(B, T, H // wh, W // ww, -1)
        else:
            qkv = ops.linear(x, self.qkv.weight, self.qkv.bias, out_dtype=torch.float16)
            qkv_pooled = None
            if self.uses_pooled:
                if not isinstance(pooled, ops.SplitMat):      # reference layout (B,nWh,nWw,T,C) -> (B,T,nWh,nWw,C)
                    pooled = pooled.permute(0, 3, 1, 2, 4).contiguous()
                qkv_pooled = ops.linear(pooled, self.qkv.weight, self.qkv.bias, out_dtype=torch.float16)
        out = ops.focal_window_attention(qkv, qkv_pooled, self.num_heads, self.window_size, self.expand_size,
                                         self.pooled_kernel(), self.scale, out_dtype="split")
        if keep is not None:
            keep.update(x=x, qkv=qkv, qkv_pooled=qkv_pooled, out=out)
        return ops.linear(out, self.proj.weight, self.proj.bias, residual=residual)

    def params(self):
        """The parameters in ``_WindowAttentionGrad``'s order: qkv weight and bias (None without qkv_bias), proj weight
        and bias."""
        return self.qkv.weight, self.qkv.bias, self.proj.weight, self.proj.bias

    def forward(self, x_all, mask_all=None):
        """Reference boundary: x_all = [x (B,T,H,W,C), pooled (B,nWh,nWw,T,C)] -> (B*nW, T*wh*ww, C)."""
        del mask_all  # always [None, None] on the path (tfocal_transformer.py:475)
        out = self.attend(x_all[0], x_all[1] if len(x_all) > 1 else None)
        return window_partition(out, self.window_size)


class _WindowAttentionGrad(torch.autograd.Function):
    """``WindowAttention.attend``'s launches with a backward into qkv, proj, x, pooled and the residual.  The forward
    splits the token rows and the pooled rows once, into one operand (kept for qkv's weight gradient), and runs the
    same qkv, attention and proj launches as the untracked call.  Backward, with g = the output's gradient:
      dW_proj = g^T . O (the attention's kept split output), db_proj = sum g;  dO = g . W_proj (``linear`` with W^T);
      dqkv = the attention backward (token rows and pooled rows in one buffer);
      dW_qkv = dqkv^T . [x; pooled] and db_qkv = sum dqkv over both sets of rows in one reduction;
      [dx; dpooled] = dqkv . W_qkv (``linear`` with W^T); the residual receives g."""

    @staticmethod
    def forward(ctx, mod, x, pooled, residual, wq, bq, wp, bp):
        B, T, H, W, C = x.shape
        wh, ww = mod.window_size
        n_tok = B * T * H * W
        rows = x.reshape(n_tok, C)
        if pooled is not None:                                  # reference layout (B,nWh,nWw,T,C) -> (B,T,nWh,nWw,C)
            rows = torch.cat([rows, pooled.permute(0, 3, 1, 2, 4).reshape(-1, C)])
        xs = ops.SplitMat(*ops.split_bf16(rows))
        qkv = ops.linear(ops.SplitMat(xs.hi[:n_tok], xs.lo[:n_tok]), wq, bq, out_dtype=torch.float16).view(B, T, H, W, -1)
        qkv_pooled = None
        if pooled is not None:
            qkv_pooled = ops.linear(ops.SplitMat(xs.hi[n_tok:], xs.lo[n_tok:]), wq, bq, out_dtype=torch.float16)
            qkv_pooled = qkv_pooled.view(B, T, H // wh, W // ww, -1)
        out = ops.focal_window_attention(qkv, qkv_pooled, mod.num_heads, mod.window_size, mod.expand_size,
                                         mod.pooled_kernel(), mod.scale, out_dtype="split")
        ctx.mod, ctx.keep, ctx.shape = mod, {"x": xs, "qkv": qkv, "qkv_pooled": qkv_pooled, "out": out}, x.shape
        ctx.save_for_backward(wq, wp)
        return ops.linear(out, wp, bp, residual=residual)

    @staticmethod
    def backward(ctx, grad):
        if ctx.keep is None:
            raise _second_backward("WindowAttention")
        wq, wp = ctx.saved_tensors
        keep, mod = ctx.keep, ctx.mod
        ctx.keep = None
        need_x, need_pool, need_res = ctx.needs_input_grad[1:4]
        nwq, nbq, nwp, nbp = ctx.needs_input_grad[4:]
        B, T, H, W, C = ctx.shape
        g = None
        if nwp or nbp or need_x or need_pool or nwq or nbq:
            g = ops.SplitMat(*ops.split_bf16(grad.reshape(-1, C)))
        drows, dwq, dbq, dwp, dbp = _attention_backward(mod, keep, g, wq, wp, ctx.shape, need_x or need_pool, nwq, nbq,
                                                        nwp, nbp)
        dx = dpool = None
        n_tok = B * T * H * W
        if need_x:
            dx = drows[:n_tok].view(B, T, H, W, C)
        if need_pool:
            wh, ww = mod.window_size
            dpool = drows[n_tok:].view(B, T, H // wh, W // ww, C).permute(0, 2, 3, 1, 4).contiguous()
        return None, dx, dpool, grad if need_res else None, dwq, dbq, dwp, dbp


def _attention_backward(mod, keep, g, wq, wp, shape, need_rows, nwq, nbq, nwp, nbp):
    """The backward of ``WindowAttention.attend``'s launches at the split output gradient g (B*T*H*W, C), with ``keep``
    = the kept joint split input "x" (token rows, then pooled rows ordered (B,T,nWh,nWw)), the fp16 "qkv" /
    "qkv_pooled" and the attention's split output "out".  Returns (drows, dW_qkv, db_qkv, dW_proj, db_proj), each None
    when not asked for; drows (rows of x, C) fp32 = [dx; dpooled] in x's joint layout (``need_rows``).
      dW_proj = g^T . O, db_proj = sum g;  dO = g . W_proj (``linear`` with W^T);
      dqkv = the attention backward (token rows and pooled rows in one buffer), split once for both of its uses;
      dW_qkv = dqkv^T . [x; pooled] and db_qkv = sum dqkv over both sets of rows in one reduction;
      [dx; dpooled] = dqkv . W_qkv (``linear`` with W^T)."""
    B, T, H, W, C = shape
    drows = dwq = dbq = dwp = dbp = None
    if nwp or nbp:
        dwp, dbp = ops.linear_wgrad(g, keep["out"].view(-1, C), with_bias=nbp)
        dwp = dwp if nwp else None
    if need_rows or nwq or nbq:
        dout = ops.linear(g, wp, transpose=True).view(B, T, H, W, C)
        dqkv = ops.focal_window_attention_backward(keep["qkv"], keep["qkv_pooled"], dout, mod.num_heads,
                                                   mod.window_size, mod.expand_size, mod.pooled_kernel(), mod.scale)
        dqkv = ops.SplitMat(*ops.split_bf16(dqkv))        # one split serves qkv's weight and input gradients
        if nwq or nbq:
            dwq, dbq = ops.linear_wgrad(dqkv, keep["x"], with_bias=nbq)
            dwq = dwq if nwq else None
        if need_rows:
            drows = ops.linear(dqkv, wq, transpose=True)
    return drows, dwq, dbq, dwp, dbp


class TemporalFocalTransformerBlock(nn.Module):
    """LN -> window pool -> focal attention -> +res -> LN -> fusion FFN -> +res (tfocal_transformer.py:402-536)."""

    def __init__(self, dim, num_heads, window_size=(5, 9), mlp_ratio=4., qkv_bias=True, pool_method="fc",
                 focal_level=2, focal_window=(5, 9), norm_layer=nn.LayerNorm, n_vecs=None, t2t_params=None,
                 hq=False):
        super().__init__()
        self.dim, self.num_heads, self.window_size = dim, num_heads, tuple(window_size)
        self.expand_size = tuple(i // 2 for i in window_size)
        self.mlp_ratio, self.pool_method = mlp_ratio, pool_method
        self.focal_level, self.focal_window = focal_level, tuple(focal_window)
        self.hq = hq
        self.pool_layers = nn.ModuleList()
        if pool_method != "none":
            for k in range(focal_level - 1):
                ws = tuple(math.floor(i / (2 ** k)) for i in self.window_size)
                layer = nn.Linear(ws[0] * ws[1], 1)
                layer.weight.data.fill_(1.0 / (ws[0] * ws[1]))
                layer.bias.data.fill_(0)
                self.pool_layers.append(layer)
        self.norm1 = norm_layer(dim)
        self.attn = WindowAttention(dim, self.expand_size, self.window_size, focal_window, focal_level, num_heads,
                                    qkv_bias, pool_method)
        self.norm2 = norm_layer(dim)
        self.mlp = FusionFeedForward(dim, n_vecs=n_vecs, t2t_params=t2t_params)

    def params(self):
        """The parameters in ``_TransformerBlockGrad``'s order: norm1 weight and bias, pool_layers[0] weight and bias
        (None without pooling), attn.qkv weight and bias (None without qkv_bias), attn.proj weight and bias, norm2
        weight and bias, mlp.conv1[0] weight and bias, mlp.conv2[1] weight and bias."""
        pool = (self.pool_layers[0].weight, self.pool_layers[0].bias) if self.attn.uses_pooled else (None, None)
        return ((self.norm1.weight, self.norm1.bias) + pool + self.attn.params() + (self.norm2.weight, self.norm2.bias)
                + (self.mlp.conv1[0].weight, self.mlp.conv1[0].bias, self.mlp.conv2[1].weight, self.mlp.conv2[1].bias))

    def _forward(self, x, output_size, keep=None):
        """The launch sequence of ``forward`` (untracked); ``keep`` (a dict or None) receives what
        ``_TransformerBlockGrad.backward`` reads: x1 = the attention's output (+ x), the attention's operands and the
        feed-forward's (which then runs its training forward: the same bits)."""
        shortcut = x
        B, T, H, W, C = x.shape
        attn_keep = None if keep is None else keep.setdefault("attn", {})
        if self.attn.uses_pooled:
            if H % self.window_size[0] or W % self.window_size[1]:
                raise ValueError(f"token grid {H}x{W} must be a multiple of the window {self.window_size}")
            # norm1 + focal window pooling in one kernel (pooled tokens accumulated in registers next to the LayerNorm);
            # token rows and pooled rows share one operand buffer, so one qkv GEMM serves both
            lin = self.pool_layers[0]
            rows, _ = ops.layer_norm_pool(x, self.norm1.weight, self.norm1.bias, self.norm1.eps, lin.weight, lin.bias,
                                          self.window_size)
            x = self.attn.attend(rows, None, residual=shortcut, joint_shape=(B, T, H, W), keep=attn_keep)
        else:
            xn_split = ops.layer_norm(x, self.norm1.weight, self.norm1.bias, self.norm1.eps, out="split")
            x = self.attn.attend(xn_split, None, residual=shortcut, keep=attn_keep)
        y = ops.layer_norm(x, self.norm2.weight, self.norm2.bias, self.norm2.eps, out="split")
        if keep is None:
            return self.mlp(y.view(B, T * H * W, C), output_size, residual=x.view(B, T * H * W, C)).view(B, T, H, W, C)
        mlp = self.mlp
        size = tuple(output_size or mlp.t2t_params["output_size"])
        out, keep["mlp"] = _ffn_forward(mlp, y.view(B * T * H * W, C), size, mlp.conv1[0].weight, mlp.conv1[0].bias,
                                        mlp.conv2[1].weight, mlp.conv2[1].bias, x)
        keep["x1"] = x
        return out.view(B, T, H, W, C)

    def forward(self, x):
        """tokens (B,T,H,W,C) -> (B,T,H,W,C); HQ: [tokens, output_size] -> (tokens, output_size).  Trainable
        (``_TransformerBlockGrad``) when grad mode is on and the tokens or a parameter requires grad; the result is the
        same bits as the untracked call."""
        if self.hq:  # x = [tokens, (h, w)] -> (tokens, (h, w))   (_hq.py:492-495,562-565)
            tokens, output_size = x[0], x[1]
        else:
            tokens, output_size = x, None
        params = self.params()
        if _tracked([tokens], [p for p in params if p is not None]):
            out = _TransformerBlockGrad.apply(self, tokens, output_size, *params)
        else:
            out = self._forward(tokens, output_size)
        return (out, output_size) if self.hq else out


class _TransformerBlockGrad(torch.autograd.Function):
    """``TemporalFocalTransformerBlock``'s launches (``_forward`` with ``keep``) with a backward into every parameter
    and the tokens x.  With g = the output's gradient and x1 = x + attention(LN1(x)):
      1. the feed-forward's backward (``_ffn_backward``) gives dy = the gradient of LN2's output and both Linears';
      2. dx1 = g + LN2'(x1; dy) (``layer_norm_backward``, fp32 and split), dgamma2, dbeta2;
      3. the attention's backward (``_attention_backward``) at dx1 gives [dxn; dpooled] and qkv's and proj's gradients;
      4. dx = dx1 + LN1'(x; dxn + w_pool dpooled) (``layer_norm_pool_backward``; without pooling ``layer_norm_backward``
         with the residual dx1), dgamma1, dbeta1, d w_pool, d b_pool.
    The walk stops at the lowest part that needs a gradient; a frozen part launches no weight gradient."""

    @staticmethod
    def forward(ctx, mod, x, output_size, *params):
        keep = {}
        out = mod._forward(x, output_size, keep)
        ctx.mod, ctx.keep = mod, keep
        ctx.save_for_backward(x, *[p for p in params if p is not None])
        ctx.have = [p is not None for p in params]
        return out

    @staticmethod
    def backward(ctx, grad):
        if ctx.keep is None:
            raise _second_backward("TemporalFocalTransformerBlock")
        saved = list(ctx.saved_tensors)
        x = saved.pop(0)
        params = [saved.pop(0) if h else None for h in ctx.have]
        keep = ctx.keep
        ctx.keep = None
        dx, grads = _block_backward(ctx.mod, keep, x, params, grad, ctx.needs_input_grad[1], ctx.needs_input_grad[3:])
        return (None, dx, None) + tuple(grads)


def _block_backward(mod, keep, x, params, grad, need_x, needs):
    """The backward of ``TemporalFocalTransformerBlock._forward(x, output_size, keep)`` at the output's gradient grad:
    (dx or None, the 14 parameter gradients in ``params()`` order, None where ``needs`` is False)."""
    n1w, n1b, pw, pb, wq, bq, wp, bp, n2w, n2b, w1, b1, w2, b2 = params
    (nn1w, nn1b, npw, npb, nwq, nbq, nwp, nbp, nn2w, nn2b, nw1, nb1, nw2, nb2) = needs
    grads = [None] * 14
    B, T, H, W, C = x.shape
    need_norm1 = nn1w or nn1b or npw or npb
    need_rows = need_x or need_norm1                         # [dxn; dpooled]: the attention's input gradient
    need_dx1 = need_rows or nwq or nbq or nwp or nbp         # the gradient of x1 past LN2 (the attention's output)
    need_dy = need_dx1 or nn2w or nn2b
    dy, *grads[10:14] = _ffn_backward(keep["mlp"], grad, w1, w2, need_dy, nw1, nb1, nw2, nb2)
    if not need_dy:
        return None, grads
    dx1, grads[8], grads[9] = ops.layer_norm_backward(keep["x1"].view(-1, C), dy, n2w, mod.norm2.eps,
                                                      residual=grad.reshape(-1, C), out="both" if need_dx1 else None,
                                                      need_weight=nn2w, need_bias=nn2b)
    if not need_dx1:
        return None, grads
    dx1_32, dx1_split = dx1
    drows, grads[4], grads[5], grads[6], grads[7] = _attention_backward(mod.attn, keep["attn"], dx1_split, wq, wp,
                                                                        x.shape, need_rows, nwq, nbq, nwp, nbp)
    if not need_rows:
        return None, grads
    if mod.attn.uses_pooled:
        dx, grads[0], grads[1], dpw, grads[3] = ops.layer_norm_pool_backward(
            x, drows, dx1_32.view(x.shape), n1w, n1b, mod.norm1.eps, pw, mod.window_size, need_x=need_x,
            need_norm=nn1w or nn1b, need_pool=npw or npb)
        grads[2] = None if dpw is None else dpw.view(pw.shape)
    else:
        dx, grads[0], grads[1] = ops.layer_norm_backward(x.view(-1, C), drows, n1w, mod.norm1.eps, residual=dx1_32,
                                                         out="f32" if need_x else None, need_weight=nn1w,
                                                         need_bias=nn1b)
    grads = [gr if need else None for gr, need in zip(grads, needs)]
    return (None if dx is None else dx.view(x.shape)), grads
