"""TEST INFRASTRUCTURE — CPU restatement of E2FGVI's InpaintGenerator.forward (the oracle).

Plain PyTorch on the CPU, functional over a reference ``state_dict``; dtype-generic (run it in fp64 for a
rounding-free yardstick).  Every function cites the reference lines it follows.  The three operators the CUDA
kernels replace are restated EXPLICITLY (gathers + einsum), not through grid_sample / a DCN library, so they are
an independent statement of the maths:

* ``flow_warp``                 flow_comp.py:345-383
* ``modulated_deform_conv2d``   mmcv op called at feat_prop.py:55-58 (DCNv2; layout pinned vs torchvision)
* ``focal_window_attention``    tfocal_transformer.py:226-396 (literal roll / partition / index / mask / softmax)

Pinned against the real reference by ``tests/test_oracle_vs_reference.py`` (in the build container) and by the
committed goldens made with ``oracle/gen_golden.py``.  Parity at the mmcv boundary itself is unpinned (mmcv is
not installable offline) — see ``oracle/__init__.py``.
"""
import math

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------------- sampling
def bilinear_gather(x, py, px, padding_mode="zeros"):
    """x (N,C,H,W); py, px (N,Ho,Wo) absolute pixel coordinates -> (N,C,Ho,Wo).

    zeros : each of the 4 corners contributes only if it lies inside the image (grid_sample zeros padding ==
            DCN's per-corner rule).   border: the coordinate is clamped to [0, size-1] first."""
    N, C, H, W = x.shape
    if padding_mode == "border":
        py = py.clamp(0, H - 1)
        px = px.clamp(0, W - 1)
    elif padding_mode != "zeros":
        raise NotImplementedError(padding_mode)
    y0 = torch.floor(py)
    x0 = torch.floor(px)
    ly, lx = py - y0, px - x0
    y0, x0 = y0.long(), x0.long()
    flat = x.reshape(N, C, H * W)
    out = torch.zeros((N, C) + tuple(py.shape[1:]), dtype=x.dtype)
    for dy, wy in ((0, 1 - ly), (1, ly)):
        for dx, wx in ((0, 1 - lx), (1, lx)):
            yy, xx = y0 + dy, x0 + dx
            inside = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).reshape(N, 1, -1).expand(N, C, -1)
            val = torch.gather(flat, 2, idx).reshape(out.shape)
            out = out + val * (wy * wx * inside.to(x.dtype)).unsqueeze(1)
    return out


def flow_warp(x, flow, interpolation="bilinear", padding_mode="zeros", align_corners=True):
    """flow_comp.py:345-383.  With align_corners=True the reference's normalise -> grid_sample denormalise
    round trip is the identity, so the sample point is (x + flow[...,0], y + flow[...,1])."""
    if x.size()[-2:] != flow.size()[1:3]:
        raise ValueError(f"The spatial sizes of input ({x.size()[-2:]}) and "
                         f"flow ({flow.size()[1:3]}) are not the same.")
    assert interpolation == "bilinear" and align_corners
    _, _, h, w = x.shape
    gy, gx = torch.meshgrid(torch.arange(h, dtype=x.dtype), torch.arange(w, dtype=x.dtype), indexing="ij")
    return bilinear_gather(x, gy[None] + flow[..., 1], gx[None] + flow[..., 0], padding_mode)


def modulated_deform_conv2d(x, offset, mask, weight, bias=None, stride=1, padding=1, dilation=1, groups=1,
                            deform_groups=1):
    """DCNv2 forward as mmcv / torchvision define it (call site feat_prop.py:55-58).

    For output pixel p, tap k=(i,j), deform group g: sample x[:, g*cpg:(g+1)*cpg] bilinearly (zero outside) at
    (p_y*stride - pad + i*dil + offset[(g*K+k)*2], p_x*stride - pad + j*dil + offset[(g*K+k)*2+1]), multiply by
    mask[g*K+k]; then out = weight[Cout, Cin*K] . col + bias with col index c*K + k."""
    assert groups == 1
    N, Cin, H, W = x.shape
    Cout, _, kh, kw = weight.shape
    K = kh * kw
    Ho = (H + 2 * padding - dilation * (kh - 1) - 1) // stride + 1
    Wo = (W + 2 * padding - dilation * (kw - 1) - 1) // stride + 1
    cpg = Cin // deform_groups
    by, bx = torch.meshgrid(torch.arange(Ho, dtype=x.dtype) * stride - padding,
                            torch.arange(Wo, dtype=x.dtype) * stride - padding, indexing="ij")
    col = torch.empty(N, deform_groups, cpg, K, Ho, Wo, dtype=x.dtype)
    for g in range(deform_groups):
        xg = x[:, g * cpg:(g + 1) * cpg]
        for k in range(K):
            i, j = divmod(k, kw)
            py = by[None] + i * dilation + offset[:, (g * K + k) * 2]
            px = bx[None] + j * dilation + offset[:, (g * K + k) * 2 + 1]
            col[:, g, :, k] = bilinear_gather(xg, py, px, "zeros") * mask[:, g * K + k].unsqueeze(1)
    out = torch.einsum("ok,nkp->nop", weight.reshape(Cout, Cin * K), col.reshape(N, Cin * K, Ho * Wo))
    out = out.reshape(N, Cout, Ho, Wo)
    return out if bias is None else out + bias.view(1, -1, 1, 1)


# --------------------------------------------------------------------------------------------- helpers
def _p(sd, prefix):
    return sd[prefix + ".weight"], sd.get(prefix + ".bias")


def _conv(sd, prefix, x, stride=1, padding=1, groups=1):
    w, b = _p(sd, prefix)
    return F.conv2d(x, w, b, stride, padding, 1, groups)


def _linear(sd, prefix, x):
    w, b = _p(sd, prefix)
    return F.linear(x, w, b)


# --------------------------------------------------------------------------------------------- SPyNet
def spynet(sd, prefix, ref, supp):
    """flow_comp.py:84-169: resize to a multiple of 32, 6-level pyramid, per level x2 upsample, border warp,
    five 7x7 convs (ReLU between), resize back and rescale (u by w/w_up, v by h/h_up)."""
    h, w = ref.shape[2:4]
    w_up = w if w % 32 == 0 else 32 * (w // 32 + 1)
    h_up = h if h % 32 == 0 else 32 * (h // 32 + 1)
    ref = F.interpolate(ref, size=(h_up, w_up), mode="bilinear", align_corners=False)
    supp = F.interpolate(supp, size=(h_up, w_up), mode="bilinear", align_corners=False)
    mean, std = sd[prefix + ".mean"], sd[prefix + ".std"]
    refs, supps = [(ref - mean) / std], [(supp - mean) / std]
    for _ in range(5):
        refs.append(F.avg_pool2d(refs[-1], 2, 2, count_include_pad=False))
        supps.append(F.avg_pool2d(supps[-1], 2, 2, count_include_pad=False))
    refs, supps = refs[::-1], supps[::-1]
    n = ref.size(0)
    flow = ref.new_zeros(n, 2, h_up // 32, w_up // 32)
    for level in range(6):
        up = flow if level == 0 else F.interpolate(flow, scale_factor=2, mode="bilinear", align_corners=True) * 2.0
        y = torch.cat([refs[level], flow_warp(supps[level], up.permute(0, 2, 3, 1), padding_mode="border"), up], 1)
        for k in range(5):
            y = _conv(sd, f"{prefix}.basic_module.{level}.basic_module.{k}.conv", y, 1, 3)
            if k < 4:
                y = F.relu(y)
        flow = up + y
    flow = F.interpolate(flow, size=(h, w), mode="bilinear", align_corners=False)
    scale = flow.new_tensor([float(w) / float(w_up), float(h) / float(h_up)]).view(1, 2, 1, 1)
    return flow * scale


def bidirect_flow(sd, masked_local_frames):
    """e2fgvi.py:210-234."""
    b, l_t, c, h, w = masked_local_frames.shape
    small = F.interpolate(masked_local_frames.reshape(-1, c, h, w), scale_factor=1 / 4, mode="bilinear",
                          align_corners=True, recompute_scale_factor=True).view(b, l_t, c, h // 4, w // 4)
    f1 = small[:, :-1].reshape(-1, c, h // 4, w // 4)
    f2 = small[:, 1:].reshape(-1, c, h // 4, w // 4)
    fwd = spynet(sd, "update_spynet", f1, f2).view(b, l_t - 1, 2, h // 4, w // 4)
    bwd = spynet(sd, "update_spynet", f2, f1).view(b, l_t - 1, 2, h // 4, w // 4)
    return fwd, bwd


# --------------------------------------------------------------------------------------------- propagation
def deform_align(sd, prefix, x, extra_feat, flow_1, flow_2, max_residue_magnitude=10.0, deform_groups=16,
                 return_parts=False):
    """SecondOrderDeformableAlignment.forward, feat_prop.py:35-58."""
    y = torch.cat([extra_feat, flow_1, flow_2], dim=1)
    for k in (0, 2, 4):
        y = F.leaky_relu(_conv(sd, f"{prefix}.conv_offset.{k}", y), 0.1)
    head = _conv(sd, f"{prefix}.conv_offset.6", y)
    o1, o2, mask = torch.chunk(head, 3, dim=1)
    offset = max_residue_magnitude * torch.tanh(torch.cat((o1, o2), dim=1))
    off1, off2 = torch.chunk(offset, 2, dim=1)
    off1 = off1 + flow_1.flip(1).repeat(1, off1.size(1) // 2, 1, 1)
    off2 = off2 + flow_2.flip(1).repeat(1, off2.size(1) // 2, 1, 1)
    offset = torch.cat([off1, off2], dim=1)
    mask = torch.sigmoid(mask)
    out = modulated_deform_conv2d(x, offset, mask, sd[prefix + ".weight"], sd[prefix + ".bias"], 1, 1, 1, 1,
                                  deform_groups)
    return (out, head, offset, mask) if return_parts else out


def bidirectional_propagation(sd, prefix, x, flows_backward, flows_forward, taps=None):
    """BidirectionalPropagation.forward, feat_prop.py:81-149 (flow_idx is i-1 in both directions, :94-103)."""
    b, t, c, h, w = x.shape
    feats = {"spatial": [x[:, i] for i in range(t)]}
    for name in ("backward_", "forward_"):
        feats[name] = []
        frame_idx = list(range(t))
        flow_idx = list(range(-1, t - 1))
        if name == "backward_":
            frame_idx = frame_idx[::-1]
            flows = flows_backward
        else:
            flows = flows_forward
        feat_prop = x.new_zeros(b, c, h, w)
        for i, idx in enumerate(frame_idx):
            feat_current = feats["spatial"][idx]
            if i > 0:
                flow_n1 = flows[:, flow_idx[i]]
                cond_n1 = flow_warp(feat_prop, flow_n1.permute(0, 2, 3, 1))
                feat_n2 = torch.zeros_like(feat_prop)
                flow_n2 = torch.zeros_like(flow_n1)
                cond_n2 = torch.zeros_like(cond_n1)
                if i > 1:
                    feat_n2 = feats[name][-2]
                    flow_n2 = flows[:, flow_idx[i - 1]]
                    flow_n2 = flow_n1 + flow_warp(flow_n2, flow_n1.permute(0, 2, 3, 1))
                    cond_n2 = flow_warp(feat_n2, flow_n2.permute(0, 2, 3, 1))
                cond = torch.cat([cond_n1, feat_current, cond_n2], dim=1)
                xin = torch.cat([feat_prop, feat_n2], dim=1)
                feat_prop = deform_align(sd, f"{prefix}.deform_align.{name}", xin, cond, flow_n1, flow_n2)
                if taps is not None:
                    taps.append({"dir": name, "step": i, "x": xin, "cond": cond, "flow_1": flow_n1,
                                 "flow_2": flow_n2, "out": feat_prop})
            feat = [feat_current] + [feats[k][idx] for k in feats if k not in ("spatial", name)] + [feat_prop]
            y = F.leaky_relu(_conv(sd, f"{prefix}.backbone.{name}.0", torch.cat(feat, dim=1)), 0.1)
            feat_prop = feat_prop + _conv(sd, f"{prefix}.backbone.{name}.2", y)
            feats[name].append(feat_prop)
        if name == "backward_":
            feats[name] = feats[name][::-1]
    outs = [_conv(sd, f"{prefix}.fusion", torch.cat([feats["backward_"][i], feats["forward_"][i]], 1), 1, 0)
            for i in range(t)]
    return torch.stack(outs, dim=1) + x


# --------------------------------------------------------------------------------------------- transformer
def _partition(x, ws):
    """window_partition, tfocal_transformer.py:101-114: (B,T,H,W,C) -> (B*nW, T*wh*ww, C)."""
    B, T, H, W, C = x.shape
    x = x.view(B, T, H // ws[0], ws[0], W // ws[1], ws[1], C)
    return x.permute(0, 2, 4, 1, 3, 5, 6).reshape(-1, T * ws[0] * ws[1], C)


def _unpartition(win, ws, T, H, W):
    """window_reverse, tfocal_transformer.py:132-147."""
    B = win.shape[0] // ((H // ws[0]) * (W // ws[1]))
    x = win.view(B, H // ws[0], W // ws[1], T, ws[0], ws[1], -1)
    return x.permute(0, 3, 1, 4, 2, 5, 6).reshape(B, T, H, W, -1)


def focal_window_attention(qkv, qkv_pooled, num_heads, window_size, expand_size, focal_kernel, scale,
                           valid_ind_rolled):
    """softmax(q k_all^T) v_all of WindowAttention.forward, tfocal_transformer.py:222-396, literally:
    own-window keys, the four (-/+eh, -/+ew) circular rolls filtered by ``valid_ind_rolled``, and the pooled
    windows unfolded with zero padding whose padded entries get -100 added to the logit.
    qkv (B,T,H,W,3C), qkv_pooled (B,T,nWh,nWw,3C) or None -> (B,T,H,W,C) (already window-reversed)."""
    B, T, H, W, C3 = qkv.shape
    C = C3 // 3
    hd = C // num_heads
    wh, ww = window_size
    eh, ew = expand_size
    area = wh * ww
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]

    def heads(win):  # (B*nW, T*area, C) -> (B*nW, heads, T*area, hd)
        return win.view(win.shape[0], -1, num_heads, hd).permute(0, 2, 1, 3)

    qw, kw_, vw = heads(_partition(q, window_size)), heads(_partition(k, window_size)), heads(_partition(v, window_size))
    keys, vals = [kw_], [vw]
    if eh > 0 or ew > 0:
        def rolled(t):
            parts = []
            for sh, sw in ((-eh, -ew), (-eh, ew), (eh, -ew), (eh, ew)):  # tl, tr, bl, br (:235-254)
                r = torch.roll(t, shifts=(sh, sw), dims=(2, 3))
                parts.append(_partition(r, window_size).view(-1, T, area, num_heads, hd))
            r = torch.cat(parts, 2).permute(0, 3, 1, 2, 4)[:, :, :, valid_ind_rolled]  # (:256-273)
            return r.reshape(r.shape[0], num_heads, -1, hd)
        keys.append(rolled(k))
        vals.append(rolled(v))
    n_rolled = sum(t.shape[2] for t in keys)
    pooled_mask = None
    if qkv_pooled is not None:
        nWh, nWw = qkv_pooled.shape[2:4]
        fh, fw = focal_kernel
        pad = (fh // 2, fw // 2)
        ones = torch.ones(T, 1, nWh, nWw, dtype=qkv.dtype)
        um = F.unfold(ones, (fh, fw), padding=pad).view(1, T, fh, fw, -1).permute(4, 1, 2, 3, 0)
        um = um.reshape(nWh * nWw, -1)                                   # (nW, T*fh*fw)  (:301-316)
        pooled_mask = torch.where(um == 0, torch.full_like(um, -100.0), torch.zeros_like(um))

        def pooled(t):  # (B,T,nWh,nWw,C) -> (B*nW, heads, T*fh*fw, hd)   (:319-333)
            t = t.permute(0, 1, 4, 2, 3).reshape(B * T, C, nWh, nWw)
            u = F.unfold(t, (fh, fw), padding=pad).view(B, T, C, fh, fw, -1).permute(0, 5, 1, 3, 4, 2)
            u = u.reshape(-1, T, fh * fw, num_heads, hd).permute(0, 3, 1, 2, 4)
            return u.reshape(u.shape[0], num_heads, -1, hd)
        keys.append(pooled(qkv_pooled[..., C:2 * C]))
        vals.append(pooled(qkv_pooled[..., 2 * C:]))
    k_all, v_all = torch.cat(keys, 2), torch.cat(vals, 2)
    attn = (qw * scale) @ k_all.transpose(-2, -1)                        # (:359-362)
    if pooled_mask is not None:
        nW = pooled_mask.shape[0]
        m = pooled_mask[None, :, None, None, :].expand(attn.shape[0] // nW, nW, 1, 1, -1).reshape(-1, 1, 1,
                                                                                               pooled_mask.shape[-1])
        attn[:, :, :, n_rolled:] = attn[:, :, :, n_rolled:] + m          # (:377-380)
    attn = torch.softmax(attn, dim=-1)
    out = (attn @ v_all).transpose(1, 2).reshape(attn.shape[0], T * area, C)
    return _unpartition(out.view(-1, T, wh, ww, C), window_size, T, H, W)


def _fold_average(sd_unused, y, output_size, n_vecs):
    """fold / fold(ones) -> unfold of FusionFeedForward, tfocal_transformer.py:89-98 (HQ: _hq.py:99-117)."""
    b, n, c = y.shape
    yy = y.view(-1, n_vecs, c).permute(0, 2, 1)
    norm = F.fold(torch.ones(1, 49, n_vecs, dtype=y.dtype), output_size, (7, 7), padding=(3, 3), stride=(3, 3))
    img = F.fold(yy, output_size, (7, 7), padding=(3, 3), stride=(3, 3)) / norm
    return F.unfold(img, (7, 7), padding=(3, 3), stride=(3, 3)).permute(0, 2, 1).reshape(b, n, c)


def transformer_block(sd, prefix, x, output_size, num_heads=4, window_size=(5, 9), focal_window=(5, 9), taps=None):
    """TemporalFocalTransformerBlock.forward, tfocal_transformer.py:466-536."""
    B, T, H, W, C = x.shape
    wh, ww = window_size
    shortcut = x
    xn = F.layer_norm(x, (C,), sd[prefix + ".norm1.weight"], sd[prefix + ".norm1.bias"])
    # window pooling: Linear(wh*ww -> 1) over each window's tokens (:508-516)
    xw = xn.view(B, T, H // wh, wh, W // ww, ww, C).permute(0, 2, 4, 1, 6, 3, 5).reshape(B, H // wh, W // ww, T, C,
                                                                                          wh * ww)
    pooled = F.linear(xw, sd[prefix + ".pool_layers.0.weight"], sd[prefix + ".pool_layers.0.bias"]).flatten(-2)
    qkv = _linear(sd, prefix + ".attn.qkv", xn)
    qkv_pooled = _linear(sd, prefix + ".attn.qkv", pooled.permute(0, 3, 1, 2, 4))
    fk = tuple(2 * (i // 2) + 1 for i in focal_window)
    att = focal_window_attention(qkv, qkv_pooled, num_heads, window_size, (wh // 2, ww // 2), fk,
                                 (C // num_heads) ** -0.5, sd[prefix + ".attn.valid_ind_rolled"])
    if taps is not None:
        taps.append({"qkv": qkv, "qkv_pooled": qkv_pooled, "out": att})
    x = shortcut + _linear(sd, prefix + ".attn.proj", att)
    y = F.layer_norm(x, (C,), sd[prefix + ".norm2.weight"], sd[prefix + ".norm2.bias"])
    y = _linear(sd, prefix + ".mlp.conv1.0", y.view(B, T * H * W, C))
    y = _fold_average(None, y, output_size, H * W)
    y = _linear(sd, prefix + ".mlp.conv2.1", F.gelu(y))
    return x + y.view(B, T, H, W, C)


# --------------------------------------------------------------------------------------------- generator
_ENC = ((2, 1), (1, 1), (2, 1), (1, 1), (1, 1), (1, 2), (1, 4), (1, 8), (1, 1))  # (stride, groups) e2fgvi.py:75-94


def encoder(sd, x):
    """Encoder.forward, e2fgvi.py:96-109 (group-wise concat of the layer-8 input from layer 10 on)."""
    bt = x.size(0)
    out, x0 = x, None
    for k, (stride, groups) in enumerate(_ENC):
        if k == 4:
            x0 = out
        if k > 4:
            h, w = x0.shape[-2:]
            out = torch.cat([x0.view(bt, groups, -1, h, w), out.view(bt, groups, -1, h, w)], 2).view(bt, -1, h, w)
        out = F.leaky_relu(_conv(sd, f"encoder.layers.{2 * k}", out, stride, 1, groups), 0.2)
    return out


def decoder(sd, x):
    """e2fgvi.py:143-150 with deconv :112-130."""
    up = lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=True)  # noqa: E731
    y = F.leaky_relu(_conv(sd, "decoder.0.conv", up(x)), 0.2)
    y = F.leaky_relu(_conv(sd, "decoder.2", y), 0.2)
    y = F.leaky_relu(_conv(sd, "decoder.4.conv", up(y)), 0.2)
    return _conv(sd, "decoder.6", y)


def inpaint_generator_forward(sd, masked_frames, num_local_frames, hq=None, taps=None):
    """InpaintGenerator.forward, e2fgvi.py:236-263 (HQ: e2fgvi_hq.py:235-262).  ``sd``: reference state_dict.
    Returns (pred (b*t,3,H,W), (flows_forward, flows_backward))."""
    if hq is None:
        hq = "sc.bias_conv.weight" in sd
    l_t = num_local_frames
    b, t, ori_c, ori_h, ori_w = masked_frames.shape
    pred_flows = bidirect_flow(sd, (masked_frames[:, :l_t] + 1) / 2)
    enc = encoder(sd, masked_frames.reshape(b * t, ori_c, ori_h, ori_w))
    _, c, h, w = enc.shape
    enc = enc.view(b, t, c, h, w)
    prop_taps = [] if taps is not None else None
    local = bidirectional_propagation(sd, "feat_prop_module", enc[:, :l_t], pred_flows[0], pred_flows[1], prop_taps)
    enc = torch.cat((local, enc[:, l_t:]), dim=1)
    blk_taps = [] if taps is not None else None
    tok = transformer(sd, soft_split(sd, enc.reshape(-1, c, h, w), b), (h, w), blk_taps)
    enc = enc + soft_comp(sd, tok, t, (h, w), hq).view(b, t, -1, h, w)
    out = torch.tanh(decoder(sd, enc.reshape(b * t, c, h, w)))
    if taps is not None:
        taps.update({"propagation": prop_taps, "blocks": blk_taps, "local_feat": local, "tokens": tok})
    return out, pred_flows


def soft_split(sd, x, b):
    """SoftSplit.forward, tfocal_transformer.py:39-46 (HQ _hq.py:32-46): x (b*t, c, h, w) -> tokens (b, t, fh, fw, 512)."""
    h, w = x.shape[-2:]
    f_h, f_w = (h + 6 - 7) // 3 + 1, (w + 6 - 7) // 3 + 1
    tok = F.unfold(x, (7, 7), padding=(3, 3), stride=(3, 3)).permute(0, 2, 1)
    return _linear(sd, "ss.embedding", tok).view(b, -1, f_h, f_w, 512)


def transformer(sd, tok, output_size, taps=None):
    """The eight TemporalFocalTransformerBlocks (e2fgvi.py:188-198, :255)."""
    for i in range(8):
        tok = transformer_block(sd, f"transformer.{i}", tok, output_size, taps=taps)
    return tok


def soft_comp(sd, tok, t, output_size, hq):
    """SoftComp.forward, tfocal_transformer.py:65-72 (HQ _hq.py:67-79): tokens (b, t, fh, fw, 512) -> (b*t, c, h, w)."""
    b = tok.shape[0]
    feat = _linear(sd, "sc.embedding", tok.reshape(b, -1, 512))
    feat = feat.view(b * t, -1, feat.size(2)).permute(0, 2, 1)
    feat = F.fold(feat, output_size, (7, 7), padding=(3, 3), stride=(3, 3))
    return _conv(sd, "sc.bias_conv", feat) if hq else feat + sd["sc.bias"][None]


def generator_trunk(sd, frames, b, t, hq):
    """tanh(decoder(enc + sc(transformer(ss(enc, b)), t))) with enc = encoder(frames): InpaintGenerator.forward
    (e2fgvi.py:245-263, HQ e2fgvi_hq.py) with the flow completion and the propagation left out (the propagation taken
    as the identity).  frames (b*t, 3, H, W) -> prediction (b*t, 3, H, W)."""
    enc = encoder(sd, frames)
    h, w = enc.shape[-2:]
    tok = transformer(sd, soft_split(sd, enc, b), (h, w))
    return torch.tanh(decoder(sd, enc + soft_comp(sd, tok, t, (h, w), hq)))
