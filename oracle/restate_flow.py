"""Float64 restatement of the differentiable flow path: ``InpaintGenerator.forward_bidirect_flow`` (model/e2fgvi.py:210-234)
and ``FlowCompletionLoss`` (model/modules/flow_comp.py:11-46) in plain torch, so that autograd gives its gradients.

It follows the reference op for op: the 1/4 bilinear downsample, SPyNet's resize to multiples of 32, the pyramid, per
level the x2 upsample, ``flow_warp`` with border padding through ``F.grid_sample`` (its normalise / denormalise round
trip and its backward conventions included), five 7x7 convs and the resize back.  The ReLUs can take their slopes from
outside (``slopes``: per level, per ReLU a 0/1 mask), so that a comparison is not decided by pre-activations that lie
within rounding of 0, where fp32 and fp64 legitimately pick different sides.  Runs on any device.
"""
import torch
import torch.nn.functional as F


class _ReluWithSlopes(torch.autograd.Function):
    """relu(x) whose derivative is the given 0/1 mask instead of (x > 0)."""

    @staticmethod
    def forward(ctx, x, mask):
        ctx.save_for_backward(mask)
        return x.clamp_min(0)

    @staticmethod
    def backward(ctx, g):
        (mask,) = ctx.saved_tensors
        return g * mask, None


def flow_warp(x, flow):
    """flow_comp.py:345-383 with padding_mode='border', align_corners=True."""
    n, _, h, w = x.shape
    gy, gx = torch.meshgrid(torch.arange(0, h, dtype=x.dtype, device=x.device),
                            torch.arange(0, w, dtype=x.dtype, device=x.device), indexing="ij")
    grid = torch.stack((gx, gy), 2)
    grid_flow = grid + flow
    gfx = 2.0 * grid_flow[:, :, :, 0] / max(w - 1, 1) - 1.0
    gfy = 2.0 * grid_flow[:, :, :, 1] / max(h - 1, 1) - 1.0
    return F.grid_sample(x, torch.stack((gfx, gfy), dim=3), mode="bilinear", padding_mode="border", align_corners=True)


def spynet(params, mean, std, ref, supp, slopes=None, record=None):
    """SPyNet.forward (flow_comp.py:136-169).  params[level][k] = (weight, bias); slopes[level][k] (k < 4): 0/1 mask
    of the ReLU after conv k or None; ``record`` (a list) receives the (pre-activation > 0) masks."""
    h, w = ref.shape[2:4]
    w_up = w if w % 32 == 0 else 32 * (w // 32 + 1)
    h_up = h if h % 32 == 0 else 32 * (h // 32 + 1)
    ref = F.interpolate(ref, size=(h_up, w_up), mode="bilinear", align_corners=False)
    supp = F.interpolate(supp, size=(h_up, w_up), mode="bilinear", align_corners=False)
    refs, supps = [(ref - mean) / std], [(supp - mean) / std]
    for _ in range(5):
        refs.append(F.avg_pool2d(refs[-1], 2, 2, count_include_pad=False))
        supps.append(F.avg_pool2d(supps[-1], 2, 2, count_include_pad=False))
    refs, supps = refs[::-1], supps[::-1]
    flow = ref.new_zeros(ref.size(0), 2, h_up // 32, w_up // 32)
    for level in range(6):
        up = flow if level == 0 else F.interpolate(flow, scale_factor=2, mode="bilinear", align_corners=True) * 2.0
        y = torch.cat([refs[level], flow_warp(supps[level], up.permute(0, 2, 3, 1)), up], 1)
        rec = []
        for k in range(5):
            wt, b = params[level][k]
            y = F.conv2d(y, wt, b, 1, 3)
            if k < 4:
                rec.append(y.detach() > 0)
                m = None if slopes is None else slopes[level][k]
                y = F.relu(y) if m is None else _ReluWithSlopes.apply(y, m.to(y.dtype))
        if record is not None:
            record.append(rec)
        flow = up + y
    flow = F.interpolate(flow, size=(h, w), mode="bilinear", align_corners=False)
    return torch.stack((flow[:, 0] * (float(w) / float(w_up)), flow[:, 1] * (float(h) / float(h_up))), dim=1)


def forward_bidirect_flow(params, mean, std, frames, slopes=None, record=None):
    """e2fgvi.py:210-234 on frames (b, l_t, 3, h, w) in [0, 1].  Both directions run as one batch (forward pairs, then
    backward pairs), which is the order of ``slopes`` / ``record``."""
    b, l_t, c, h, w = frames.shape
    small = F.interpolate(frames.reshape(-1, c, h, w), scale_factor=1 / 4, mode="bilinear", align_corners=True,
                          recompute_scale_factor=True).view(b, l_t, c, h // 4, w // 4)
    a = small[:, :-1].reshape(-1, c, h // 4, w // 4)
    z = small[:, 1:].reshape(-1, c, h // 4, w // 4)
    n = a.size(0)
    both = spynet(params, mean, std, torch.cat([a, z]), torch.cat([z, a]), slopes, record)
    return both[:n].reshape(b, l_t - 1, 2, h // 4, w // 4), both[n:].reshape(b, l_t - 1, 2, h // 4, w // 4)


def flow_completion_loss(gt_params, mean, std, pred_flows, gt_frames):
    """FlowCompletionLoss.forward: L1 per direction against the frozen SPyNet's flows on the ground truth, summed."""
    with torch.no_grad():
        gf, gb = forward_bidirect_flow(gt_params, mean, std, gt_frames)
    return (pred_flows[0] - gf).abs().mean() + (pred_flows[1] - gb).abs().mean()


def params_from_state_dict(sd, prefix, dtype=torch.float64, device=None, requires_grad=False):
    """[[(weight, bias)] * 5] * 6 leaf tensors from a state dict's ``<prefix>.basic_module.*`` entries (``prefix`` ""
    for a SPyNet's own state dict)."""
    prefix = prefix + "." if prefix else ""
    out = []
    for level in range(6):
        row = []
        for k in range(5):
            key = f"{prefix}basic_module.{level}.basic_module.{k}.conv"
            wt = sd[key + ".weight"].to(device=device, dtype=dtype).detach().clone().requires_grad_(requires_grad)
            b = sd[key + ".bias"].to(device=device, dtype=dtype).detach().clone().requires_grad_(requires_grad)
            row.append((wt, b))
        out.append(row)
    return out
