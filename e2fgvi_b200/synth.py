"""Deterministic synthetic weights and frames.

No released checkpoint or dataset is reachable offline, so parity and benchmarks run on random-init weights and
synthetic frames (BASELINE.json).  Every tensor is drawn on the CPU from a ``torch.Generator`` seeded by
(seed, key), so the same values are produced in this container (where the goldens are made from the real
reference) and on the GPU box.

Two weight families:
* ``"default"``  — the reference's construction-time family: N(0,0.02) convs/linears with zero bias
  (e2fgvi.py:29-68), zeroed last offset conv (feat_prop.py:32-33), uniform DCN weight, kaiming SPyNet.
  Activations shrink to ~1e-2 and offsets equal the flow, so this family alone is a weak parity test (SURVEY §7).
* ``"stress"``   — fan-in-scaled weights so activations stay O(1), non-zero biases, a live last offset conv
  (offsets = flow + up to +-10 px, masks spread over (0,1)), perturbed LayerNorm / pooling weights.
"""
import hashlib
import math

import torch

FAMILIES = ("default", "stress")


def _gen(seed, key):
    h = hashlib.sha256(f"{seed}:{key}".encode()).digest()
    g = torch.Generator(device="cpu")
    g.manual_seed(int.from_bytes(h[:8], "little") & 0x7FFFFFFFFFFFFFFF)
    return g


def _normal(shape, std, g, mean=0.0):
    return torch.empty(shape, dtype=torch.float32).normal_(mean, std, generator=g)


def _fan_in(shape):
    return int(math.prod(shape[1:])) if len(shape) > 1 else int(shape[0])


def synth_state_dict(model, family="default", seed=0):
    """Return a full ``state_dict`` (CPU, fp32 / int64) for ``model`` with deterministic synthetic values."""
    if family not in FAMILIES:
        raise ValueError(f"family must be one of {FAMILIES}")
    ref = model.state_dict()
    out = {}
    stress = family == "stress"
    for key in sorted(ref.keys()):
        t = ref[key]
        shape = tuple(t.shape)
        g = _gen(seed, key)
        leaf = key.rsplit(".", 1)[-1]
        if not t.is_floating_point():  # attn.valid_ind_rolled: structural, keep the constructed value
            out[key] = t.detach().cpu().clone()
            continue
        if key.startswith("update_spynet."):
            if leaf in ("mean", "std"):
                out[key] = t.detach().cpu().clone()
            elif leaf == "weight":  # kaiming-normal fan_out / relu, what mmcv's ConvModule does by default
                fan_out = shape[0] * shape[2] * shape[3]
                out[key] = _normal(shape, math.sqrt(2.0 / fan_out), g)
                if stress and ".basic_module.4.conv." in key:
                    out[key] *= 0.06  # keeps |flow| at a few pixels so warps sample inside the map
            else:
                out[key] = _normal(shape, 0.02, g) if stress else torch.zeros(shape)
            continue
        if ".norm1." in key or ".norm2." in key:
            if leaf == "weight":
                out[key] = 1.0 + (_normal(shape, 0.1, g) if stress else 0.0) * torch.ones(shape)
            else:
                out[key] = _normal(shape, 0.1, g) if stress else torch.zeros(shape)
            continue
        if key == "sc.bias":
            out[key] = _normal(shape, 0.1, g) if stress else torch.zeros(shape)
            continue
        if ".pool_layers." in key:
            if leaf == "weight":
                out[key] = (1.0 / shape[1] + _normal(shape, 0.01, g)) if stress else _normal(shape, 0.02, g)
            else:
                out[key] = _normal(shape, 0.05, g) if stress else torch.zeros(shape)
            continue
        is_dcn = ".deform_align." in key and ".conv_offset." not in key
        is_last_offset = ".conv_offset.6." in key
        if leaf == "weight":
            fan = _fan_in(shape)
            if is_dcn:
                bound = 1.0 / math.sqrt(fan)
                w = torch.empty(shape).uniform_(-bound, bound, generator=g)
                out[key] = w * (math.sqrt(3.0) if stress else 1.0)  # stress: unit-variance-preserving
            elif is_last_offset:
                out[key] = _normal(shape, 0.6 / math.sqrt(fan), g) if stress else torch.zeros(shape)
            elif stress:
                out[key] = _normal(shape, 1.0 / math.sqrt(fan), g)
            else:
                out[key] = _normal(shape, 0.02, g)
        elif leaf == "bias":
            if is_last_offset:
                out[key] = _normal(shape, 0.3, g) if stress else torch.zeros(shape)
            else:
                out[key] = _normal(shape, 0.05, g) if stress else torch.zeros(shape)
        else:
            raise KeyError(f"no synthetic rule for {key}")
    return out


def synth_frames(b, t, h, w, seed=0, holes=True):
    """``masked_frames`` (b,t,3,h,w) fp32 in [-1,1]: smooth moving texture + noise, with a zeroed rectangle per
    frame (what test.py:155 feeds the model: imgs*(1-mask))."""
    g = _gen(seed, f"frames:{b}:{t}:{h}:{w}")
    yy = torch.linspace(0, 1, h).view(1, 1, 1, h, 1)
    xx = torch.linspace(0, 1, w).view(1, 1, 1, 1, w)
    tt = torch.arange(t, dtype=torch.float32).view(1, t, 1, 1, 1)
    ph = torch.rand((b, 1, 3, 1, 1), generator=g) * 6.28
    base = 0.5 * torch.sin(6.28 * (2.0 * xx + 0.03 * tt) + ph) * torch.cos(6.28 * (1.5 * yy - 0.02 * tt))
    x = (base + 0.5 * (torch.rand((b, t, 3, h, w), generator=g) * 2 - 1)).clamp_(-1, 1)
    if holes:
        hh, ww = max(h // 4, 1), max(w // 4, 1)
        for bi in range(b):
            for ti in range(t):
                y0 = int(torch.randint(0, h - hh + 1, (1,), generator=g))
                x0 = int(torch.randint(0, w - ww + 1, (1,), generator=g))
                x[bi, ti, :, y0:y0 + hh, x0:x0 + ww] = 0.0
    return x.contiguous()


def synth_video(n, h, w, seed=0):
    """A synthetic RGB video and its hole masks for the video-level driver (test.py:125-141):
    ``frames`` (n,h,w,3) uint8 — drifting sinusoid texture + noise — and ``masks`` (n,h,w) uint8 in {0,1} — a
    rectangle that moves across the frame (before the reference's 4x cross dilation)."""
    import numpy as np
    g = _gen(seed, f"video:{n}:{h}:{w}")
    yy = torch.linspace(0, 1, h).view(1, h, 1, 1)
    xx = torch.linspace(0, 1, w).view(1, 1, w, 1)
    tt = torch.arange(n, dtype=torch.float32).view(n, 1, 1, 1)
    ph = torch.rand((1, 1, 1, 3), generator=g) * 6.28
    base = 0.5 + 0.35 * torch.sin(6.28 * (2.0 * xx + 0.02 * tt) + ph) * torch.cos(6.28 * (1.5 * yy - 0.015 * tt))
    x = (base + 0.15 * (torch.rand((n, h, w, 3), generator=g) - 0.5)).clamp_(0, 1)
    frames = (x * 255).round().to(torch.uint8).numpy()
    masks = np.zeros((n, h, w), dtype=np.uint8)
    hh, ww = max(h // 3, 1), max(w // 4, 1)
    for i in range(n):
        y0 = int((h - hh) * (0.5 + 0.4 * math.sin(0.5 * i)))
        x0 = int((w - ww) * (i / max(n - 1, 1)))
        masks[i, y0:y0 + hh, x0:x0 + ww] = 1
    return frames, masks


def synth_i3d_state_dict(seed=0):
    """A full ``InceptionI3d`` state dict (the reference's 344 keys, CPU) with deterministic synthetic values: conv
    weights N(0, 2 / fan_in) (He), so activations stay O(1) through the 57 ReLU layers; BatchNorm weight 1 + N(0, 0.1),
    bias N(0, 0.1), running mean N(0, 0.1) and running var 1 + U(-0.3, 0.3), so that the host-side folding is exercised;
    ``num_batches_tracked`` kept; the classifier's conv weight and bias N(0, 0.02)."""
    from .i3d import InceptionI3d
    out = {}
    for key, t in InceptionI3d().state_dict().items():
        shape = tuple(t.shape)
        g = _gen(seed, "i3d:" + key)
        leaf = key.rsplit(".", 1)[-1]
        if not t.is_floating_point():
            out[key] = t.detach().clone()
        elif key.startswith("logits."):
            out[key] = _normal(shape, 0.02, g)
        elif ".conv3d." in key:
            out[key] = _normal(shape, math.sqrt(2.0 / _fan_in(shape)), g)
        elif leaf == "weight":
            out[key] = 1.0 + _normal(shape, 0.1, g)
        elif leaf in ("bias", "running_mean"):
            out[key] = _normal(shape, 0.1, g)
        elif leaf == "running_var":
            out[key] = 1.0 + torch.empty(shape).uniform_(-0.3, 0.3, generator=g)
        else:
            raise KeyError(f"no synthetic rule for {key}")
    return out


def synth_activations(n, d, seed=0):
    """(n, d) float64 synthetic activation rows for Fréchet-distance checks: non-negative and correlated, like I3D's
    post-ReLU feature means."""
    g = _gen(seed, f"activations:{n}:{d}")
    mix = torch.randn((d, d), generator=g, dtype=torch.float64) / math.sqrt(d)
    z = torch.randn((n, d), generator=g, dtype=torch.float64)
    return (z @ mix + 0.5).clamp_(min=0).numpy()


def synth_composite_pair(h, w, c, seed, holes=True):
    """A uint8 frame and an evaluate.py-like composite: multiples of 1/4, equal to the frame outside the holes."""
    import numpy as np
    rng = np.random.default_rng(seed)
    ori = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
    comp = ori.astype(np.float32)
    if holes:
        y0, x0 = h // 4, w // 3
        quarters = rng.integers(0, 255 * 4 + 1, (h // 2, w // 3, c)).astype(np.float32) / 4
        comp[y0:y0 + h // 2, x0:x0 + w // 3] = quarters
    return ori, comp


def write_eval_dataset(root, videos, size=(54, 96), drop_mask=None):
    """A DAVIS-layout dataset as evaluate.py reads it: R/davis/{test.json, JPEGImages/<v>.zip, test_masks/<v>/%05d.png}.
    Zip members are PNG (lossless: decoding does not depend on the OpenCV build); masks are at frame size and, as
    DAVIS's, palette images (index 1 = hole, colour (128, 0, 0)); the holes are the top quarter of ``synth_video``'s
rectangles.  ``videos``: name -> frame count; video k comes from
    ``synth_video(n, *size, seed=40 + k)``.  Returns R and {name: (frames, masks)}."""
    import json
    import os
    import zipfile
    import cv2
    import numpy as np
    from PIL import Image
    data = os.path.join(root, "davis")
    os.makedirs(os.path.join(data, "JPEGImages"))
    with open(os.path.join(data, "test.json"), "w") as f:
        json.dump(videos, f)
    out = {}
    for k, (name, n) in enumerate(videos.items()):
        frames, masks = synth_video(n, *size, seed=40 + k)
        for m in masks:                                   # the top quarter of each rectangle: small goldens
            rows = np.nonzero(m.any(1))[0]
            m[rows[0] + (len(rows) + 3) // 4:] = 0
        with zipfile.ZipFile(os.path.join(data, "JPEGImages", f"{name}.zip"), "w") as z:
            for i in range(n):
                z.writestr(f"{i:05d}.png", cv2.imencode(".png", cv2.cvtColor(frames[i], cv2.COLOR_RGB2BGR))[1].tobytes())
        mdir = os.path.join(data, "test_masks", name)
        os.makedirs(mdir)
        for i in range(n):
            if (name, i) != drop_mask:
                im = Image.fromarray(masks[i], mode="P")
                im.putpalette([0, 0, 0, 128, 0, 0] + [0] * 762)
                im.save(os.path.join(mdir, f"{i:05d}.png"))
        out[name] = (frames, masks)
    return root, out


def synth_dis_state_dict(seed=0, use_spectral_norm=True, in_channels=3):
    """State dict of ``Discriminator(in_channels, use_spectral_norm=...)`` with deterministic values: fan-in-scaled
    weights (activations stay O(1) through the six layers), small biases, and under spectral norm ``weight_u`` /
    ``weight_v`` from ten power iterations on the weight."""
    chans = (in_channels, 32, 64, 128, 128, 128, 128)
    sd = {}
    for i in range(6):
        cout, cin = chans[i + 1], chans[i]
        shape = (cout, cin, 3, 5, 5)
        w = _normal(shape, math.sqrt(2.0 / _fan_in(shape)), _gen(seed, f"dis.{i}.w"))
        p = f"conv.{2 * i}."
        if i < 5 and use_spectral_norm:
            sd[p + "weight_orig"] = w
            # near the top singular pair (as after some training), so that eval()-mode sigma is not arbitrarily small
            u = _normal((cout,), 1.0, _gen(seed, f"dis.{i}.u")).double()
            wm = w.double().reshape(cout, -1)
            for _ in range(10):
                v = wm.t() @ u
                v = v / v.norm()
                u = wm @ v
                u = u / u.norm()
            sd[p + "weight_u"] = u.float()
            sd[p + "weight_v"] = v.float()
        else:
            sd[p + "weight"] = w
            sd[p + "bias"] = _normal((cout,), 0.1, _gen(seed, f"dis.{i}.b"))
    return sd


def synth_spynet_state_dict(seed=0, prefix="", flow_scale=1.0):
    """State dict of a ``SPyNet`` (``prefix`` e.g. "update_spynet." or "fix_spynet.") with deterministic values:
    fan-in-scaled (He) weights so that activations stay O(1) through each level's five convs, small biases, and the last
    conv of every level scaled by ``flow_scale`` so that the flows reach several pixels (about 10 at 64x128 for 1.0, 3 for
    0.25): enough for warps that clamp at the border and for coarse-level flows that move whole pixels."""
    from .model.modules.flow_comp import _LEVEL_CONVS, _NUM_LEVELS
    sd = {}
    for level in range(_NUM_LEVELS):
        for k, (cin, cout) in enumerate(_LEVEL_CONVS):
            shape = (cout, cin, 7, 7)
            std = math.sqrt(2.0 / _fan_in(shape)) * (flow_scale if k == len(_LEVEL_CONVS) - 1 else 1.0)
            key = f"{prefix}basic_module.{level}.basic_module.{k}.conv."
            sd[key + "weight"] = _normal(shape, std, _gen(seed, f"spy.{level}.{k}.w"))
            sd[key + "bias"] = _normal((cout,), 0.05, _gen(seed, f"spy.{level}.{k}.b"))
    sd[prefix + "mean"] = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    sd[prefix + "std"] = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    return sd
