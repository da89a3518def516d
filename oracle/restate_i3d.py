"""Functional restatement of the reference's InceptionI3d.extract_features(x, 'Logits') (core/metrics.py:196-570) in
torch ops, from a state dict: F.pad "same" padding, conv3d, eval-mode batch norm (eps 1e-3), ReLU, zero-padded max
pools, the Inception concatenations and x.mean(4).mean(3).mean(2).  Runs on any device; the GPU tests compare the
kernels with it layer by layer and tools/i3d_bench.py times it on cuDNN."""
import torch
import torch.nn.functional as F

from e2fgvi_b200.i3d import ENDPOINTS, MIXED, POOLS, compute_pad


def _same(x, kernel, stride):
    pads = []
    for k, s, n in zip(kernel[::-1], stride[::-1], x.shape[:1:-1]):   # (w, h, t) for F.pad
        pads += list(compute_pad(k, s, n))
    return F.pad(x, pads)


def unit3d(sd, prefix, x, kernel=(1, 1, 1), stride=(1, 1, 1)):
    x = F.conv3d(_same(x, kernel, stride), sd[prefix + ".conv3d.weight"], None, stride)
    x = F.batch_norm(x, sd[prefix + ".bn.running_mean"], sd[prefix + ".bn.running_var"], sd[prefix + ".bn.weight"],
                     sd[prefix + ".bn.bias"], False, 0.0, 1e-3)
    return F.relu(x)


def max_pool(x, kernel, stride):
    return F.max_pool3d(_same(x, kernel, stride), kernel, stride)


def mixed(sd, name, x):
    b0 = unit3d(sd, name + ".b0", x)
    b1 = unit3d(sd, name + ".b1b", unit3d(sd, name + ".b1a", x), (3, 3, 3))
    b2 = unit3d(sd, name + ".b2b", unit3d(sd, name + ".b2a", x), (3, 3, 3))
    b3 = unit3d(sd, name + ".b3b", max_pool(x, (3, 3, 3), (1, 1, 1)))
    return torch.cat([b0, b1, b2, b3], 1)


def extract_features(sd, x, endpoints=None):
    """x (B, 3, T, H, W) fp32 in [0, 1] -> (B, 1024); ``endpoints`` (a dict) receives every endpoint's output."""
    sd = {k: v.to(x.device) for k, v in sd.items()}
    mixed_names = {m[0] for m in MIXED}
    for name in ENDPOINTS:
        if name == "Conv3d_1a_7x7":
            x = unit3d(sd, name, x, (7, 7, 7), (2, 2, 2))
        elif name in POOLS:
            x = max_pool(x, *POOLS[name])
        elif name == "Conv3d_2b_1x1":
            x = unit3d(sd, name, x)
        elif name == "Conv3d_2c_3x3":
            x = unit3d(sd, name, x, (3, 3, 3))
        else:
            assert name in mixed_names
            x = mixed(sd, name, x)
        if endpoints is not None:
            endpoints[name] = x
    return x.mean(4).mean(3).mean(2)
