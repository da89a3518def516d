"""InceptionI3d — the feature extractor behind evaluate.py's VFID (reference core/metrics.py:192-570) on the sm_90a
kernels of ``csrc/i3d.cu`` and ``csrc/conv.cu``.

The module keeps the reference's parameter layout (its ``state_dict`` has the same 344 keys, shapes and dtypes, so
``i3d_rgb_imagenet.pt`` loads with ``strict=True``) and computes ``extract_features(x, 'Logits')``: the network up to
``Mixed_5c`` and ``x.mean(4).mean(3).mean(2)``, a 1024-d vector per video.  BatchNorm is applied with its running
statistics (eval mode), folded into the conv weights and bias on the host.  The classifier head (``logits``) exists
only so that checkpoints load; ``forward`` and every other endpoint raise.  There is no CPU path.
"""
import ctypes

import torch
import torch.nn as nn

from . import _lib, ops

BN_EPS = 1e-3

# (name, in_channels, [b0, b1a, b1b, b2a, b2b, b3b]) of the nine Inception modules, reference core/metrics.py:450-518
MIXED = (
    ("Mixed_3b", 192, (64, 96, 128, 16, 32, 32)),
    ("Mixed_3c", 256, (128, 128, 192, 32, 96, 64)),
    ("Mixed_4b", 480, (192, 96, 208, 16, 48, 64)),
    ("Mixed_4c", 512, (160, 112, 224, 24, 64, 64)),
    ("Mixed_4d", 512, (128, 128, 256, 24, 64, 64)),
    ("Mixed_4e", 512, (112, 144, 288, 32, 64, 64)),
    ("Mixed_4f", 528, (256, 160, 320, 32, 128, 128)),
    ("Mixed_5b", 832, (256, 160, 320, 32, 128, 128)),
    ("Mixed_5c", 832, (384, 192, 384, 48, 128, 128)),
)
# max pools in network order: name -> (kernel, stride)
POOLS = {
    "MaxPool3d_2a_3x3": ((1, 3, 3), (1, 2, 2)),
    "MaxPool3d_3a_3x3": ((1, 3, 3), (1, 2, 2)),
    "MaxPool3d_4a_3x3": ((3, 3, 3), (2, 2, 2)),
    "MaxPool3d_5a_2x2": ((2, 2, 2), (2, 2, 2)),
}
ENDPOINTS = ("Conv3d_1a_7x7", "MaxPool3d_2a_3x3", "Conv3d_2b_1x1", "Conv3d_2c_3x3", "MaxPool3d_3a_3x3", "Mixed_3b",
             "Mixed_3c", "MaxPool3d_4a_3x3", "Mixed_4b", "Mixed_4c", "Mixed_4d", "Mixed_4e", "Mixed_4f",
             "MaxPool3d_5a_2x2", "Mixed_5b", "Mixed_5c")


def compute_pad(k, stride, s):
    """The reference's "same" padding of one axis of size s: (front, back)."""
    pad = max(k - stride, 0) if s % stride == 0 else max(k - s % stride, 0)
    return pad // 2, pad - pad // 2


def same_pad(kernel, stride, size):
    """(t_front, t_back, h_front, h_back, w_front, w_back) and the output size for kernel / stride / size triples."""
    pads, out = [], []
    for k, s, n in zip(kernel, stride, size):
        f, b = compute_pad(k, s, n)
        pads += [f, b]
        out.append((n + f + b - k) // s + 1)
    return pads, tuple(out)


def _ints(v):
    return (ctypes.c_int * len(v))(*v)


class Unit3D(nn.Module):
    """Parameters of the reference's Unit3D: ``conv3d`` (no bias unless ``use_bias``) and ``bn`` (BatchNorm3d,
    eps 1e-3) when ``use_batch_norm``."""

    def __init__(self, in_channels, output_channels, kernel_shape=(1, 1, 1), stride=(1, 1, 1), use_batch_norm=True,
                 use_bias=False):
        super().__init__()
        self.kernel_shape, self.stride = tuple(kernel_shape), tuple(stride)
        self.conv3d = nn.Conv3d(in_channels, output_channels, kernel_shape, stride, padding=0, bias=use_bias)
        if use_batch_norm:
            self.bn = nn.BatchNorm3d(output_channels, eps=BN_EPS, momentum=0.01)


class InceptionModule(nn.Module):
    def __init__(self, in_channels, out_channels):
        super().__init__()
        c = out_channels
        self.b0 = Unit3D(in_channels, c[0])
        self.b1a = Unit3D(in_channels, c[1])
        self.b1b = Unit3D(c[1], c[2], (3, 3, 3))
        self.b2a = Unit3D(in_channels, c[3])
        self.b2b = Unit3D(c[3], c[4], (3, 3, 3))
        self.b3b = Unit3D(in_channels, c[5])
        self.out_channels = c[0] + c[2] + c[4] + c[5]


class _Act:
    """An NDHWC activation [B][T][H][W][C]: fp32 and / or its bf16 (hi, lo) split."""

    __slots__ = ("f32", "hi", "lo", "size", "c")

    def __init__(self, f32, hi, lo, size, c):
        self.f32, self.hi, self.lo, self.size, self.c = f32, hi, lo, size, c


class InceptionI3d(nn.Module):
    """Drop-in for the reference's ``InceptionI3d(num_classes, in_channels=3)`` as ``evaluate.py`` uses it."""

    def __init__(self, num_classes=400, in_channels=3, spatial_squeeze=True, final_endpoint="Logits",
                 name="inception_i3d", dropout_keep_prob=0.5):
        super().__init__()
        if in_channels != 3:
            raise NotImplementedError("InceptionI3d: the stem kernel takes 3 input channels")
        if final_endpoint != "Logits":
            raise NotImplementedError("InceptionI3d: only the 'Logits' network (extract_features) is implemented")
        # registration order follows the reference, so state_dict() lists the keys in the same order
        self.logits = Unit3D(384 + 384 + 128 + 128, num_classes, use_batch_norm=False, use_bias=True)
        self.Conv3d_1a_7x7 = Unit3D(in_channels, 64, (7, 7, 7), (2, 2, 2))
        self.Conv3d_2b_1x1 = Unit3D(64, 64)
        self.Conv3d_2c_3x3 = Unit3D(64, 192, (3, 3, 3))
        for name_, cin, c in MIXED:
            self.add_module(name_, InceptionModule(cin, c))

    # ------------------------------------------------------------------------------------------------ parameters
    def load_state_dict(self, state_dict, strict=True, assign=False):
        result = super().load_state_dict(state_dict, strict=strict, assign=assign)
        ops.invalidate_weight_caches()
        return result

    @staticmethod
    def _folded(unit, stem=False):
        """(w_hi, w_lo, bias) of a Unit3D with its BatchNorm folded in, packed in the K order of the conv kernel;
        cached until one of the parameters changes (``ops.invalidate_weight_caches`` drops it)."""
        bn = unit.bn
        params = [unit.conv3d.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var]

        def build():
            w = unit.conv3d.weight.detach().double()
            scale = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
            bias = (bn.bias.detach().double() - bn.running_mean.detach().double() * scale).float().contiguous()
            w = (w * scale.view(-1, 1, 1, 1, 1)).float()
            cout, cin = w.shape[:2]
            if stem:          # [co][kt][ky][16 px][4 ch]: one 64-wide K chunk per (kt, ky), zeros past kx 7 / channel 3
                packed = torch.zeros((cout, 7, 7, 16, 4), dtype=torch.float32, device=w.device)
                packed[..., :7, :3] = w.permute(0, 2, 3, 4, 1)
                hi, lo = ops.split_bf16(packed.view(cout, -1))
            else:             # [co][tap (kt, ky, kx)][cin padded to 64-channel chunks]
                taps = w[0, 0].numel()
                kp = (cin + 63) // 64 * 64
                packed = torch.zeros((cout, taps, kp), dtype=torch.float32, device=w.device)
                packed[:, :, :cin] = w.reshape(cout, cin, taps).transpose(1, 2)
                hi, lo = ops.split_bf16(packed.view(cout, -1))
            return hi, lo, bias

        return ops._derived(params, ("i3d_fold", stem), build)

    # ------------------------------------------------------------------------------------------------ layers
    @staticmethod
    def _alloc(b, size, c, dev, f32=True, split=True):
        shape = (b,) + tuple(size) + (c,)
        o = torch.empty(shape, dtype=torch.float32, device=dev) if f32 else None
        hi = torch.empty(shape, dtype=torch.bfloat16, device=dev) if split else None
        lo = torch.empty(shape, dtype=torch.bfloat16, device=dev) if split else None
        return _Act(o, hi, lo, tuple(size), c)

    @staticmethod
    def _ptr(t, coff=0):
        return None if t is None else t.data_ptr() + coff * t.element_size()

    def _conv(self, unit, x, b, out, coff=0):
        """Unit3D (conv, folded BN, ReLU) of x into channels [coff, coff + cout) of ``out``."""
        w_hi, w_lo, bias = self._folded(unit)
        k = unit.kernel_shape[0]
        pads, size = same_pad((k,) * 3, (1, 1, 1), x.size)
        assert size == out.size
        cout = unit.conv3d.weight.shape[0]
        with ops._timed(f"conv3d_{k}x{k}x{k}", 2.0 * b * size[0] * size[1] * size[2] * cout * x.c * k ** 3):
            st = _lib.load().e2f_conv3d_bf16x3(x.hi.data_ptr(), x.lo.data_ptr(), x.c, w_hi.data_ptr(), w_lo.data_ptr(),
                                               bias.data_ptr(), self._ptr(out.f32, coff), self._ptr(out.hi, coff),
                                               self._ptr(out.lo, coff), out.c, b, x.size[0], x.size[1], x.size[2], cout,
                                               k, _ints(pads), 1, ops._stream())
        _lib.check(st, "e2f_conv3d_bf16x3")
        return out

    def _pool(self, name, x, b, split=True):
        k, s = POOLS[name]
        pads, size = same_pad(k, s, x.size)
        out = self._alloc(b, size, x.c, x.f32.device, split=split)
        with ops._timed("maxpool3d", 4.0 * x.f32.numel()):
            st = _lib.load().e2f_maxpool3d(x.f32.data_ptr(), out.f32.data_ptr(), self._ptr(out.hi), self._ptr(out.lo), b,
                                           x.size[0], x.size[1], x.size[2], x.c, _ints(k), _ints(s), _ints(pads),
                                           ops._stream())
        _lib.check(st, "e2f_maxpool3d")
        return out

    def _mixed(self, mod, x, b):
        c = [mod.b0, mod.b1a, mod.b1b, mod.b2a, mod.b2b, mod.b3b]
        ch = [u.conv3d.weight.shape[0] for u in c]
        dev = x.hi.device
        out = self._alloc(b, x.size, mod.out_channels, dev)
        self._conv(mod.b0, x, b, out, 0)
        t1 = self._conv(mod.b1a, x, b, self._alloc(b, x.size, ch[1], dev, f32=False))
        self._conv(mod.b1b, t1, b, out, ch[0])
        t2 = self._conv(mod.b2a, x, b, self._alloc(b, x.size, ch[3], dev, f32=False))
        self._conv(mod.b2b, t2, b, out, ch[0] + ch[2])
        # b3a: 3x3x3 / stride 1 max pool of the module input, written as the split operand of b3b only
        pads, _ = same_pad((3, 3, 3), (1, 1, 1), x.size)
        p3 = self._alloc(b, x.size, x.c, dev, f32=False)
        with ops._timed("maxpool3d", 4.0 * x.f32.numel()):
            st = _lib.load().e2f_maxpool3d(x.f32.data_ptr(), None, p3.hi.data_ptr(), p3.lo.data_ptr(), b, x.size[0],
                                           x.size[1], x.size[2], x.c, _ints((3, 3, 3)), _ints((1, 1, 1)), _ints(pads),
                                           ops._stream())
        _lib.check(st, "e2f_maxpool3d")
        self._conv(mod.b3b, p3, b, out, ch[0] + ch[2] + ch[4])
        return out

    def _run(self, src, x_u8, b, t, h, w, endpoints=None):
        """The network from the packed stem input to the (b, 1024) features.  ``endpoints``: an optional dict that
        receives every endpoint's fp32 NDHWC output (tests compare them layer by layer)."""
        lib = _lib.load()
        dev = src.device
        keep = endpoints is not None
        n = int(lib.e2f_i3d_stem_elems(b, t, h, w))
        s_hi = torch.empty(n, dtype=torch.bfloat16, device=dev)
        s_lo = torch.empty(n, dtype=torch.bfloat16, device=dev)
        with ops._timed("i3d_stem_pack", float(src.numel() * src.element_size() + 4 * n)):
            st = lib.e2f_i3d_stem_pack(src.data_ptr(), x_u8, s_hi.data_ptr(), s_lo.data_ptr(), b, t, h, w, ops._stream())
        _lib.check(st, "e2f_i3d_stem_pack")
        unit = self.Conv3d_1a_7x7
        w_hi, w_lo, bias = self._folded(unit, stem=True)
        _, size = same_pad((7, 7, 7), (2, 2, 2), (t, h, w))
        x = self._alloc(b, size, 64, dev, split=False)
        with ops._timed("conv3d_stem", 2.0 * b * size[0] * size[1] * size[2] * 64 * 3 * 343):
            st = lib.e2f_i3d_stem_conv(s_hi.data_ptr(), s_lo.data_ptr(), w_hi.data_ptr(), w_lo.data_ptr(), bias.data_ptr(),
                                       x.f32.data_ptr(), None, None, 64, b, t, h, w, 64, ops._stream())
        _lib.check(st, "e2f_i3d_stem_conv")

        def note(name, a):
            if keep:
                endpoints[name] = a.f32

        note("Conv3d_1a_7x7", x)
        x = self._pool("MaxPool3d_2a_3x3", x, b)
        note("MaxPool3d_2a_3x3", x)
        x = self._conv(self.Conv3d_2b_1x1, x, b, self._alloc(b, x.size, 64, dev, f32=keep))
        note("Conv3d_2b_1x1", x)
        x = self._conv(self.Conv3d_2c_3x3, x, b, self._alloc(b, x.size, 192, dev, split=False))
        note("Conv3d_2c_3x3", x)
        x = self._pool("MaxPool3d_3a_3x3", x, b)
        note("MaxPool3d_3a_3x3", x)
        for name, _, _ in MIXED:
            if name == "Mixed_4b":
                x = self._pool("MaxPool3d_4a_3x3", x, b)
                note("MaxPool3d_4a_3x3", x)
            elif name == "Mixed_5b":
                x = self._pool("MaxPool3d_5a_2x2", x, b)
                note("MaxPool3d_5a_2x2", x)
            x = self._mixed(getattr(self, name), x, b)
            note(name, x)
        feats = torch.empty((b, x.c), dtype=torch.float32, device=dev)
        with ops._timed("mean_thw", 4.0 * x.f32.numel()):
            st = lib.e2f_mean_thw(x.f32.data_ptr(), feats.data_ptr(), b, x.size[0], x.size[1], x.size[2], x.c,
                                  ops._stream())
        _lib.check(st, "e2f_mean_thw")
        return feats

    # ------------------------------------------------------------------------------------------------ public
    @torch.no_grad()
    def extract_features(self, x, target_endpoint="Logits"):
        """The reference's ``extract_features(x, 'Logits')``: x fp32 (B, 3, T, H, W) in [0, 1] on the GPU -> (B, 1024)."""
        if target_endpoint != "Logits":
            raise NotImplementedError(f"InceptionI3d.extract_features: only target_endpoint='Logits', got {target_endpoint!r}")
        ops._need_cuda(x)
        if x.dim() != 5 or x.shape[1] != 3:
            raise ValueError(f"extract_features: expected (B, 3, T, H, W), got {tuple(x.shape)}")
        b, _, t, h, w = x.shape
        return self._run(x.contiguous().float(), 0, b, t, h, w)

    @torch.no_grad()
    def features_u8(self, frames):
        """uint8 RGB frames (B, T, H, W, 3) or (T, H, W, 3) on the GPU (what ``VideoInpainter`` returns) -> (B, 1024)
        features, equal to ``extract_features(frames / 255)`` bit for bit.  No host round trip."""
        ops._need_cuda(frames)
        if frames.dtype != torch.uint8 or frames.shape[-1] != 3 or frames.dim() not in (4, 5):
            raise ValueError(f"features_u8: expected uint8 (B, T, H, W, 3) or (T, H, W, 3), got {frames.dtype} "
                             f"{tuple(frames.shape)}")
        if frames.dim() == 4:
            frames = frames.unsqueeze(0)
        b, t, h, w, _ = frames.shape
        return self._run(frames.contiguous(), 1, b, t, h, w)

    def forward(self, x):
        raise NotImplementedError("InceptionI3d.forward (the classifier) is not implemented; use extract_features")
