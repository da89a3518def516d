"""Micro-benchmark of the implicit-GEMM conv kernel on every distinct conv shape of the path at B=8 clips
(T=8 -> 64 frames, 112 SPyNet pairs).  Prints us/launch and algorithmic TFLOP/s (2*MACs, fp32-equivalent)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from e2fgvi_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
# name, N, [cin...], H, W, cout, groups, ks, stride, out
SHAPES = [
    ("spynet L5 8->32 k7", 112, [8], 64, 128, 32, 1, 7, 1, "split"),
    ("spynet L5 32->64 k7", 112, [32], 64, 128, 64, 1, 7, 1, "split"),
    ("spynet L5 64->32 k7", 112, [64], 64, 128, 32, 1, 7, 1, "split"),
    ("spynet L5 32->16 k7", 112, [32], 64, 128, 16, 1, 7, 1, "split"),
    ("spynet L5 16->2 k7", 112, [16], 64, 128, 2, 1, 7, 1, "f32"),
    ("enc0 3->64 s2", 64, [3], 240, 432, 64, 1, 3, 2, "split"),
    ("enc1 64->64", 64, [64], 120, 216, 64, 1, 3, 1, "split"),
    ("enc2 64->128 s2", 64, [64], 120, 216, 128, 1, 3, 2, "split"),
    ("enc3 128->256", 64, [128], 60, 108, 256, 1, 3, 1, "split"),
    ("enc4 256->384", 64, [256], 60, 108, 384, 1, 3, 1, "split"),
    ("enc5 640->512 g2", 64, [256, 384], 60, 108, 512, 2, 3, 1, "split"),
    ("enc6 768->384 g4", 64, [256, 512], 60, 108, 384, 4, 3, 1, "split"),
    ("enc7 640->256 g8", 64, [256, 384], 60, 108, 256, 8, 3, 1, "split"),
    ("enc8 512->128", 64, [256, 256], 60, 108, 128, 1, 3, 1, "f32"),
    ("offset0 388->128", 8, [128, 128, 128, 4], 60, 108, 128, 1, 3, 1, "split"),
    ("offset1 128->128", 8, [128], 60, 108, 128, 1, 3, 1, "split"),
    ("offset3 128->432", 8, [128], 60, 108, 432, 1, 3, 1, "f32"),
    ("backbone 384->128", 8, [128, 128, 128], 60, 108, 128, 1, 3, 1, "split"),
    ("dec0 128->128 @120", 64, [128], 120, 216, 128, 1, 3, 1, "split"),
    ("dec1 128->64 @120", 64, [128], 120, 216, 64, 1, 3, 1, "f32"),
    ("dec2 64->64 @240", 64, [64], 240, 432, 64, 1, 3, 1, "split"),
    ("dec3 64->3 @240", 64, [64], 240, 432, 3, 1, 3, 1, "f32"),
    # experiments (not layers of the path): epilogue / weight-tile effects
    ("x dec3 64->32 f32", 64, [64], 240, 432, 32, 1, 3, 1, "f32"),
    ("x dec3 64->8 f32", 64, [64], 240, 432, 8, 1, 3, 1, "f32"),
    ("x dec2 64->64 f32", 64, [64], 240, 432, 64, 1, 3, 1, "f32"),
    # per-tile fixed cost: same output (64 images at 60 x 108 = 54 tiles of 12 x 10 each), K = 9 cin / 64 blocks per
    # tile; the intercept of time against K is what a tile costs besides its MMAs (epilogue, pipeline refill).  Not in
    # the total; the fit uses K <= 72 (at cin 1024 the time leaves the straight line)
] + [(f"x ksweep {c}->{co}", 64, [c], 60, 108, co, 1, 3, 1, "split") for co in (128, 64) for c in (64, 128, 256, 512, 1024)]
SWEEP_TILES, SWEEP_MAX_KB = 64 * 54, 72
only = sys.argv[1] if len(sys.argv) > 1 else ""
g = torch.Generator(device="cpu").manual_seed(0)
total = 0.0
sweep = {}
for name, n, cins, h, w, cout, groups, ks, stride, out in SHAPES:
    if only and only not in name:
        continue
    srcs = [ops.split_nhwc(torch.randn(n, c, h, w, device=dev)) for c in cins]
    variants = [("", srcs)]
    if len(cins) == 1 and cins[0] <= 32 and groups == 1:
        variants.append((" [rows]", ops.pack_rows(torch.randn(n, cins[0], h, w, device=dev), lead=ks // 2)))
    wt = torch.randn(cout, sum(cins) // groups, ks, ks, device=dev) * 0.05
    bias = torch.randn(cout, device=dev)
    for tag, src in variants:
        run = lambda: ops.conv3x3(src, wt, bias, groups=groups, negative_slope=0.2, out=out, stride=stride)  # noqa: E731
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 10
        e0.record()
        for _ in range(reps):
            run()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / reps * 1e3
        ho, wo = (h + 2 * (ks // 2) - ks) // stride + 1, (w + 2 * (ks // 2) - ks) // stride + 1
        flops = 2.0 * n * ho * wo * cout * (sum(cins) // groups) * ks * ks
        print(f"CONV {name + tag:30s} {us:9.1f} us  {flops / us / 1e6:8.1f} TFLOP/s")
        if name.startswith("x ksweep"):
            if 9 * cins[0] // 64 <= SWEEP_MAX_KB:
                sweep.setdefault(cout, []).append((9 * cins[0] // 64, us))
        else:
            total += us if tag or len(variants) == 1 else 0.0
    del srcs, variants
print(f"CONV total {total / 1e3:.2f} ms")
sms = torch.cuda.get_device_properties(dev).multi_processor_count
for cout, pts in sweep.items():
    if len(pts) < 2:
        continue
    kb = torch.tensor([p[0] for p in pts], dtype=torch.float64)
    us = torch.tensor([p[1] for p in pts], dtype=torch.float64)
    slope = float(((kb - kb.mean()) * (us - us.mean())).sum() / ((kb - kb.mean()) ** 2).sum())
    icpt = float(us.mean() - slope * kb.mean())
    per_cta = SWEEP_TILES / sms                        # tiles per persistent CTA
    print(f"CONV ksweep Cout {cout}: {icpt:.1f} us + {slope:.2f} us per K block of every tile; per tile "
          f"{icpt / per_cta:.2f} us fixed + {slope / per_cta:.3f} us per K block ({per_cta:.1f} tiles per CTA)")
