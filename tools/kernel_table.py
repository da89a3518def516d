"""Markdown table of bench.py's per-kernel rooflines (live CUDA-event timing inside the timed region).
    python tools/kernel_table.py <bench JSON line file> [workload]"""
import json
import sys

d = json.load(open(sys.argv[1]))
w = d if len(sys.argv) < 3 else d["workloads"][sys.argv[2]]
steps = w.get("steps", d.get("steps", 1))
print("| kernel (op kind) | launches / step | avg launch | share of step | bound | achieved | of measured peak | DRAM traffic / launch (ncu) |")
print("|---|---|---|---|---|---|---|---|")
for k, v in sorted(w["roofline_kernels"].items(), key=lambda kv: -kv[1]["share_of_step"]):
    tr = v.get("traffic")
    extra = f" ({v['tensor_pipe_frac']:.2f} of the pipe with the 3-term split)" if "tensor_pipe_frac" in v else ""
    print(f"| `{k}` | {v['launches_timed'] / steps:.0f} | {v['avg_launch_ms'] * 1e3:.0f} µs | {100 * v['share_of_step']:.1f} % | {v['bound']} | "
          f"{v['achieved']:.0f} {v['unit']} | {v['frac']:.3f}{extra} | {'-' if tr is None else f'{tr / 1e6:.0f} MB'} |")
