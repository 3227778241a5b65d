"""Cost of the absolute screen-space gradient (`absgrad_out`, DESIGN.md §5m) against the same backward without it.

    python tools/bench_absgrad.py [--steps 20] [--warmup 5]

Workloads: bench.py's C3 (3 M codebook-quantised Gaussians, 1920x1080) and a dense 3 M scene of SH degree 3 rendered from its raw
parameters.  Per workload the arms `plain` and `absgrad` run forward + backward of the same view on the default (atomic) path,
alternating step by step; each step is timed with a CUDA event pair, L2 is flushed (256 MB write) between steps outside the pair, and
the median of the steps is reported.  A separate profiled pass per arm gives per-kernel times (render_backward, absgrad_finish).
Prints the card's name and power limit, then one JSON line per (workload, arm).
"""
import argparse
import json
import statistics

import torch

import benchkit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    dev = benchkit.device("bench_absgrad")
    benchkit.banner()
    flush = benchkit.l2_flush(dev)
    c3 = benchkit.bench_workload("C3", dev)
    cam = c3.cams[0]
    dense = benchkit.dense_raw_workload(c3.W, c3.H, dev)

    for name, wl in (("C3", c3), ("dense3M_deg3_raw", dense)):
        absgrad = torch.empty(wl.scene.P, 3, device=dev)
        arms = {"plain": lambda i: benchkit.forward_backward(wl, cam),
                "absgrad": lambda i: benchkit.forward_backward(wl, cam, bwd={"absgrad_out": absgrad})}
        times = benchkit.time_arms(arms, args.steps, args.warmup, flush)
        kernels = benchkit.kernel_ms(arms, 10, flush, warm=0)
        R = benchkit.forward_backward(wl, cam, backward=False)[0][0]
        base = statistics.median(times["plain"])
        for k in arms:
            med = statistics.median(times[k])
            rb = kernels[k].get("render_backward", 0.0)
            print(json.dumps({"workload": name, "arm": k, "P": int(wl.scene.P), "R": int(R),
                              "fwd_bwd_ms_median": round(med, 4), "ratio_to_plain": round(med / base, 4),
                              "render_backward_ms": rb,
                              "render_backward_ratio": round(rb / kernels["plain"].get("render_backward", rb or 1.0), 4),
                              "kernels_ms": kernels[k]}), flush=True)


if __name__ == "__main__":
    main()
