"""Cost of the deterministic backward (`deterministic=True`, DESIGN.md §5i) against the default atomic one.

    python tools/bench_deterministic.py [--steps 20] [--warmup 5]

Workloads: bench.py's C3 (3 M codebook-quantised Gaussians, 1920x1080) and a dense 3 M scene rendered from its raw parameters
(`raw=`, SH degree 3).  Per workload the arms `default` and `deterministic` run forward + backward of the same view, alternating step
by step; each step is timed with a CUDA event pair, L2 is flushed (256 MB write) between steps outside the pair, and the median of
the steps is reported.  A separate profiled pass per arm gives per-kernel times (render_backward, det_scan, det_gather, det_clear =
the memset of the slots).  Prints the card's name and power limit, then one JSON line per (workload, arm) with R and the
deterministic workspace size.
"""
import argparse
import json
import statistics

import benchkit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    dev = benchkit.device("bench_deterministic")
    benchkit.banner()
    flush = benchkit.l2_flush(dev)
    from gs_b200 import lib as gsl
    L = gsl.lib()
    c3 = benchkit.bench_workload("C3", dev)
    cam = c3.cams[0]
    dense = benchkit.dense_raw_workload(c3.W, c3.H, dev)

    for name, wl in (("C3", c3), ("dense3M_raw", dense)):
        arms = {"default": lambda i: benchkit.forward_backward(wl, cam),
                "deterministic": lambda i: benchkit.forward_backward(wl, cam, bwd={"deterministic": True})}
        times = benchkit.time_arms(arms, args.steps, args.warmup, flush)
        kernels = benchkit.kernel_ms(arms, 5, flush, warm=0)
        P, R = int(wl.scene.P), int(benchkit.forward_backward(wl, cam, backward=False)[0][0])
        base = statistics.median(times["default"])
        for k in arms:
            med = statistics.median(times[k])
            print(json.dumps({"workload": name, "arm": k, "P": P, "R": R,
                              "det_workspace_bytes": int(L.gsb_deterministic_workspace_bytes(P, R, 0)) if k == "deterministic" else 0,
                              "fwd_bwd_ms_median": round(med, 4), "ratio_to_default": round(med / base, 4),
                              "kernels_ms": kernels[k]}), flush=True)


if __name__ == "__main__":
    main()
