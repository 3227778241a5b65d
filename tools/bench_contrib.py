"""Cost of the contribution statistics (`_C.contributions`, gsb_contributions, DESIGN.md §5p) next to the forward they read.

    python tools/bench_contrib.py [--steps 20] [--warmup 3]

Two workloads at 1920x1080: bench.py's C3 (3 M quantised Gaussians, mixed SH degrees) and a dense 3 M degree-3 scene rendered from
its raw parameters; one view per step over four cameras, each step timed with a CUDA event pair, L2 flushed (256 MB write) in front
of it.  Arms, alternated step by step so that drift of the shared machine hits all of them alike:
  fwd          the colour forward
  fwd_contrib  the forward, then the contribution pass on its blobs (unweighted)
  fwd_map      the same with a pixel-weight map
  feat_bwd     the route to weight_sum without this pass: the forward with features = ones [P, 1], then the backward with
               dL_dfeatures_out = the map (its dL_dfeatures is the map-weighted sum, summed with float atomics)
A profiled pass gives the per-kernel device times (`contributions`, `render_forward`, `features_backward`, ...).  Prints the
card's name and power limit, then one JSON line per arm.
"""
import argparse
import json

import torch

import benchkit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    dev = benchkit.device("bench_contrib")
    benchkit.banner()
    flush = benchkit.l2_flush(dev)
    from diff_gaussian_rasterization import _C
    c3 = benchkit.bench_workload("C3", dev)
    dense = benchkit.dense_raw_workload(1920, 1080, dev)
    dense.cams = c3.cams
    for label, wl in (("C3", c3), ("dense3M_raw", dense)):
        P, W, H = wl.scene.P, wl.W, wl.H
        wmap = torch.rand(H, W, generator=torch.Generator().manual_seed(7)).to(dev)
        ones = torch.ones(P, 1, device=dev)
        zero = torch.zeros(3, H, W, device=dev)

        def contrib(weights):
            def fn(i):
                out, _ = benchkit.forward_backward(wl, wl.cams[i % 4], backward=False)
                _C.contributions(out[3], out[4], out[5], out[0], W, H, P, pixel_weights=weights)
            return fn

        arms = {
            "fwd": lambda i: benchkit.forward_backward(wl, wl.cams[i % 4], backward=False),
            "fwd_contrib": contrib(None),
            "fwd_map": contrib(wmap),
            "feat_bwd": lambda i: benchkit.forward_backward(wl, wl.cams[i % 4], dict(features=ones),
                                                            dict(features=ones, dL_dfeatures_out=wmap.view(1, H, W)), dL=zero),
        }
        times = benchkit.time_arms(arms, args.steps, args.warmup, flush)
        kernels = benchkit.kernel_ms(arms, 4, flush, warm=1)
        base = sorted(times["fwd"])[len(times["fwd"]) // 2]
        for k, v in times.items():
            ms = sorted(v)
            med = ms[len(ms) // 2]
            print(json.dumps({"workload": label, "arm": k, "W": W, "H": H, "P": P, "steps": len(ms), "median_ms": round(med, 3),
                              "min_ms": round(ms[0], 3), "max_ms": round(ms[-1], 3), "over_fwd_ms": round(med - base, 3),
                              "kernels_ms": kernels[k]}), flush=True)


if __name__ == "__main__":
    main()
