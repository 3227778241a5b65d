"""Cost of the deterministic SH-culling statistics and k-means (DESIGN.md §5j) against the default atomic paths.

    python tools/bench_deterministic_tools.py [--reps 10] [--warmup 2]

Workloads: `calculate_colours_variance` over 32 cameras at 1920x1080 on a dense 3 M Gaussian scene of SH degree 3 (one call = 32
statistics forwards + 32 statistics updates), and `kmeans_cuda` with 256 centres drawn from 9 M values (tol 1e-4, at most 500
iterations: the codebook call of gaussian_model.py) for uniform, normal and 70 % exact-zero values.  Per workload the arms
`default` and `deterministic` alternate call by call; each call is timed with a CUDA event pair, L2 is flushed (256 MB write)
between calls outside the pair, and the median over the calls is reported.  Prints the card's name and power limit, then one
JSON line per (workload, arm) and the ratio deterministic / default.
"""
import argparse
import json
import math
import statistics

import numpy as np
import torch

import benchkit
from diff_gaussian_rasterization import _C  # on sys.path through benchkit
from gs_b200 import synth


def _cameras(n, W, H, dev):
    cams = []
    for yaw in np.linspace(-30.0, 30.0, n):
        th = math.radians(yaw)
        R = np.array([[math.cos(th), 0, math.sin(th)], [0, 1, 0], [-math.sin(th), 0, math.cos(th)]])
        C = R @ np.array([0.0, 0.0, -4.0])
        cams.append(synth.make_camera(W, H, R, -R.T @ C).to(dev))
    return dict(positions=torch.stack([c.camera_center for c in cams]), views=torch.stack([c.world_view_transform for c in cams]),
                projs=torch.stack([c.full_proj_transform for c in cams]),
                tanx=torch.tensor([math.tan(c.FoVx * 0.5) for c in cams], device=dev),
                tany=torch.tensor([math.tan(c.FoVy * 0.5) for c in cams], device=dev),
                H=torch.full((n,), H, dtype=torch.int32, device=dev), W=torch.full((n,), W, dtype=torch.int32, device=dev))


def _report(workload, times, extra=None):
    med = {a: statistics.median(t) for a, t in times.items()}
    for a, t in times.items():
        print(json.dumps({"workload": workload, "arm": a, "median_ms": round(med[a], 3), "min_ms": round(min(t), 3),
                          "max_ms": round(max(t), 3), "calls": len(t), **(extra or {})}), flush=True)
    print(json.dumps({"workload": workload, "deterministic_over_default": round(med["deterministic"] / med["default"], 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = benchkit.device("bench_deterministic_tools")
    assert args.reps >= 10, "the medians are taken over at least 10 calls per arm"
    benchkit.banner()
    flush = benchkit.l2_flush(dev)

    def time_both(fn):
        """{arm: [ms per call]} of fn(arm) for the arms default and deterministic."""
        return benchkit.time_arms({a: (lambda i, a=a: fn(a)) for a in ("default", "deterministic")}, args.reps, args.warmup, flush)

    # ---- SH-culling statistics: 32 cameras at 1080p, dense 3 M degree-3 scene
    W, H = 1920, 1080
    sc = synth.make_scene(3_000_000, 3, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.006)).to(dev)
    ct = _cameras(32, W, H, dev)

    def colours(arm):
        return _C.calculate_colours_variance(ct["positions"], sc.means3D, sc.opacity, sc.scales, sc.rotations, ct["views"], ct["projs"],
                                             ct["tanx"], ct["tany"], ct["H"], ct["W"], sc.sh, sc.degrees, 3,
                                             deterministic=arm == "deterministic")
    _report("colours_variance_3M_32x1080p", time_both(colours))
    del sc, ct
    torch.cuda.empty_cache()

    # ---- k-means: 256 centres on 9 M values
    n = 9_000_000
    g = torch.Generator(device=dev).manual_seed(0)
    dists = {"uniform": torch.rand(n, 1, device=dev, generator=g) * 2 - 1,
             "normal": torch.randn(n, 1, device=dev, generator=g)}
    z = 0.05 * torch.randn(n, 1, device=dev, generator=g)
    z[torch.rand(n, 1, device=dev, generator=g) < 0.7] = 0.0
    dists["zeros70"] = z
    for name, v in dists.items():
        c = v.view(-1)[torch.randint(n, (256,), device=dev, generator=g)].contiguous()
        iters = {}

        def kmeans(arm):
            ids, cc = _C.kmeans_cuda(v, c, 1e-4, 500, deterministic=arm == "deterministic")
            iters[arm] = cc
        t = time_both(kmeans)
        gap = float((iters["deterministic"] - iters["default"]).abs().max())
        _report(f"kmeans_9M_256_{name}", t, {"max_centre_gap_vs_default": gap})


if __name__ == "__main__":
    main()
