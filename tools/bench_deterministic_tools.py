"""Cost of the deterministic SH-culling statistics and k-means (DESIGN.md §5j) against the default atomic paths.

    python tools/bench_deterministic_tools.py [--reps 10] [--warmup 2]

Workloads: `calculate_colours_variance` over 32 cameras at 1920x1080 on a dense 3 M Gaussian scene of SH degree 3 (one call = 32
statistics forwards + 32 statistics updates), and `kmeans_cuda` with 256 centres drawn from 9 M values (tol 1e-4, at most 500
iterations: the codebook call of gaussian_model.py) for uniform, normal and 70 % exact-zero values.  Per workload the arms
`default` and `deterministic` alternate call by call; each call is timed with a CUDA event pair and the median over the calls is
reported.  Prints the card's name and power limit, then one JSON line per (workload, arm) and the ratio deterministic / default.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
from diff_gaussian_rasterization import _C  # noqa: E402
from gs_b200 import synth  # noqa: E402


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


def _time(fn, arms, reps, warmup):
    """{arm: [ms per call]}, the arms interleaved call by call."""
    for _ in range(warmup):
        for a in arms:
            fn(a)
    torch.cuda.synchronize()
    out = {a: [] for a in arms}
    for _ in range(reps):
        for a in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(a)
            e1.record()
            e1.synchronize()
            out[a].append(e0.elapsed_time(e1))
    return out


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
    assert torch.cuda.is_available(), "bench_deterministic_tools needs a GPU"
    assert args.reps >= 10, "the medians are taken over at least 10 calls per arm"
    dev = torch.device("cuda", 0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "n/a"}), flush=True)
    arms = ("default", "deterministic")

    # ---- SH-culling statistics: 32 cameras at 1080p, dense 3 M degree-3 scene
    W, H = 1920, 1080
    sc = synth.make_scene(3_000_000, 3, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.006)).to(dev)
    ct = _cameras(32, W, H, dev)

    def colours(arm):
        return _C.calculate_colours_variance(ct["positions"], sc.means3D, sc.opacity, sc.scales, sc.rotations, ct["views"], ct["projs"],
                                             ct["tanx"], ct["tany"], ct["H"], ct["W"], sc.sh, sc.degrees, 3,
                                             deterministic=arm == "deterministic")
    _report("colours_variance_3M_32x1080p", _time(colours, arms, args.reps, args.warmup))
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
        t = _time(kmeans, arms, args.reps, args.warmup)
        gap = float((iters["deterministic"] - iters["default"]).abs().max())
        _report(f"kmeans_9M_256_{name}", t, {"max_centre_gap_vs_default": gap})


if __name__ == "__main__":
    main()
