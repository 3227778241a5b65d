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
import math
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
import bench  # noqa: E402  (workload and cameras of the benchmark, unchanged)
from diff_gaussian_rasterization import _C  # noqa: E402
from gs_b200 import lib as gsl  # noqa: E402
from gs_b200 import synth  # noqa: E402

E = torch.Tensor([])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_absgrad needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "n/a"}), flush=True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

    name, W, H, scene, quant, prune = bench.build_workload(SimpleNamespace(config="C3", points=0), dev, 0, 1)
    cam = bench.bench_cameras(W, H, 4)[0].to(dev)
    sd, qd = scene.to(dev), quant.to(dev)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    bg = torch.zeros(3, device=dev)
    G = synth.grad_image(W, H, 1000).to(dev)
    abs_c3 = torch.empty(sd.P, 3, device=dev)

    def c3_step(ab):
        fa = (bg, sd.means3D, E, sd.opacity, E, E, 1.0, E, cam.world_view_transform, cam.full_proj_transform, tx, ty, H, W, E, sd.degrees,
              cam.camera_center, False, False)
        R, color, radii, gb, bb, ib = _C.rasterize_gaussians(*fa, quant=qd)
        _C.rasterize_gaussians_backward(bg, sd.means3D, radii, E, E, E, 1.0, E, cam.world_view_transform, cam.full_proj_transform, tx, ty,
                                        G, E, sd.degrees, cam.camera_center, gb, R, bb, ib, 0.0, False, quant=qd,
                                        **({"absgrad_out": abs_c3} if ab else {}))
        return R

    dsc = synth.make_scene(3_000_000, 7, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.01))
    xyz, op = dsc.means3D.to(dev), dsc.opacity.to(dev)
    raw = (dsc.sh[:, :1].contiguous().to(dev), dsc.sh[:, 1:16].contiguous().to(dev), torch.log(dsc.scales).to(dev),
           dsc.rotations.contiguous().to(dev))
    deg = dsc.degrees.to(dev)
    abs_dense = torch.empty(dsc.P, 3, device=dev)

    def dense_step(ab):
        fa = (bg, xyz, E, op, E, E, 1.0, E, cam.world_view_transform, cam.full_proj_transform, tx, ty, H, W, E, deg, cam.camera_center,
              False, False)
        R, color, radii, gb, bb, ib = _C.rasterize_gaussians(*fa, raw=raw)
        _C.rasterize_gaussians_backward(bg, xyz, radii, E, E, E, 1.0, E, cam.world_view_transform, cam.full_proj_transform, tx, ty, G, E,
                                        deg, cam.camera_center, gb, R, bb, ib, 0.0, False, raw=raw,
                                        **({"absgrad_out": abs_dense} if ab else {}))
        return R

    for wl, step, P in (("C3", c3_step, sd.P), ("dense3M_deg3_raw", dense_step, dsc.P)):
        times = {False: [], True: []}
        R = 0
        for i in range(args.warmup + args.steps):
            for ab in ((False, True) if i % 2 == 0 else (True, False)):
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                R = step(ab)
                b.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[ab].append(a.elapsed_time(b))
        kernels = {}
        for ab in (False, True):
            gsl.profile_enable(True)
            gsl.profile_read()
            n = 10
            for _ in range(n):
                flush.zero_()
                step(ab)
            torch.cuda.synchronize()
            kernels[ab] = {kn: round(t / n, 4) for kn, (t, _) in gsl.profile_read().items()}
            gsl.profile_enable(False)
        base = statistics.median(times[False])
        for ab in (False, True):
            med = statistics.median(times[ab])
            rb = kernels[ab].get("render_backward", 0.0)
            print(json.dumps({"workload": wl, "arm": "absgrad" if ab else "plain", "P": int(P), "R": int(R),
                              "fwd_bwd_ms_median": round(med, 4), "ratio_to_plain": round(med / base, 4),
                              "render_backward_ms": rb,
                              "render_backward_ratio": round(rb / kernels[False].get("render_backward", rb or 1.0), 4),
                              "kernels_ms": kernels[ab]}), flush=True)


if __name__ == "__main__":
    main()
