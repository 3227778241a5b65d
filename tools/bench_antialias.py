"""Cost of anti-aliased rendering (antialiasing=True, gsb_forward_antialiased / gsb_backward_antialiased) against the colour step.

    python tools/bench_antialias.py [--config C3] [--steps 20] [--warmup 5]

bench.py's workload (C3: 3 M quantised Gaussians, 1920x1080, device-resident), one view per step over its cameras; each step
is timed with a CUDA event pair, and L2 is flushed (256 MB write) between steps outside the pair.  Arms:
  a          colour forward + backward (gsb_forward / gsb_backward, what bench.py times)
  b          the same with anti-aliasing
  c          b plus the inverse-depth and alpha maps and the gradients w.r.t. viewmatrix, projmatrix and campos
The arms alternate step by step so that drift of the shared machine hits all alike.  A separate profiled pass per arm gives
per-kernel times (gsb_profile_*).  Prints the card's name and power limit, then one JSON line per arm and a summary line.
"""
import argparse
import json
import math
import os
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

EMPTY = torch.Tensor([])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=["C1", "C2", "C3"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_antialias needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "n/a"}), flush=True)

    name, W, H, scene, quant, prune = bench.build_workload(SimpleNamespace(config=args.config, points=0), dev, 0, 1)
    cams = [c.to(dev) for c in bench.bench_cameras(W, H, 4)]
    sd = scene.to(dev)
    qd = None if quant is None else quant.to(dev)
    prune_d = None if prune is None else prune.to(dev)
    bg0 = torch.zeros(3, device=dev)
    G = synth.grad_image(W, H, 1000).to(dev)
    Gm = synth.grad_image(W, H, 1001)[:2].to(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

    def fwd_args(c):
        tx, ty = math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5)
        if qd is not None:
            return (bg0, sd.means3D, EMPTY, EMPTY, EMPTY, EMPTY, 1.0, EMPTY, c.world_view_transform, c.full_proj_transform, tx, ty, H, W,
                    EMPTY, sd.degrees, c.camera_center, False, False)
        return (bg0, sd.means3D, EMPTY, sd.opacity, sd.scales, sd.rotations, 1.0, EMPTY, c.world_view_transform, c.full_proj_transform,
                tx, ty, H, W, sd.sh, sd.degrees, c.camera_center, False, False)

    def fb(c, aa, extras):
        a = fwd_args(c)
        out = _C.rasterize_gaussians(*a, prune_mask=prune_d, quant=qd, antialiasing=aa, return_maps=extras)
        R, color, radii, gb, bb, ib = out[:6]
        kw = dict(dL_dinvdepth=Gm[0:1], dL_dalpha=Gm[1:2], camera_grads=True) if extras else {}
        return _C.rasterize_gaussians_backward(a[0], a[1], radii, a[2], a[4], a[5], 1.0, EMPTY, a[8], a[9], a[10], a[11], G, a[14], a[15],
                                               a[16], gb, R, bb, ib, 0.0, False, prune_mask=prune_d, quant=qd, antialiasing=aa, **kw)

    arms = {"a": lambda c: fb(c, False, False), "b": lambda c: fb(c, True, False), "c": lambda c: fb(c, True, True)}
    for i in range(max(args.warmup, 2)):
        for fn in arms.values():
            flush.zero_()
            fn(cams[i % len(cams)])
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for i in range(args.steps):
        for k, fn in arms.items():
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(cams[i % len(cams)])
            e1.record()
            times[k].append((e0, e1))
    torch.cuda.synchronize()
    ms = {k: sorted(a.elapsed_time(b) for a, b in v) for k, v in times.items()}
    kernels = {}
    gsl.profile_enable(True)
    for k, fn in arms.items():
        for i in range(2):
            flush.zero_()
            fn(cams[i % len(cams)])
        torch.cuda.synchronize()
        gsl.profile_read()
        n = min(args.steps, 8)
        for i in range(n):
            flush.zero_()
            fn(cams[i % len(cams)])
        torch.cuda.synchronize()
        kernels[k] = {kn: round(t / n, 4) for kn, (t, _) in gsl.profile_read().items()}
    gsl.profile_enable(False)
    med = {k: v[len(v) // 2] for k, v in ms.items()}
    for k in arms:
        v = ms[k]
        print(json.dumps({"arm": k, "config": name, "W": W, "H": H, "P": sd.P, "steps": len(v), "median_ms": round(med[k], 4),
                          "mean_ms": round(sum(v) / len(v), 4), "min_ms": round(v[0], 4), "max_ms": round(v[-1], 4),
                          "kernels_ms_per_step": kernels[k]}), flush=True)
    print(json.dumps({"b_over_a": round(med["b"] / med["a"], 4), "c_over_a": round(med["c"] / med["a"], 4)}), flush=True)


if __name__ == "__main__":
    main()
