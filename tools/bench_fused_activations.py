"""Cost of the activation glue between the model's parameters and the rasterizer (DESIGN.md §5h).

    python tools/bench_fused_activations.py [--points 3000000] [--repeats 20]

Setup: P fp32 Gaussians with the reference's leaf parameters (_features_rest [P,15,3]), SH degrees 0/1/2/3 for 50/20/15/15 %,
one 1920x1080 view.  Arms, interleaved repeat by repeat, each timed by CUDA events (median of --repeats):
  activated  render() + backward() through get_features / get_scaling / get_rotation (torch.cat, exp, F.normalize and their backwards)
  fused      the same with pipe.fused_activations (the kernels read the parameters and write their gradients)
and both again followed by one GaussianAdam step, to show the share of a training iteration.  Also prints the per-kernel device
time of one iteration of each arm (torch.profiler), the peak memory over forward + backward, the card's name and power limit.
"""
import argparse
import json
import math
import os
import statistics
import sys
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

import benchkit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
from gaussian_renderer import render  # noqa: E402
from gs_b200 import synth  # noqa: E402
from gs_b200.optim import GaussianAdam  # noqa: E402

NAMES = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")


class Model:
    def __init__(self, scene, dev):
        self._xyz = scene.means3D.to(dev).requires_grad_()
        self._features_dc = scene.sh[:, :1].to(dev).contiguous().requires_grad_()
        self._features_rest = scene.sh[:, 1:].to(dev).contiguous().requires_grad_()
        self._opacity = scene.opacity.to(dev).requires_grad_()
        self._scaling = torch.log(scene.scales).to(dev).requires_grad_()
        self._rotation = scene.rotations.to(dev).requires_grad_()
        self._degrees = scene.degrees.to(dev)
        self.scaling_activation, self.rotation_activation = torch.exp, F.normalize
        self.active_sh_degree = self.max_sh_degree = 3

    get_xyz = property(lambda s: s._xyz)
    get_scaling = property(lambda s: s.scaling_activation(s._scaling))
    get_rotation = property(lambda s: s.rotation_activation(s._rotation))
    get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), dim=1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=3_000_000)
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda")
    name, pl = torch.cuda.get_device_name(), benchkit.banner().get("power_limit", "unknown")
    W, H = 1920, 1080
    scene = synth.make_scene(args.points, 3, sh_degree=3, mixed_degrees=True)
    m = Model(scene, dev)
    cam = synth.make_camera(W, H).to(dev)
    bg = torch.zeros(3, device=dev)
    w = synth.grad_image(W, H, 1).to(dev)
    opt = GaussianAdam([{"params": [getattr(m, n)], "lr": 1e-12} for n in NAMES], lr=0.0, eps=1e-15)
    pipes = {f: SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False, fused_activations=f) for f in (False, True)}

    def step(fused, adam):
        for n in NAMES:
            getattr(m, n).grad = None
        pkg = render(cam, m, pipes[fused], bg)
        (pkg["render"] * w).sum().backward()
        if adam:
            opt.step()

    arms = [("activated", False, False), ("fused", True, False), ("activated+adam", False, True), ("fused+adam", True, True)]
    for _, f, a in arms:                                      # warm-up (allocator, first-launch attributes, Adam state)
        for _ in range(3):
            step(f, a)
    torch.cuda.synchronize()
    times = {k: [] for k, _, _ in arms}
    for _ in range(args.repeats):
        for k, f, a in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(f, a)
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1))
    med = {k: statistics.median(v) for k, v in times.items()}
    peaks = {}
    for k, f, _ in arms[:2]:
        for n in NAMES:
            getattr(m, n).grad = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        step(f, False)
        torch.cuda.synchronize()
        peaks[k] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    kernels = {}
    for k, f, _ in arms[:2]:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            step(f, False)
            torch.cuda.synchronize()
        rows = sorted(((e.key, e.device_time_total / 1000.0, e.count) for e in prof.key_averages() if e.device_time_total > 0),
                      key=lambda r: -r[1])
        kernels[k] = rows
    for k in ("activated", "fused"):
        print(f"\n{k}: per-kernel device time of one render + backward (ms, launches)")
        for key, ms, cnt in kernels[k][:16]:
            print(f"  {ms:8.3f}  {cnt:3d}  {key[:110]}")
    print()
    for k, v in med.items():
        print(f"{k:16s} median {v:8.3f} ms  (min {min(times[k]):.3f}, max {max(times[k]):.3f})")
    print(f"saving: {med['activated'] - med['fused']:.3f} ms per render + backward, "
          f"{med['activated+adam'] - med['fused+adam']:.3f} ms per iteration with the Adam step "
          f"({100 * (med['activated+adam'] - med['fused+adam']) / med['activated+adam']:.1f} % of it)")
    print(f"peak memory over forward + backward: activated {peaks['activated']:.0f} MiB, fused {peaks['fused']:.0f} MiB")
    print(json.dumps(dict(device=name, power_limit=pl, points=args.points, image=[W, H], median_ms=med, peak_mib=peaks)))


if __name__ == "__main__":
    main()
