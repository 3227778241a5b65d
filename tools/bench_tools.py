"""Timing of the reduced-3dgs tool rows (SURVEY §8(f)) — ours vs the unmodified reference (oracle/_ref/_refC.so) on the same GPU.
One JSON line per row; device time by CUDA events around the public `_C` call (host code included: these entry points loop
over cameras / iterations on the host in both implementations).

    python tools/bench_tools.py [--points 500000] [--cams 8] [--values 9000000]
"""
import argparse
import json
import math
import os
import sys
import time

import torch

import benchkit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from diff_gaussian_rasterization import _C  # noqa: E402
from gs_b200 import synth  # noqa: E402
import build_ref  # noqa: E402
import cases  # noqa: E402


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    best = 1e30
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=500_000)
    ap.add_argument("--cams", type=int, default=8)
    ap.add_argument("--values", type=int, default=9_000_192)
    ap.add_argument("--knn", type=int, default=30)
    a = ap.parse_args()
    benchkit.banner()
    refC = build_ref.load()
    dev = "cuda"
    W, H = 1920, 1080
    scene = synth.config_scene("C2", a.points).to(dev)
    cams = [c.to(dev) for c in synth.orbit_cameras(a.cams, W, H)] if False else []
    for i in range(a.cams):
        th = math.radians((i - a.cams / 2) * 2.0)
        import numpy as np
        Rc2w = np.array([[math.cos(th), 0, math.sin(th)], [0, 1, 0], [-math.sin(th), 0, math.cos(th)]])
        C = Rc2w @ np.array([0.0, 0.0, -4.0])
        cams.append(synth.make_camera(W, H, Rc2w, -Rc2w.T @ C))
    ct = {k: v.to(dev) for k, v in cases.tools_camera_tensors(cams).items()}
    P = scene.P
    rows = []

    def row(name, ours_fn, ref_fn, unit_count, unit, check):
        t_o, o = timed(ours_fn)
        line = {"row": name, "ours_ms": round(t_o, 3), "unit": unit, "ours_rate": round(unit_count / t_o * 1e3 / 1e6, 2)}
        if refC is not None:
            t_r, r = timed(ref_fn)
            line.update(reference_ms=round(t_r, 3), speedup=round(t_r / t_o, 2), parity=check(o, r))
        rows.append(line)
        print(json.dumps(line), flush=True)

    cv = lambda m: m.calculate_colours_variance(ct["positions"], scene.means3D, scene.opacity, scene.scales, scene.rotations, ct["views"],
                                                ct["projs"], ct["tanx"], ct["tany"], ct["H"], ct["W"], scene.sh, scene.degrees, 3)
    rel = lambda x, y: float((torch.nan_to_num(x - y).abs().max() / (torch.nan_to_num(y).abs().max() + 1e-30)).item())
    row(f"calculate_colours_variance ({P} Gaussians, {a.cams} cameras 1080p)", lambda: cv(_C), lambda: cv(refC), a.cams * W * H,
        "Mpix/s (camera pixels)", lambda o, r: {"max_rel_err": max(rel(x, y) for x, y in zip(o, r))})
    px = lambda m: m.find_minimum_projected_pixel_size(ct["projs"], ct["inv_projs"], scene.means3D, ct["H"], ct["W"])
    row(f"find_minimum_projected_pixel_size ({P} x {a.cams} cameras)", lambda: px(_C), lambda: px(refC), P * a.cams, "M point-cameras/s",
        lambda o, r: {"bit_identical": bool(torch.equal(o, r))})
    nb = torch.randint(P, (P, a.knn), device=dev, dtype=torch.int32)
    rad = px(_C) * 4.0
    se = lambda m: m.sphere_ellipsoid_intersection(scene.means3D, scene.scales, scene.rotations, nb, rad, a.knn)
    row(f"sphere_ellipsoid_intersection ({P} x {a.knn} neighbours)", lambda: se(_C), lambda: se(refC), P * a.knn, "M pairs/s",
        lambda o, r: {"identical": bool(torch.equal(o[0], r[0]) and torch.equal(o[1], r[1]))})
    red, mask = se(_C)
    mr = lambda m: m.allocate_minimum_redundancy_value(red, nb, mask, a.knn)
    row(f"allocate_minimum_redundancy_value ({P} x {a.knn})", lambda: mr(_C), lambda: mr(refC), P * a.knn, "M pairs/s",
        lambda o, r: {"identical": bool(torch.equal(o[0], r[0]))})
    c, v, centers = cases.build_kmeans_inputs("k1", n=a.values)
    v, centers = v.to(dev), centers.to(dev)
    km = lambda m: m.kmeans_cuda(v, centers, 1e-4, 500)
    cost = lambda o: float((v.view(-1) - o[1][o[0].view(-1).long()]).abs().double().mean())
    row(f"kmeans_cuda ({a.values} values, 256 centres, tol 1e-4, <= 500 iterations)", lambda: km(_C), lambda: km(refC), a.values, "M values/s",
        lambda o, r: {"cost_ours": cost(o), "cost_reference": cost(r)})


if __name__ == "__main__":
    main()
