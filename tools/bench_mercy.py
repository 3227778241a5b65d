"""Cost of resolution-aware redundancy pruning (gs_b200.densify.calculate_redundancy_metric + mercy_points; DESIGN.md §5k)
against the reference's glue over this library's `_C` / `simple_knn._C` (tests/mercy_restatement.py), which is what a user of
the drop-ins runs today.

    python tools/bench_mercy.py [--points 1000000 3000000] [--cameras 100] [--repeats 5]

C3 positions (synth.config_scene("C3")'s first draws), log-normal scales around 4 mm, 100 orbit cameras at 1080p, K = 30,
mercy_type 'redundancy_opacity_opacity' on a GaussianAdam model with the reference's six params.  The arms alternate repeat by
repeat; each call ends in a host synchronisation and is timed by a host clock (median of --repeats).  max_memory_allocated
above the model is reported for the whole call (set by the prune's new model) and for calculate_redundancy_metric alone.
Prints the card's name and power limit and one JSON line per measurement.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

import benchkit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("reduced-3dgs_b200", "tests", os.path.join("tests", "golden")):
    sys.path.insert(0, os.path.join(ROOT, p))
import knn_cases as KC  # noqa: E402
import mercy_restatement as mr  # noqa: E402
from gs_b200 import densify, synth  # noqa: E402
from gs_b200.optim import GaussianAdam  # noqa: E402

GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
          "rotation": "_rotation"}


class Model:
    _codebook_dict = None


def build(xyz, seed):
    P = xyz.shape[0]
    g = torch.Generator(device="cuda").manual_seed(seed)
    m = Model()
    m._xyz = torch.nn.Parameter(xyz.clone())
    m._features_dc = torch.nn.Parameter(torch.randn(P, 1, 3, device="cuda", generator=g))
    m._features_rest = torch.nn.Parameter(torch.randn(P, 15, 3, device="cuda", generator=g) * 0.1)
    m._opacity = torch.nn.Parameter(torch.randn(P, 1, device="cuda", generator=g) * 2)
    m._scaling = torch.nn.Parameter(np.log(0.004) + 0.6 * torch.randn(P, 3, device="cuda", generator=g))
    m._rotation = torch.nn.Parameter(torch.randn(P, 4, device="cuda", generator=g))
    m._degrees = torch.randint(0, 4, (P, 1), device="cuda", generator=g, dtype=torch.int32)
    m.xyz_gradient_accum = torch.zeros((P, 1), device="cuda")
    m.denom = torch.zeros((P, 1), device="cuda")
    m.max_radii2D = torch.zeros((P,), device="cuda")
    m.optimizer = GaussianAdam([{"params": [getattr(m, a)], "lr": 1e-3, "name": n} for n, a in GROUPS.items()], lr=0.0, eps=1e-15)
    for a in GROUPS.values():
        getattr(m, a).grad = torch.randn(getattr(m, a).shape, device="cuda", generator=g) * 1e-3
    m.optimizer.step()
    for a in GROUPS.values():
        getattr(m, a).grad = None
    return m


def scene_of(m, cams):
    s = mr.RedScene(m._xyz, torch.exp(m._scaling), torch.nn.functional.normalize(m._rotation), [])
    s.cams = cams
    return s


def ref_arm(m, cams):
    red, _ = mr.calculate_redundancy_metric(scene_of(m, cams))
    m._splatted_num_accum = red.unsqueeze(1)
    mr.mercy_points(m, {}, 1.0, 3, "redundancy_opacity_opacity", prune_points=lambda mask: densify.prune_points(m, mask))


def native_arm(m, cams):
    red, _ = densify.calculate_redundancy_metric(scene_of(m, cams))
    m._splatted_num_accum = red.unsqueeze(1)
    densify.mercy_points(m, {}, 1.0, 3, "redundancy_opacity_opacity")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--cameras", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mercy needs a GPU"
    benchkit.banner()
    cams = [mr.Cam(c, torch.device("cuda")) for c in synth.orbit_cameras(a.cameras, 1920, 1080)]
    for P in a.points:
        xyz = KC.c3_positions(P).cuda()
        times = {"ref": [], "native": []}
        peaks = {}
        for r in range(a.repeats + 1):
            for name, fn in (("ref", ref_arm), ("native", native_arm)) if r % 2 == 0 else (("native", native_arm), ("ref", ref_arm)):
                m = build(xyz, r)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                fn(m, cams)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                peaks[name] = torch.cuda.max_memory_allocated() - base
                if r > 0:                                  # the first round warms up both arms
                    times[name].append(dt * 1e3)
                del m
        red_peak = {}
        m = build(xyz, 0)
        for name, fn in (("ref", mr.calculate_redundancy_metric), ("native", densify.calculate_redundancy_metric)):
            fn(scene_of(m, cams))
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            out = fn(scene_of(m, cams))
            torch.cuda.synchronize()
            red_peak[name] = torch.cuda.max_memory_allocated() - base
            del out
        del m
        res = {k: statistics.median(v) for k, v in times.items()}
        print(json.dumps({"P": P, "cameras": a.cameras, "K": 30, "ref_ms": round(res["ref"], 2), "native_ms": round(res["native"], 2),
                          "speedup": round(res["ref"] / res["native"], 3), "ref_peak_MB": round(peaks["ref"] / 2**20, 1),
                          "native_peak_MB": round(peaks["native"] / 2**20, 1),
                          "ref_redundancy_peak_MB": round(red_peak["ref"] / 2**20, 1),
                          "native_redundancy_peak_MB": round(red_peak["native"] / 2**20, 1),
                          "ref_spread_ms": [round(min(times["ref"]), 2), round(max(times["ref"]), 2)],
                          "native_spread_ms": [round(min(times["native"]), 2), round(max(times["native"]), 2)]}), flush=True)


if __name__ == "__main__":
    main()
