"""Cost of densification (gs_b200.densify; DESIGN.md §5g) against the reference's torch path (tests/densify_restatement.py).

    python tools/bench_densify.py [--points 3000000] [--repeats 5]

C3 size: 3 M Gaussians with the reference's six params (59 floats per row), both Adam moments and masks that clone about 5 %,
split about 5 % and prune about 3 % (the realised fractions are printed).  Arms, alternated repeat by repeat:
  ref     the reference's densify_and_prune (restated in torch: boolean indexing, repeat, normal, bmm, four concatenations / prunes)
  native  gs_b200.densify.densify_and_prune (plan, one read-back, normal, one emit)
Both end in a host synchronisation, so each call is timed by a host clock around synchronised work (median of --repeats); the
model is rebuilt before each call outside the timed window.  Bytes from shapes: the native path reads every source row once
(params, moments: 3 x 59 floats) and writes every output row once, plus the statistics.  Also the per-iteration statistics
(train.py:134-135 against add_densification_stats(..., radii)), timed by CUDA events over 50 calls each.  Prints the card's
name and power limit, peak memory of each arm, and one JSON line per measurement.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

import benchkit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import densify_restatement as rs  # noqa: E402
from gs_b200 import densify  # noqa: E402
from gs_b200.optim import GaussianAdam  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
          "rotation": "_rotation"}


class Model:
    _codebook_dict = None


def build(P, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    m = Model()
    m._xyz = torch.nn.Parameter(torch.randn(P, 3, device="cuda", generator=g) * 3)
    m._features_dc = torch.nn.Parameter(torch.randn(P, 1, 3, device="cuda", generator=g))
    m._features_rest = torch.nn.Parameter(torch.randn(P, 15, 3, device="cuda", generator=g) * 0.1)
    u = torch.rand(P, device="cuda", generator=g)
    m._opacity = torch.nn.Parameter(torch.where(u < 0.03, -7.0, 1.0 + u).unsqueeze(1))
    sc = torch.rand(P, 3, device="cuda", generator=g) * 2 - 6
    sc[torch.rand(P, device="cuda", generator=g) < 0.5] += 3.5
    m._scaling = torch.nn.Parameter(sc)
    m._rotation = torch.nn.Parameter(torch.randn(P, 4, device="cuda", generator=g))
    m._degrees = torch.randint(0, 4, (P, 1), device="cuda", generator=g, dtype=torch.int32)
    m.percent_dense = 0.01
    m.optimizer = GaussianAdam([{"params": [getattr(m, a)], "lr": 1e-3, "name": n} for n, a in GROUPS.items()], lr=0.0, eps=1e-15)
    for a in GROUPS.values():
        getattr(m, a).grad = torch.randn(getattr(m, a).shape, device="cuda", generator=g) * 1e-3
    m.optimizer.step()
    for a in GROUPS.values():
        getattr(m, a).grad = None
    hot = torch.rand(P, device="cuda", generator=g) < 0.10
    m.denom = torch.randint(1, 6, (P, 1), device="cuda", generator=g).float()
    m.xyz_gradient_accum = torch.where(hot.unsqueeze(1), 3e-4, 1e-5) * m.denom
    m.max_radii2D = torch.zeros(P, device="cuda")
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=3_000_000)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_densify needs a GPU"
    benchkit.banner()
    P = args.points
    fns = {"ref": rs.densify_and_prune, "native": densify.densify_and_prune}
    times = {k: [] for k in fns}
    peak = {}
    info = {}
    for rep in range(args.repeats + 1):                   # the first round warms up
        for arm, fn in fns.items():
            m = build(P, 1)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            d = {}
            t0 = time.perf_counter()
            fn(m, 0.0002, 0.005, 10.0, 20, d)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if rep:
                times[arm].append(dt)
            peak[arm] = torch.cuda.max_memory_allocated() - base
            info[arm] = (int(d["n_points_cloned"]), int(d["n_points_split"]), int(d["n_points_pruned"]), m._xyz.shape[0])
            del m
    C, S, pruned, P_out = info["native"]
    assert info["ref"] == info["native"], info
    print(json.dumps({"P": P, "cloned": C / P, "split": S / P, "pruned": pruned / (P + C + S), "P_out": P_out}), flush=True)
    row = 59 * 4
    nbytes = P * 3 * row + P_out * 3 * row + P * (4 + 4 * 4 + 16 + 12) + P_out * 4 + 2 * S * 12
    for arm in fns:
        ms = statistics.median(times[arm]) * 1e3
        print(json.dumps({"arm": arm, "ms_median": round(ms, 3), "ms_all": [round(t * 1e3, 3) for t in times[arm]],
                          "peak_extra_MB": round(peak[arm] / 2**20, 1),
                          "native_bytes_GB": round(nbytes / 1e9, 3), "share_of_3.35TB/s": round(nbytes / HBM_BYTES_PER_S / (ms * 1e-3), 3)}),
              flush=True)

    # per-iteration statistics: train.py:134-135 against one add_densification_stats(..., radii)
    m = build(P, 2)
    r = build(P, 2)
    g = torch.Generator(device="cuda").manual_seed(3)
    vs = torch.zeros(P, 3, device="cuda", requires_grad=True)
    vis = torch.rand(P, device="cuda", generator=g) < 0.83
    vs.grad = torch.randn(P, 3, device="cuda", generator=g) * 1e-3 * vis.unsqueeze(1)
    radii = (torch.rand(P, device="cuda", generator=g) * 50).int() * vis
    for arm, fn in (("stats_ref", lambda: rs.add_densification_stats(r, vs, vis, radii)),
                    ("stats_native", lambda: densify.add_densification_stats(m, vs, vis, radii))):
        for _ in range(5):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 50
        sbytes = P * (12 + 1 + 4 + 3 * 8)                # grad rows (3 floats read), visibility, radii, 3 statistics read + written
        print(json.dumps({"arm": arm, "ms": round(ms, 4), "share_of_3.35TB/s": round(sbytes / HBM_BYTES_PER_S / (ms * 1e-3), 3)}), flush=True)
    for k in ("xyz_gradient_accum", "denom", "max_radii2D"):
        assert torch.equal(getattr(m, k), getattr(r, k)), k


if __name__ == "__main__":
    main()
