"""`render_backward` of this tree against a checkout of the parent commit, measured in one command.

    git archive HEAD~1 | tar -x -C _trees/parent && python _trees/parent/reduced-3dgs_b200/csrc/build.py
    python tools/bench_render_backward.py --parent-tree _trees/parent [--steps 20] [--warmup 5] [--reps 2]

The parent checkout lies inside the repository (`_trees/` is git-ignored) and is built before the call.  The two trees are measured
alternately (parent, this, parent, this, ...), each arm in a process of its own that imports bench.py and the library from its
tree.  Workloads: bench.py's C3 (3 M codebook-quantised Gaussians) and a dense 3 M scene rendered from its raw parameters
(`raw=`, SH degree 3), both 1920x1080, forward + backward of bench.py's first camera.  Every step is timed with a CUDA event
pair, L2 is flushed (256 MB write) between steps outside the pair, the library's per-kernel event pairs give `render_backward`
per step; medians and min..max of the timed steps are reported.  The gradients of the last step (the inputs are the same in
every step) are kept as seeded row samples, and per gradient array the largest difference between the two trees is printed
relative to the array's largest magnitude, next to the same figure for two runs of the parent.  Prints the card's name and
power limit.  Without a GPU it fails.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKLOADS = ("C3", "dense3M_raw")


def measure(tree, steps, warmup, dump):
    """One arm: this process imports everything from `tree`, prints one JSON line per workload and writes the gradient samples."""
    sys.path[:0] = [tree, os.path.join(tree, "reduced-3dgs_b200")]
    import numpy as np
    import torch
    assert torch.cuda.is_available(), "bench_render_backward needs a GPU"
    import bench
    from diff_gaussian_rasterization import _C
    from gs_b200 import lib as gsl
    from gs_b200 import synth
    assert os.path.realpath(gsl.__file__).startswith(os.path.realpath(tree) + os.sep), gsl.__file__
    E = torch.Tensor([])
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

    name, W, H, scene, quant, prune = bench.build_workload(SimpleNamespace(config="C3", points=0), dev, 0, 1)
    cam = bench.bench_cameras(W, H, 4)[0].to(dev)
    sd, qd = scene.to(dev), quant.to(dev)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    bg = torch.zeros(3, device=dev)
    G = synth.grad_image(W, H, 1000).to(dev)

    def c3_step():
        fa = (bg, sd.means3D, E, sd.opacity, E, E, 1.0, E, cam.world_view_transform, cam.full_proj_transform, tx, ty, H, W, E, sd.degrees,
              cam.camera_center, False, False)
        R, color, radii, gb, bb, ib = _C.rasterize_gaussians(*fa, quant=qd)
        return R, _C.rasterize_gaussians_backward(bg, sd.means3D, radii, E, E, E, 1.0, E, cam.world_view_transform, cam.full_proj_transform,
                                                  tx, ty, G, E, sd.degrees, cam.camera_center, gb, R, bb, ib, 0.0, False, quant=qd)

    dsc = synth.make_scene(3_000_000, 7, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.01))
    xyz, op = dsc.means3D.to(dev), dsc.opacity.to(dev)
    raw = (dsc.sh[:, :1].contiguous().to(dev), dsc.sh[:, 1:16].contiguous().to(dev), torch.log(dsc.scales).to(dev),
           dsc.rotations.contiguous().to(dev))
    deg = dsc.degrees.to(dev)

    def dense_step():
        fa = (bg, xyz, E, op, E, E, 1.0, E, cam.world_view_transform, cam.full_proj_transform, tx, ty, H, W, E, deg, cam.camera_center,
              False, False)
        R, color, radii, gb, bb, ib = _C.rasterize_gaussians(*fa, raw=raw)
        return R, _C.rasterize_gaussians_backward(bg, xyz, radii, E, E, E, 1.0, E, cam.world_view_transform, cam.full_proj_transform,
                                                  tx, ty, G, E, deg, cam.camera_center, gb, R, bb, ib, 0.0, False, raw=raw)

    samples = {}
    gsl.profile_enable(True)
    for wl, step, P in zip(WORKLOADS, (c3_step, dense_step), (sd.P, dsc.P)):
        step_ms, rb_ms = [], []
        for i in range(warmup + steps):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            R, grads = step()
            b.record()
            torch.cuda.synchronize()
            prof = gsl.profile_read()
            if i >= warmup:
                step_ms.append(a.elapsed_time(b))
                rb_ms.append(prof["render_backward"][0])
        rows = torch.as_tensor(np.sort(np.random.default_rng(P).choice(P, bench.DUMP_ROWS, replace=False)), device=dev)
        for i, g in enumerate(grads):                                          # every per-Gaussian output (raw= appends its own)
            if torch.is_tensor(g) and g.dim() and g.shape[0] == P:
                samples[f"{wl}/{bench.GRAD_NAMES[i] if i < len(bench.GRAD_NAMES) else i}"] = g[rows].float().cpu().numpy()
        print(json.dumps({"workload": wl, "R": int(R), "steps": steps,
                          "render_backward_ms": {"median": round(statistics.median(rb_ms), 4), "min": round(min(rb_ms), 4), "max": round(max(rb_ms), 4)},
                          "step_ms": {"median": round(statistics.median(step_ms), 4), "min": round(min(step_ms), 4), "max": round(max(step_ms), 4)}}),
              flush=True)
    gsl.profile_enable(False)
    np.savez(dump, **samples)


def largest_gaps(a, b):
    """Per gradient array: max |a - b| / max |a|."""
    import numpy as np
    return {k: float(np.abs(a[k].astype(np.float64) - b[k]).max() / max(float(np.abs(a[k]).max()), 1e-30)) for k in a.files}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-tree", help="built checkout of the parent commit, inside the repository")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=2, help="(parent, this tree) pairs")
    ap.add_argument("--measure", metavar="TREE", help=argparse.SUPPRESS)      # one arm (the subprocess mode)
    ap.add_argument("--dump", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.measure:
        return measure(args.measure, args.steps, args.warmup, args.dump)
    if not args.parent_tree:
        ap.error("--parent-tree is required")
    if args.steps < 20 or args.reps < 2:
        ap.error("a median of at least 20 steps and at least 2 pairs")
    parent = os.path.realpath(os.path.join(ROOT, args.parent_tree))
    if not parent.startswith(os.path.realpath(ROOT) + os.sep):
        ap.error("the parent tree must lie inside the repository")
    for tree in (parent, ROOT):
        so = os.path.join(tree, "reduced-3dgs_b200", "gs_b200", "libgs_b200.so")
        if not os.path.isfile(so):
            ap.error(f"{so} is missing: build the tree first")
    import numpy as np
    import torch
    assert torch.cuda.is_available(), "bench_render_backward needs a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "n/a"}), flush=True)

    res = {}                                                                   # (arm, rep) -> {workload: line}
    with tempfile.TemporaryDirectory() as tmp:
        for rep in range(args.reps):
            for arm, tree in (("parent", parent), ("this", ROOT)):
                dump = os.path.join(tmp, f"{arm}{rep}.npz")
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--measure", tree, "--dump", dump, "--steps", str(args.steps),
                                      "--warmup", str(args.warmup)], stdout=subprocess.PIPE, text=True, check=True).stdout
                res[arm, rep] = {}
                for line in out.splitlines():
                    if line.startswith("{"):
                        d = json.loads(line)
                        res[arm, rep][d["workload"]] = d
                        print(json.dumps({"arm": arm, "rep": rep, **d}), flush=True)
        for wl in WORKLOADS:
            for rep in range(args.reps):
                p, t = res["parent", rep][wl], res["this", rep][wl]
                print(json.dumps({"workload": wl, "pair": rep,
                                  "render_backward_this_over_parent": round(t["render_backward_ms"]["median"] / p["render_backward_ms"]["median"], 4),
                                  "step_this_over_parent": round(t["step_ms"]["median"] / p["step_ms"]["median"], 4)}), flush=True)
        p0, p1, t0 = (np.load(os.path.join(tmp, f)) for f in ("parent0.npz", "parent1.npz", "this0.npz"))
        own, gap = largest_gaps(p0, p1), largest_gaps(p0, t0)
        for k in p0.files:
            print(json.dumps({"gradient": k, "this_vs_parent": float(f"{gap[k]:.3g}"), "parent_vs_parent": float(f"{own[k]:.3g}")}), flush=True)


if __name__ == "__main__":
    main()
