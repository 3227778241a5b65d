"""`render_backward`, `preprocess` and `preprocess_backward` of this tree against a checkout of the parent commit, measured in one command.

    git archive HEAD~1 | tar -x -C _trees/parent && python _trees/parent/reduced-3dgs_b200/csrc/build.py
    python tools/bench_render_backward.py --parent-tree _trees/parent [--steps 20] [--warmup 5] [--reps 2]

The parent checkout lies inside the repository (`_trees/` is git-ignored) and is built before the call.  The two trees are measured
alternately (parent, this, parent, this, ...), each arm in a process of its own that imports bench.py and the library from its
tree.  Workloads, one per input format of the per-Gaussian kernels: bench.py's C3 (3 M codebook-quantised Gaussians), a dense 3 M
scene rendered from its raw parameters (`raw=`, SH degree 3) and the same scene activated by torch before the call, all
1920x1080, forward + backward of bench.py's first camera.  Every step is timed with a CUDA event
pair, L2 is flushed (256 MB write) between steps outside the pair, the library's per-kernel event pairs give `render_backward`,
`preprocess` and `preprocess_backward` per step; medians and min..max of the timed steps are reported.  The gradients of the last step (the inputs are the same in
every step) are kept as seeded row samples, and per gradient array the largest difference between the two trees is printed
relative to the array's largest magnitude, next to the same figure for two runs of the parent.  Prints the card's name and
power limit.  Without a GPU it fails.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import benchkit     # from this script's directory: the parent tree need not have it

ROOT = benchkit.ROOT
WORKLOADS = ("C3", "dense3M_raw", "dense3M_activated")
KERNELS = ("render_backward", "preprocess", "preprocess_backward")


def measure(tree, steps, warmup, dump):
    """One arm: this process imports everything from `tree`, prints one JSON line per workload and writes the gradient samples."""
    sys.path[:0] = [tree, os.path.join(tree, "reduced-3dgs_b200")]
    import numpy as np
    import torch
    dev = benchkit.device("bench_render_backward")
    import bench
    from gs_b200 import lib as gsl
    assert os.path.realpath(gsl.__file__).startswith(os.path.realpath(tree) + os.sep), gsl.__file__
    assert os.path.realpath(bench.__file__).startswith(os.path.realpath(tree) + os.sep), bench.__file__
    flush = benchkit.l2_flush(dev)
    c3 = benchkit.bench_workload("C3", dev)
    cam = c3.cams[0]

    samples = {}
    gsl.profile_enable(True)
    raw = benchkit.dense_raw_workload(c3.W, c3.H, dev)
    for name, wl in zip(WORKLOADS, (c3, raw, benchkit.activated_workload(raw))):
        prof, last = [], []

        def step(i):
            # the library's event pairs of the previous step, so prof[k + 1] belongs to step k.  The read runs inside this step's
            # event pair, while the L2 flush in front of it still runs on the GPU; host time it takes beyond the flush counts in
            # step_ms (the kernels' own pairs do not see it)
            prof.append(gsl.profile_read())
            last[:] = benchkit.forward_backward(wl, cam)

        step_ms = benchkit.time_arms({name: step}, steps, warmup, flush)[name]
        prof.append(gsl.profile_read())
        kernel_ms = {k: [p.get(k, (0.0, 0))[0] for p in prof[warmup + 1:]] for k in KERNELS}
        R, grads, P = last[0][0], last[1], wl.scene.P
        rows = torch.as_tensor(np.sort(np.random.default_rng(P).choice(P, bench.DUMP_ROWS, replace=False)), device=dev)
        for i, g in enumerate(grads):                                          # every per-Gaussian output (raw= appends its own)
            if torch.is_tensor(g) and g.dim() and g.shape[0] == P:
                samples[f"{name}/{bench.GRAD_NAMES[i] if i < len(bench.GRAD_NAMES) else i}"] = g[rows].float().cpu().numpy()
        spread = lambda v: {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}
        print(json.dumps({"workload": name, "R": int(R), "steps": steps, **{f"{k}_ms": spread(v) for k, v in kernel_ms.items()},
                          "step_ms": spread(step_ms)}), flush=True)
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
    benchkit.banner()

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
                                  **{f"{k}_this_over_parent": round(t[f"{k}_ms"]["median"] / p[f"{k}_ms"]["median"], 4) for k in KERNELS},
                                  "step_this_over_parent": round(t["step_ms"]["median"] / p["step_ms"]["median"], 4)}), flush=True)
        p0, p1, t0 = (np.load(os.path.join(tmp, f)) for f in ("parent0.npz", "parent1.npz", "this0.npz"))
        own, gap = largest_gaps(p0, p1), largest_gaps(p0, t0)
        for k in p0.files:
            print(json.dumps({"gradient": k, "this_vs_parent": float(f"{gap[k]:.3g}"), "parent_vs_parent": float(f"{own[k]:.3g}")}), flush=True)


if __name__ == "__main__":
    main()
