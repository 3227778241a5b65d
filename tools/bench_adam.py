"""Cost of the optimizer step (GaussianAdam, gsb_adam_step; DESIGN.md §5f) against torch.optim.Adam and against the render step.

    python tools/bench_adam.py [--steps 20] [--warmup 3]

C3 (bench.py's workload: 3 M Gaussians, SH degrees 0/1/2/3 mixed 50/20/15/15 %), the reference's six parameter tensors
(xyz [P,3], f_dc [P,1,3], f_rest [P,15,3], opacity [P,1], scaling [P,3], rotation [P,4]: 59 floats per Gaussian) with its
learning rates and eps = 1e-15; visibility = radii > 0 of one 1920x1080 view's forward, degrees = the scene's.  Arms:
  a  torch.optim.Adam, default (foreach)        d  GaussianAdam, step(visibility=...)
  b  torch.optim.Adam(fused=True)               e  GaussianAdam, step(visibility=..., degrees=...)
  c  GaussianAdam, dense                        f  the render forward + backward of that view (bench.py's step), for scale
Each step is timed by a CUDA event pair, L2 is flushed (256 MB write) between steps outside the pair, the arms alternate step
by step; median of --steps.  Bytes are computed from shapes: 28 B per updated element (read p, g, m, v; write p, m, v), plus
1 B of visibility per row for each tensor and 4 B of degree per row for the banded tensor.  Prints the card's name and power
limit, one JSON line per arm, and checks afterwards that (c) and (a) hold the same bytes.
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
from gs_b200 import synth  # noqa: E402
from gs_b200.optim import GaussianAdam  # noqa: E402

EMPTY = torch.Tensor([])
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
LRS = {"xyz": 1.6e-4, "f_dc": 2.5e-3, "f_rest": 2.5e-3 / 20, "opacity": 0.05, "scaling": 5e-3, "rotation": 1e-3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_adam needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "n/a"}), flush=True)

    name, W, H, scene, quant, prune = bench.build_workload(SimpleNamespace(config="C3", points=0), dev, 0, 1)
    cam = bench.bench_cameras(W, H, 4)[0].to(dev)
    sd = scene.to(dev)
    qd = quant.to(dev)
    P = sd.P
    bg0 = torch.zeros(3, device=dev)
    G = synth.grad_image(W, H, 1000).to(dev)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    fa = (bg0, sd.means3D, EMPTY, EMPTY, EMPTY, EMPTY, 1.0, EMPTY, cam.world_view_transform, cam.full_proj_transform, tx, ty, H, W,
          EMPTY, sd.degrees, cam.camera_center, False, False)

    def render_step():
        R, color, radii, gb, bb, ib = _C.rasterize_gaussians(*fa, quant=qd)[:6]
        _C.rasterize_gaussians_backward(fa[0], fa[1], radii, fa[2], fa[4], fa[5], 1.0, EMPTY, fa[8], fa[9], fa[10], fa[11], G, fa[14],
                                        fa[15], fa[16], gb, R, bb, ib, 0.0, False, quant=qd)
        return radii

    visibility = render_step() > 0
    degrees = sd.degrees.contiguous()
    base = {"xyz": sd.means3D, "f_dc": sd.sh[:, :1], "f_rest": sd.sh[:, 1:], "opacity": sd.opacity, "scaling": torch.log(sd.scales),
            "rotation": sd.rotations}
    gen = torch.Generator(device=dev).manual_seed(0)
    grads = {k: torch.randn(v.shape, device=dev, generator=gen) * 1e-3 for k, v in base.items()}
    del scene

    def groups():
        out = []
        for k, v in base.items():
            p = torch.nn.Parameter(v.detach().clone().contiguous())
            p.grad = grads[k]
            grp = {"params": [p], "lr": LRS[k], "name": k}
            if k == "f_rest":
                grp["sh_offset"] = 1
            out.append(grp)
        return out

    opts = {"a": torch.optim.Adam(groups(), lr=0.0, eps=1e-15), "b": torch.optim.Adam(groups(), lr=0.0, eps=1e-15, fused=True),
            "c": GaussianAdam(groups(), lr=0.0, eps=1e-15), "d": GaussianAdam(groups(), lr=0.0, eps=1e-15),
            "e": GaussianAdam(groups(), lr=0.0, eps=1e-15)}
    arms = {"a": opts["a"].step, "b": opts["b"].step, "c": opts["c"].step, "d": lambda: opts["d"].step(visibility=visibility),
            "e": lambda: opts["e"].step(visibility=visibility, degrees=degrees), "f": render_step}

    vis_rows = int(visibility.sum())
    deg = degrees.view(-1).clamp(0, 3)
    rest_active = int((3 * ((deg + 1) ** 2 - 1))[visibility].sum())
    floats_per_row = 59
    nb = {"a": 28 * floats_per_row * P, "b": 28 * floats_per_row * P, "c": 28 * floats_per_row * P,
          "d": 28 * floats_per_row * vis_rows + 6 * P,
          "e": 28 * ((floats_per_row - 45) * vis_rows + rest_active) + 6 * P + 4 * P}

    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    for _ in range(max(args.warmup, 1)):
        for fn in arms.values():
            flush.zero_()
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.steps):
        for k, fn in arms.items():
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            times[k].append((e0, e1))
    torch.cuda.synchronize()
    print(json.dumps({"P": P, "visible_rows": vis_rows, "visible_fraction": round(vis_rows / P, 4),
                      "degree_mix": [round(float((deg == d).float().mean()), 4) for d in range(4)]}), flush=True)
    med = {}
    for k in arms:
        v = sorted(a.elapsed_time(b) for a, b in times[k])
        med[k] = v[len(v) // 2]
        line = {"arm": k, "steps": len(v), "median_ms": round(med[k], 4), "min_ms": round(v[0], 4), "max_ms": round(v[-1], 4)}
        if k in nb:
            gbs = nb[k] / (med[k] * 1e-3) / 1e9
            line.update({"bytes": nb[k], "GB_per_s": round(gbs, 1), "fraction_of_3.35TBps": round(gbs * 1e9 / HBM_BYTES_PER_S, 3)})
        print(json.dumps(line), flush=True)
    print(json.dumps({"a_over_c": round(med["a"] / med["c"], 3), "b_over_c": round(med["b"] / med["c"], 3),
                      "c_over_f": round(med["c"] / med["f"], 3), "e_over_f": round(med["e"] / med["f"], 3)}), flush=True)
    # (c) and (a) took the same steps from the same start: every byte of params and moments must agree
    for ga, gc in zip(opts["a"].param_groups, opts["c"].param_groups):
        pa, pc = ga["params"][0], gc["params"][0]
        sa, sc = opts["a"].state[pa], opts["c"].state[pc]
        for x, y in ((pa, pc), (sa["exp_avg"], sc["exp_avg"]), (sa["exp_avg_sq"], sc["exp_avg_sq"])):
            assert torch.equal(x.detach().view(torch.int32), y.detach().view(torch.int32)), ga["name"]
    print(json.dumps({"dense_equals_torch_adam": True}), flush=True)


if __name__ == "__main__":
    main()
