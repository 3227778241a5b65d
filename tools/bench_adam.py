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

import torch

import benchkit
from gs_b200.optim import GaussianAdam  # on sys.path through benchkit

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
LRS = {"xyz": 1.6e-4, "f_dc": 2.5e-3, "f_rest": 2.5e-3 / 20, "opacity": 0.05, "scaling": 5e-3, "rotation": 1e-3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    dev = benchkit.device("bench_adam")
    benchkit.banner()

    wl = benchkit.bench_workload("C3", dev)
    sd = wl.scene
    P = sd.P

    def render_step():
        return benchkit.forward_backward(wl, wl.cams[0])[0][2]

    visibility = render_step() > 0
    degrees = sd.degrees.contiguous()
    base = {"xyz": sd.means3D, "f_dc": sd.sh[:, :1], "f_rest": sd.sh[:, 1:], "opacity": sd.opacity, "scaling": torch.log(sd.scales),
            "rotation": sd.rotations}
    gen = torch.Generator(device=dev).manual_seed(0)
    grads = {k: torch.randn(v.shape, device=dev, generator=gen) * 1e-3 for k, v in base.items()}

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
    arms = {"a": lambda i: opts["a"].step(), "b": lambda i: opts["b"].step(), "c": lambda i: opts["c"].step(),
            "d": lambda i: opts["d"].step(visibility=visibility), "e": lambda i: opts["e"].step(visibility=visibility, degrees=degrees),
            "f": lambda i: render_step()}

    vis_rows = int(visibility.sum())
    deg = degrees.view(-1).clamp(0, 3)
    rest_active = int((3 * ((deg + 1) ** 2 - 1))[visibility].sum())
    floats_per_row = 59
    nb = {"a": 28 * floats_per_row * P, "b": 28 * floats_per_row * P, "c": 28 * floats_per_row * P,
          "d": 28 * floats_per_row * vis_rows + 6 * P,
          "e": 28 * ((floats_per_row - 45) * vis_rows + rest_active) + 6 * P + 4 * P}

    times = benchkit.time_arms(arms, args.steps, args.warmup, benchkit.l2_flush(dev))
    print(json.dumps({"P": P, "visible_rows": vis_rows, "visible_fraction": round(vis_rows / P, 4),
                      "degree_mix": [round(float((deg == d).float().mean()), 4) for d in range(4)]}), flush=True)
    med = {}
    for k in arms:
        v = sorted(times[k])
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
