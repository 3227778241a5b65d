"""Cost of the inverse-depth and alpha maps (return_maps) against the colour step and against the emulation they replace.

    python tools/bench_maps.py [--config C3] [--steps 20] [--warmup 5]

bench.py's workload (C3: 3 M quantised Gaussians, 1920x1080, device-resident), one view per step over its cameras; each step
is timed with a CUDA event pair, and L2 is flushed (256 MB write) between steps outside the pair.  Arms:
  a          colour forward + backward (gsb_forward / gsb_backward, what bench.py times)
  b          colour + both maps forward + backward (the requests' map fields), loss on all three
  c          the emulation of the reference's callers: (a) plus one override_color forward + backward per map
             (colour (1/z, 0, 0) for invdepth, colour (1, 1, 1) on a black background for alpha)
The arms alternate step by step so that drift of the shared machine hits all of them alike.  A separate profiled pass per arm
gives per-kernel times (gsb_profile_*).  Prints the card's name and power limit, then one JSON line per arm and a summary line.
"""
import argparse
import json

import torch

import benchkit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=["C1", "C2", "C3"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    dev = benchkit.device("bench_maps")
    benchkit.banner()
    flush = benchkit.l2_flush(dev)
    wl = benchkit.bench_workload(args.config, dev)
    cams, sd, W, H = wl.cams, wl.scene, wl.W, wl.H
    g = torch.Generator().manual_seed(1001)
    Gd = torch.randn(1, H, W, generator=g).to(dev)
    Ga = torch.randn(1, H, W, generator=g).to(dev)
    ones = torch.ones(sd.P, 3, device=dev)
    dLd3 = torch.zeros(3, H, W, device=dev)
    dLd3[0] = Gd[0]
    dLa3 = torch.zeros(3, H, W, device=dev)
    dLa3[0] = Ga[0]

    def arm_a(i):
        benchkit.forward_backward(wl, cams[i % len(cams)])

    def arm_b(i):
        benchkit.forward_backward(wl, cams[i % len(cams)], dict(return_maps=True), dict(dL_dinvdepth=Gd, dL_dalpha=Ga))

    def arm_c(i):
        c = cams[i % len(cams)]
        benchkit.forward_backward(wl, c)
        V = c.world_view_transform                       # the callers' per-Gaussian depth: view-space z of the means
        z = sd.means3D @ V[:3, 2] + V[3, 2]
        col = torch.zeros(sd.P, 3, device=dev)
        col[:, 0] = 1.0 / z
        benchkit.forward_backward(wl, c, dL=dLd3, colors=col)
        benchkit.forward_backward(wl, c, dL=dLa3, colors=ones)

    arms = {"a": arm_a, "b": arm_b, "c": arm_c}
    ms = {k: sorted(v) for k, v in benchkit.time_arms(arms, args.steps, args.warmup, flush).items()}
    kernels = benchkit.kernel_ms(arms, min(args.steps, 8), flush)
    med = {k: v[len(v) // 2] for k, v in ms.items()}
    for k in arms:
        v = ms[k]
        print(json.dumps({"arm": k, "config": wl.name, "W": W, "H": H, "P": sd.P, "steps": len(v), "median_ms": round(med[k], 4),
                          "mean_ms": round(sum(v) / len(v), 4), "min_ms": round(v[0], 4), "max_ms": round(v[-1], 4),
                          "kernels_ms_per_step": kernels[k]}), flush=True)
    print(json.dumps({"b_over_a": round(med["b"] / med["a"], 4), "c_over_a": round(med["c"] / med["a"], 4),
                      "b_over_c": round(med["b"] / med["c"], 4)}), flush=True)


if __name__ == "__main__":
    main()
