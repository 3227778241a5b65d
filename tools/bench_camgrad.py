"""Cost of the camera gradients (camera_grads=True, gsb_backward's camera outputs) against the colour step.

    python tools/bench_camgrad.py [--config C3] [--steps 20] [--warmup 5]

bench.py's workload (C3: 3 M quantised Gaussians, 1920x1080, device-resident), one view per step over its cameras; each step
is timed with a CUDA event pair, and L2 is flushed (256 MB write) between steps outside the pair.  Arms:
  a          colour forward + backward (gsb_forward / gsb_backward, what bench.py times)
  b          the same plus the gradients w.r.t. viewmatrix, projmatrix and campos (gsb_backward's camera outputs)
The arms alternate step by step so that drift of the shared machine hits both alike.  A separate profiled pass per arm gives
per-kernel times (gsb_profile_*): preprocess_backward and camera_grad (the one-CTA finishing kernel) are the ones that change.
Prints the card's name and power limit, then one JSON line per arm and a summary line.
"""
import argparse
import json

import benchkit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=["C1", "C2", "C3"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    dev = benchkit.device("bench_camgrad")
    benchkit.banner()
    flush = benchkit.l2_flush(dev)
    wl = benchkit.bench_workload(args.config, dev)
    cams = wl.cams

    arms = {"a": lambda i: benchkit.forward_backward(wl, cams[i % len(cams)], bwd=dict(camera_grads=False)),
            "b": lambda i: benchkit.forward_backward(wl, cams[i % len(cams)], bwd=dict(camera_grads=True))}
    ms = {k: sorted(v) for k, v in benchkit.time_arms(arms, args.steps, args.warmup, flush).items()}
    kernels = benchkit.kernel_ms(arms, min(args.steps, 8), flush)
    med = {k: v[len(v) // 2] for k, v in ms.items()}
    for k in arms:
        v = ms[k]
        print(json.dumps({"arm": k, "config": wl.name, "W": wl.W, "H": wl.H, "P": wl.scene.P, "steps": len(v),
                          "median_ms": round(med[k], 4), "mean_ms": round(sum(v) / len(v), 4), "min_ms": round(v[0], 4),
                          "max_ms": round(v[-1], 4), "kernels_ms_per_step": kernels[k]}), flush=True)
    pb = {k: kernels[k].get("preprocess_backward", 0.0) for k in arms}
    print(json.dumps({"b_over_a": round(med["b"] / med["a"], 4), "b_minus_a_ms": round(med["b"] - med["a"], 4),
                      "preprocess_backward_b_minus_a_ms": round(pb["b"] - pb["a"], 4),
                      "camera_grad_ms": kernels["b"].get("camera_grad", 0.0)}), flush=True)


if __name__ == "__main__":
    main()
