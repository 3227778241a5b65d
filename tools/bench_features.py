"""Cost of per-Gaussian feature channels (`features=[P, F]`) against the colour step and against the workaround they replace.

    python tools/bench_features.py [--config C3] [--steps 10] [--warmup 3] [--F 1,3,8,16,32,64] [--ch 0|8|16]

bench.py's workload (C3: 3 M quantised Gaussians, mixed SH degrees, 1920x1080, device-resident), one view per step over its
cameras; each step is timed with a CUDA event pair, and L2 is flushed (256 MB write) between steps outside the pair.  Arms:
  base         colour forward (fwd) / forward + backward (fb), what bench.py times
  feat_F       the same plus F feature channels (the requests' `features` field), loss on colour and features
  override_F   the workaround: the colour step plus one colors_precomp render (forward, and backward) per 3 channels
The arms alternate step by step so that drift of the shared machine hits all of them alike.  --ch sets GSB_FEATURES_CH (the
channels per CTA of both feature kernels; 0 = the built-in choice).  A profiled pass gives the feature kernels' own device time.
Prints the card's name and power limit, then one JSON line per arm.
"""
import argparse
import json
import os

import torch

import benchkit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=["C1", "C2", "C3"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--F", default="1,3,8,16,32,64")
    ap.add_argument("--ch", type=int, default=0, choices=[0, 8, 16])
    args = ap.parse_args()
    if args.ch:
        os.environ["GSB_FEATURES_CH"] = str(args.ch)          # read once, when the library first launches a feature kernel
    dev = benchkit.device("bench_features")
    benchkit.banner(ch=args.ch)
    flush = benchkit.l2_flush(dev)
    wl = benchkit.bench_workload(args.config, dev)
    cams, sd, W, H = wl.cams, wl.scene, wl.W, wl.H
    Fs = [int(f) for f in args.F.split(",")]
    g = torch.Generator().manual_seed(1100)
    feats = torch.randn(sd.P, max(Fs), generator=g).to(dev)
    Gf = torch.randn(max(Fs), H, W, generator=g).to(dev)
    fslice = {F: feats[:, :F].contiguous() for F in Fs}
    groups = {F: [torch.nn.functional.pad(feats[:, k:min(k + 3, F)], (0, 3 - (min(k + 3, F) - k))).contiguous() for k in range(0, F, 3)]
              for F in Fs}

    def arm_base(bwd):
        return lambda i: benchkit.forward_backward(wl, cams[i % len(cams)], backward=bwd)

    def arm_feat(F, bwd):
        return lambda i: benchkit.forward_backward(wl, cams[i % len(cams)], dict(features=fslice[F]),
                                                   dict(features=fslice[F], dL_dfeatures_out=Gf[:F]), backward=bwd)

    def arm_override(F, bwd):
        def fn(i):
            c = cams[i % len(cams)]
            benchkit.forward_backward(wl, c, backward=bwd)
            for k, col in enumerate(groups[F]):
                benchkit.forward_backward(wl, c, dL=Gf[3 * k:3 * k + 3] if 3 * k + 3 <= F else wl.G, colors=col, backward=bwd)
        return fn

    arms = {}
    for bwd, tag in ((False, "fwd"), (True, "fb")):
        arms[f"base_{tag}"] = arm_base(bwd)
        for F in Fs:
            arms[f"feat{F}_{tag}"] = arm_feat(F, bwd)
            arms[f"override{F}_{tag}"] = arm_override(F, bwd)
    times = benchkit.time_arms(arms, args.steps, args.warmup, flush)
    # the feature kernels' own device time
    kernels = benchkit.kernel_ms({k: arms[k] for F in Fs for k in (f"feat{F}_fwd", f"feat{F}_fb")}, 4, flush, warm=1,
                                 keep=lambda kn: kn.startswith("features"))
    med = {}
    for k, v in times.items():
        ms = sorted(v)
        med[k] = ms[len(ms) // 2]
        tag = k.rsplit("_", 1)[1]
        line = {"arm": k, "config": wl.name, "W": W, "H": H, "P": sd.P, "steps": len(ms), "median_ms": round(med[k], 3),
                "min_ms": round(ms[0], 3), "max_ms": round(ms[-1], 3), "over_base": round(med[k] / med[f"base_{tag}"], 4)}
        if k in kernels:
            line["feature_kernels_ms"] = kernels[k]
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
