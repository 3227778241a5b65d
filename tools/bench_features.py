"""Cost of per-Gaussian feature channels (`features=[P, F]`) against the colour step and against the workaround they replace.

    python tools/bench_features.py [--config C3] [--steps 10] [--warmup 3] [--F 1,3,8,16,32,64] [--ch 0|8|16]

bench.py's workload (C3: 3 M quantised Gaussians, mixed SH degrees, 1920x1080, device-resident), one view per step over its
cameras; each step is timed with a CUDA event pair, and L2 is flushed (256 MB write) between steps outside the pair.  Arms:
  base         colour forward (fwd) / forward + backward (fb), what bench.py times
  feat_F       the same plus F feature channels (gsb_forward_features / gsb_backward_features), loss on colour and features
  override_F   the workaround: the colour step plus one colors_precomp render (forward, and backward) per 3 channels
The arms alternate step by step so that drift of the shared machine hits all of them alike.  --ch sets GSB_FEATURES_CH (the
channels per CTA of both feature kernels; 0 = the built-in choice).  A profiled pass gives the feature kernels' own device time.
Prints the card's name and power limit, then one JSON line per arm.
"""
import argparse
import json
import math
import os
import subprocess
import sys
from types import SimpleNamespace


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
    import torch
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
    import bench  # workload and cameras of the benchmark, unchanged
    from diff_gaussian_rasterization import _C
    from gs_b200 import lib as gsl
    from gs_b200 import synth

    EMPTY = torch.Tensor([])
    assert torch.cuda.is_available(), "bench_features needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "n/a", "ch": args.ch}), flush=True)

    name, W, H, scene, quant, prune = bench.build_workload(SimpleNamespace(config=args.config, points=0), dev, 0, 1)
    cams = [c.to(dev) for c in bench.bench_cameras(W, H, 4)]
    sd = scene.to(dev)
    qd = None if quant is None else quant.to(dev)
    Fs = [int(f) for f in args.F.split(",")]
    g = torch.Generator().manual_seed(1100)
    feats = torch.randn(sd.P, max(Fs), generator=g).to(dev)
    G = synth.grad_image(W, H, 1000).to(dev)
    Gf = torch.randn(max(Fs), H, W, generator=g).to(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    bg0 = torch.zeros(3, device=dev)
    fslice = {F: feats[:, :F].contiguous() for F in Fs}
    groups = {F: [torch.nn.functional.pad(feats[:, k:min(k + 3, F)], (0, 3 - (min(k + 3, F) - k))).contiguous() for k in range(0, F, 3)]
              for F in Fs}

    def fwd_args(c, colors=EMPTY):
        tx, ty = math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5)
        if qd is not None:
            return (bg0, sd.means3D, colors, EMPTY, EMPTY, EMPTY, 1.0, EMPTY, c.world_view_transform, c.full_proj_transform, tx, ty, H, W,
                    EMPTY, sd.degrees, c.camera_center, False, False)
        return (bg0, sd.means3D, colors, sd.opacity, sd.scales, sd.rotations, 1.0, EMPTY, c.world_view_transform, c.full_proj_transform,
                tx, ty, H, W, EMPTY if colors.numel() else sd.sh, sd.degrees, c.camera_center, False, False)

    def run(a, dL, bwd, fkw=None, bkw=None):
        out = _C.rasterize_gaussians(*a, quant=qd, **(fkw or {}))
        if bwd:
            R, color, radii, gb, bb, ib = out[:6]
            _C.rasterize_gaussians_backward(a[0], a[1], radii, a[2], a[4], a[5], 1.0, EMPTY, a[8], a[9], a[10], a[11], dL, a[14], a[15],
                                            a[16], gb, R, bb, ib, 0.0, False, quant=qd, **(bkw or {}))

    def arm_base(bwd):
        return lambda c: run(fwd_args(c), G, bwd)

    def arm_feat(F, bwd):
        return lambda c: run(fwd_args(c), G, bwd, dict(features=fslice[F]), dict(features=fslice[F], dL_dfeatures_out=Gf[:F]))

    def arm_override(F, bwd):
        def fn(c):
            run(fwd_args(c), G, bwd)
            for k, col in enumerate(groups[F]):
                run(fwd_args(c, col), Gf[3 * k:3 * k + 3] if 3 * k + 3 <= F else G, bwd)
        return fn

    arms = {}
    for bwd, tag in ((False, "fwd"), (True, "fb")):
        arms[f"base_{tag}"] = arm_base(bwd)
        for F in Fs:
            arms[f"feat{F}_{tag}"] = arm_feat(F, bwd)
            arms[f"override{F}_{tag}"] = arm_override(F, bwd)
    for i in range(max(args.warmup, 1)):
        for fn in arms.values():
            flush.zero_()
            fn(cams[i % len(cams)])
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for i in range(args.steps):
        for k, fn in arms.items():
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(cams[i % len(cams)])
            e1.record()
            times[k].append((e0, e1))
    torch.cuda.synchronize()
    # the feature kernels' own device time, in a separate pass with the event brackets on
    kernels = {}
    gsl.profile_enable(True)
    for F in Fs:
        for tag in ("fwd", "fb"):
            k = f"feat{F}_{tag}"
            arms[k](cams[0])
            torch.cuda.synchronize()
            gsl.profile_read()
            for i in range(4):
                flush.zero_()
                arms[k](cams[i % len(cams)])
            torch.cuda.synchronize()
            kernels[k] = {kn: round(t / 4, 4) for kn, (t, _) in gsl.profile_read().items() if kn.startswith("features")}
    gsl.profile_enable(False)
    med = {}
    for k, v in times.items():
        ms = sorted(a.elapsed_time(b) for a, b in v)
        med[k] = ms[len(ms) // 2]
        tag = k.rsplit("_", 1)[1]
        line = {"arm": k, "config": name, "W": W, "H": H, "P": sd.P, "steps": len(ms), "median_ms": round(med[k], 3),
                "min_ms": round(ms[0], 3), "max_ms": round(ms[-1], 3), "over_base": round(med[k] / med[f"base_{tag}"], 4)}
        if k in kernels:
            line["feature_kernels_ms"] = kernels[k]
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
