"""What the rasterizer's A/B bench tools share: the card banner, the L2 flush, bench.py's workload, the dense raw-parameter
scene and its activated form, one forward + backward call, and the timed loops.

Importing this module puts the repository root and `reduced-3dgs_b200` on sys.path.  bench.py and the library are imported only
when a function needs them, so a caller that puts another tree in front of sys.path first (tools/bench_render_backward.py
--measure) gets that tree's.
"""
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

E = torch.Tensor([])


def device(tool):
    """cuda:0 as the current device.  Without a GPU the tool fails."""
    assert torch.cuda.is_available(), f"{tool} needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    return dev


def banner(**extra):
    """Prints one JSON line: the card's name as torch sees it, the NVIDIA driver's "name, power limit, max SM clock" line and the
    `extra` keys.  -> {"name", "power_limit", "max_sm_clock"} from the driver's line ({} when its query tool is missing)."""
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True).stdout.strip().splitlines()
    except OSError:
        smi = []
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "n/a", **extra}), flush=True)
    return dict(zip(("name", "power_limit", "max_sm_clock"), smi[0].split(", "))) if smi else {}


def l2_flush(dev):
    """A 256 MB buffer; zeroing it between steps evicts the 50 MB L2, so no step starts on the previous one's data."""
    return torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def bench_workload(config, dev):
    """bench.py's workload `config` on `dev`: name, W, H, scene, quant, prune, its first four cameras, bench.py's loss gradient
    image G and a black background."""
    import bench
    from gs_b200 import synth
    name, W, H, scene, quant, prune = bench.build_workload(SimpleNamespace(config=config, points=0), dev, 0, 1)
    return SimpleNamespace(name=name, W=W, H=H, scene=scene.to(dev), quant=None if quant is None else quant.to(dev),
                           prune=None if prune is None else prune.to(dev), raw=None,
                           cams=[c.to(dev) for c in bench.bench_cameras(W, H, 4)], G=synth.grad_image(W, H, 1000).to(dev),
                           bg=torch.zeros(3, device=dev))


def dense_raw_workload(W, H, dev):
    """A dense 3 M scene of SH degree 3 on `dev`, rendered from its raw parameters (`raw=`) at W x H, with the G and background
    of bench_workload."""
    from gs_b200 import synth
    s = synth.make_scene(3_000_000, 7, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.01))
    raw = (s.sh[:, :1].contiguous().to(dev), s.sh[:, 1:16].contiguous().to(dev), torch.log(s.scales).to(dev),
           s.rotations.contiguous().to(dev))
    scene = SimpleNamespace(P=s.P, means3D=s.means3D.to(dev), opacity=s.opacity.to(dev), degrees=s.degrees.to(dev))
    return SimpleNamespace(W=W, H=H, scene=scene, quant=None, prune=None, raw=raw,
                           G=synth.grad_image(W, H, 1000).to(dev), bg=torch.zeros(3, device=dev))


def activated_workload(wl):
    """The raw-parameter workload `wl` (dense_raw_workload) with its activations applied by torch before the call: scales =
    exp(_scaling), rotations = F.normalize(_rotation), sh = cat(_features_dc, _features_rest), the same Gaussians in the reference's
    input format."""
    dc, rest, scaling, rotation = wl.raw
    scene = SimpleNamespace(P=wl.scene.P, means3D=wl.scene.means3D, opacity=wl.scene.opacity, degrees=wl.scene.degrees,
                            scales=torch.exp(scaling), rotations=torch.nn.functional.normalize(rotation), sh=torch.cat((dc, rest), 1))
    return SimpleNamespace(W=wl.W, H=wl.H, scene=scene, quant=None, prune=None, raw=None, G=wl.G, bg=wl.bg)


def forward_backward(wl, cam, fwd=None, bwd=None, dL=None, colors=E, backward=True):
    """`_C.rasterize_gaussians` of workload `wl` from camera `cam` on its background, then (with `backward`)
    `_C.rasterize_gaussians_backward` of the loss gradient `dL` (default wl.G).  `fwd` / `bwd` are the calls' extra keywords;
    `colors` (colors_precomp, which replaces the SH) goes to both.  -> (forward outputs, backward outputs or None)."""
    from diff_gaussian_rasterization import _C
    s, bg = wl.scene, wl.bg
    dense = wl.quant is None and wl.raw is None
    opacity = E if wl.quant is not None else s.opacity
    scales, rotations = (s.scales, s.rotations) if dense else (E, E)
    sh = s.sh if dense and not colors.numel() else E
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    V, Pm, campos = cam.world_view_transform, cam.full_proj_transform, cam.camera_center
    kw = dict(prune_mask=wl.prune, quant=wl.quant, raw=wl.raw)
    out = _C.rasterize_gaussians(bg, s.means3D, colors, opacity, scales, rotations, 1.0, E, V, Pm, tx, ty, wl.H, wl.W, sh, s.degrees,
                                 campos, False, False, **kw, **(fwd or {}))
    if not backward:
        return out, None
    R, color, radii, gb, bb, ib = out[:6]
    return out, _C.rasterize_gaussians_backward(bg, s.means3D, radii, colors, scales, rotations, 1.0, E, V, Pm, tx, ty,
                                                wl.G if dL is None else dL, sh, s.degrees, campos, gb, R, bb, ib, 0.0, False,
                                                **kw, **(bwd or {}))


def time_arms(arms, steps, warmup, flush):
    """{name: [ms of each timed step]} of `arms` ({name: fn(i)}).  `warmup` untimed rounds (i = 0 .. warmup-1), then `steps` timed
    ones (i = 0 .. steps-1 again, so a tool that picks its camera by i sees the same sequence whatever the warm-up); each round
    runs every arm once, in the reverse order of the previous round (ABC, CBA, ...), so that drift of the shared machine hits all
    arms alike.  Each step is a CUDA event pair with L2 flushed in front of it and a synchronise after it."""
    names = list(arms)
    ms = {k: [] for k in names}
    for i in range(warmup + steps):
        for k in names if i % 2 == 0 else names[::-1]:
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arms[k](i if i < warmup else i - warmup)
            e1.record()
            torch.cuda.synchronize()
            if i >= warmup:
                ms[k].append(e0.elapsed_time(e1))
    return ms


def kernel_ms(arms, n, flush, warm=2, keep=None):
    """{name: {kernel: ms per step}} from the library's per-kernel event pairs (gsb_profile_*), in a pass of its own per arm:
    `warm` steps, then `n` counted steps, L2 flushed in front of each.  `keep(kernel name)` selects the kernels reported."""
    from gs_b200 import lib as gsl
    out = {}
    gsl.profile_enable(True)
    for k, fn in arms.items():
        for i in range(warm):
            flush.zero_()
            fn(i)
        torch.cuda.synchronize()
        gsl.profile_read()
        for i in range(n):
            flush.zero_()
            fn(i)
        torch.cuda.synchronize()
        out[k] = {kn: round(t / n, 4) for kn, (t, _) in gsl.profile_read().items() if keep is None or keep(kn)}
    gsl.profile_enable(False)
    return out
