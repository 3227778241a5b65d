"""Cost of Mip-Splatting's 3D smoothing filter (DESIGN.md §5o): computing it, and rendering with it.

    python tools/bench_filter3d.py [--steps 10] [--warmup 3]

Part 1, compute_3D_filter at P = 3 M (bench.py's C3 centres) from 64 and 300 orbit cameras at 1920x1080:
  native     gs_b200.mip.compute_3D_filter (gsb_filter_3d: two launches)
  torch      Mip-Splatting's GaussianModel.compute_3D_filter loop as it is written (mip_splatting_loop below: one `xyz @ R + T` per
             camera and its other ops), the cost a training script pays today; its per-camera torch.tensor(camera.R / camera.T)
             host copies are left out (R and T are slices of the device-resident world_view_transform), which only favours it
Part 2, one forward + backward (gsb_forward / gsb_backward), one view per step over bench.py's cameras:
  C3         bench.py's workload (3 M quantised Gaussians, 1920x1080) without and with a filter
  raw        a dense 3 M raw-parameter scene of SH degree 3 (benchkit.dense_raw_workload) without and with a filter
The filter is compute_3D_filter's from the workload's cameras.  Arms alternate step by step, L2 is flushed (256 MB write) before
each timed step (benchkit.time_arms).  Prints the card's name and power limit, then one JSON line per arm and the ratios.
"""
import argparse
import json
import math
from types import SimpleNamespace

import torch

import benchkit


def orbit(n, W, H, radius=4.0):
    """n cameras on a circle around the origin, looking at it, as the objects compute_3D_filter reads."""
    cams = []
    for i in range(n):
        a = 2 * math.pi * i / n
        R = torch.tensor([[math.cos(a), 0, -math.sin(a)], [0, 1, 0], [math.sin(a), 0, math.cos(a)]])
        view = torch.eye(4)
        view[:3, :3] = R.T
        view[3, 2] = radius
        cams.append(SimpleNamespace(world_view_transform=view.cuda(), image_width=W, image_height=H, FoVx=1.0,
                                    FoVy=2 * math.atan(math.tan(0.5) * H / W)))
    return cams


@torch.no_grad()
def mip_splatting_loop(xyz, cameras):
    """Mip-Splatting's compute_3D_filter (Yu et al. 2024) op for op, with R and T read from world_view_transform (its transpose holds
    R^T in the upper 3 x 3 and T in the last row) -> filter [P, 1]."""
    distance = torch.ones((xyz.shape[0]), device=xyz.device) * 100000.0
    valid_points = torch.zeros((xyz.shape[0]), device=xyz.device, dtype=torch.bool)
    focal_length = 0.
    for camera in cameras:
        V = camera.world_view_transform
        R, T = V[:3, :3], V[3, :3]
        xyz_cam = xyz @ R + T[None, :]
        xyz_to_cam = torch.norm(xyz_cam, dim=1)  # noqa: F841  (computed and unused in Mip-Splatting too)
        valid_depth = xyz_cam[:, 2] > 0.2
        x, y, z = xyz_cam[:, 0], xyz_cam[:, 1], xyz_cam[:, 2]
        z = torch.clamp(z, min=0.001)
        focal_x = camera.image_width / (2 * math.tan(camera.FoVx / 2))
        focal_y = camera.image_height / (2 * math.tan(camera.FoVy / 2))
        x = x / z * focal_x + camera.image_width / 2.0
        y = y / z * focal_y + camera.image_height / 2.0
        in_screen = torch.logical_and(torch.logical_and(x >= -0.15 * camera.image_width, x <= camera.image_width * 1.15),
                                      torch.logical_and(y >= -0.15 * camera.image_height, y <= 1.15 * camera.image_height))
        valid = torch.logical_and(valid_depth, in_screen)
        distance[valid] = torch.min(distance[valid], z[valid])
        valid_points = torch.logical_or(valid_points, valid)
        if focal_length < focal_x:
            focal_length = focal_x
    distance[~valid_points] = distance[valid_points].max()
    filter_3D = distance / focal_length * (0.2 ** 0.5)
    return filter_3D[..., None]


def summary(ms):
    v = sorted(ms)
    return dict(steps=len(v), median_ms=round(v[len(v) // 2], 4), min_ms=round(v[0], 4), max_ms=round(v[-1], 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    dev = benchkit.device("bench_filter3d")
    benchkit.banner()
    flush = benchkit.l2_flush(dev)
    from gs_b200 import mip
    wl = benchkit.bench_workload("C3", dev)
    model = SimpleNamespace(get_xyz=wl.scene.means3D)
    ratios = {}
    for n in (64, 300):
        cams = orbit(n, wl.W, wl.H)
        arms = {"native": lambda i: mip.compute_3D_filter(model, cams), "torch": lambda i: mip_splatting_loop(model.get_xyz, cams)}
        ms = benchkit.time_arms(arms, args.steps, args.warmup, flush)
        for k, v in ms.items():
            print(json.dumps({"part": "compute_3D_filter", "arm": k, "P": wl.scene.P, "cameras": n, **summary(v)}), flush=True)
        ratios[f"torch_over_native_{n}"] = round(summary(ms["torch"])["median_ms"] / summary(ms["native"])["median_ms"], 2)

    for name, w in (("C3", wl), ("raw", benchkit.dense_raw_workload(wl.W, wl.H, dev))):
        w.cams = wl.cams
        f = mip.compute_3D_filter(SimpleNamespace(get_xyz=w.scene.means3D), w.cams).view(-1)
        op = {} if w.quant is not None else dict(opacity=w.scene.opacity)

        def fb(i, filt):
            cam = w.cams[i % len(w.cams)]
            kw = dict(filter_3D=f) if filt else {}
            benchkit.forward_backward(w, cam, dict(kw), dict(kw, **op) if filt else {})
        arms = {"plain": lambda i: fb(i, False), "filter": lambda i: fb(i, True)}
        ms = benchkit.time_arms(arms, args.steps, args.warmup, flush)
        kernels = benchkit.kernel_ms(arms, min(args.steps, 6), flush)
        for k, v in ms.items():
            print(json.dumps({"part": "forward_backward", "workload": name, "arm": k, "P": w.scene.P, **summary(v),
                              "kernels_ms_per_step": kernels[k]}), flush=True)
        ratios[f"{name}_filter_over_plain"] = round(summary(ms["filter"])["median_ms"] / summary(ms["plain"])["median_ms"], 4)
    print(json.dumps(ratios), flush=True)


if __name__ == "__main__":
    main()
