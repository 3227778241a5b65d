"""GPU: the differentiable path end to end — a few Adam steps through the drop-in packages (gaussian_renderer.render +
utils.loss_utils.l1_ssim_loss, the loop body of the reference's train.py:93-155) must pull a perturbed scene back towards the
images of the scene it was perturbed from, without and with anti-aliasing (pipe.antialiasing).  This is a behavioural check of
the gradients' SIGN and SCALE across all parameter groups (means, opacity logits, log-scales, quaternions, SH), complementary to
the element-wise parity tests."""
import math
from types import SimpleNamespace

import pytest
import torch

import ours as O
from gs_b200 import synth

pytestmark = pytest.mark.gpu

# per case: target scene seed, its log-scale mean, perturbation seed
_CASES = {False: (71, 0.04, 5), True: (231, 0.02, 232)}


@pytest.mark.parametrize("antialiasing", [False, True], ids=["plain", "aa"])
def test_adam_steps_reduce_the_loss(antialiasing):
    from gaussian_renderer import render
    from utils.loss_utils import l1_ssim_loss
    dev = torch.device("cuda")
    W, H = 256, 192
    scene_seed, ls, seed = _CASES[antialiasing]
    target_scene = synth.make_scene(6_000, scene_seed, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(ls), M=16)
    cams = [O.yaw_cam(W, H, yaw) for yaw in (-10.0, 0.0, 10.0)]
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False, antialiasing=antialiasing)
    bg = torch.tensor([0.1, 0.1, 0.1], device=dev)
    with torch.no_grad():
        gts = [render(c, O.Model(target_scene, dev), pipe, bg)["render"].clone() for c in cams]
    g = torch.Generator().manual_seed(seed)
    start = synth.Scene(target_scene.means3D + 0.01 * torch.randn(target_scene.means3D.shape, generator=g),
                        target_scene.opacity + 0.5 * torch.randn(target_scene.opacity.shape, generator=g),
                        target_scene.scales * torch.exp(0.2 * torch.randn(target_scene.scales.shape, generator=g)),
                        torch.nn.functional.normalize(target_scene.rotations + 0.1 * torch.randn(target_scene.rotations.shape, generator=g)),
                        target_scene.sh + 0.1 * torch.randn(target_scene.sh.shape, generator=g), target_scene.degrees)
    model = O.Model(start, dev)
    opt = torch.optim.Adam([{"params": [model._xyz], "lr": 2e-4}, {"params": [model._opacity], "lr": 5e-2},
                            {"params": [model._log_scaling], "lr": 5e-3}, {"params": [model._rotation], "lr": 1e-3},
                            {"params": [model._features], "lr": 1e-2}])
    losses = []
    for it in range(90):
        k = it % len(cams)
        opt.zero_grad(set_to_none=True)
        pkg = render(cams[k], model, pipe, bg)
        loss = l1_ssim_loss(pkg["render"], gts[k], 0.2)
        loss.backward()
        for p in model.params():
            assert p.grad is not None and torch.isfinite(p.grad).all()
        opt.step()
        losses.append(float(loss.detach()))
    first, last = sum(losses[:3]) / 3, sum(losses[-3:]) / 3
    print(f"\n[{'antialias ' if antialiasing else ''}training] loss {first:.4f} -> {last:.4f}")
    assert last < 0.8 * first, (first, last)
    # the densification statistic the reference reads after backward (train.py:139, gaussian_model.py:693-695) is populated
    assert pkg["viewspace_points"].grad is not None and float(pkg["viewspace_points"].grad[:, :2].norm(dim=1).max()) > 0
    assert int(pkg["visibility_filter"].sum()) > 0 and pkg["radii"].dtype == torch.int32
