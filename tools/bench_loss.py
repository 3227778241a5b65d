"""Loss row timing: fused L1 + D-SSIM (ours) vs the reference's formulation (five grouped 11x11 conv2d + element-wise ops +
autograd, utils/loss_utils.py:33-65) on the same GPU, 3x1080x1920, forward + backward."""
import json, os, sys
import torch
import torch.nn.functional as F
import benchkit
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
from utils import loss_utils as LU


def ref_loss(x, y, lam, window):
    """The SSIM definition of Wang et al. with the reference's window / padding / constants, written with torch ops."""
    C = x.shape[0]
    conv = lambda t: F.conv2d(t[None], window, padding=5, groups=C)[0]
    mu1, mu2 = conv(x), conv(y)
    s1, s2, s12 = conv(x * x) - mu1 * mu1, conv(y * y) - mu2 * mu2, conv(x * y) - mu1 * mu2
    ssim = (((2 * mu1 * mu2 + 1e-4) * (2 * s12 + 9e-4)) / ((mu1 * mu1 + mu2 * mu2 + 1e-4) * (s1 + s2 + 9e-4))).mean()
    return (1 - lam) * (x - y).abs().mean() + lam * (1 - ssim)


def timed(fn, reps=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    benchkit.banner()
    g = torch.Generator().manual_seed(0)
    x = torch.rand(3, 1080, 1920, generator=g).cuda().requires_grad_(True)
    y = torch.rand(3, 1080, 1920, generator=g).cuda()
    w1 = torch.tensor([torch.exp(torch.tensor(-(i - 5) ** 2 / 4.5)) for i in range(11)]); w1 = w1 / w1.sum()
    window = (w1[:, None] @ w1[None, :]).expand(3, 1, 11, 11).contiguous().cuda()

    def ours():
        x.grad = None
        LU.l1_ssim_loss(x, y, 0.2).backward()

    def ref():
        x.grad = None
        ref_loss(x, y, 0.2, window).backward()
    ours(); go = x.grad.clone(); ref(); gr = x.grad.clone()
    t_o, t_r = timed(ours), timed(ref)
    print(json.dumps({"row": "L1 + D-SSIM loss fwd+bwd, 3x1080x1920", "ours_ms": round(t_o, 4), "torch_conv2d_formulation_ms": round(t_r, 4),
                      "speedup": round(t_r / t_o, 1), "grad_max_rel_diff": float((go - gr).abs().max() / gr.abs().max())}))


if __name__ == "__main__":
    main()
