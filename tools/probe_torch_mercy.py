"""GPU probe: the torch arithmetic of the reference's GaussianModel.mercy_points on CUDA (DESIGN.md §5k).

    python tools/probe_torch_mercy.py

Settles: (1) how torch's fp32 mean / unbiased var of integer-valued tensors compare with the correctly rounded values (fp64 of
the exact sums), over the sizes the tests use; (2) torch.median's NaN and tie behaviour; (3) the dtype of torch.quantile's
rank (fp32 q * fp32(n - 1) against the fp64 product); (4) whether the CUDA lerp is contracted to FMA; (5) the generator offset
of a 0-row torch.rand.  Prints one line per finding.
"""
import numpy as np
import torch


def fma32(a, b, c):
    return np.float32(np.float64(a) * np.float64(b) + np.float64(c))       # exact product, one rounding of the sum (fp32 args)


def main():
    assert torch.cuda.is_available(), "the probe needs a GPU"
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    # (1) mean / var
    for P in (301, 10_000, 100_000, 1_000_000, 3_000_000):
        dm = dv = 0
        trials = 20
        for _ in range(trials):
            c = (torch.poisson(torch.full((P,), 4.0, device=dev), generator=g) + 1).to(torch.int32)
            f = c.float()
            m, v = f.mean(dim=0, keepdim=True), f.var(dim=0, keepdim=True)
            x = c.cpu().numpy().astype(np.int64)
            S, Q = int(x.sum()), int((x * x).sum())
            em, ev = np.float32(S / P), np.float32((P * Q - S * S) / (P * (P - 1)))
            dm += int(m.item() != em)
            dv += int(v.item() != ev)
        print(f"mean/var P={P:>9}: torch fp32 mean differs from the correctly rounded one in {dm}/{trials}, var in {dv}/{trials}")
    # (2) median
    t = torch.tensor([0.3, float("nan"), 0.1, 0.2], device=dev)
    print("median with a NaN:", t.median().item(), "| ties [1,1,2,2] ->", torch.tensor([1., 1., 2., 2.], device=dev).median().item(),
          "| empty ->", torch.empty(0, device=dev).median().item())
    # (3) quantile rank
    mism32 = mism64 = 0
    for n in list(range(2, 4000, 7)) + [100_003, 1_000_003, 3_000_001, (1 << 24) - 1]:
        v = torch.sort(torch.rand(n, device=dev, generator=g))[0]
        for q in (0.03, 0.045):
            got = v.quantile(q).item()
            s = v.cpu().numpy()
            for rank, name in ((np.float32(q) * np.float32(n - 1), 32), (np.float64(np.float32(q)) * (n - 1), 64)):
                lo, hi = int(rank), int(np.ceil(rank))
                w = np.float32(rank - lo)
                d = np.float32(s[hi] - s[lo])
                want = fma32(w, d, s[lo]) if abs(w) < 0.5 else fma32(-d, np.float32(1) - w, s[hi])
                if name == 32:
                    mism32 += int(np.float32(got) != want)
                else:
                    mism64 += int(np.float32(got) != want)
    print(f"quantile: fp32 rank formula mismatches {mism32}, fp64 rank formula mismatches {mism64}")
    # (4) lerp contraction
    n = 1 << 20
    a = torch.rand(n, device=dev, generator=g)
    b = torch.rand(n, device=dev, generator=g)
    w = torch.rand(n, device=dev, generator=g)
    got = torch.lerp(a, b, w).cpu().numpy()
    A, B, W = a.cpu().numpy(), b.cpu().numpy(), w.cpu().numpy()
    D = (B - A).astype(np.float32)
    small = np.abs(W) < 0.5
    fused = np.where(small, (W.astype(np.float64) * D + A).astype(np.float32),
                     (-D.astype(np.float64) * (np.float32(1) - W) + B).astype(np.float32))
    plain = np.where(small, A + (W * D).astype(np.float32), B - (D * (np.float32(1) - W)).astype(np.float32)).astype(np.float32)
    print(f"lerp: FMA form mismatches {int((got != fused).sum())}/{n}, unfused form mismatches {int((got != plain).sum())}/{n}")
    # (5) 0-row rand
    torch.cuda.manual_seed(7)
    s0 = torch.cuda.get_rng_state()
    torch.rand((0,), device=dev)
    s1 = torch.cuda.get_rng_state()
    x = torch.rand(4, device=dev)
    torch.cuda.manual_seed(7)
    y = torch.rand(4, device=dev)
    print(f"rand of 0 rows: generator state unchanged {torch.equal(s0, s1)}; next draws equal to a fresh seed {torch.equal(x, y)}")


if __name__ == "__main__":
    main()
