"""Time the drop-in simple_knn._C (gsb_knn) against the unmodified reference (oracle/_ref/_refKnn.so) on the same GPU.

    python tools/bench_knn.py [--sizes 100000,1000000,3000000] [--reps 5] [--ref-reps-3m 1]

Rows: distCUDA2, distIndex2 (K = 30) and distIndexQ (K = 30; a seeded 10 % of the points as queries in random order, half of
the points as candidates) for P in --sizes, on the C3 positions and on the clustered multi-scale cloud of tests/golden/knn_cases.py.  Each time is the median of --reps calls, CUDA events around the public call (after one warm-up call of
every shape); the reference arm runs --ref-reps-3m times at P >= 3 M.  Each row also gives the parity verdict: distCUDA2 bit-equal,
and the per-row-sorted distIndex2 / distIndexQ distances bit-equal.  The card's name and power limit are printed in the same run.  One JSON line
per row.
"""
import argparse
import json
import os
import sys

import torch

import benchkit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("reduced-3dgs_b200", "oracle", os.path.join("tests", "golden")):
    sys.path.insert(0, os.path.join(ROOT, p))
import knn_cases as KC  # noqa: E402


def _time(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000,3000000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-reps-3m", type=int, default=1)
    ap.add_argument("--K", type=int, default=30)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_knn needs a GPU"
    import build_ref_knn
    from simple_knn import _C as ours
    ref = build_ref_knn.load()
    assert ref is not None, "oracle/_ref/_refKnn.so missing: build it with oracle/build_ref_knn.py"
    benchkit.banner()
    K = args.K
    for P in [int(s) for s in args.sizes.split(",")]:
        for name, pts in KC.large_inputs(P).items():
            pts = pts.cuda()
            ref_reps = args.ref_reps_3m if P >= 3_000_000 else args.reps
            o2, r2 = ours.distCUDA2(pts), ref.distCUDA2(pts)          # warm-up of every shape
            od, oi = ours.distIndex2(pts, K)
            rd, ri = ref.distIndex2(pts, K)
            row = {"P": P, "cloud": name, "K": K}
            row["distCUDA2_ours_ms"] = _time(lambda: ours.distCUDA2(pts), args.reps)
            row["distCUDA2_ref_ms"] = _time(lambda: ref.distCUDA2(pts), ref_reps)
            row["distIndex2_ours_ms"] = _time(lambda: ours.distIndex2(pts, K), args.reps)
            row["distIndex2_ref_ms"] = _time(lambda: ref.distIndex2(pts, K), ref_reps)
            g = torch.Generator().manual_seed(P)
            qi = torch.randperm(P, generator=g)[: P // 10].to(torch.int32).cuda()
            ni = torch.randperm(P, generator=g)[: P // 2].to(torch.int32).cuda()
            oq, rq = ours.distIndexQ(pts, qi, ni, K), ref.distIndexQ(pts, qi, ni, K)
            row["distIndexQ_ours_ms"] = _time(lambda: ours.distIndexQ(pts, qi, ni, K), args.reps)
            row["distIndexQ_ref_ms"] = _time(lambda: ref.distIndexQ(pts, qi, ni, K), ref_reps)
            row["distIndexQ_speedup"] = row["distIndexQ_ref_ms"] / row["distIndexQ_ours_ms"]
            row["distIndexQ_sorted_dists_equal"] = bool(torch.equal(KC.sorted_rows_t(oq[0], oq[1], K)[0].view(torch.int32),
                                                                    KC.sorted_rows_t(rq[0], rq[1], K)[0].view(torch.int32)))
            del oq, rq
            row["distCUDA2_speedup"] = row["distCUDA2_ref_ms"] / row["distCUDA2_ours_ms"]
            row["distIndex2_speedup"] = row["distIndex2_ref_ms"] / row["distIndex2_ours_ms"]
            row["distCUDA2_equal"] = bool(torch.equal(o2.view(torch.int32), r2.view(torch.int32)))
            sd_o, _ = KC.sorted_rows_t(od, oi, K)
            sd_r, _ = KC.sorted_rows_t(rd, ri, K)
            row["sorted_dists_equal"] = bool(torch.equal(sd_o.view(torch.int32), sd_r.view(torch.int32)))
            print(json.dumps(row), flush=True)
            del pts, o2, r2, od, oi, rd, ri, sd_o, sd_r
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
