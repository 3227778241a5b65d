"""Golden records of the REFERENCE'S kNN (oracle/_ref/_refKnn.so, the unmodified simple_knn._C) for tests/test_gpu_knn.py and
tests/test_knn_oracle.py.  Cases: tests/golden/knn_cases.py.

Run on a GPU where the reference modules have been built (oracle/build_ref.py, oracle/build_ref_knn.py):
    python tests/golden/make_golden_knn.py OUT_DIR
then copy OUT_DIR/*.npz into tests/golden/.

    kn1*.npz      the raw outputs as the reference returns them (flat, in its own slot order), plus, per K, the rows with a tie at
                  the K-th distance (from a K+1 search)
    kn_edge*.npz  the same for the edge cases
    kn_red*.npz   the redundancy pipeline's min_redundancy and redundancy, the digest of the per-row-sorted neighbour distances and
                  the rows with boundary ties
    kn_large*.npz per 3 M-point cloud: digests of distCUDA2 and of the per-row-sorted distIndex2 distances (K = 30), seeded sample
                  rows of the per-row-sorted (distance, index) pairs, and the rows with boundary ties
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (HERE, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "reduced-3dgs_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import knn_cases as KC  # noqa: E402
import refsummary as S  # noqa: E402


def _np(t):
    return t.detach().cpu().numpy()


def _knn_arrays(ref, pts, K, prefix):
    d, i = ref.distIndex2(pts, K)
    d1, _ = ref.distIndex2(pts, K + 1)
    return {prefix + "_d": _np(d), prefix + "_i": _np(i), prefix + "_ties": KC.boundary_ties(_np(d1), K)}


def ref_kn1(ref):
    c = KC.KNN_CASES["kn1"]
    pts, q, n = KC.kn1_inputs()
    pts, q, n = pts.cuda(), q.cuda(), n.cuda()
    out = {"d2": _np(ref.distCUDA2(pts))}
    for K in c["ks"]:
        out.update(_knn_arrays(ref, pts, K, f"k{K}"))
    d, i = ref.distIndexQ(pts, q, n, c["q_k"])
    d1, _ = ref.distIndexQ(pts, q, n, c["q_k"] + 1)
    out.update(q_d=_np(d), q_i=_np(i), q_ties=KC.boundary_ties(_np(d1), c["q_k"]))
    return out


def ref_edge(ref):
    out = {}
    for name, pts in KC.edge_inputs().items():
        pts = pts.cuda()
        out[name + "_d2"] = _np(ref.distCUDA2(pts))
        out.update(_knn_arrays(ref, pts, KC.EDGE_K, name))
    return out


def ref_red(ref, refC):
    K = KC.KNN_CASES["kn_red"]["K"]
    c, scene, cams = KC.red_inputs()
    min_red, red, _ = KC.redundancy_pipeline(ref, refC, scene, cams, c["radius_scale"], K)
    xyz = scene.means3D.cuda()
    d, i = ref.distIndex2(xyz, K)
    d1, _ = ref.distIndex2(xyz, K + 1)
    sd, _ = KC.sorted_rows_t(d, i, K)
    ties = KC.boundary_ties(_np(d1), K)
    return {"min_redundancy": _np(min_red), "redundancy": _np(red), "sorted_d": np.str_(S.digest(sd)), "ties": ties,
            "n_ties": np.int64(ties.size)}


def ref_large(ref):
    c = KC.KNN_CASES["kn_large"]
    K = c["K"]
    out = {}
    for name, pts in KC.large_inputs().items():
        pts = pts.cuda()
        P = pts.shape[0]
        out[name + "_d2"] = np.str_(S.digest(ref.distCUDA2(pts)))
        d, i = ref.distIndex2(pts, K)
        sd, si = KC.sorted_rows_t(d, i, K)
        out[name + "_sorted_d"] = np.str_(S.digest(sd))
        rows = torch.as_tensor(S.sample_index(P, c["rows"]), device=pts.device)
        out[name + "_rows_d"], out[name + "_rows_i"] = _np(sd[rows]), _np(si[rows])
        del d, i, sd, si
        d1, _ = ref.distIndex2(pts, K + 1)
        out[name + "_ties"] = KC.boundary_ties(_np(d1), K)
        del d1
        torch.cuda.empty_cache()
        print(f"  {name}: {out[name + '_ties'].size} rows with boundary ties", flush=True)
    return out


def main():
    import build_ref
    import build_ref_knn
    out_dir = sys.argv[1]
    os.makedirs(out_dir, exist_ok=True)
    ref = build_ref_knn.load()
    assert ref is not None, "oracle/_ref/_refKnn.so missing (run oracle/build_ref_knn.py where the reference sources exist)"
    refC = build_ref.load()
    assert refC is not None, "oracle/_ref/_refC.so missing"
    for name, fn in (("kn1", lambda: ref_kn1(ref)), ("kn_edge", lambda: ref_edge(ref)), ("kn_red", lambda: ref_red(ref, refC)),
                     ("kn_large", lambda: ref_large(ref))):
        arrays = fn()
        S.save_parts(os.path.join(out_dir, name), arrays)
        print(name, "written", flush=True)


if __name__ == "__main__":
    main()
