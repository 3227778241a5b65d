"""CPU: the fp64 oracle's anti-aliased backward (antialiasing=True, DESIGN.md §5e) and the AA scenes of tests/backward_edges.py.
  1. the oracle's fp64 AA backward is the float64 autograd of the AA forward (render64.py) at the fp32 forward state (its sigmoid,
     s, q, cov3D, means2D, conic, o^, colours and final T), on a small scene with needles on both sides of the clamp of
     q = det0 / det1: to 1e-12 in dL_dmeans2D / dL_dcolors / dL_dopacity, to 1e-7 (float constants) through the covariance;
  2. every AA scene, and every BE.CASES scene rendered with AA, reaches what it is built for (aa_needles: enough clamped and
     near-clamp needles among those checked in every array), and the oracle's fp32 AA backward leaves culled Gaussians at zero;
  3. a backward that takes s and the clamp decision from a differently associated fp32 q (the one the CUDA preprocess backward
     formed before it reused the forward's arithmetic, without the compiler's contraction) is caught per element on aa_needles;
     restricted to the well-conditioned needles whose s it moves by less than 1e-4, the global 2e-4-of-scale bar (on the arrays
     where the fp32 reference itself meets it) lets it through;
  4. the clamp: adding the dq terms where q_f is clamped, flipping the decision next to the clamp, or dropping the dq terms is
     flagged by what test_gpu_antialias_edges.py checks on aa_needles (backward_edges.compare_aa).
Only the oracle runs here: no GPU."""
import math
import time

import numpy as np
import pytest
import torch

import backward_edges as BE
from render64 import render64
from gs_b200 import synth

F64 = torch.float64
_cache = {}


def _run(name):
    if name not in _cache:
        case = BE.build(name, aa=True)
        t = time.perf_counter()
        o, o64, o32 = BE.oracle(case, aa=True)
        excl = BE.excluded(case, o)
        print("\n[%s, aa] oracle %.2f s; %d visible, %d excluded, %d borderline pixels" % (
            name, time.perf_counter() - t, int((o["radii"] > 0).sum()), int(excl.sum()), int(o["borderline"].sum())))
        _cache[name] = case, o, o64, o32, excl
    return _cache[name]


def _global_ok(o64, got, arrays=BE.ARRAYS):
    return all(np.abs(np.asarray(got[n], np.float64).reshape(-1) - np.asarray(o64[n], np.float64).reshape(-1)).max()
               <= BE.GLOBAL * np.abs(o64[n]).max() for n in arrays if o64[n].size)


# ---- 1. the oracle against autograd -------------------------------------------------------------------------------------------

def _small_needles():
    """48x32: 24 round splats of 1..4 px and 24 needles (thinness 1e-2..1e-4, random rotations) on both sides of the clamp."""
    W, H = 48, 32
    cam = synth.make_camera(W, H)
    g = torch.Generator().manual_seed(6200)
    P = 48
    u = torch.rand(P, 6, generator=g, dtype=torch.float64).numpy()
    px, py = 2 + (W - 4) * u[:, 0], 2 + (H - 4) * u[:, 1]
    depth = 3.0 + 3.0 * u[:, 2]
    sigma = 1.0 + 3.0 * u[:, 3]
    t = np.where(np.arange(P) < 24, 0.5 + 0.5 * u[:, 4], 10.0 ** (-2.0 - 2.0 * u[:, 4]))
    aniso = np.stack([np.ones(P), t, t], 1)
    p = 0.3 + 0.69 * u[:, 5]
    sh = torch.randn(P, 4, 3, generator=g).numpy()
    sh[:, 1:] *= 0.2
    scene = BE.pixel_scene(cam, px, py, depth, sigma, np.log(p / (1 - p)), sh, g, aniso)
    return BE.Case("small_needles", scene, cam, torch.tensor([0.3, 0.2, 0.1]), synth.grad_image(W, H, 6201))


def test_oracle_aa_backward_is_the_autograd_of_the_aa_forward():
    case = _small_needles()
    o, o64, _ = BE.oracle(case, aa=True)
    vis = o["radii"] > 0
    qf = o["aa_q"]
    assert int(vis.sum()) >= 40 and int((vis & (qf <= BE.AA_MIN_RATIO)).sum()) >= 3
    assert int((vis & (qf > BE.AA_MIN_RATIO) & (BE.cancellation(case, o) > 1e3)).sum()) >= 3
    s = case.scene
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(F64)
    leaf = lambda v: v.to(F64).detach().clone().requires_grad_(True)
    x = dict(means=leaf(s.means3D), logit=leaf(s.opacity), view=leaf(case.cam.world_view_transform), proj=leaf(case.cam.full_proj_transform),
             campos=leaf(case.cam.camera_center), scales=leaf(s.scales), rots=leaf(s.rotations), sh=leaf(s.sh), deg=s.degrees)
    tiles = [torch.from_numpy(o["point_list"][int(r0):int(r1)].astype(np.int64)) for r0, r1 in o["ranges"]]
    at = dict(sigmoid=t(o["aa_sigmoid"]), s=t(o["aa_s"]), q=t(o["aa_q"]), cov3D=t(o["cov3D"]), means2D=t(o["means2D"]),
              conic_opacity=t(o["conic_opacity"]), rgb=t(o["rgb"]), final_T=t(o["final_T"]))
    col, _, _, nc, mid, (margin_a, margin_t) = render64(x, case.cam, case.bg, torch.from_numpy(vis), tiles, at=at)
    assert np.array_equal(nc.numpy(), o["n_contrib"].astype(np.int64)), "the restatement took the oracle's decisions"
    assert margin_a > 1e-7 and margin_t > 1e-9, (margin_a, margin_t)
    (col * case.dL.to(F64)).sum().backward()
    ref = dict(dL_dmeans2D=mid["ndc"].grad, dL_dcolors=mid["rgb"].grad, dL_dopacity=x["logit"].grad, dL_dmeans3D=x["means"].grad,
               dL_dsh=x["sh"].grad, dL_dscales=x["scales"].grad, dL_drotations=x["rots"].grad)
    got = dict(o64, dL_dmeans2D=o64["dL_dmeans2D"][:, :2])
    errs = {}
    for k, r in ref.items():
        r = r.numpy().reshape(o64[k].shape[0], -1)
        e = np.abs(np.asarray(got[k]).reshape(r.shape) - r)
        errs[k] = float(e.max() / np.abs(r).max())
    print("\n[oracle vs autograd] max |o64 - autograd| / max |autograd|: " + ", ".join("%s %.2e" % kv for kv in errs.items()))
    # at the same state the two agree to float64 rounding in the screen-space gradients; past the 2D covariance the oracle uses the
    # float constants of the kernels (the 0.3f dilation, the SH coefficients rounded to float), the restatement their float64 values
    for k, e in errs.items():
        assert e <= (1e-12 if k in ("dL_dmeans2D", "dL_dcolors", "dL_dopacity") else 1e-7), (k, e)
    # and the AA terms are what it checks: leaving out the q branch moves the needles' scales far beyond that
    at_no_q = dict(at, q=torch.zeros_like(at["q"]))
    for v in x.values():
        if isinstance(v, torch.Tensor) and v.grad is not None:
            v.grad = None
    col2, _, _, _, _, _ = render64(x, case.cam, case.bg, torch.from_numpy(vis), tiles, at=at_no_q)
    (col2 * case.dL.to(F64)).sum().backward()
    r2 = x["scales"].grad.numpy()
    assert np.abs(r2 - ref["dL_dscales"].numpy()).max() > 1e-2 * np.abs(ref["dL_dscales"].numpy()).max()


# ---- 2. coverage of every AA scene --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", BE.AA_CASES + BE.CASES)
def test_aa_scene_reaches_its_boundary(name):
    case, o, o64, o32, excl = _run(name)
    BE.assert_reaches(case, o, excl)
    # the oracle's fp32 backward through compare_aa: the per-element part holds by construction (its bar is at least 8 E32, E32 =
    # |o32 - o64|), so this pins only the excluded Gaussians' global bar and exact zeros for the culled ones
    failures = BE.compare_aa(name, case, o, o64, o32, o32, ~excl, glob=(excl, BE.EXCLUDED_BAR))
    assert not failures, BE.describe(failures, o, o64, o32, case.W, case.H)


def test_aa_needles_check_the_clamp_and_the_gradient_through_q():
    """What compare_aa checks on aa_needles reaches the clamp: an oracle fp32 backward that (a) adds the dq terms also where q_f <=
    2.5e-5, (b) flips the clamp decision of the needles within 1e-3 of it, or (c) drops the dq terms is flagged in the covariance
    chain of the well-conditioned needles."""
    case, o, o64, o32, excl = _run("aa_needles")
    thr, qf = BE.AA_MIN_RATIO, o["aa_q"]
    up = np.nextafter(thr, np.float32(1))
    near = np.abs(qf / np.float64(thr) - 1.0) <= 1e-3
    mutants = {"clamp ignored": np.where(qf <= thr, up, qf), "clamp flipped near 2.5e-5": np.where(near, np.where(qf > thr, thr, up), qf),
               "no gradient through q": np.zeros_like(qf)}
    well = BE.well_conditioned(case, o)
    for label, q in mutants.items():
        _, _, m32 = BE.oracle(case, fwd=dict(o, aa_q=q.astype(np.float32)), aa=True)
        failures = BE.compare_aa(label, case, o, o64, o32, m32, ~excl)
        rows = np.unique(np.concatenate([f[2] for f in failures])) if failures else np.zeros(0, np.int64)
        assert {"dL_dcov3D", "dL_dscales"} <= {f[0] for f in failures}, label
        assert well[rows].any(), label


# ---- 3. the mismatched s ------------------------------------------------------------------------------------------------------

def _f(v):
    return np.float32(v)


def _q_unfused(case, o):
    """q = det0 / det1 as the preprocess backward formed it from its own products (plain fp32 multiplies and adds, left to right,
    without the forward's fused multiply-add or the undilated determinant's fma): T = W J, TV = T V, ua = TV0 . T0, cb = TV1 . T0,
    uc = TV1 . T1, det1 = (ua + 0.3)(uc + 0.3) - cb^2, q = (ua uc - cb^2) / det1."""
    kw = case.cam_kw()
    v = kw["viewmatrix"].numpy().astype(np.float32).reshape(-1)
    m = case.scene.means3D.numpy().astype(np.float32)
    mx, my, mz = m[:, 0], m[:, 1], m[:, 2]
    tx = v[0] * mx + v[4] * my + v[8] * mz + v[12]
    ty = v[1] * mx + v[5] * my + v[9] * mz + v[13]
    tz = v[2] * mx + v[6] * my + v[10] * mz + v[14]
    tanx, tany = _f(kw["tan_fovx"]), _f(kw["tan_fovy"])
    limx, limy = _f(1.3) * tanx, _f(1.3) * tany
    tx = np.minimum(limx, np.maximum(-limx, tx / tz)) * tz
    ty = np.minimum(limy, np.maximum(-limy, ty / tz)) * tz
    hx, hy = _f(case.W) / (_f(2.0) * tanx), _f(case.H) / (_f(2.0) * tany)
    J00, J02 = hx / tz, -(hx * tx) / (tz * tz)
    J11, J12 = hy / tz, -(hy * ty) / (tz * tz)
    T0 = [v[4 * r] * J00 + v[4 * r + 2] * J02 for r in range(3)]
    T1 = [v[4 * r + 1] * J11 + v[4 * r + 2] * J12 for r in range(3)]
    c = o["cov3D"].astype(np.float32)
    V = [[c[:, 0], c[:, 1], c[:, 2]], [c[:, 1], c[:, 3], c[:, 4]], [c[:, 2], c[:, 4], c[:, 5]]]
    TV0 = [T0[0] * V[k][0] + T0[1] * V[k][1] + T0[2] * V[k][2] for k in range(3)]
    TV1 = [T1[0] * V[k][0] + T1[1] * V[k][1] + T1[2] * V[k][2] for k in range(3)]
    ua = TV0[0] * T0[0] + TV0[1] * T0[1] + TV0[2] * T0[2]
    cb = TV1[0] * T0[0] + TV1[1] * T0[1] + TV1[2] * T0[2]
    uc = TV1[0] * T1[0] + TV1[1] * T1[1] + TV1[2] * T1[2]
    denom = (ua + _f(0.3)) * (uc + _f(0.3)) - cb * cb
    with np.errstate(divide="ignore", invalid="ignore"):
        return ((ua * uc - cb * cb) / denom).astype(np.float32)


def _with_s(o, vis, q, use):
    """The forward state with s and the clamp decision taken from `q` for the Gaussians of `use`: that backward's sigmoid is o^ / s
    (its own s), its clamp decision its own q."""
    s = np.sqrt(np.maximum(BE.AA_MIN_RATIO, q)).astype(np.float32)
    use = use & vis
    bad = dict(o, aa_q=np.where(use, q, o["aa_q"]).astype(np.float32), aa_s=np.where(use, s, o["aa_s"]).astype(np.float32))
    bad["aa_sigmoid"] = np.where(use, o["conic_opacity"][:, 3] / bad["aa_s"], o["aa_sigmoid"]).astype(np.float32)
    return bad


def test_per_element_check_rejects_a_mismatched_s():
    case, o, o64, o32, excl = _run("aa_needles")
    vis = o["radii"] > 0
    q = _q_unfused(case, o)
    s = np.sqrt(np.maximum(BE.AA_MIN_RATIO, q)).astype(np.float32)
    rel = np.abs(s.astype(np.float64) / o["aa_s"] - 1.0)
    flips = int(((q > BE.AA_MIN_RATIO) != (o["aa_q"] > BE.AA_MIN_RATIO))[vis].sum())
    print("\n[mismatched s] |s_unfused / s_f - 1|: median %.2e max %.2e; clamp decisions flipped: %d" % (
        float(np.median(rel[vis])), float(rel[vis].max()), flips))
    # 1. every Gaussian: on the needles the gap reaches 1e-1 of s, and the per-element check flags dL_dopacity and the
    #    covariance chain
    _, _, m32 = BE.oracle(case, fwd=_with_s(o, vis, q, np.ones_like(vis)), aa=True)
    names = {f[0] for f in BE.compare_aa("mismatched s", case, o, o64, o32, m32, ~excl)}
    assert "dL_dopacity" in names and "dL_dscales" in names
    # 2. the global 2e-4-of-scale bar cannot judge this scene in dL_drotations: the fp32 reference arithmetic itself is 2e-3 of the
    #    scale off there.  On the other arrays it passes, and there a mismatched s on only the well-conditioned needles whose s moves
    #    by less than 1e-4 gets through the global bar while the per-element check flags dL_dopacity
    assert not _global_ok(o64, o32, ["dL_drotations"])
    judged = [n for n in BE.ARRAYS if n != "dL_drotations"]
    assert _global_ok(o64, o32, judged)
    mild = BE.well_conditioned(case, o) & (rel < 1e-4) & (rel > 0)
    assert int((mild & ~excl).sum()) >= 10
    _, _, m32 = BE.oracle(case, fwd=_with_s(o, vis, q, mild), aa=True)
    failures = BE.compare_aa("mismatched s, well-conditioned, |ds / s| < 1e-4", case, o, o64, o32, m32, ~excl)
    assert "dL_dopacity" in {f[0] for f in failures}
    assert _global_ok(o64, m32, judged), "the global bar lets it through"
