"""GPU: the inverse-depth / alpha maps' backward (render_backward_kernel<MAPS = true, *, *> and the MAPS branch of the preprocess
backward) and the feature channels' backward (features_backward_kernel<CH>) against the fp64 oracle, element by element, on the
boundary scenes of tests/backward_edges.py.  The oracle side is the exact composition of the colour oracle of
tests/maps_features64.py.
  - maps: BE.CASES + BE.AA_CASES, deterministic False and True, maps alone (colour dL = 0, so the maps' terms are the whole row)
    and maps + colour; camera gradients with maps on four scenes (camera_chain with the dinvd / tz term); the absolute screen-space
    gradient with maps (render_backward_kernel<true, *, true>) against absgrad64.pair_sums;
  - features: F in {1, 8, 9, 16, 17, 67, 256} (CH = 8 single chunk, CH = 16 single chunk, several chunks), features alone and
    features + colour, every gradient array and dL_dfeatures; on `large` F = 17 only; CH = 8 with several chunks
    (GSB_FEATURES_CH=8, read once per process) in one subprocess;
  - everything at once: colour + maps + F = 17 features + camera gradients, anti-aliased, on odd_17x15, staircase and aa_needles
    (one accumulator record per Gaussian holds all of it).
Integers (radii, keys, point_list, ranges, n_contrib off borderline pixels) are asserted equal to the oracle's first.  The bar is
backward_edges.compare's (max(8 E32, 1e-4 |o64|_row, 1e-6 max|o64|), BE.BAR_CASE for dense_faint, BE.excluded Gaussians at
BE.EXCLUDED_BAR of the array's scale), every check is followed by a second pass with the colour, map and feature gradients zeroed
on the borderline pixels, which holds every Gaussian per element, and culled rows must be exactly zero.  pytest -s prints, per
case and array, max e / max(E32, 1e-4 |o64|_row, 1e-6 max|o64|) and max e / bar.
Feature upstream gradients are of full rank up to F = 17 on staircase, odd_17x15 and saturation (ceil(F / 3) oracle backwards:
a channel-mixing bug cannot hide in a rank-3 structure there) and of rank 3 (maps_features64.rank3: one oracle backward)
elsewhere and for F > 17."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import absgrad64
import backward_edges as BE
import maps_features64 as MF
import ours
from camera_chain import chain, check
from diff_gaussian_rasterization import _C

pytestmark = pytest.mark.gpu

ALL = BE.CASES + BE.AA_CASES
FEATURE_F = [1, 8, 9, 16, 17, 67, 256]
LARGE_F = [17]                              # `large`: one oracle backward costs seconds on the CPU
FULL_RANK_MAX = 17
FULL_RANK_CASES = {"staircase", "odd_17x15", "saturation"}
CAMERA_CASES = ["staircase", "odd_17x15", "saturation", "large"]
ALL_AT_ONCE = ["odd_17x15", "staircase", "aa_needles"]
CH8_NODES = ["staircase-17", "odd_17x15-67", "saturation-256"]
MAP_SEED, FEAT_SEED, GRAD_SEED = 41, 43, 47
# Per-case bars (R_REL, A_ABS) beyond BE.BAR_CASE, observed on one H100 80GB HBM3 at 700 W:
# - staircase / staircase_ties, maps: the invdepth channel's colour 1/z varies little along a tile's list of faint Gaussians, so
#   dL/dalpha = dL_dinvdepth (T 1/z_i - S_i / (1 - alpha_i)) cancels, and the kernel's T (recovered back to front with MUFU.RCP
#   over up to 1 000 entries) carries that cancellation into dL_dscales / dL_drotations: up to 1.2e-4 / 1.4e-4 of the row with
#   the maps alone (1.16 / 1.40 of the default bar); with a colour loss, whose channels do not cancel, 0.58 of it.
# - aa_needles, features: on needles dL_dscales and dL_drotations are ill-conditioned in fp32 (see BE.AA_WELL_CONDITIONED): under a
#   feature loss the dL_drotations of needle 146 (a c / det0 < 1e2) is 5.2e-4 of its row off with F = 1 (the fp32 reference's own
#   error there is 1e-4 of it: 1.26 of the default bar 8 E32, the same on two runs), and dL_dscales of the needles with
#   a c / det0 >= 1e2 reaches 2.0e-4 of the row (1.97 of the default bar, F = 256 + colour).
# - aa_needles, camera: the same needles' terms make up 1.8e-4 of sum |c_i| (bar 2e-4) in the view gradient, whose kernel side
#   moves with the atomic order; held to 4e-4.
# - large, maps + colour and features + colour: the dL_dopacity of a 35..200 px Gaussian sums ~1e5 signed pixel terms whose total
#   cancels; adding the maps' or the features' terms to the colour's raises their absolute sum, not the total: Gaussian 20023 came
#   out 1.4e-4 of its (one-element) row off with maps + colour (1.16 of the default bar, default and deterministic alike), 0.92 of
#   it with F = 17 + colour.
MAPS_BAR_CASE = {"staircase": (3e-4, 1e-6), "staircase_ties": (3e-4, 1e-6), "large": (3e-4, 1e-6)}
CAMERA_BAR_CASE = {"aa_needles": 4e-4}
FEATURES_BAR_CASE = {"aa_needles": (1e-3, 1e-6), "large": (3e-4, 1e-6)}

_states = {}


class _State:
    pass


def _state(name, aa=False):
    """Oracle forward, colour backward (and its borderline-masked twin), excluded Gaussians and our forward of a case, checked for
    equal integers; cached across the tests of this file."""
    key = (name, aa or name in BE.AA_CASES)
    if key in _states:
        return _states[key]
    s = _State()
    s.case = case = BE.build(name, aa=aa)
    s.aa = aa = case.meta["aa"]
    t0 = time.perf_counter()
    s.o, c64, c32 = BE.oracle(case, aa=aa)
    s.colour = (c64, c32)
    s.excl = BE.excluded(case, s.o)
    BE.assert_reaches(case, s.o, s.excl)
    s.border = s.o["borderline"]
    s.dL_masked = None
    if s.excl.any():
        s.dL_masked = case.dL.clone()
        s.dL_masked[:, torch.from_numpy(s.border)] = 0.0
        s.colour_masked = BE.oracle(case, dL=s.dL_masked, fwd=s.o, aa=aa)[1:]
    s.oracle_s = time.perf_counter() - t0
    s.args, s.out, fwd = ours.run_forward(case.scene, case.cam, case.bg, aa=aa)
    o = s.o
    assert int(fwd["num_rendered"]) == int(o["num_rendered"])
    for k in ("radii", "keys", "point_list", "ranges"):
        assert np.array_equal(np.asarray(o[k]).reshape(-1), fwd[k].reshape(-1)), k
    assert np.array_equal(o["n_contrib"][~s.border], fwd["n_contrib"][~s.border]), "n_contrib"
    s.fwd = fwd
    s.bar = BE.BAR_CASE.get(name, (BE.R_REL, BE.A_ABS))
    _states[key] = s
    return s


def _check(s, label, pair, got, every=False, arrays=BE.ARRAYS, bar=None):
    """backward_edges.compare (compare_aa when anti-aliased) of `got` against the composition `pair` = (o64, o32): the excluded
    Gaussians to the global bar, or with `every` (a borderline-masked pass) every Gaussian per element.  -> a description of the
    failures ("" if none), so that one run prints every case's ratios."""
    o, (o64, o32) = s.o, pair
    chk = np.ones_like(s.excl) if every else ~s.excl
    glob = None if every else (s.excl, BE.EXCLUDED_BAR)
    bar = bar or s.bar
    if s.aa:
        failures = BE.compare_aa(label, s.case, o, o64, o32, got, chk, glob, bar=bar, arrays=arrays)
    else:
        _, failures = BE.compare(label, o, o64, o32, got, chk, glob, bar=bar, arrays=arrays)
    return "" if not failures else "\n[%s]\n%s" % (label, BE.describe(failures, o, o64, got, s.case.W, s.case.H))


def _zero_dL(s):
    return torch.zeros(3, s.case.H, s.case.W)


def _label(s, what):
    return "%s%s, %s" % (s.case.name, ", aa" if s.aa else "", what)


# ---- maps -----------------------------------------------------------------------------------------------------------------------

def _maps(s):
    """The maps' upstream gradients of a case, their borderline-masked twins and the maps-only compositions of both (cached)."""
    if not hasattr(s, "maps"):
        case = s.case
        Gd, Ga = MF.map_gradients(case.W, case.H, MAP_SEED)
        s.maps = (Gd, Ga), MF.compose(case, s.o, maps=(Gd, Ga), aa=s.aa)
        s.maps_masked = None
        if s.dL_masked is not None:
            Gdm, Gam = MF.masked(Gd, s.border), MF.masked(Ga, s.border)
            s.maps_masked = (Gdm, Gam), MF.compose(case, s.o, maps=(Gdm, Gam), aa=s.aa)
    return s.maps, s.maps_masked


@pytest.mark.parametrize("name", ALL)
def test_maps_backward_per_element_against_fp64_oracle(name):
    s = _state(name)
    case = s.case
    t0 = time.perf_counter()
    ((Gd, Ga), maps), mm = _maps(s)
    (Gdm, Gam), masked = mm if mm is not None else ((None, None), None)
    t1 = time.perf_counter()
    runs = [("maps", maps, _zero_dL(s), 0.0, masked, _zero_dL(s))]
    runs.append(("maps + colour", MF.with_colour(maps, s.colour), case.dL, case.lam,
                 None if masked is None else MF.with_colour(masked, s.colour_masked), s.dL_masked))
    bar = MAPS_BAR_CASE.get(name)
    failed = ""
    for det in (False, True):
        for what, pair, dL, lam, mpair, mdL in runs:
            label = _label(s, what + (", deterministic" if det else ""))
            got = ours.run_backward(s.args, s.out, dL, lam, aa=s.aa, deterministic=det, dL_dinvdepth=Gd, dL_dalpha=Ga)
            failed += _check(s, label, pair, got, bar=bar)
            if mpair is not None:
                got = ours.run_backward(s.args, s.out, mdL, lam, aa=s.aa, deterministic=det, dL_dinvdepth=Gdm, dL_dalpha=Gam)
                failed += _check(s, label + ", borderline dL = 0", mpair, got, every=True, bar=bar)
    assert not failed, failed
    print("[%s] oracle %.2f s (colour %.2f s), total %.2f s" % (_label(s, "maps"), t1 - t0 + s.oracle_s, s.oracle_s,
                                                                time.perf_counter() - t0))


@pytest.mark.parametrize("name", CAMERA_CASES)
def test_camera_grads_with_maps_against_the_chain_of_the_fp64_oracle(name):
    s = _state(name)
    case = s.case
    ((Gd, Ga), maps), _ = _maps(s)
    m64, _ = MF.with_colour(maps, s.colour)
    got = ours.run_backward(s.args, s.out, case.dL, case.lam, dL_dinvdepth=Gd, dL_dalpha=Ga, camera_grads=True)
    kw = case.cam_kw()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    sc = case.scene
    per = chain(case.cam.world_view_transform, case.cam.full_proj_transform, case.cam.camera_center, case.W, case.H, kw["tan_fovx"],
                kw["tan_fovy"], sc.means3D, t(s.o["cov3D"]), sc.sh, sc.degrees, t(s.o["clamped"]), t(s.o["radii"] > 0).cuda(),
                t(m64["dL_dmeans2D"]), t(m64["dL_dconic"]), t(s.colour[0]["dL_dcolors"]), g_invd=t(m64["dinvd"]))
    check([torch.from_numpy(got[k]).cuda() for k in ("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos")], per, 2e-4, name + ", maps + colour")


@pytest.mark.parametrize("name", ALL)
def test_absgrad_with_maps_against_float64_per_gaussian(name):
    """render_backward_kernel<true, *, true>: the absolute screen-space gradient with the maps' gradients, against absgrad64's
    restatement with dL_dinvdepth / dL_dalpha (pinned to the maps composition by test_maps_features_edges_oracle.py), with
    test_gpu_absgrad's bar."""
    s = _state(name)
    case = s.case
    (Gd, Ga), _ = _maps(s)[0]
    _, abs64 = absgrad64.pair_sums(s.fwd, case.bg.numpy(), case.dL.numpy(), case.W, case.H, dL_dinvdepth=Gd, dL_dalpha=Ga)
    (bg, means3D, colors, opacity, scales, rotations, mod, cov, view, proj, tx, ty, H, W, sh, degrees, campos, _, _) = s.args
    R, color, radii, geom, binning, img = s.out
    dmap = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).view(1, H, W).cuda()
    rel, a_abs = s.bar
    vis = s.fwd["radii"] > 0
    chk = vis & ~s.excl
    for det in (False, True):
        ab = torch.full((case.scene.P, 3), float("nan"), device="cuda")
        _C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, mod, cov, view, proj, tx, ty, case.dL.cuda(), sh,
                                        degrees, campos, geom, R, binning, img, case.lam, False, antialiasing=s.aa, deterministic=det,
                                        dL_dinvdepth=dmap(Gd), dL_dalpha=dmap(Ga), absgrad_out=ab)
        got = ab.cpu().double().numpy()
        assert (got[:, 2] == 0).all() and (got[~vis] == 0).all()
        got = got[:, :2]
        err = np.abs(got - abs64).max(axis=1)
        bar = np.maximum(rel * np.abs(abs64).max(axis=1), a_abs * np.abs(abs64).max())
        worst = float((err[chk] / np.maximum(bar[chk], 1e-30)).max()) if chk.any() else 0.0
        print(f"\n[{_label(s, 'absgrad with maps')} det={det}] {int(chk.sum())} Gaussians per element, worst err / bar {worst:.3f}")
        assert (err[chk] <= bar[chk]).all(), (name, det, worst)
        if (s.excl & vis).any():
            assert err[s.excl & vis].max() <= BE.EXCLUDED_BAR * np.abs(abs64).max(), name


# ---- features -------------------------------------------------------------------------------------------------------------------

def _feature_inputs(s, F):
    """-> (features [P, F], G [F, H, W] for the kernel, G for the oracle (G itself, or (A, h) of rank 3), its masked twins)."""
    case = s.case
    feat = np.random.default_rng(FEAT_SEED + F).standard_normal((case.scene.P, F)).astype(np.float32)
    if s.case.name not in FULL_RANK_CASES or F > FULL_RANK_MAX:
        A, h, G = MF.rank3(F, case.H, case.W, GRAD_SEED + F)
        return feat, G, (A, h), MF.masked(G, s.border), (A, MF.masked(h, s.border))
    G = MF.full_rank(F, case.H, case.W, GRAD_SEED + F)
    Gm = MF.masked(G, s.border)
    return feat, G, G, Gm, Gm


def _features_cases():
    return [pytest.param(n, F, id="%s-%d" % (n, F)) for n in ALL for F in (LARGE_F if n == "large" else FEATURE_F)]


@pytest.mark.parametrize("name, F", _features_cases())
def test_features_backward_per_element_against_fp64_oracle(name, F):
    s = _state(name)
    case = s.case
    t0 = time.perf_counter()
    feat, G, Go, Gm, Gom = _feature_inputs(s, F)
    fo = MF.compose(case, s.o, features=(feat, Go), aa=s.aa)
    masked = MF.compose(case, s.o, features=(feat, Gom), aa=s.aa) if s.dL_masked is not None else None
    t1 = time.perf_counter()
    arrays = BE.ARRAYS + ["dL_dfeatures"]
    runs = [("F = %d" % F, fo, _zero_dL(s), 0.0, masked, _zero_dL(s)),
            ("F = %d + colour" % F, MF.with_colour(fo, s.colour), case.dL, case.lam,
             None if masked is None else MF.with_colour(masked, s.colour_masked), s.dL_masked)]
    bar = FEATURES_BAR_CASE.get(name)
    failed = ""
    for what, pair, dL, lam, mpair, mdL in runs:
        got = ours.run_backward(s.args, s.out, dL, lam, aa=s.aa, features=feat, dL_dfeatures_out=G)
        failed += _check(s, _label(s, what), pair, got, arrays=arrays, bar=bar)
        if mpair is not None:
            got = ours.run_backward(s.args, s.out, mdL, lam, aa=s.aa, features=feat, dL_dfeatures_out=Gm)
            failed += _check(s, _label(s, what + ", borderline dL = 0"), mpair, got, every=True, arrays=arrays, bar=bar)
    assert not failed, failed
    print("[%s] oracle %.2f s, total %.2f s" % (_label(s, "F = %d" % F), t1 - t0, time.perf_counter() - t0))


def test_features_ch8_with_several_chunks():
    """The 8-channel chunk layout with several chunks (F > 8 under GSB_FEATURES_CH=8, read once per process), in one subprocess."""
    if os.environ.get("GSB_FEATURES_CH"):
        pytest.skip("already in the forced-width process")
    here = os.path.abspath(__file__)
    nodes = ["%s::test_features_backward_per_element_against_fp64_oracle[%s]" % (here, n) for n in CH8_NODES]
    env = dict(os.environ, GSB_FEATURES_CH="8")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "-p", "no:cacheprovider", *nodes], cwd=ours.ROOT, env=env,
                       capture_output=True, text=True, timeout=1800)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stdout[-8000:] + r.stderr[-4000:]
    assert ("%d passed" % len(CH8_NODES)) in r.stdout


# ---- everything at once ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ALL_AT_ONCE)
def test_colour_maps_features_camera_and_aa_at_once(name):
    s = _state(name, aa=True)
    case = s.case
    assert s.aa
    Gd, Ga = MF.map_gradients(case.W, case.H, MAP_SEED)
    feat, G, Go, Gm, Gom = _feature_inputs(s, 17)
    pair = MF.compose(case, s.o, colour=s.colour, maps=(Gd, Ga), features=(feat, Go), aa=True)
    got = ours.run_backward(s.args, s.out, case.dL, case.lam, aa=True, dL_dinvdepth=Gd, dL_dalpha=Ga, features=feat,
                            dL_dfeatures_out=G, camera_grads=True)
    arrays = BE.ARRAYS + ["dL_dfeatures"]
    bar = FEATURES_BAR_CASE.get(name)
    failed = _check(s, _label(s, "colour + maps + F = 17"), pair, got, arrays=arrays, bar=bar)
    if s.dL_masked is not None:
        mpair = MF.compose(case, s.o, colour=s.colour_masked, maps=(MF.masked(Gd, s.border), MF.masked(Ga, s.border)),
                           features=(feat, Gom), aa=True)
        mgot = ours.run_backward(s.args, s.out, s.dL_masked, case.lam, aa=True, dL_dinvdepth=MF.masked(Gd, s.border),
                                 dL_dalpha=MF.masked(Ga, s.border), features=feat, dL_dfeatures_out=Gm)
        failed += _check(s, _label(s, "colour + maps + F = 17, borderline dL = 0"), mpair, mgot, every=True, arrays=arrays, bar=bar)
    assert not failed, failed
    # the camera: o^ = sigmoid * s carries dL/do^ = dL_dopacity / (s sigmoid (1 - sigmoid)) through q = det0 / det1
    o, o64 = s.o, pair[0]
    vis = o["radii"] > 0
    sig, sa = o["aa_sigmoid"].astype(np.float64), o["aa_s"].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        g_ohat = np.where(vis, o64["dL_dopacity"][:, 0] / (sa * sig * (1.0 - sig)), 0.0)
    clamped_q = o["aa_q"] <= BE.AA_MIN_RATIO
    kw = case.cam_kw()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    sc = case.scene
    per = chain(case.cam.world_view_transform, case.cam.full_proj_transform, case.cam.camera_center, case.W, case.H, kw["tan_fovx"],
                kw["tan_fovy"], sc.means3D, t(o["cov3D"]), sc.sh, sc.degrees, t(o["clamped"]), t(vis).cuda(), t(o64["dL_dmeans2D"]),
                t(o64["dL_dconic"]), t(s.colour[0]["dL_dcolors"]), g_invd=t(o64["dinvd"]), aa=(t(g_ohat), t(sig), t(clamped_q)))
    check([torch.from_numpy(got[k]).cuda() for k in ("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos")], per,
          CAMERA_BAR_CASE.get(name, 2e-4), name + ", aa, colour + maps + F = 17")
