"""GPU: the per-Gaussian preprocess, forward (gsb_preprocess.cu) and backward (preprocess_backward_kernel, gsb_backward.cu), on
the general camera of tests/preprocess_edges.py (fx = 1.08 fy, rotated about three axes, off-axis centre, 333x197), with the
production SH layout M = 16 (degree 3, a partial last warp), mixed and lower degrees in M = 16 with junk in the inactive bands,
scale_modifier = 0.7, precomputed covariances and colours, the quantised scene and the raw-parameter call.  Three references:
  1. the oracle's forward: integers, depth bits, means2D, cov3D, rgb, clamped and conic[:3] exactly, n_contrib off the
     borderline pixels, colour within 1e-4;
  2. the oracle's fp64 backward, element by element (backward_edges.compare: max(8 E32, 1e-4 |o64|_row, 1e-6 max|o64|), the
     excluded Gaussians at 1e-3 of the array's scale and per element on a second backward with dL = 0 on the borderline pixels);
  3. preprocess_edges.restate_chain, float64 autograd of restate64 fed the kernel's own screen-space gradients:
     |ours - chain| <= max(1e-5 |chain|_row, 1e-6 max|chain|) for dL_dsh, dL_dmeans3D, dL_dcov3D, dL_dscales, dL_drotations.
     The render backward's error drops out, so this bar is 10x tighter than (2)'s relative one.
The SH direction term of dL_dmeans3D is checked on its own: two deterministic backwards, one with SH and one with
colors_precomp = the first forward's rgb (same image, same render-backward bits), differ by that term alone, which must match
float64 autograd of the SH colour within 2 ulp of the total + 1e-5 of the term's row.  The camera gradients on the general camera
are held to camera_chain's 1e-5 bar.  SH, rotations and scales given as contiguous views 1, 2 and 3 floats into their storage give
the aligned call's bytes, forward and backward: the kernels read rotation and SH rows with 128-bit loads, so the Python layer hands
over 16-byte aligned inputs (lib.aligned16), and the backward writes an accumulate_into dL_dsh at any offset (its float4 write-back
only where that tensor is aligned), which is checked too, as are the raw parameters.
Observed on one H100 80GB HBM3 (700 W power limit; pytest -s prints the ratios, as max e / bar):
  - (2): at most 0.18 of the bar in every case and array (precomp dL_dopacity, 0.177; mod dL_dsh on the masked pass, 0.175);
  - (3): at most 0.26 over two runs (mod dL_dscales 0.254 and 0.185, raw dL_drotations 0.214, raw dL_dscales 0.187; dL_dsh
    <= 0.032, dL_dmeans3D <= 0.029, dL_dcov3D <= 0.15);
  - the SH direction term: at most 0.245 (mixed_unsorted), with 366 / 270 / 145 / 79 Gaussians whose term is >= 10 % of their
    dL_dmeans3D row in sh3 / mod / mixed_unsorted / sh2_in_16;
  - the camera chain: 3.9e-8 of sum |c_i| (bar 1e-5).
The file takes ~15 s.
"""
import math

import numpy as np
import pytest
import torch

import backward_edges as BE
import camera_chain
import ours
import preprocess_edges as PE
from diff_gaussian_rasterization import _C

pytestmark = pytest.mark.gpu
DEV = "cuda"
EMPTY = torch.Tensor([])
_cache = {}


def _case(name):
    """The case with its device-side activations (the quantised scene de-quantised and the raw one activated on the GPU, as the
    kernels do) and the oracle on it."""
    if name not in _cache:
        case = PE.build(name)
        if name == "quant":
            d = case.meta["quant"].to(DEV).dequantise()
            case.scene = PE.synth.Scene(*[getattr(d, f).cpu() for f in ("means3D", "opacity", "scales", "rotations", "sh", "degrees")])
        if name == "raw":
            PE.activate_raw(case, DEV)
        _cache[name] = (case,) + PE.oracle(case)
    return _cache[name]


def _args(case, colors=None, raw=None):
    """Positional arguments of rasterize_gaussians for the case, and its keywords (quant / raw)."""
    s = case.scene
    pre = case.meta.get("precomp")
    extra = {"cov3D_precomp": pre[0], "colors_precomp": pre[1]} if pre is not None else {}
    if colors is not None:
        extra["colors_precomp"] = colors
    args = list(ours.forward_args(s, case.cam, case.bg, extra))
    args[6] = case.mod
    kw = {}
    if "quant" in case.meta:
        kw["quant"] = case.meta["quant"].to(DEV)
    if "raw" in case.meta:
        args[4] = args[5] = args[14] = EMPTY
        kw["raw"] = raw if raw is not None else tuple(t.to(DEV) for t in case.meta["raw"])
    return args, kw


def _forward(case, args, kw):
    dbg = {}
    out = _C.rasterize_gaussians(*args, debug_out=dbg, **kw)
    st = _C.export_state(out[3], out[4], out[5], out[0], case.W, case.H, P=case.scene.P)
    torch.cuda.synchronize()
    return out, dbg, st


def _backward(case, args, kw, out, dL=None, **extra):
    """The backward as a dict of device tensors named as the oracle's (the raw call's SH gradient concatenated)."""
    (bg, means3D, colors, _, scales, rotations, mod, cov, view, proj, tx, ty, H, W, sh, degrees, campos, _, _) = args
    R, _, radii, geom, binning, img = out[:6]
    dL = case.dL if dL is None else dL
    g = _C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, mod, cov, view, proj, tx, ty, dL.to(DEV), sh,
                                        degrees, campos, geom, R, binning, img, case.lam, False, want_conic=True, **kw, **extra)
    torch.cuda.synchronize()
    if "raw" in kw:
        res = dict(zip(["dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D"], g[:5]))
        res["dL_dsh"] = torch.cat([g[5], g[6]], 1) if g[5] is not None else None
        res.update(dL_dscales=g[7], dL_drotations=g[8], dL_dconic=g[9])
        rest = g[10:]
    else:
        res = dict(zip(BE.ARRAYS, g[:9]))
        rest = g[9:]
    return res, rest


def _np(g):
    return {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in g.items()}


# ---- 1. forward against the oracle -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", PE.CASES)
def test_forward_against_oracle(name):
    case, o, _, _ = _case(name)
    PE.assert_reaches(case, o)
    args, kw = _args(case)
    out, dbg, st = _forward(case, args, kw)
    assert int(out[0]) == int(o["num_rendered"])
    assert np.array_equal(out[2].cpu().numpy(), o["radii"])
    vis = o["radii"] > 0
    assert np.array_equal(dbg["depths"].cpu().numpy()[vis].view(np.uint32), o["depths"][vis].view(np.uint32))
    for k in ("keys", "point_list", "ranges"):
        assert np.array_equal(st[k].cpu().numpy().astype(np.int64).reshape(-1), np.asarray(o[k]).astype(np.int64).reshape(-1)), k
    for k in ("means2D", "cov3D", "rgb"):
        assert np.array_equal(dbg[k].cpu().numpy()[vis], np.asarray(o[k], np.float32)[vis]), k
    assert np.array_equal(dbg["clamped"].cpu().numpy()[vis].astype(bool), o["clamped"][vis].astype(bool))
    assert np.array_equal(dbg["conic_opacity"].cpu().numpy()[vis, :3], o["conic_opacity"][vis, :3])
    nb = ~o["borderline"]
    assert np.array_equal(st["n_contrib"].cpu().numpy()[nb], o["n_contrib"][nb].astype(np.int32)), "n_contrib"
    assert np.abs(out[1].cpu().numpy() - o["color"]).max() <= 1e-4


# ---- 2. backward against the oracle's fp64 backward --------------------------------------------------------------------------

def _oracle_arrays(case):
    skip = {"dL_dcolors", "dL_dcov3D"} if "raw" in case.meta else set()
    return [n for n in BE.ARRAYS if n not in skip]


@pytest.mark.parametrize("name", PE.CASES)
def test_backward_per_element_against_fp64_oracle(name):
    case, o, o64, o32 = _case(name)
    excl = BE.excluded(case, o)
    args, kw = _args(case)
    out, _, _ = _forward(case, args, kw)
    got = _np(_backward(case, args, kw, out)[0])
    arrays = _oracle_arrays(case)
    _, failures = BE.compare(name, o, o64, o32, got, ~excl, glob=(excl, BE.EXCLUDED_BAR), arrays=arrays)
    assert not failures, "\n" + BE.describe(failures, o, o64, got, case.W, case.H)
    if excl.any():
        dL = case.dL.clone()
        dL[:, torch.from_numpy(o["borderline"])] = 0.0
        _, m64, m32 = PE.oracle(case, dL=dL)
        mgot = _np(_backward(case, args, kw, out, dL=dL)[0])
        _, failures = BE.compare(name + ", borderline dL = 0", o, m64, m32, mgot, np.ones_like(excl), arrays=arrays)
        assert not failures, "\n" + BE.describe(failures, o, m64, mgot, case.W, case.H)
    if case.meta.get("precomp") is None:
        # the inactive bands (junk in mixed_unsorted) and culled rows carry exactly zero
        deg = case.scene.degrees.view(-1).numpy()
        inactive = np.arange(16)[None, :] >= ((deg + 1) ** 2)[:, None]
        assert not got["dL_dsh"][inactive].any()


# ---- 3. backward against the float64 restatement, fed the kernel's own screen-space gradients --------------------------------

def _screen(case, args, kw, out, deterministic=False):
    """(backward dict, dL_dcolors) of one backward; the raw call returns no dL_dcolors, so it comes from the activated call's
    deterministic backward on the same (device-activated) scene, whose render backward is the raw one's bit for bit."""
    got, _ = _backward(case, args, kw, out, deterministic=deterministic)
    g_col = got["dL_dcolors"]
    if "raw" in case.meta:
        a2 = list(args)
        s = case.scene
        a2[4], a2[5], a2[14] = s.scales.to(DEV), s.rotations.to(DEV), s.sh.to(DEV)
        out2, _, _ = _forward(case, a2, {})
        g_col = _backward(case, a2, {}, out2, deterministic=True)[0]["dL_dcolors"]
    return _np(got), g_col.cpu().numpy()


@pytest.mark.parametrize("name", PE.CASES)
def test_backward_against_restated_chain(name):
    case, o, _, _ = _case(name)
    args, kw = _args(case)
    out, dbg, _ = _forward(case, args, kw)
    got, g_col = _screen(case, args, kw, out, deterministic="raw" in case.meta)
    vis = out[2].cpu().numpy() > 0
    ref = PE.restate_chain(case, vis, dbg["clamped"].cpu().numpy(), got["dL_dmeans2D"], got["dL_dconic"], g_col)
    _, failures = PE.compare_restated(name, vis, ref, got)
    assert not failures, [(n, w, r[:8].tolist()) for n, w, r in failures]


@pytest.mark.parametrize("name", ["sh3", "mixed_unsorted", "mod", "sh2_in_16"])
def test_sh_direction_term_of_dmeans3D(name):
    case, _, _, _ = _case(name)
    args, kw = _args(case)
    out, dbg, _ = _forward(case, args, kw)
    with_sh, _ = _backward(case, args, kw, out, deterministic=True)
    args_c, _ = _args(case, colors=dbg["rgb"].cpu())
    out_c, dbg_c, _ = _forward(case, args_c, kw)
    assert torch.equal(out_c[1], out[1]), "colors_precomp = rgb renders the same image"
    no_sh, _ = _backward(case, args_c, kw, out_c, deterministic=True)
    assert torch.equal(no_sh["dL_dmeans2D"], with_sh["dL_dmeans2D"]) and torch.equal(no_sh["dL_dconic"], with_sh["dL_dconic"])
    tot = with_sh["dL_dmeans3D"].cpu().numpy()
    diff = tot.astype(np.float64) - no_sh["dL_dmeans3D"].cpu().numpy().astype(np.float64)
    vis = out[2].cpu().numpy() > 0
    term = PE.sh_direction_term(case, vis, dbg["clamped"].cpu().numpy(), with_sh["dL_dcolors"].cpu().numpy())
    bar = PE.DIR_ULP * np.spacing(np.abs(tot)).astype(np.float64) + PE.DIR_REL * np.abs(term).max(axis=1, keepdims=True)
    e = np.abs(diff - term)
    q = e / np.maximum(bar, 1e-38)
    share = np.abs(term).max(axis=1) / np.maximum(np.abs(tot).max(axis=1), 1e-30)
    print("\n[%s] SH direction term: max e / (%g ulp + %g |term|_row) = %.3g; %d Gaussians with a share >= %g" % (
        name, PE.DIR_ULP, PE.DIR_REL, float(q[vis].max()), int((vis & (share >= PE.MIN_DIR_SHARE)).sum()), PE.MIN_DIR_SHARE))
    assert (e <= bar)[vis].all(), np.nonzero(~(e <= bar).all(axis=1) & vis)[0][:8]


def test_camera_grads_on_the_general_camera():
    case, _, _, _ = _case("sh3")
    args, kw = _args(case)
    out, dbg, _ = _forward(case, args, kw)
    got, cam_g = _backward(case, args, kw, out, camera_grads=True)
    cam = case.cam
    per = camera_chain.chain(cam.world_view_transform, cam.full_proj_transform, cam.camera_center, case.W, case.H,
                             math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), case.scene.means3D, dbg["cov3D"], case.scene.sh,
                             case.scene.degrees, dbg["clamped"], out[2] > 0, got["dL_dmeans2D"], got["dL_dconic"], got["dL_dcolors"])
    camera_chain.check(cam_g, per, 1e-5, "general camera, sh3")


# ---- 16-byte loads of the caller's tensors at any float offset -----------------------------------------------------------------

def _offset(t, off):
    """A contiguous copy of `t` that starts `off` floats into its storage."""
    buf = torch.zeros(t.numel() + off, dtype=t.dtype, device=DEV)
    v = buf[off:off + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 == 4 * off
    return v


def _same_forward(a, b):
    (oa, da, sa), (ob, db, sb) = a, b
    assert oa[0] == ob[0]
    for i in (1, 2):
        assert ours.same(oa[i], ob[i]), i
    for k in da:
        assert ours.same(da[k], db[k]), k
    for k in ("keys", "point_list", "ranges", "n_contrib", "final_T"):
        assert ours.same(sa[k], sb[k]), k


@pytest.mark.parametrize("off", [1, 2, 3])
def test_offset_views_give_the_aligned_bytes(off):
    case, _, _, _ = _case("sh3")
    args, kw = _args(case)
    args = [a.to(DEV) if torch.is_tensor(a) else a for a in args]
    shifted = list(args)
    for i in (4, 5, 14):                                       # scales, rotations, sh
        shifted[i] = _offset(args[i], off)
    fa, fb = _forward(case, args, kw), _forward(case, shifted, kw)
    _same_forward(fa, fb)
    ga, _ = _backward(case, args, kw, fa[0], deterministic=True)
    gb, _ = _backward(case, shifted, kw, fb[0], deterministic=True)
    for k in ga:
        assert ours.same(ga[k], gb[k]), k
    # view-batch accumulation into offset views of a previous call's outputs
    first = [ga[n] for n in BE.GRAD_NAMES]
    acc_a = tuple(t.clone() for t in first)
    acc_b = tuple(_offset(t, off) for t in first)
    _backward(case, args, kw, fa[0], deterministic=True, accumulate_into=acc_a)
    _backward(case, shifted, kw, fb[0], deterministic=True, accumulate_into=acc_b)
    for n, x, y in zip(BE.GRAD_NAMES, acc_a, acc_b):
        assert torch.equal(x, y), n
    assert not torch.equal(acc_a[5], first[5])


@pytest.mark.parametrize("off", [1, 3])
def test_offset_raw_parameters_give_the_aligned_bytes(off):
    case, _, _, _ = _case("raw")
    raw = tuple(t.to(DEV) for t in case.meta["raw"])
    args, kw = _args(case, raw=raw)
    args_b, kw_b = _args(case, raw=tuple(_offset(t, off) for t in raw))
    fa, fb = _forward(case, args, kw), _forward(case, args_b, kw_b)
    _same_forward(fa, fb)
    ga, _ = _backward(case, args, kw, fa[0], deterministic=True)
    gb, _ = _backward(case, args_b, kw_b, fb[0], deterministic=True)
    for k in ga:
        assert (ga[k] is None and gb[k] is None) or ours.same(ga[k], gb[k]), k
