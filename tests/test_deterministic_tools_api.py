"""CPU: the deterministic SH-culling statistics and k-means (a statistics forward request with `deterministic`,
gsb_kmeans with `deterministic`):
exports, workspace sizes, every refused argument (checked before any CUDA call), the `deterministic` keyword of
`_C.calculate_colours_variance` / `_C.kmeans_cuda` against a stub library, and the float32 restatement of the k-means summation
order (oracle/kmeans_det_order.py) on hand-made cases."""
import contextlib
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from gs_b200 import lib

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import kmeans_det_order as kdo  # noqa: E402

NEW_SYMBOLS = ("gsb_statistics_workspace_bytes", "gsb_forward", "gsb_kmeans_workspace_bytes", "gsb_kmeans")


@pytest.fixture
def torch_deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


def test_symbols_are_exported():
    L = lib.lib()
    for sym in NEW_SYMBOLS:
        assert sym in lib.EXPORTED_SYMBOLS
        getattr(L, sym)


def test_workspace_sizes():
    L = lib.lib()
    for P in (0, 1, 1000, 10 ** 6, 3 * 10 ** 6):
        assert L.gsb_statistics_workspace_bytes(P) >= 8 * P
    assert L.gsb_statistics_workspace_bytes(2000) > L.gsb_statistics_workspace_bytes(1000)
    for n, K in ((0, 1), (1, 1), (4095, 256), (4097, 256), (9 * 10 ** 6, 256), (9 * 10 ** 6, 1024)):
        assert L.gsb_kmeans_workspace_bytes(n, K, 1) >= 8 * n
        assert L.gsb_kmeans_workspace_bytes(n, K, 1) >= L.gsb_kmeans_workspace_bytes(n, K, 0)
    assert L.gsb_kmeans_workspace_bytes(2 * 10 ** 6, 256, 1) > L.gsb_kmeans_workspace_bytes(10 ** 6, 256, 1)
    assert L.gsb_kmeans_workspace_bytes(10 ** 6, 1024, 1) > L.gsb_kmeans_workspace_bytes(10 ** 6, 256, 1)


def _stats(L, scene, cam=None, outs=True, ws=None):
    """A deterministic statistics forward; outs=False leaves out transmittance_sum (one statistics output without the other)."""
    buf = (C.c_float * 16)()
    p = C.addressof(buf)
    cam = cam if cam is not None else lib.GsbCamera()
    req = lib.GsbForwardRequest(scene=scene, cam=C.pointer(cam), out_color=p, radii=p, num_rendered=C.pointer(C.c_int64(0)),
                                touched_pixels=p, transmittance_sum=p if outs else None, deterministic=1, workspace=ws)
    return L.gsb_forward(C.byref(req))


def test_statistics_deterministic_rejects_bad_arguments():
    L = lib.lib()
    ws = (C.c_char * 256)()
    for scene in (None, C.pointer(lib.GsbScene(P=-1))):
        assert _stats(L, scene, ws=C.addressof(ws)) == -1 and b"P < 0" in L.gsb_last_error()
    assert _stats(L, C.pointer(lib.GsbScene(P=10)), outs=False, ws=C.addressof(ws)) == -1
    assert b"output pointers missing" in L.gsb_last_error()
    assert _stats(L, C.pointer(lib.GsbScene(P=10))) == -1 and b"workspace is NULL" in L.gsb_last_error()
    # W * H = 2^28 is out of range (the check comes before any memory is touched), just below it goes on to the camera checks
    for W, H in ((1 << 14, 1 << 14), (1 << 28, 1), (1 << 15, 1 << 14)):
        assert _stats(L, C.pointer(lib.GsbScene(P=10)), cam=lib.GsbCamera(width=W, height=H), ws=C.addressof(ws)) == -4
        assert b"2^28" in L.gsb_last_error()
    for scene, wsp in ((lib.GsbScene(P=0), None), (lib.GsbScene(P=0), C.addressof(ws))):
        assert _stats(L, C.pointer(scene), cam=lib.GsbCamera(width=(1 << 14) - 1, height=1 << 14), ws=wsp) == -1
        assert b"camera tensors missing" in L.gsb_last_error()


def _km(L, n=10, K=4, max_it=5, values=True, centers=True, ids=True, out=True, ws=True, ws_off=0):
    buf = (C.c_float * 64)()
    a = C.addressof(buf)
    return L.gsb_kmeans(a if values else None, n, a if centers else None, K, 1e-4, max_it, 1, a if ids else None, a if out else None,
                        (a + ws_off) if ws else None, None)


def test_kmeans_deterministic_rejects_bad_arguments():
    L = lib.lib()
    for kw in (dict(n=-1), dict(K=0), dict(K=-3), dict(max_it=-1)):
        assert _km(L, **kw) == -1 and b"bad sizes" in L.gsb_last_error()
    for kw in (dict(centers=False), dict(out=False), dict(values=False), dict(ids=False), dict(ws=False)):
        assert _km(L, **kw) == -1 and b"NULL argument" in L.gsb_last_error()
    # n == 0 needs no values, ids or workspace: it goes on to the launcher (which refuses K above the maximum before any CUDA call)
    assert _km(L, n=0, K=1025, values=False, ids=False, ws=False) == -1 and b"1..1024" in L.gsb_last_error()
    assert _km(L, ws_off=4) == -1 and b"16-byte aligned" in L.gsb_last_error()
    assert _km(L, n=1 << 30) == -4 and b"2^30" in L.gsb_last_error()
    assert _km(L, K=1025) == -1 and b"1..1024" in L.gsb_last_error()


# ---------------------------------------------------------------------------------------------- plumbing against a stub library
class _StubLib:
    """Records every C-ABI call of _C's colour-variance and k-means wrappers and succeeds without touching memory."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("gsb_"):
            raise AttributeError(name)

        def fn(*args):
            self.calls.append((name, args))
            return 1024 if name.endswith("_bytes") else 0
        return fn


def _canon(args, named):
    """Arguments with pointers to the caller's tensors replaced by their names, ctypes by-reference structs by their bytes with
    pointer fields replaced likewise, and pointers to buffers allocated inside the call by their order of appearance."""
    fresh = {}

    def p(v):
        if v in named:
            return named[v]
        return fresh.setdefault(v, f"fresh{len(fresh)}")

    def field(s, f, t):
        v = getattr(s, f)
        if isinstance(v, C._Pointer):
            return "non-null" if v else None
        if isinstance(v, C._CFuncPtr):
            return "callback"
        return p(v) if t is C.c_void_p and v else v

    out = []
    for a in args:
        if isinstance(a, int) and a > (1 << 16):
            out.append(p(a))
        elif type(a).__name__ == "CArgObject":
            s = a._obj
            if isinstance(s, C.Structure):
                out.append(tuple((f, field(s, f, t)) for f, t in s._fields_ if not isinstance(getattr(s, f), C.Array)))
            else:
                out.append(type(s).__name__)
        elif isinstance(a, C._CFuncPtr):
            out.append("callback")
        else:
            out.append(a)
    return tuple(out)


@contextlib.contextmanager
def _stubbed(monkeypatch):
    from diff_gaussian_rasterization import _C
    stub = _StubLib()
    monkeypatch.setattr(_C._lib, "lib", lambda: stub)
    monkeypatch.setattr(_C._lib, "current_stream", lambda device: 0)
    monkeypatch.setattr(_C, "_device_of", lambda t: torch.device("cpu"))
    monkeypatch.setattr(_C, "on_device", lambda device: contextlib.nullcontext())
    yield _C, stub


def _colour_inputs(P=6, n_cams=2):
    g = torch.Generator().manual_seed(0)
    r = lambda *s: torch.rand(*s, generator=g)
    return dict(cam_positions=r(n_cams, 3), means3D=r(P, 3), opacity=r(P, 1), scales=r(P, 3), rotations=r(P, 4),
                cam_viewmatrices=r(n_cams, 4, 4), cam_projmatrices=r(n_cams, 4, 4), tan_fovxs=torch.full((n_cams,), 0.5),
                tan_fovys=torch.full((n_cams,), 0.4), image_height=torch.full((n_cams,), 24), image_width=torch.full((n_cams,), 32),
                sh=r(P, 16, 3), degrees=torch.full((P, 1), 3, dtype=torch.int32), max_sh_deg=3)


def _colour_calls(monkeypatch, raw=False, **kw):
    """The library calls of calculate_colours_variance, canonicalised; raw=True: the forward requests as the library received them."""
    x = _colour_inputs()
    with _stubbed(monkeypatch) as (_C, stub):
        _C.calculate_colours_variance(*x.values(), **kw)
    if raw:
        return [args[0]._obj for name, args in stub.calls if name == "gsb_forward"]
    named = {t.data_ptr(): k for k, t in x.items() if isinstance(t, torch.Tensor)}
    named.update({x["cam_positions"][i].data_ptr(): f"campos{i}" for i in range(2)})
    named.update({x["cam_viewmatrices"][i].data_ptr(): f"view{i}" for i in range(2)})
    named.update({x["cam_projmatrices"][i].data_ptr(): f"proj{i}" for i in range(2)})
    return [(name, _canon(args, named)) for name, args in stub.calls]


def _deterministic(monkeypatch, **kw):
    """The `deterministic` field of the first statistics forward request of calculate_colours_variance."""
    return _colour_calls(monkeypatch, raw=True, **kw)[0].deterministic


def _kmeans_calls(monkeypatch, **kw):
    g = torch.Generator().manual_seed(1)
    values, centers = torch.rand(100, 1, generator=g), torch.rand(8, generator=g)
    with _stubbed(monkeypatch) as (_C, stub):
        _C.kmeans_cuda(values, centers, 1e-4, 500, **kw)
    named = {values.data_ptr(): "values", centers.data_ptr(): "centers"}
    return [(name, _canon(args, named)) for name, args in stub.calls]


def _names(calls):
    return [n for n, _ in calls]


def _kmeans_run(monkeypatch, **kw):
    """The name of kmeans_cuda's last library call and the `deterministic` argument it passed."""
    name, args = _kmeans_calls(monkeypatch, **kw)[-1]
    return name, args[6]


def test_flag_off_keeps_the_old_calls(monkeypatch, torch_deterministic):
    torch.use_deterministic_algorithms(False)
    col = _colour_calls(monkeypatch)
    assert _names(col) == ["gsb_forward", "gsb_sh_statistics_update"] * 2
    assert col == _colour_calls(monkeypatch, deterministic=False)
    # the statistics forward's request: scene, camera, 3 x (callback, NULL), out_color, radii, &R, touched, tsum, stream 0, and
    # no other option
    fwd = dict(col[0][1][0])
    assert len(col[0][1]) == 1 and fwd["geom_alloc"] == "callback" and fwd["geom_user"] is None and fwd["stream"] is None
    assert all(fwd[k] is not None for k in ("scene", "cam", "out_color", "radii", "num_rendered", "touched_pixels", "transmittance_sum"))
    assert all(not fwd[k] for k in ("debug", "out_invdepth", "out_alpha", "antialiasing", "raw", "deterministic", "workspace", "features"))
    km = _kmeans_calls(monkeypatch)
    assert _names(km) == ["gsb_kmeans_workspace_bytes", "gsb_kmeans"]
    assert km[0][1] == (100, 8, 0)
    assert km[1][1] == ("values", 100, "centers", 8, pytest.approx(1e-4), 500, 0, "fresh0", "fresh1", "fresh2", 0)
    assert km == _kmeans_calls(monkeypatch, deterministic=False)


def test_torch_flag_selects_the_deterministic_paths(monkeypatch, torch_deterministic):
    torch.use_deterministic_algorithms(True)
    col = _colour_calls(monkeypatch)
    assert _names(col) == ["gsb_statistics_workspace_bytes"] + ["gsb_forward", "gsb_sh_statistics_update"] * 2
    assert col[0][1] == (6,)
    torch.use_deterministic_algorithms(False)
    ref = _colour_calls(monkeypatch)
    # the old request plus `deterministic` and ONE workspace, the same for every camera
    for (name, det), (_, old) in zip(col[1::2], ref[0::2]):
        det, old = dict(det[0]), dict(old[0])
        assert det.pop("deterministic") == 1 and det.pop("workspace") is not None
        assert old.pop("deterministic") == 0 and old.pop("workspace") is None and det == old
    torch.use_deterministic_algorithms(True)
    reqs = _colour_calls(monkeypatch, raw=True)
    assert len(reqs) == 2 and reqs[0].workspace and reqs[0].workspace == reqs[1].workspace
    torch.use_deterministic_algorithms(True)
    km = _kmeans_calls(monkeypatch)
    assert _names(km) == ["gsb_kmeans_workspace_bytes", "gsb_kmeans"]
    assert km[0][1] == (100, 8, 1)
    assert km[1][1] == ("values", 100, "centers", 8, pytest.approx(1e-4), 500, 1, "fresh0", "fresh1", "fresh2", 0)


def test_flag_is_read_at_call_time(monkeypatch, torch_deterministic):
    torch.use_deterministic_algorithms(False)
    assert _kmeans_run(monkeypatch) == ("gsb_kmeans", 0)
    torch.use_deterministic_algorithms(True)
    assert _kmeans_run(monkeypatch) == ("gsb_kmeans", 1)
    torch.use_deterministic_algorithms(False)
    assert _deterministic(monkeypatch) == 0


def test_explicit_bool_wins(monkeypatch, torch_deterministic):
    torch.use_deterministic_algorithms(True)
    assert _kmeans_run(monkeypatch, deterministic=False) == ("gsb_kmeans", 0)
    assert _deterministic(monkeypatch, deterministic=False) == 0
    torch.use_deterministic_algorithms(False)
    assert _kmeans_run(monkeypatch, deterministic=True) == ("gsb_kmeans", 1)
    assert _deterministic(monkeypatch, deterministic=True) == 1


def test_keyword_only(monkeypatch):
    x = _colour_inputs()
    with _stubbed(monkeypatch) as (_C, _):
        with pytest.raises(TypeError):
            _C.kmeans_cuda(torch.zeros(4, 1), torch.zeros(2), 1e-4, 5, True)
        with pytest.raises(TypeError):
            _C.calculate_colours_variance(*x.values(), True)


# ---------------------------------------------------------------------------------------------- the k-means restatement
F32 = np.float32


def _naive_sums(sorted_values, ids, K):
    """cluster_sums written out element by element, straight from the definition (slow; small inputs only)."""
    n = len(sorted_values)
    part = {}
    for b in range((n + kdo.BLOCK - 1) // kdo.BLOCK):
        for k in sorted(set(ids[b * kdo.BLOCK:(b + 1) * kdo.BLOCK].tolist())):
            leaves = []
            for t in range(kdo.CHUNKS_PER_BLOCK):
                s = F32(-0.0)
                for p in range(b * kdo.BLOCK + t * kdo.CHUNK, min(n, b * kdo.BLOCK + (t + 1) * kdo.CHUNK)):
                    if ids[p] == k:
                        s = F32(s + sorted_values[p])
                leaves.append(s)
            while len(leaves) > 1:
                leaves = [F32(leaves[i] + leaves[i + 1]) for i in range(0, len(leaves), 2)]
            part[(b, k)] = leaves[0]
    out = np.zeros(K, F32)
    for k in range(K):
        lanes = [F32(-0.0)] * kdo.LANES
        for (b, kk), v in sorted(part.items()):
            if kk == k:
                lanes[b % kdo.LANES] = F32(lanes[b % kdo.LANES] + v)
        while len(lanes) > 1:
            lanes = [F32(lanes[i] + lanes[i + 1]) for i in range(0, len(lanes), 2)]
        out[k] = F32(lanes[0] + F32(0.0))
    return out


def _bits(a):
    return np.asarray(a, F32).view(np.uint32)


def test_sort_key_order():
    v = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1.5, -2.0, 1e-45], F32)
    s = kdo.sort_values(v)
    assert _bits(s[0]) >> 31 == 1 and np.isnan(s[0]) and s[1] == -np.inf and s[2] == -2.0
    assert _bits(s[3]) == _bits(F32(-0.0)) and _bits(s[4]) == 0 and s[-2] == np.inf and np.isnan(s[-1])
    assert _bits(kdo.key_float(kdo.float_key(v))).tolist() == _bits(v).tolist()


def test_assign_ties_and_non_finite():
    c = np.array([1.0, 3.0, 1.0, 2.0, 3.0], F32)             # duplicates: the first index wins
    v = np.array([1.0, 0.0, 2.5, 3.5, 1.5, np.nan, np.inf, -np.inf], F32)
    # 2.5: |2 - 2.5| = |3 - 2.5| -> index 1 (3.0 first) vs 3 (2.0): equal distances, smallest index is 1
    assert kdo.assign(v, c).tolist() == [0, 0, 1, 1, 0, 0, 0, 0]
    assert kdo.assign(np.array([5.0], F32), np.array([7.0], F32)).tolist() == [0]
    # a value whose distance to every centre overflows has no nearest centre either
    assert kdo.assign(np.array([3e38], F32), np.array([-3e38, -2e38], F32)).tolist() == [0]


@pytest.mark.parametrize("case", ["small", "ties", "nonfinite", "k1", "zeros", "multiblock"])
def test_cluster_sums_match_the_definition(case):
    rng = np.random.default_rng(7)
    if case == "small":                                      # n below one chunk
        v, c = rng.normal(size=11).astype(F32), np.array([-1, 0, 1], F32)
    elif case == "ties":
        v, c = rng.normal(size=300).astype(F32), np.array([0.5, -0.5, 0.5, 0.5, -0.5], F32)
    elif case == "nonfinite":
        v = rng.normal(size=700).astype(F32)
        v[::37] = np.nan
        v[5::41] = np.inf
        v[7::43] = -np.inf
        v[9::47] = -np.nan
        c = np.array([0.3, -1.0, 2.0], F32)
    elif case == "k1":
        v, c = rng.normal(size=5000).astype(F32), np.array([0.25], F32)
    elif case == "zeros":
        v = rng.normal(size=6000).astype(F32)
        v[rng.random(6000) < 0.7] = 0.0
        v[:40] = -0.0
        c = np.linspace(-2, 2, 9).astype(F32)
    else:                                                    # runs across block boundaries
        v, c = rng.uniform(-1, 1, size=3 * kdo.BLOCK + 123).astype(F32), np.array([-0.5, 0.0, 0.5], F32)
    sv = kdo.sort_values(v)
    ids = kdo.assign(sv, c)
    got = kdo.cluster_sums(sv, ids, len(c))
    want = _naive_sums(sv, ids, len(c))
    # bit for bit, except that a NaN is any NaN (the device's additions return the canonical one; the centre becomes 0 anyway)
    assert np.isnan(got).tolist() == np.isnan(want).tolist()
    assert _bits(got[~np.isnan(got)]).tolist() == _bits(want[~np.isnan(want)]).tolist()
    finite = np.isfinite(sv)
    for k in range(len(c)):
        m = (ids == k) & finite
        if m.sum() == (ids == k).sum():
            assert got[k] == pytest.approx(float(np.sum(sv[m], dtype=np.float64)), rel=1e-5, abs=1e-4)


def test_cluster_sum_signs():
    # an empty cluster and a cluster of -0 values both end at +0, as the default path's zeroed accumulator
    sv = kdo.sort_values(np.array([-0.0, -0.0, 5.0], F32))
    got = kdo.cluster_sums(sv, np.array([0, 0, 2]), 3)
    assert _bits(got).tolist() == [0, 0, _bits(F32(5.0))]


def test_kmeans_restatement_edges():
    ids, c, it = kdo.kmeans(np.zeros(0, F32), np.array([1.0, 2.0], F32), 1e-4, 500)
    assert ids.shape == (0,) and c.tolist() == [1.0, 2.0] and it == 0
    v = np.array([0.0, 1.0, 10.0, 11.0], F32)
    ids, c, it = kdo.kmeans(v, np.array([0.0, 10.0], F32), 1e-4, 0)
    assert it == 0 and ids.tolist() == [0, 0, 1, 1] and c.tolist() == [0.0, 10.0]
    ids, c, it = kdo.kmeans(v, np.array([0.0, 10.0], F32), 1e-4, 500)
    assert c.tolist() == [0.5, 10.5] and ids.tolist() == [0, 0, 1, 1] and it == 2
    # K = 1, and an empty cluster (its centre becomes 0)
    ids, c, it = kdo.kmeans(v, np.array([3.0], F32), 1e-4, 500)
    assert c.tolist() == [5.5] and ids.tolist() == [0, 0, 0, 0]
    ids, c, it = kdo.kmeans(v, np.array([0.0, 10.0, 100.0], F32), 1e-4, 1)
    assert c.tolist() == [0.5, 10.5, 0.0] and it == 1
