"""CPU: the request checks of the rasterizer's two calls, gsb_forward and gsb_backward (include/gs_b200.h, "Request checks").  The
table holds fourteen request presets, six forwards and eight backwards: the plain request and one per option or combination of
options a caller uses.  For each refusal a preset's options can express, the call returns the same code, starts gsb_last_error()
with its direction ("forward: " / "backward: "), and refuses before any CUDA call: the requests below hold host buffers where
device memory belongs, and on a machine without a GPU any CUDA call would fail with GSB_ECUDA instead of the expected code."""
import ctypes as C

import pytest

from gs_b200 import lib

EINVAL, ERANGE = -1, -4
_BUF = (C.c_float * 64)()
A = C.addressof(_BUF)


def _scene(P=10):
    s = lib.GsbScene(P=P)
    s.means3D = s.opacities = s.degrees = A
    return s


def _camera(width=16, height=16):
    c = lib.GsbCamera(width=width, height=height)
    c.viewmatrix = c.projmatrix = c.campos = c.background = A
    return c


def _raw(Cn=3):
    return lib.GsbRawParams(A, A if Cn else None, Cn, A, A)


def _p(s):
    return None if s is None else C.pointer(s)


# Option values every refusal starts from: a scene and camera that pass every check up to the scene's own tensors, and each option
# either absent or complete.  A preset lists the options it takes, and the values that make it the request it stands for.
BASE = dict(scene=_scene(), cam=_camera(), R=5, maps=(None, None), aa=0, raw=None, raw_grads=None, stats=(None, None), stats_ws=None,
            fwd_features=None, cam_out=(None, None, None), det_ws=None, features=None, absgrad=None)
FWD_FEATURES = lib.GsbFeatures(4, A, A, None, None)
BWD_FEATURES = lib.GsbFeatures(4, A, None, A, A)


def _forward(a):
    req = lib.GsbForwardRequest(scene=_p(a["scene"]), cam=C.pointer(a["cam"]), out_color=A, radii=A, num_rendered=C.pointer(C.c_int64(0)),
                                out_invdepth=a["maps"][0], out_alpha=a["maps"][1], antialiasing=a["aa"], raw=_p(a["raw"]),
                                touched_pixels=a["stats"][0], transmittance_sum=a["stats"][1], features=_p(a["fwd_features"]))
    if a["stats_ws"] is not None:
        req.deterministic, req.workspace = 1, a["stats_ws"]
    return lib.lib().gsb_forward(C.byref(req))


def _backward(a):
    req = lib.GsbBackwardRequest(scene=_p(a["scene"]), cam=C.pointer(a["cam"]), num_rendered=a["R"], radii=A, geom_blob=A, binning_blob=A,
                                 image_blob=A, dL_dout_color=A, grads=C.pointer(lib.GsbGrads()), dL_dinvdepth=a["maps"][0],
                                 dL_dalpha=a["maps"][1], antialiasing=a["aa"], raw=_p(a["raw"]), raw_grads=_p(a["raw_grads"]),
                                 features=_p(a["features"]), dL_dmeans2D_abs=a["absgrad"])
    req.dL_dviewmatrix, req.dL_dprojmatrix, req.dL_dcampos = a["cam_out"]
    if a["det_ws"] is not None:
        req.deterministic, req.det_workspace = 1, a["det_ws"]
    return lib.lib().gsb_backward(C.byref(req))


# name -> (direction, options the preset takes, its option values)
PRESETS = {
    "forward": (_forward, {"fwd_features"}, {}),
    "forward-statistics": (_forward, {"fwd_features", "stats"}, dict(stats=(A, A))),
    "forward-statistics-deterministic": (_forward, {"fwd_features", "stats"}, dict(stats=(A, A), stats_ws=A)),
    "forward-maps": (_forward, {"fwd_features", "maps"}, dict(maps=(A, A))),
    "forward-antialiased": (_forward, {"fwd_features", "maps"}, dict(aa=1)),
    "forward-raw": (_forward, {"fwd_features", "maps", "raw"}, dict(raw=_raw())),
    "backward": (_backward, {"R"}, {}),
    "backward-maps": (_backward, {"R"}, dict(maps=(A, A))),
    "backward-camera": (_backward, {"R", "cam_out"}, {}),
    "backward-antialiased": (_backward, {"R", "cam_out"}, dict(aa=1)),
    "backward-raw": (_backward, {"R", "cam_out", "raw", "raw_grads"}, dict(raw=_raw(), raw_grads=lib.GsbRawGrads(A, A, A, A))),
    "backward-deterministic": (_backward, {"R", "cam_out", "raw", "raw_grads", "det_ws"}, dict(det_ws=A)),
    "backward-absgrad": (_backward, {"R", "cam_out", "raw", "raw_grads", "det_ws", "absgrad"}, dict(absgrad=A)),
    "backward-features": (_backward, {"R", "cam_out", "raw", "raw_grads", "det_ws", "features"}, {}),
}

# refusal -> (the options it needs, the option values that differ from the preset's, code, message substring)
REFUSALS = {
    "scene_null": (set(), dict(scene=None), EINVAL, b"scene is NULL or P < 0"),
    "P_negative": (set(), dict(scene=_scene(P=-1)), EINVAL, b"scene is NULL or P < 0"),
    "bad_image_size": (set(), dict(cam=_camera(width=0)), EINVAL, b"bad image size 0x16"),
    "one_map_output": ({"maps"}, dict(maps=(A, None)), EINVAL, b"map output"),
    "camera_output_without_workspace": ({"cam_out"}, dict(cam_out=(None, A, None)), EINVAL, b"workspace is NULL"),
    "raw_grads_without_raw": ({"raw_grads"}, dict(raw=None, raw_grads=lib.GsbRawGrads(A, A, A, A)), EINVAL, b"raw_grads given without raw"),
    "raw_C4": ({"raw"}, dict(raw=_raw(Cn=4)), EINVAL, b"C = 4"),
    "num_rendered_negative": ({"R"}, dict(R=-1), EINVAL, b"num_rendered < 0"),
    "num_rendered_2_30_deterministic": ({"det_ws"}, dict(R=1 << 30, det_ws=A), ERANGE, b"2^30"),
    "deterministic_with_features": ({"features"}, dict(det_ws=A, features=BWD_FEATURES), EINVAL, b"no deterministic form"),
    # combinations a request can express and no former entry point could
    "statistics_with_maps": ({"stats"}, dict(maps=(A, A)), EINVAL, b"statistics go without the maps"),
    "statistics_with_antialiasing": ({"stats"}, dict(aa=1), EINVAL, b"statistics go without the maps"),
    "statistics_with_raw": ({"stats"}, dict(raw=_raw()), EINVAL, b"statistics go without the maps"),
    "absgrad_with_features": ({"absgrad"}, dict(features=BWD_FEATURES), EINVAL, b"no feature form"),
    # statistics are both outputs or neither, at any P
    "one_statistics_output": ({"stats"}, dict(stats=(A, None)), EINVAL, b"statistics output pointers missing"),
    "one_statistics_output_P0": ({"stats"}, dict(stats=(None, A), scene=_scene(P=0)), EINVAL, b"statistics output pointers missing"),
    # the feature image of a forward
    "forward_features_F0": ({"fwd_features"}, dict(fwd_features=lib.GsbFeatures(0, A, A, None, None)), EINVAL, b"F = 0"),
    "forward_features_F257": ({"fwd_features"}, dict(fwd_features=lib.GsbFeatures(257, A, A, None, None)), EINVAL, b"F = 257"),
    "forward_features_null": ({"fwd_features"}, dict(fwd_features=lib.GsbFeatures(4, None, A, None, None)), EINVAL,
                              b"features->features is NULL"),
    "forward_features_out_null": ({"fwd_features"}, dict(fwd_features=lib.GsbFeatures(4, A, None, None, None)), EINVAL, b"out is NULL"),
}

CASES = [(refusal, name) for refusal, (needs, _, _, _) in REFUSALS.items() for name, (_, takes, _) in PRESETS.items() if needs <= takes]


def test_fourteen_presets_through_two_calls():
    assert len(PRESETS) == 14
    assert sum(call is _forward for call, _, _ in PRESETS.values()) == 6
    assert [s for s in lib.EXPORTED_SYMBOLS if s.startswith(("gsb_forward", "gsb_backward"))] == ["gsb_forward", "gsb_backward"]


def test_every_refusal_is_expressed_where_expected():
    by_refusal = {}
    for refusal, name in CASES:
        by_refusal.setdefault(refusal, []).append(name)
    assert {r: len(n) for r, n in by_refusal.items()} == {
        "scene_null": 14, "P_negative": 14, "bad_image_size": 14, "one_map_output": 3, "camera_output_without_workspace": 6,
        "raw_grads_without_raw": 4, "raw_C4": 5, "num_rendered_negative": 8, "num_rendered_2_30_deterministic": 3,
        "deterministic_with_features": 1, "statistics_with_maps": 2, "statistics_with_antialiasing": 2, "statistics_with_raw": 2,
        "absgrad_with_features": 1, "one_statistics_output": 2, "one_statistics_output_P0": 2, "forward_features_F0": 6,
        "forward_features_F257": 6, "forward_features_null": 6, "forward_features_out_null": 6}


@pytest.mark.parametrize("refusal, name", CASES, ids=[f"{r}-{n}" for r, n in CASES])
def test_request_is_refused_before_any_cuda_call(refusal, name):
    L = lib.lib()
    _, args, code, msg = REFUSALS[refusal]
    call, _, preset = PRESETS[name]
    a = dict(BASE, **preset)
    a.update(args)
    launches = L.gsb_launch_count()
    assert call(a) == code
    err = L.gsb_last_error()
    assert err.startswith(name.split("-")[0].encode() + b": "), err
    assert msg in err, err
    assert L.gsb_launch_count() == launches
