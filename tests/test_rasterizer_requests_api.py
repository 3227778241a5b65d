"""CPU: the request checks of the rasterizer's fourteen request entry points (six forwards, eight backwards; include/gs_b200.h,
"Request checks").  For each refusal an entry point's arguments can express, every such entry point returns the same code, names
itself at the start of gsb_last_error() (the camera and scene checks, the same for every entry point of a direction, name the
direction instead), and refuses before any CUDA call: the calls below pass host buffers where device memory belongs, and on a
machine without a GPU any CUDA call would fail with GSB_ECUDA instead of the expected code."""
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


# Arguments every refusal starts from: a scene and camera that pass every check up to the scene's own tensors, and each option
# either absent or complete.  `takes` below lists the options an entry point has; ENTRY_BASE what it needs to be complete.
BASE = dict(scene=_scene(), cam=_camera(), R=5, maps=(None, None), cam_out=(None, None, None), raw=None, raw_grads=None, det_ws=None,
            features=None)
ENTRY_BASE = {
    "gsb_forward_maps": dict(maps=(A, A)),
    "gsb_forward_raw": dict(raw=_raw()),
    "gsb_backward_raw": dict(raw=_raw(), raw_grads=lib.GsbRawGrads(A, A, A, A)),
    "gsb_backward_deterministic": dict(det_ws=A),
}


def _p(s):
    return None if s is None else C.byref(s)


def _fwd(a, *tail):
    return (_p(a["scene"]), C.byref(a["cam"]), lib.ALLOC_FN(0), None, lib.ALLOC_FN(0), None, lib.ALLOC_FN(0), None, A, A,
            C.byref(C.c_int64(0))) + tail


def _bwd(a, *tail):
    return (_p(a["scene"]), C.byref(a["cam"]), a["R"], A, A, A, A, A, C.byref(lib.GsbGrads())) + tail


def _cam_tail(a):
    return (A, A, 0.0, *a["cam_out"], None)


def _raw_tail(a):
    return _cam_tail(a) + (_p(a["raw"]), _p(a["raw_grads"]), 0)


# name -> (options the entry point takes, its argument list)
ENTRIES = {
    "gsb_forward": (set(), lambda a: _fwd(a, None, None)),
    "gsb_forward_statistics": (set(), lambda a: _fwd(a, A, A, None)),
    "gsb_forward_statistics_deterministic": (set(), lambda a: _fwd(a, A, A, A, None)),
    "gsb_forward_maps": ({"maps"}, lambda a: _fwd(a, None, *a["maps"], None)),
    "gsb_forward_antialiased": ({"maps"}, lambda a: _fwd(a, None, *a["maps"], None)),
    "gsb_forward_raw": ({"maps", "raw"}, lambda a: _fwd(a, None, *a["maps"], _p(a["raw"]), 0, None)),
    "gsb_backward": ({"R"}, lambda a: _bwd(a, 0.0, None)),
    "gsb_backward_maps": ({"R"}, lambda a: _bwd(a, A, A, 0.0, None)),
    "gsb_backward_camera": ({"R", "cam_out"}, lambda a: _bwd(a, *_cam_tail(a), None)),
    "gsb_backward_antialiased": ({"R", "cam_out"}, lambda a: _bwd(a, *_cam_tail(a), None)),
    "gsb_backward_raw": ({"R", "cam_out", "raw", "raw_grads"}, lambda a: _bwd(a, *_raw_tail(a), None)),
    "gsb_backward_deterministic": ({"R", "cam_out", "raw", "raw_grads", "det_ws"}, lambda a: _bwd(a, *_raw_tail(a), a["det_ws"], None)),
    "gsb_backward_absgrad": ({"R", "cam_out", "raw", "raw_grads", "det_ws"}, lambda a: _bwd(a, *_raw_tail(a), a["det_ws"], A, None)),
    "gsb_backward_features": ({"R", "cam_out", "raw", "raw_grads", "det_ws", "features"},
                              lambda a: _bwd(a, *_raw_tail(a), a["det_ws"], _p(a["features"]), None)),
}

# refusal -> (the options it needs, the arguments that differ from the entry point's complete call, code, message substring)
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
    "deterministic_with_features": ({"features"}, dict(det_ws=A, features=lib.GsbFeatures(4, A, None, A, A)), EINVAL,
                                    b"no deterministic form"),
}
# refusals whose message names the direction ("forward request" / "backward request") rather than the entry point
BY_DIRECTION = {"bad_image_size"}
# gsb_backward_raw cannot go without raw: its own requirement comes first
MESSAGE = {("raw_grads_without_raw", "gsb_backward_raw"): b"raw parameters are NULL"}

CASES = [(refusal, name) for refusal, (needs, _, _, _) in REFUSALS.items() for name, (takes, _) in ENTRIES.items() if needs <= takes]


def test_the_fourteen_entry_points_are_exported():
    assert len(ENTRIES) == 14
    for name in ENTRIES:
        assert name in lib.EXPORTED_SYMBOLS


def test_every_refusal_is_expressed_where_expected():
    by_refusal = {}
    for refusal, name in CASES:
        by_refusal.setdefault(refusal, []).append(name)
    assert {r: len(n) for r, n in by_refusal.items()} == {
        "scene_null": 14, "P_negative": 14, "bad_image_size": 14, "one_map_output": 3, "camera_output_without_workspace": 6,
        "raw_grads_without_raw": 4, "raw_C4": 5, "num_rendered_negative": 8, "num_rendered_2_30_deterministic": 3,
        "deterministic_with_features": 1}


@pytest.mark.parametrize("refusal, name", CASES, ids=[f"{r}-{n}" for r, n in CASES])
def test_request_is_refused_before_any_cuda_call(refusal, name):
    L = lib.lib()
    _, args, code, msg = REFUSALS[refusal]
    a = dict(BASE, **ENTRY_BASE.get(name, {}))
    a.update(args)
    launches = L.gsb_launch_count()
    assert getattr(L, name)(*ENTRIES[name][1](a)) == code
    err = L.gsb_last_error()
    prefix = f"{name.split('_')[1]} request" if refusal in BY_DIRECTION else name[len("gsb_"):]
    assert err.startswith(prefix.encode() + b": "), err
    assert MESSAGE.get((refusal, name), msg) in err, err
    assert L.gsb_launch_count() == launches

