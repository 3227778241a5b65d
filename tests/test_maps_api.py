"""CPU: argument checks of the map requests (out_invdepth / out_alpha of gsb_forward, dL_dinvdepth / dL_dalpha of gsb_backward) and
the Python layer's refusal of CPU tensors with return_maps; every call below is rejected before the first CUDA call."""
import ctypes as C

import pytest
import torch

import stub_c
from gs_b200 import lib


def test_map_entry_points_reject_bad_scenes():
    L = lib.lib()
    cb = lib.ALLOC_FN(lambda user, n: 0)
    R = C.c_int64(0)
    cam = lib.GsbCamera()
    buf = (C.c_float * 16)()
    m = C.addressof(buf)
    for scene in (None, lib.GsbScene(P=-1)):
        sp = None if scene is None else C.pointer(scene)
        fwd = lib.GsbForwardRequest(scene=sp, cam=C.pointer(cam), geom_alloc=cb, binning_alloc=cb, image_alloc=cb, num_rendered=C.pointer(R),
                                    out_invdepth=m, out_alpha=m)
        st = L.gsb_forward(C.byref(fwd))
        assert st < 0 and len(L.gsb_last_error()) > 0
        st = L.gsb_backward(C.byref(lib.GsbBackwardRequest(scene=sp, cam=C.pointer(cam), dL_dinvdepth=m, dL_dalpha=m)))
        assert st < 0 and len(L.gsb_last_error()) > 0


def test_render_with_maps_refuses_cpu_tensors():
    from gaussian_renderer import render
    with pytest.raises(RuntimeError):
        render(stub_c.camera(16, 16), stub_c.Model(), stub_c.pipe(), torch.zeros(3), return_maps=True)
