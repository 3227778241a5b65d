"""CPU: argument checks of the map entry points (gsb_forward_maps / gsb_backward_maps) and the Python layer's refusal of CPU
tensors with return_maps; every call below is rejected before the first CUDA call."""
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
    for scene in (None, lib.GsbScene(P=-1)):
        sp = None if scene is None else C.byref(scene)
        st = L.gsb_forward_maps(sp, C.byref(cam), cb, None, cb, None, cb, None, None, None, C.byref(R), None, None, None, None)
        assert st < 0 and len(L.gsb_last_error()) > 0
        st = L.gsb_backward_maps(sp, C.byref(cam), 0, None, None, None, None, None, None, None, None, 0.0, None)
        assert st < 0 and len(L.gsb_last_error()) > 0
    # a valid scene without the map outputs
    scene = lib.GsbScene(P=0)
    st = L.gsb_forward_maps(C.byref(scene), C.byref(cam), cb, None, cb, None, cb, None, None, None, C.byref(R), None, None, None, None)
    assert st < 0 and b"map" in L.gsb_last_error()


def test_render_with_maps_refuses_cpu_tensors():
    from gaussian_renderer import render
    with pytest.raises(RuntimeError):
        render(stub_c.camera(16, 16), stub_c.Model(), stub_c.pipe(), torch.zeros(3), return_maps=True)
