"""CPU: argument checks of the map entry points (gsb_forward_maps / gsb_backward_maps) and the Python layer's refusal of CPU
tensors with return_maps; every call below is rejected before the first CUDA call."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch

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


class _CpuModel:
    def __init__(self, P=4):
        self.get_xyz = torch.zeros(P, 3)
        self._opacity = torch.zeros(P, 1)
        self._degrees = torch.zeros(P, 1, dtype=torch.int32)
        self.get_scaling = torch.full((P, 3), 0.1)
        self.get_rotation = torch.tensor([[1.0, 0, 0, 0]]).repeat(P, 1)
        self.get_features = torch.zeros(P, 1, 3)
        self.active_sh_degree = self.max_sh_degree = 0


def test_render_with_maps_refuses_cpu_tensors():
    from gaussian_renderer import render
    cam = SimpleNamespace(FoVx=1.0, FoVy=1.0, image_height=16, image_width=16, world_view_transform=torch.eye(4),
                          full_proj_transform=torch.eye(4), camera_center=torch.zeros(3))
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    with pytest.raises(RuntimeError):
        render(cam, _CpuModel(), pipe, torch.zeros(3), return_maps=True)
