"""CPU: the C-ABI shared library loads and exports every symbol include/gs_b200.h declares (no compute calls)."""
import ctypes
import os
import re

from gs_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "gs_b200.h")).read()
    return re.findall(r"GSB_API\s+[\w\s\*]+?\b(gsb_\w+)\s*\(", text)


def test_every_declared_symbol_is_exported():
    L = lib.lib()
    syms = declared_symbols()
    assert len(syms) >= 12
    for s in syms:
        assert getattr(L, s) is not None, s
    assert set(lib.EXPORTED_SYMBOLS) == set(syms)


def test_host_only_entry_points():
    L = lib.lib()
    assert b"sm_90a" in L.gsb_version()
    g1, g2 = L.gsb_geom_bytes(1000), L.gsb_geom_bytes(2000)
    assert 0 < g1 < g2 and g2 - g1 >= 1000 * 104          # rec 48 + rect 8 + clamped 1 + depth bits 4 + accumulator 48, modulo alignment
    assert L.gsb_image_bytes(1920, 1080) >= 1920 * 1080 * 8
    # what the forward requests follows the scene's histogram plan: never above the scene-independent bound, and no table at all
    # once the tile histogram exceeds shared memory (8K image: global-atomics binning)
    assert 1920 * 1080 * 8 <= L.gsb_image_bytes_for(3_000_000, 1920, 1080, 1) <= L.gsb_image_bytes(1920, 1080)
    assert L.gsb_image_bytes_for(1000, 7680, 4320, 0) < 7680 * 4320 * 8 + 40 * (480 * 270) + 4096
    assert L.gsb_binning_bytes(10 ** 6) >= 10 ** 6 * 20
    assert L.gsb_launch_count() >= 0


def test_struct_layouts_match_header():
    # field order / sizes of the ctypes mirrors against the C declarations (x86-64 SysV)
    assert ctypes.sizeof(lib.GsbQuant) == 6 * 8
    assert ctypes.sizeof(lib.GsbCamera) == 4 * 4 + 4 * 8 + 8
    assert ctypes.sizeof(lib.GsbGrads) == 9 * 8 + 8 + 8 and lib.GsbGrads.dL_dmeans2D_view.offset == 9 * 8 + 8
    assert ctypes.sizeof(lib.GsbDebug) == 7 * 8
    assert lib.GsbScene.means3D.offset == 8 and lib.GsbScene.scale_modifier.offset == 8 + 8 * 8
    assert lib.GsbScene.band_count.offset == lib.GsbScene.scale_modifier.offset + 8
    assert ctypes.sizeof(lib.GsbScene) == lib.GsbScene.quant.offset + 8
    assert ctypes.sizeof(lib.GsbForwardRequest) == 22 * 8 and lib.GsbForwardRequest.stream.offset == 21 * 8
    assert ctypes.sizeof(lib.GsbBackwardRequest) == 24 * 8 and lib.GsbBackwardRequest.stream.offset == 23 * 8


def test_sass_is_hopper_only():
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", lib.SO_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out


def test_argument_validation_needs_no_gpu():
    """Error behaviour of the C ABI (the reference throws std::runtime_error / AT_ERROR; here: negative code + gsb_last_error()).
    Every call below is rejected before the first CUDA call, so it runs on the CPU-only box."""
    import ctypes as C
    L = lib.lib()
    scene, cam = lib.GsbScene(), lib.GsbCamera()
    scene.P, scene.M = -1, 0
    cb = lib.ALLOC_FN(lambda user, n: 0)
    R = C.c_int64(0)
    fwd = lib.GsbForwardRequest(scene=C.pointer(scene), cam=C.pointer(cam), geom_alloc=cb, binning_alloc=cb, image_alloc=cb,
                                num_rendered=C.pointer(R))
    st = L.gsb_forward(C.byref(fwd))
    assert st < 0 and len(L.gsb_last_error()) > 0
    st = L.gsb_backward(C.byref(lib.GsbBackwardRequest(scene=C.pointer(scene), cam=C.pointer(cam))))
    assert st < 0
    assert L.gsb_mark_visible(-1, None, None, None, None, None) < 0
    assert L.gsb_mark_visible(5, None, None, None, None, None) < 0
    assert L.gsb_kmeans(None, 10, None, 256, 0.1, 5, 0, None, None, None, None) < 0 and b"kmeans" in L.gsb_last_error()
    assert L.gsb_kmeans(None, -1, None, 256, 0.1, 5, 0, None, None, None, None) < 0
    assert L.gsb_sphere_ellipsoid_intersection(-3, None, None, None, None, None, 4, None, None, None) < 0
    assert L.gsb_min_projected_pixel_size(7, None, 1, None, None, None, None, None, None) < 0
    assert L.gsb_min_redundancy_value(7, None, None, None, 4, None, None) < 0
    assert L.gsb_sh_statistics_update(10, 4, *([None] * 13)) < 0 and b"16" in L.gsb_last_error()      # needs the full SH layout
    assert L.gsb_l1_ssim_forward(None, None, 3, 8, 8, None, None, None) < 0
    assert L.gsb_l1_ssim_backward(None, None, 3, 8, 8, None, 1.0, None, 1.0, None, None, None) < 0
    assert L.gsb_forward(C.byref(lib.GsbForwardRequest(geom_alloc=cb, binning_alloc=cb, image_alloc=cb, num_rendered=C.pointer(R)))) < 0
    # size helpers are monotone and include the per-kind fixed parts
    assert L.gsb_kmeans_workspace_bytes(10 ** 6, 256, 0) > 8 * 10 ** 6
    assert L.gsb_l1_ssim_blocks(3, 1080, 1920) == 3 * 68 * 120


def test_python_layer_refuses_cpu_tensors():
    """There is no CPU / PyTorch fallback: CPU tensors raise instead of silently taking another path."""
    import pytest
    import torch
    from diff_gaussian_rasterization import _C
    z = torch.zeros(4, 3)
    with pytest.raises(RuntimeError):
        _C.rasterize_gaussians(torch.zeros(3), z, torch.empty(0), torch.zeros(4, 1), z, torch.zeros(4, 4), 1.0, torch.empty(0),
                               torch.eye(4), torch.eye(4), 1.0, 1.0, 16, 16, torch.zeros(4, 1, 3), torch.zeros(4, 1, dtype=torch.int32),
                               torch.zeros(3), False, False)
    with pytest.raises(RuntimeError):
        _C.kmeans_cuda(torch.zeros(8, 1), torch.zeros(4), 0.1, 2)
    with pytest.raises(RuntimeError):
        _C.find_minimum_projected_pixel_size(torch.eye(4)[None], torch.eye(4)[None], z, torch.tensor([8]), torch.tensor([8]))
    from utils import loss_utils
    with pytest.raises(RuntimeError):
        loss_utils.l1_loss(torch.zeros(3, 8, 8), torch.zeros(3, 8, 8))
