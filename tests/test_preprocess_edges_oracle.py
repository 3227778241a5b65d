"""CPU: the scenes of tests/preprocess_edges.py reach what they are built for on the general camera (fx != fy, rotated about
three axes, off-axis centre, odd non-square image), the float64 restatement of the preprocess backward agrees with the oracle's
fp64 backward, and the comparisons reject planted near-misses that the axis-aligned fx == fy camera cannot see.  Only the oracle
runs here: no GPU."""
import numpy as np
import pytest
import torch

import backward_edges as BE
import preprocess_edges as PE
from gs_b200 import lib

_cache = {}


def _run(name):
    if name not in _cache:
        case = PE.build(name)
        o, o64, o32 = PE.oracle(case)
        _cache[name] = case, o, o64, o32
    return _cache[name]


def _restated(case, o, o64, **plant):
    return PE.restate_chain(case, o["radii"] > 0, o["clamped"], o64["dL_dmeans2D"], o64["dL_dconic"], o64["dL_dcolors"], **plant)


@pytest.mark.parametrize("name", PE.CASES)
def test_scene_reaches_its_edges(name):
    case, o, o64, o32 = _run(name)
    PE.assert_reaches(case, o, o64)
    excl = BE.excluded(case, o)
    vis = o["radii"] > 0
    assert excl[vis].mean() <= BE.EXCLUDED_DEFAULT, excl[vis].mean()
    # the oracle's fp32 backward passes the per-element net of backward_edges (K >= 1)
    _, failures = BE.compare(name, o, o64, o32, o32, ~excl, glob=(excl, BE.EXCLUDED_BAR), verbose=False)
    assert not failures, BE.describe(failures, o, o64, o32, case.W, case.H)


@pytest.mark.parametrize("name", PE.CASES)
def test_restated_chain_agrees_with_the_fp64_oracle(name):
    """The independent float64 chain, fed the oracle's own screen-space gradients, reproduces its fp64 backward within the bar the
    kernels are held to."""
    case, o, o64, _ = _run(name)
    ref = _restated(case, o, o64)
    _, failures = PE.compare_restated(name, o["radii"] > 0, ref, o64)
    assert not failures, [(n, w, r[:5].tolist()) for n, w, r in failures]


@pytest.mark.parametrize("plant, array", [(dict(swap_focal=True), "dL_dcov3D"), (dict(transpose_view=True), "dL_dmeans3D"),
                                          (dict(flip_dRx=True), "dL_dmeans3D"), (dict(drop_sparsity=True), "dL_dsh")])
def test_comparison_rejects_planted_near_misses(plant, array):
    """fx <-> fy swapped, the view matrix's rotation block transposed, the x-derivative of one degree-3 SH term negated, the SH
    sparsity term dropped: each makes the restated chain miss the oracle's own gradients."""
    case, o, o64, _ = _run("sh3")
    ref = _restated(case, o, o64, **plant)
    _, failures = PE.compare_restated(str(plant), o["radii"] > 0, ref, o64)
    assert array in [n for n, _, _ in failures], failures


def test_the_default_camera_hides_what_the_general_one_shows():
    """On synth.make_camera (R = I, fx == fy) the swapped focal lengths and the transposed view matrix change nothing, so only the
    general camera can catch them."""
    case, o, o64, _ = _run("sh3")
    fx, fy = PE.focal(case.cam)
    assert abs(fx / fy - 1.0) > 0.05
    flat = PE.build("sh3")
    flat.cam = PE.synth.make_camera(flat.W, flat.H)
    fo, f64, _ = PE.oracle(flat)
    for plant in (dict(swap_focal=True), dict(transpose_view=True)):
        ref = _restated(flat, fo, f64, **plant)
        _, failures = PE.compare_restated(str(plant) + " on make_camera", fo["radii"] > 0, ref, f64)
        assert not failures, failures


@pytest.mark.parametrize("off", [0, 1, 2, 3])
def test_inputs_are_handed_over_16_byte_aligned(off):
    """A contiguous view `off` floats into its storage reaches the kernels as a 16-byte aligned tensor with the same values (a copy
    only when it is not aligned already): they read rotation and SH rows with 128-bit loads."""
    buf = torch.arange(4 * 37 + off, dtype=torch.float32)
    v = buf[off:].view(37, 4)
    assert v.is_contiguous() and (v.data_ptr() % 16 == 0) == (off == 0)
    for got in (lib.f32(v, v.device), lib.aligned16(v)):
        assert got.data_ptr() % 16 == 0 and torch.equal(got, v)
        assert (got.data_ptr() == v.data_ptr()) == (off == 0)
