"""CPU checks of the mesh-extraction yardstick (tests/mesh_ref.py): emit_ref against the independent restatement oracle/mc.py at
every res, its vertices within the fp64 bar, and the bar against near-miss vertex formulas.  No GPU needed."""
import numpy as np
import pytest

import mesh_ref as MR
from util import ROOT  # noqa: F401

VS = 0.3


@pytest.mark.parametrize("res", range(2, 17))
def test_emit_ref_matches_the_restatement(res):
    rng = np.random.default_rng(100 + res)
    n = 6
    sdf = MR.random_lattices(rng, n, res)
    centres = MR.random_centres(rng, n, VS)
    ref = MR.emit_ref(sdf, centres, VS)
    assert ref["totals"][0] == ref["verts"].shape[0] and ref["totals"][1] == ref["faces"].shape[0]
    assert ref["nvert"][1] == 0 and ref["nvert"][2] == 0 and ref["nvert"][0] > 0     # kinds: crossing, all positive, all negative
    voxels = [0, 1, 3] if res <= 8 else [0, 3]
    MR.check_against_oracle(ref, sdf, centres, VS, voxels)


@pytest.mark.parametrize("res", (2, 3, 8, 16))
def test_emit_ref_within_the_fp64_bar(res):
    rng = np.random.default_rng(7 + res)
    sdf = MR.random_lattices(rng, 12, res)
    centres = MR.random_centres(rng, 12, VS)
    ref = MR.emit_ref(sdf, centres, VS)
    v, bar, ok = MR.vertex_fp64(sdf, centres, VS)
    assert ok.all() and v.shape == ref["verts"].shape
    ratio = MR.fp64_ratio(ref["verts"], sdf, centres, VS)
    assert 0 < ratio <= 1.0, ratio
    # the bar is not loose by orders of magnitude: the worst vertex uses a fair share of it
    assert ratio > 0.05, ratio


def _mutants(sdf, centres, res):
    """Near-miss vertex formulas, each in the layout of emit_ref's vertices."""
    s0, s1, axis, ijk = MR._edges(sdf)
    cross = (s0 < 0) != (s1 < 0)
    vv, ee = np.nonzero(cross)
    a, b, ax, p, c = s0[vv, ee], s1[vv, ee], axis[ee], ijk[ee], centres[vv]
    other = centres[(vv + 1) % len(centres)]
    return {
        "wrong end": MR.vertices_f32(b, a, ax, p, c, res, VS),
        "1/res": MR.vertices_f32(a, b, ax, p, c, res, VS, inv=np.float32(1) / np.float32(res)),
        "axes swapped": MR.vertices_f32(a, b, ax, p, c, res, VS, swap=(0, 2)),
        "wrong voxel": MR.vertices_f32(a, b, ax, p, other, res, VS),
    }


@pytest.mark.parametrize("res", (2, 8, 16))
def test_the_bar_rejects_near_misses(res):
    rng = np.random.default_rng(31 + res)
    sdf = MR.random_lattices(rng, 9, res)
    centres = MR.random_centres(rng, 9, VS)
    for name, got in _mutants(sdf, centres, res).items():
        ratio = MR.fp64_ratio(got, sdf, centres, VS)
        assert ratio > 100, (name, ratio)


def test_edge_values_and_empty_input():
    """emit_ref on NaN / inf / signed-zero / subnormal lattices follows the kernel's rules (NaN and -0 are outside), and on no
    voxels returns empty arrays."""
    sdf = np.ones((3, 2, 2, 2), np.float32)
    sdf[0, 0, 0, 0] = -0.0                        # -0 is not inside: no crossing
    sdf[1, 0, 0, 0] = -1.0
    sdf[1, 1, 0, 0] = np.nan                      # NaN is outside: the edge to it crosses, at a NaN position
    sdf[2, 0, 0, 0] = -1e-45
    sdf[2, 0, 0, 1] = 0.0
    ref = MR.emit_ref(sdf, np.zeros((3, 3), np.float32), VS)
    assert ref["nvert"].tolist() == [0, 3, 3] and ref["ntri"].tolist() == [0, 1, 1]
    v1 = ref["verts"][0:3]
    assert np.isnan(v1[0, 0]) and not np.isnan(v1[0, 1:]).any() and not np.isnan(v1[1:]).any()
    # the subnormal corner: its crossing towards the +0 neighbour (axis 2, the voxel's last vertex) sits on that neighbour (t = 1)
    assert ref["verts"][5, 2] == np.float32(0.5) * np.float32(VS)
    z = MR.emit_ref(np.zeros((0, 4, 4, 4), np.float32), np.zeros((0, 3), np.float32), VS)
    assert z["verts"].shape == (0, 3) and z["faces"].shape == (0, 3) and z["totals"].tolist() == [0, 0]
