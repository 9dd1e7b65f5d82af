"""The ground segmentation's vertical-structure filter without a GPU: the NumPy restatement (tests/ground_vertical_ref.py) at cell
edges, at the height threshold and on one-row cells, its identity with ground_ref.segment when the filter is off, its results on the
canyon scan and the terrain scene, and the argument checks of the C ABI and of GroundParams."""
import ctypes
import dataclasses

import numpy as np
import pytest

import ground_ref as GR
import ground_vertical_ref as GV
from test_ground_cpu import terrain_scene


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


@pytest.fixture(scope="module")
def params(nl):
    return nl.ground.GroundParams(vertical_cell=0.2, vertical_height=0.3)


def f32(v):
    return np.float32(v)


def below(v):
    return np.nextafter(f32(v), f32(-np.inf))


def above(v):
    return np.nextafter(f32(v), f32(np.inf))


def test_cells_floor_downwards_at_negative_coordinates(params):
    p = dataclasses.replace(params, vertical_cell=0.25)                  # a binary cell width: x = -0.25 is exactly the edge of cell -1
    pts = np.array([[-0.25, -4.0, -1.7], [-0.25, -4.0, -1.2],           # cell (-1, -16), extent 0.5
                    [-0.1, -3.8, -1.7],                                   # (-1, -16) too: -0.4 and -15.2 floor downwards
                    [below(-0.25), -4.0, -1.7],                           # just past the x edge: cell (-2, -16), alone
                    [-0.25, below(-4.0), -1.7],                           # just past the y edge: cell (-1, -17), alone
                    [above(-0.25), -4.0, -1.2],                           # just inside: cell (-1, -16)
                    [0.1, -3.9, -1.0]], np.float32)                       # cell (0, -16): truncation towards zero would join it to row 2
    vert, margin, extent = GV.vertical_flags(pts, p)
    assert vert.tolist() == [True, True, True, False, False, True, False]
    assert extent[0] == pytest.approx(0.5, abs=1e-6) and extent[3] == 0.0 and extent[4] == 0.0 and extent[6] == 0.0
    assert margin[0] == 0.0 and margin[3] < 1e-6 and margin[2] > 0.1


def test_extent_equal_to_the_height_is_not_vertical(params):
    lo, hi = f32(-1.7), f32(-1.4)
    ext = float(hi) - float(lo)                                           # exact in fp64
    pts = np.array([[5.0, 0.05, lo], [5.05, 0.1, hi]], np.float32)
    for h, want in ((ext, False), (np.nextafter(ext, 0.0), True), (np.nextafter(ext, 1.0), False)):
        vert, _, extent = GV.vertical_flags(pts, dataclasses.replace(params, vertical_height=h))
        assert extent[0] == ext and vert.tolist() == [want, want], h
    vert, _, _ = GV.vertical_flags(np.array([[5.0, 0.05, -1.5], [5.05, 0.1, -1.0]], np.float32), dataclasses.replace(params, vertical_height=0.5))
    assert not vert.any()


def test_one_row_cells_and_rows_outside_the_ranges(params):
    rng = np.random.default_rng(4)
    r, th = rng.uniform(3.0, 60.0, 400), rng.permutation(400) * (2 * np.pi / 400)
    lone = np.stack([r * np.cos(th), r * np.sin(th), rng.uniform(-3.0, 3.0, 400)], 1).astype(np.float32)
    p = dataclasses.replace(params, vertical_cell=0.01)
    vert, _, extent = GV.vertical_flags(lone, p)
    assert (extent == 0.0).all() and not vert.any()                       # every row alone in its cell: extent 0
    a, b = GV.segment(lone, p), GR.segment(lone, p)
    assert np.array_equal(a["label"], b["label"]) and np.array_equal(a["cos"], b["cos"])
    # rows inside min_range neither are flagged nor count towards the extent of a cell they share with rows inside the ranges
    p = dataclasses.replace(params, vertical_cell=0.5)
    pts = np.array([[2.6, 0.1, 0.0], [2.6, 0.1, -1.7], [2.75, 0.1, -1.7], [2.8, 0.2, -1.72]], np.float32)
    assert GR.bin_points(pts, p)[0].tolist()[:2] == [-1, -1]
    vert, _, extent = GV.vertical_flags(pts, p)
    assert not vert.any() and np.isnan(extent[:2]).all() and extent[2] == pytest.approx(0.02, abs=1e-6)


def test_off_reproduces_segment_exactly(params):
    pts = terrain_scene(seed=3, n=30_000)[0]
    off = dataclasses.replace(params, vertical_cell=0.0)
    a, b = GV.segment(pts, off), GR.segment(pts, off)
    assert not a["vertical"].any()
    for k in ("label", "cos", "patch", "zone", "ring", "edge_margin", "tie", "counts"):
        assert a[k].tobytes() == b[k].tobytes(), k
    for k, v in b["patches"].items():
        assert np.array_equal(a["patches"][k], v, equal_nan=True), k
    assert (a["patches"]["n_vertical"] == 0).all()


def test_vertical_rows_are_left_out_of_the_fits(params):
    """On the canyon scan the result is ground_ref.segment of the non-vertical rows, with the vertical rows added back as non-ground."""
    import nerfloam_b200 as nl
    pts, _, _ = nl.synthetic.make_scan(n_beams=32, n_az=600)
    r = GV.segment(pts, params)
    v = r["vertical"] == 1
    assert v.any() and (r["label"][v] == 0).all() and (r["cos"][v] == 1.0).all()
    sub = GR.segment(pts[~v], params)
    assert np.array_equal(r["label"][~v], sub["label"]) and np.array_equal(r["cos"][~v], sub["cos"])
    rec = r["patches"]
    assert np.array_equal(rec["n_points"] - rec["n_vertical"], sub["patches"]["n_points"])
    assert rec["n_vertical"].sum() == v.sum() and rec["n_points"].sum() == (r["patch"] >= 0).sum()
    assert r["counts"].tolist() == [int(r["label"].sum()), len(pts) - int(r["label"].sum()), 0, 0]


def test_canyon_scan(nl, params):
    """The canyon scan of synthetic.make_scan (82 720 points) with 0.2 m columns and a 0.3 m height, measured with the restatement:
    ground recall 0.98503 (0.99955 unfiltered), 98.59 % of the true-ground cosines within 0.02 of the analytic |d_z| (85.5 %), the
    largest error 0.0607 (0.138), and 2 wall returns labelled ground (3 088).  38 534 rows are vertical.  The recall lost is the ground
    in cells that touch a wall."""
    pts, cos, _ = nl.synthetic.make_scan()
    r = GV.segment(pts, params)
    true = cos < 1.0
    lab = r["label"] == 1
    assert (lab & true).sum() >= 0.98 * true.sum()
    err = np.abs(r["cos"] - cos)[lab & true]
    assert (err < 0.02).mean() >= 0.98
    assert err.max() < 0.08
    assert (lab & ~true).sum() <= 10
    assert (r["cos"][~lab] == 1.0).all()
    assert r["counts"].tolist() == [lab.sum(), (~lab).sum(), 0, 0]


def test_terrain_scene(params):
    """Road of 4 % grade, 0.12 m kerbs, 1.6 m boxes and a wall (80 749 points, 24 042 of them 0.3 m or more above the surface),
    measured with the restatement: recall 0.98383 (0.9995 unfiltered), none of the high points labelled ground, and none of the
    4 854 ground returns within 0.5 m of a kerb flagged vertical."""
    X, truth, height = terrain_scene()
    r = GV.segment(X, params)
    lab = r["label"] == 1
    recall = (lab & truth).sum() / truth.sum()
    high = height >= 0.3
    assert recall >= 0.98, recall
    assert (lab & high).sum() == 0
    kerb = truth & (np.abs(np.abs(X[:, 1]) - 6.0) < 0.5)
    assert kerb.sum() > 1000 and not r["vertical"][kerb].any()


# ---- argument checks ----------------------------------------------------------------------------------------------------------
def test_params_reject_bad_vertical_settings(nl):
    good = nl.ground.GroundParams()
    assert good.vertical_cell == 0.0 and good.vertical_height == 0.3
    c = good.to_c()
    assert c.vertical_cell == 0.0 and c.vertical_height == 0.3
    dataclasses.replace(good, vertical_height=0.0).to_c()                 # the height is not checked while the filter is off
    for cell in (-0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="vertical_cell"):
            dataclasses.replace(good, vertical_cell=cell).to_c()
    for h in (0.0, -0.3, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="vertical_height"):
            dataclasses.replace(good, vertical_cell=0.2, vertical_height=h).to_c()
    with pytest.raises(ValueError, match="too small"):
        dataclasses.replace(good, vertical_cell=1e-8).to_c()              # 80 m / 1e-8 m > 2^30 cells
    dataclasses.replace(good, vertical_cell=80.0 / 2 ** 30).to_c()


def test_c_abi_rejects_bad_vertical_arguments(nl):
    L = nl._capi.lib()
    err = lambda: L.nl_last_error().decode()
    ws, out, pts, vws = (ctypes.c_void_p(256 * k) for k in (1, 2, 3, 4))    # never dereferenced: every call below fails its checks
    assert L.nl_ground_vertical_workspace_bytes(-1) < 0 and "n must be" in err()
    assert L.nl_ground_vertical_workspace_bytes(0) == 16 * 256
    assert L.nl_ground_vertical_workspace_bytes(1000) == 16 * 2048
    assert L.nl_ground_vertical_workspace_bytes(1024) == 16 * 2048
    assert L.nl_ground_vertical_workspace_bytes(1025) == 16 * 4096

    def params(cell=0.2, height=0.3):
        c = nl.ground.GroundParams().to_c()
        c.vertical_cell, c.vertical_height = cell, height
        return c

    def call(p, **kw):
        a = dict(n=5, pts=pts, stride=3, ws=ws, wsb=1 << 30, vws=vws, vwsb=1 << 30, label=out, cos=out, patch=None, patches=None,
                 vert=out, counts=out)
        a.update(kw)
        return L.nl_ground_segment_vertical(a["n"], a["pts"], a["stride"], p, a["ws"], a["wsb"], a["vws"], a["vwsb"], a["label"], a["cos"],
                                            a["patch"], a["patches"], a["vert"], a["counts"], None)
    for cell in (-0.2, float("nan"), float("inf")):
        assert call(params(cell)) != 0 and "vertical_cell" in err(), cell
    for h in (0.0, -1.0, float("nan"), float("inf")):
        assert call(params(0.2, h)) != 0 and "vertical_height" in err(), h
    assert call(params(1e-8)) != 0 and "too small" in err()
    for k in ("vws", "vert"):
        assert call(params(), **{k: None}) != 0 and "null" in err(), k
    assert call(params(), vwsb=16 * 256 - 1) != 0 and "vertical workspace" in err()
    assert call(params(), vws=ctypes.c_void_p(256 * 4 + 8)) != 0 and "aligned" in err()
    assert call(params(), n=-1) != 0 and "n must be" in err()
    assert call(params(), stride=5) != 0 and "stride" in err()
    # the entry point without the vertical arguments refuses the filter rather than running without it
    rc = L.nl_ground_segment(5, pts, 3, params(), ws, 1 << 30, out, out, None, None, out, None)
    assert rc != 0 and "nl_ground_segment_vertical" in err()
