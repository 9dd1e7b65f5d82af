"""Reconstruction evaluation without a GPU: the NumPy / SciPy restatement (tests/eval_ref.py) against brute force on small sets, and
the argument checks of nerf-loam_b200/evaluate.py that run before any device work."""
import math

import numpy as np
import pytest
import torch

import eval_ref as ER


@pytest.fixture(scope="module")
def ev():
    import nerfloam_b200 as nl
    return nl.evaluate


@pytest.mark.parametrize("nq,nt,trunc", [(1, 1, 0.5), (50, 1, 10.0), (300, 200, 0.1), (500, 700, 0.05), (200, 50, 100.0)])
def test_oracle_nearest_matches_brute_force(nq, nt, trunc):
    rng = np.random.default_rng(nq * 1000 + nt)
    q = rng.uniform(-1, 1, (nq, 3)).astype(np.float32)
    t = rng.uniform(-1, 1, (nt, 3)).astype(np.float32)
    np.testing.assert_allclose(ER.nearest_distances(q, t, trunc), ER.nearest_brute(q, t, trunc), rtol=0, atol=1e-12)


def test_oracle_down_sample_matches_a_dictionary():
    rng = np.random.default_rng(5)
    p = rng.uniform(0, 1, (3000, 3)).astype(np.float32)
    p[:500] = p[500:1000]                                       # duplicates
    p[1000:1100] = (np.floor(p[1000:1100] / 0.125) * 0.125).astype(np.float32)   # exactly on voxel faces
    res, origin = 0.125, np.zeros(3)
    cells = {}
    for x in p:
        k = tuple(np.floor((x.astype(np.float64) - origin) / res).astype(np.int64))
        cells.setdefault(k, []).append(x.astype(np.float64))
    want = [np.mean(cells[k], 0) for k in sorted(cells)]         # lexicographic (x, y, z) = key order
    got, keys = ER.voxel_down_sample(p, res, origin)
    assert len(got) == len(want) and np.all(np.diff(keys.astype(np.float64)) > 0)
    np.testing.assert_allclose(got, np.array(want), rtol=0, atol=1e-7)
    fast, fkeys = ER.voxel_down_sample_fast(p, res, origin)
    assert np.array_equal(keys, fkeys)
    np.testing.assert_array_max_ulp(fast, got, maxulp=1)
    with pytest.raises(ValueError):
        ER.voxel_down_sample(p - 1.0, res, origin)


def test_oracle_metrics_formulas():
    d_acc, d_comp = np.array([0.0, 0.1, 0.3]), np.array([0.2, 0.2])
    m = ER.metrics(d_acc, d_comp, 0.15)
    assert m["accuracy"] == pytest.approx(0.4 / 3) and m["completeness"] == pytest.approx(0.2)
    assert m["chamfer_l1"] == pytest.approx((0.4 / 3 + 0.2) / 2)
    assert m["chamfer_l2"] == pytest.approx(math.sqrt((0.1 / 3 + 0.04) / 2))
    assert m["precision"] == pytest.approx(200 / 3) and m["recall"] == 0.0
    assert m["fscore"] == 0.0
    assert ER.metrics(np.array([1.0]), np.array([1.0]), 0.5)["fscore"] == 0.0


def test_oracle_crop_pads_by_res():
    gt = np.array([[0, 0, 0], [1, 1, 1]], np.float32)
    s = np.array([[-0.1, 0.5, 0.5], [-0.2, 0.5, 0.5], [1.1, 1.1, 1.1], [0.5, 0.5, 1.3]], np.float32)
    kept, dropped = ER.crop(s, gt, 0.15)
    assert dropped == 2 and len(kept) == 2


V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
F = np.array([[0, 1, 2]], np.int32)
G = np.array([[0.2, 0.2, 0.0]], np.float32)


@pytest.mark.parametrize("kw", [
    dict(verts=V[:, :2]), dict(verts=V.astype(np.int32)), dict(verts=np.zeros((0, 3), np.float32)), dict(verts=[[0, 0, 0]]),
    dict(faces=F[:, :2]), dict(faces=F.astype(np.float32)), dict(faces=np.zeros((0, 3), np.int32)),
    dict(gt=np.zeros((0, 3), np.float32)), dict(gt=G.reshape(-1)), dict(gt=G.astype(np.float16)),
    dict(n_samples=0), dict(n_samples=2.5), dict(n_samples=2**31), dict(res=0.0), dict(res=-1.0), dict(res=float("nan")),
    dict(threshold=0.0), dict(threshold=float("inf")), dict(truncation=-0.5), dict(seed=-1), dict(seed=2**64), dict(seed=1.5),
])
def test_eval_mesh_rejects_bad_arguments_before_device_work(ev, kw):
    args = dict(verts=V, faces=F, gt=G, n_samples=100)
    args.update(kw)
    with pytest.raises(ValueError):
        ev.eval_mesh(args.pop("verts"), args.pop("faces"), args.pop("gt"), **args)


def test_other_entry_points_reject_bad_arguments_before_device_work(ev):
    with pytest.raises(ValueError):
        ev.sample_surface(V, F, -1)
    with pytest.raises(ValueError):
        ev.sample_surface(V, np.zeros((0, 3), np.int64), 10)
    with pytest.raises(ValueError):
        ev.sample_surface(torch.zeros(0, 3), torch.from_numpy(F), 10)
    with pytest.raises(ValueError):
        ev.voxel_down_sample(np.zeros((0, 3), np.float32), 0.1, (0, 0, 0))
    with pytest.raises(ValueError):
        ev.voxel_down_sample(G, 0.1, (0, 0))
    with pytest.raises(ValueError):
        ev.voxel_down_sample(G, 0.1, (0, float("nan"), 0))
    with pytest.raises(ValueError):
        ev.voxel_down_sample(G, 0.0, (0, 0, 0))
    with pytest.raises(ValueError):
        ev.nearest_distances(G, np.zeros((0, 3), np.float32), 1.0)
    with pytest.raises(ValueError):
        ev.nearest_distances(G, G, 0.0)
    with pytest.raises(ValueError):
        ev.nearest_distances(G[:, :2], G, 1.0)
    with pytest.raises(ValueError):
        ev.nearest_distances("not an array", G, 1.0)


def test_search_cell_bounds_the_rings_and_fits_the_key(ev):
    for lo, hi, n, trunc in [((0, 0, 0), (1, 1, 1), 10**6, 0.1), ((0, 0, 0), (100, 100, 0), 10**6, 0.5), ((0, 0, 0), (0, 0, 0), 5, 0.2),
                             ((-1e6, 0, 0), (1e6, 1, 1), 2000, 0.01)]:
        h, ring = ev.search_cell(lo, hi, n, trunc)
        assert h > 0 and 1 <= ring <= ev.MAX_RING and ring * h >= trunc
        assert max(hi[a] - lo[a] for a in range(3)) / h < ev.KEY_DIM - 1
