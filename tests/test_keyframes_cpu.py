"""Keyframe graph without a GPU: the NumPy restatement of the overlap counts (tests/keyframe_ref.py) at voxel boundaries and the grid's
edges, rank_by_overlap, KeyframeGraph's bookkeeping and every window that needs no counts, and the argument checks of the C ABI and
of keyframes.py that run before any device work."""
import ctypes
import random

import numpy as np
import pytest
import torch

import keyframe_ref as KR


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


@pytest.fixture(scope="module")
def kfm(nl):
    return nl.keyframes


IDENTITY = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32)


def test_ref_keys_on_voxel_boundaries():
    vs = 0.25                                                      # exact in binary: k * vs is a boundary
    p = np.array([[0.0, 0.0, 0.0], [0.25, 0.5, 0.75], [2.5, 0.25, 1.0]], np.float32)
    keys, out = KR.voxel_keys(p, IDENTITY, vs, 64)
    assert out == 0
    want = [(0, 0, 0), (1, 2, 3), (10, 1, 4)]
    assert keys.tolist() == [(x << 36) | (y << 18) | z for x, y, z in want]
    below = np.nextafter(p[1:], np.float32(-1))                     # one float32 step under the boundary: the voxel before it
    keys, _ = KR.voxel_keys(below, IDENTITY, vs, 64)
    assert keys.tolist() == [(x << 36) | (y << 18) | z for x, y, z in [(0, 1, 2), (9, 0, 3)]]


def test_ref_keys_outside_the_grid():
    vs, gd = 0.5, 16                                                # the grid covers [0, 8)^3
    p = np.array([[-1e-6, 1, 1], [1, 8.0, 1], [1, 1, 7.999], [np.nan, 1, 1], [1, 1, np.inf], [0, 0, 0]], np.float32)
    keys, out = KR.voxel_keys(p, IDENTITY, vs, gd)
    assert out == 4
    assert keys.tolist() == [(2 << 36) | (2 << 18) | 15, 0]
    Rt = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 2000.0, 2000.0, 2000.0], np.float32)   # translation: the same points, in the grid
    keys, out = KR.voxel_keys(np.array([[-1e-6, 1, 1]], np.float32), Rt, 0.3, 1 << 18)
    assert out == 0 and keys.tolist() == [(6666 << 36) | (6670 << 18) | 6670]


def test_ref_overlap_counts_by_hand():
    a = np.array([[0.1, 0.1, 0.1], [0.2, 0.1, 0.1], [1.1, 0.1, 0.1]], np.float32)   # voxels (0,0,0) twice, (1,0,0)
    b = np.array([[0.4, 0.4, 0.4], [2.5, 0.1, 0.1], [-1, 0, 0]], np.float32)        # (0,0,0), (2,0,0), one outside
    Rt = np.stack([IDENTITY, IDENTITY, IDENTITY])
    r = KR.overlap(a, [b, np.zeros((0, 3), np.float32)], Rt, 1.0, 8)
    assert r["frame_voxels"] == 2
    assert r["shared"].tolist() == [1, 0] and r["kf_voxels"].tolist() == [2, 0] and r["outside"].tolist() == [1, 0]


# ---- rank_by_overlap --------------------------------------------------------------------------------------------------------
def test_rank_by_iou(kfm):
    # IoU = s / (kv + fv - s) with fv = 100: 0.1, 0.5, 10/190, 0.25 -> keyframes 1 and 3, in graph order
    assert kfm.rank_by_overlap([20, 60, 10, 40], [100, 80, 100, 100], 100, 2) == [1, 3]
    assert kfm.rank_by_overlap([20, 60, 10, 40], [100, 80, 100, 100], 100, 3) == [0, 1, 3]
    # a larger shared count is not enough: 50 / (400 + 100 - 50) < 30 / (40 + 100 - 30)
    assert kfm.rank_by_overlap([50, 30], [400, 40], 100, 1) == [1]


def test_rank_ties_go_to_later_keyframes(kfm):
    assert kfm.rank_by_overlap([5, 5, 5, 5], [10, 10, 10, 10], 10, 2) == [2, 3]
    # the same IoU from different counts: 4 / (6 + 10 - 4) = 5 / (10 + 10 - 5) = 1/3, in either order
    assert kfm.rank_by_overlap([4, 5], [6, 10], 10, 1) == [1]
    assert kfm.rank_by_overlap([5, 4], [10, 6], 10, 1) == [1]
    assert kfm.rank_by_overlap([5, 4, 1], [10, 6, 10], 10, 2) == [0, 1]


def test_rank_is_in_graph_order(kfm):
    shared = [1, 9, 3, 7, 5]
    assert kfm.rank_by_overlap(shared, [10] * 5, 10, 3) == [1, 3, 4]
    assert kfm.rank_by_overlap(torch.tensor(shared), torch.tensor([10] * 5), torch.tensor(10), 5) == [0, 1, 2, 3, 4]


def test_rank_with_empty_voxel_sets(kfm):
    # |V_k| = |V_c| = 0: the denominator is 0 and the IoU is taken as 0; the tie goes to the later keyframes
    assert kfm.rank_by_overlap([0, 0, 0], [0, 0, 0], 0, 2) == [1, 2]
    assert kfm.rank_by_overlap([0, 0, 0], [0, 5, 0], 0, 1) == [2]
    assert kfm.rank_by_overlap([0, 3, 0], [0, 5, 7], 4, 1) == [1]


# ---- KeyframeGraph --------------------------------------------------------------------------------------------------------
def _frame(nl, index, x, n=40, spread=5.0, seed=None):
    g = torch.Generator().manual_seed(index if seed is None else seed)
    pts = (torch.rand((n, 3), generator=g) * 2 - 1) * spread
    pose = nl.se3pose.OptimizablePose(torch.tensor([2000.0 + x, 2000.0, 2000.0, 0.0, 0.0, 0.01]))
    return nl.frame.LidarFrame(index, pts, torch.ones(n), pose, new_keyframe=True)


def _graph(nl, kfm, n_kf, window=3):
    kg = kfm.KeyframeGraph(window_size=window, keyframe_gap=1.0, key_distance=10.0, n_rays=4, voxel_size=0.3)
    for i in range(n_kf):
        kg.insert_keyframe(_frame(nl, i, 2.0 * i))
    return kg


def test_insert_keyframe_crops_and_shares_the_pose(nl, kfm):
    kg = kfm.KeyframeGraph(window_size=3, keyframe_gap=1.0, key_distance=2.0, n_rays=4, voxel_size=0.3)
    f = _frame(nl, 7, 0.0, n=200, spread=4.0)
    kf = kg.insert_keyframe(f)
    keep = (f.points.abs() < 2.01).all(dim=1)
    assert torch.equal(kf.points, f.points[keep]) and torch.equal(kf.pointsCos, f.pointsCos[keep])
    assert 0 < kf.points.shape[0] < 200 and kf.index == 7
    assert kf.pose is f.pose                                        # later bundle adjustments move both
    assert kg.current_keyframe is kf and kg.keyframe_graph == [kf]
    with torch.no_grad():
        f.pose.data[0] += 1.0
    assert float(kf.pose.data[0]) == float(f.pose.data[0]) == 2001.0


def test_insert_keyframe_needs_two_batches_of_rays(nl, kfm):
    kg = kfm.KeyframeGraph(window_size=3, keyframe_gap=1.0, key_distance=1.0, n_rays=60, voxel_size=0.3)
    with pytest.raises(ValueError, match="valid_distance"):
        kg.insert_keyframe(_frame(nl, 1, 0.0, n=100, spread=4.0))   # ~ (2.02 / 8)^3 of 100 points survive the crop
    assert kg.keyframe_graph == [] and kg.current_keyframe is None
    kg.n_rays = 4
    kg.key_distance = 4.0
    kg.insert_keyframe(_frame(nl, 1, 0.0, n=100, spread=4.0))
    assert len(kg.keyframe_graph) == 1


def test_needs_keyframe(nl, kfm):
    kg = kfm.KeyframeGraph(window_size=3, keyframe_gap=1.5, key_distance=10.0, n_rays=4, voxel_size=0.3)
    assert kg.needs_keyframe(_frame(nl, 0, 0.0))                    # the first one always
    kg.insert_keyframe(_frame(nl, 0, 0.0))
    assert not kg.needs_keyframe(_frame(nl, 1, 1.5))                # strictly more than the gap
    assert kg.needs_keyframe(_frame(nl, 2, 1.6))
    assert kg.needs_keyframe(_frame(nl, 3, -1.6))


def test_select_previous_and_current(nl, kfm):
    kg = _graph(nl, kfm, 6)
    f = _frame(nl, 99, 12.0)
    assert kg.select_optimize_targets(f, "previous") == kg.keyframe_graph[-3:] + [f]
    assert kg.select_optimize_targets(None, "previous") == kg.keyframe_graph[-3:]
    assert kg.select_optimize_targets(f, "current") == [f]
    with pytest.raises(ValueError, match="track frame"):
        kg.select_optimize_targets(None, "current")


def test_select_random_matches_random_sample(nl, kfm):
    kg = _graph(nl, kfm, 8)
    f = _frame(nl, 99, 12.0)
    random.seed(1234)
    want = random.sample(kg.keyframe_graph, 3)
    random.seed(1234)
    assert kg.select_optimize_targets(f, "random") == want + [f]


@pytest.mark.parametrize("method", ["previous", "random", "overlap"])
def test_small_graph_returns_every_keyframe(nl, kfm, method, monkeypatch):
    monkeypatch.setattr(kfm, "_overlap_counts", lambda *a: pytest.fail("a small graph needs no counts"))
    kg = _graph(nl, kfm, 3)
    f = _frame(nl, 99, 12.0)
    assert kg.select_optimize_targets(f, method) == kg.keyframe_graph + [f]
    assert kg.select_optimize_targets(None, method) == kg.keyframe_graph


def test_tracked_frame_appended_unless_it_is_the_current_keyframe(nl, kfm):
    kg = _graph(nl, kfm, 5)
    assert kg.select_optimize_targets(kg.current_keyframe, "previous") == kg.keyframe_graph[-3:]
    f = _frame(nl, 99, 12.0)
    assert kg.select_optimize_targets(f, "previous")[-1] is f


def test_overlap_window_from_the_counts(nl, kfm, monkeypatch):
    """The 'overlap' window is rank_by_overlap of the counts (here faked on the host), against the tracked frame or, without one, the
    current keyframe."""
    kg = _graph(nl, kfm, 6)
    seen = []

    def fake(ref, keyframes, voxel_size, grid_dim):
        seen.append(ref)
        shared, kv = [9, 1, 8, 2, 3, 7], [10] * 6
        return torch.tensor(shared + kv + [0] * 6 + [10])

    monkeypatch.setattr(kfm, "_overlap_counts", fake)
    f = _frame(nl, 99, 12.0)
    g = kg.keyframe_graph
    assert kg.select_optimize_targets(f, "overlap") == [g[0], g[2], g[5], f]
    assert kg.select_optimize_targets(None, "overlap") == [g[0], g[2], g[5]]
    assert seen == [f, kg.current_keyframe]


def test_unknown_method_raises(nl, kfm):
    kg = _graph(nl, kfm, 2)
    with pytest.raises(ValueError, match="unknown"):
        kg.select_optimize_targets(_frame(nl, 99, 0.0), "nearest")


def test_python_argument_checks(nl, kfm, monkeypatch):
    f = _frame(nl, 1, 0.0)
    for gd in (3, 0, -4, 1 << 19, 2.5):
        with pytest.raises(ValueError, match="grid_dim"):
            kfm.keyframe_overlap(f, [f], 0.3, grid_dim=gd)
        with pytest.raises(ValueError, match="grid_dim"):
            kfm.KeyframeGraph(4, 1.0, 10.0, 4, 0.3, grid_dim=gd)
    for vs in (0.0, -0.3, float("inf"), float("nan")):
        with pytest.raises(ValueError, match="voxel_size"):
            kfm.keyframe_overlap(f, [f], vs)
    monkeypatch.setattr(kfm, "SLOT_BUDGET", 1 << 12)
    assert kfm._table_slots([100, 200]) == 1024 and kfm._table_slots([1000, 1000]) == 4096 and kfm._table_slots([]) == 1024
    assert kfm._table_slots([2048, 2048]) == 4096                   # two passes
    with pytest.raises(ValueError, match="does not fit"):
        kfm._table_slots([10, 2049])


def test_c_abi_rejects_bad_arguments(nl):
    L = nl._capi.lib()
    err = lambda: L.nl_last_error().decode()
    ws, out, rt, pts = (ctypes.c_void_p(256 * k) for k in (1, 2, 3, 4))     # never dereferenced: every call below fails its checks
    cnt = (ctypes.c_int64 * 2)(10, 20)
    call = lambda **kw: L.nl_keyframe_overlap(*[kw.get(k, v) for k, v in (
        ("n", 5), ("fp", pts), ("K", 2), ("kp", pts), ("kn", pts), ("hn", cnt), ("rt", rt), ("vs", 0.3), ("gd", 1 << 18),
        ("slots", 1024), ("ws", ws), ("wsb", 1 << 20), ("out", out), ("st", None))])
    assert call(n=-1) != 0 and "n_frame" in err()
    assert call(K=-1) != 0 and "n_kf" in err()
    for gd in (0, 3, 1 << 19):
        assert call(gd=gd) != 0 and "grid_dim" in err()
    for vs in (0.0, -1.0, float("inf"), float("nan")):
        assert call(vs=vs) != 0 and "voxel_size" in err()
    for slots in (0, 1000, 512, 3 << 10):
        assert call(slots=slots) != 0 and "table_slots" in err()
    for k in ("fp", "kp", "kn", "hn", "rt", "ws", "out"):
        assert call(**{k: None}) != 0 and "null" in err(), k
    assert call(n=0, fp=None, K=0, kp=None, kn=None, hn=None, rt=None) != 0 and "null" in err()     # the matrices are always read
    assert call(hn=(ctypes.c_int64 * 2)(10, -1)) != 0 and "negative" in err()
    assert call(hn=(ctypes.c_int64 * 2)(10, 513)) != 0 and "holds at most 512" in err()
    assert call(wsb=8 * (1024 + 1024) - 1) != 0 and "workspace" in err()
    assert call(ws=ctypes.c_void_p(256 + 8)) != 0 and "aligned" in err()
    assert L.nl_keyframe_overlap_workspace_bytes(-1, 1024) < 0 and "n_frame" in err()
    assert L.nl_keyframe_overlap_workspace_bytes(10, 1000) < 0 and "table_slots" in err()
    assert L.nl_keyframe_overlap_workspace_bytes(10, 1024) == 8 * (1024 + 1024)
    assert L.nl_keyframe_overlap_workspace_bytes(1000, 1 << 12) == 8 * (2048 + 4096)
