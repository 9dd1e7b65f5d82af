"""Keyframe overlap on the GPU (csrc/overlap.cu, nerf-loam_b200/keyframes.py): every count against the NumPy restatement
tests/keyframe_ref.py fed with the matrices nl_pose_matrices produced, the 'overlap' window on a drive that returns to its start, and
that window feeding bundle_adjust_frames' captured graph."""
import numpy as np
import pytest
import torch

import keyframe_ref as KR

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


def _frame(nl, index, pts, pose6):
    pts = torch.as_tensor(np.ascontiguousarray(pts, dtype=np.float32))
    return nl.frame.LidarFrame(index, pts, torch.ones(pts.shape[0]), nl.se3pose.OptimizablePose(torch.tensor(pose6, dtype=torch.float32)),
                               new_keyframe=True)


def _pose6(rng, around=2000.0, spread=3.0):
    return np.r_[around + rng.uniform(-spread, spread, 3), rng.normal(0, 0.2, 3)].astype(np.float32)


def _matrices(nl, frames):
    """[K+1,12] from nl_pose_matrices, read back: the restatement uses the same matrices as the kernel."""
    pose6 = torch.stack([f.pose.data.detach().float() for f in frames]).cuda().contiguous()
    Rt = torch.empty((len(frames), 12), dtype=torch.float32, device="cuda")
    nl._capi.check(nl._capi.lib().nl_pose_matrices(len(frames), nl._capi.ptr(pose6), nl._capi.ptr(Rt), nl._capi.stream_ptr()))
    return Rt.cpu().numpy()


def _check(nl, frame, kfs, vs, gd):
    kfm = nl.keyframes
    got = kfm.keyframe_overlap(frame, kfs, vs, grid_dim=gd)
    again = kfm.keyframe_overlap(frame, kfs, vs, grid_dim=gd)
    for a, b in zip(got, again):
        assert a.is_cuda and a.dtype == torch.int64 and torch.equal(a, b)
    want = KR.overlap(frame.points.numpy(), [k.points.numpy() for k in kfs], _matrices(nl, [frame] + kfs), vs, gd)
    assert got.shared.cpu().tolist() == want["shared"].tolist()
    assert got.kf_voxels.cpu().tolist() == want["kf_voxels"].tolist()
    assert got.outside.cpu().tolist() == want["outside"].tolist()
    assert int(got.frame_voxels) == want["frame_voxels"]
    return got, want


def _cloud(rng, n, spread=20.0):
    return rng.uniform(-spread, spread, (n, 3)).astype(np.float32)


def test_one_keyframe(nl):
    rng = np.random.default_rng(1)
    pts, _, pose = nl.synthetic.make_scan(seed=5)
    f = _frame(nl, 1, pts, nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose)).data.detach().numpy())
    kp, _, kpose = nl.synthetic.make_scan(seed=6, sensor_xyz=(1.5, 0.2, 0.0), yaw=0.05)
    k = _frame(nl, 2, kp, nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(kpose)).data.detach().numpy())
    got, want = _check(nl, f, [k], 0.3, 1 << 18)
    assert 0 < want["shared"][0] < want["kf_voxels"][0] and want["outside"][0] == 0
    _check(nl, _frame(nl, 3, _cloud(rng, 5000), _pose6(rng)), [k], 0.2, 1 << 18)


def test_keyframe_identical_to_the_scan_and_empty_and_duplicated(nl):
    rng = np.random.default_rng(2)
    pts, p6 = _cloud(rng, 30000), _pose6(rng)
    f = _frame(nl, 1, pts, p6)
    same = _frame(nl, 2, pts.copy(), p6)
    empty = _frame(nl, 3, np.zeros((0, 3), np.float32), _pose6(rng))
    dup = _frame(nl, 4, np.repeat(pts[:3000], 7, axis=0)[rng.permutation(21000)], p6)
    dup_sorted = _frame(nl, 5, np.repeat(pts[:3000], 7, axis=0), p6)        # runs of equal points: the warp's repeat test
    got, want = _check(nl, f, [same, empty, dup, dup_sorted], 0.3, 1 << 18)
    s, kv = want["shared"], want["kf_voxels"]
    assert s[0] == kv[0] == want["frame_voxels"] > 0
    assert s[1] == kv[1] == 0 and want["outside"][1] == 0
    assert s[2] == kv[2] == s[3] == kv[3] > 0


def test_points_outside_the_grid(nl):
    rng = np.random.default_rng(3)
    pts = _cloud(rng, 20000, spread=5.0)
    pts[:500, 0] -= 4000.0                                                  # world x < 0
    pts[500:900] = np.nan
    f = _frame(nl, 1, _cloud(rng, 20000, spread=5.0), _pose6(rng))
    k1 = _frame(nl, 2, pts, _pose6(rng))
    k2 = _frame(nl, 3, _cloud(rng, 10000, spread=5.0), _pose6(rng, around=8191 * 0.25))    # straddles the edge of an 8192 grid
    got, want = _check(nl, f, [k1, k2], 0.25, 1 << 13)
    assert want["outside"][0] == 900 and 0 < want["outside"][1] < 10000
    _check(nl, f, [k1, k2], 0.25, 1 << 18)


def test_many_keyframes_in_several_passes(nl, monkeypatch):
    """A lowered slot budget forces several passes over the table; more than NL_OVERLAP_MAX_CHUNK keyframes force a pass boundary
    on the keyframe count too.  Keyframes near the scan share voxels with it, far ones do not."""
    kfm = nl.keyframes
    rng = np.random.default_rng(4)
    base = _pose6(rng)
    f = _frame(nl, 1, _cloud(rng, 8000, spread=4.0), base)
    kfs = []
    for i in range(40):
        p6 = base.copy()
        p6[:3] += rng.uniform(-6, 6, 3) + (30.0 if i % 3 == 0 else 0.0)      # every third one far from the scan
        kfs.append(_frame(nl, 2 + i, _cloud(rng, int(rng.integers(0, 2000)), spread=4.0), p6))
    monkeypatch.setattr(kfm, "SLOT_BUDGET", 1 << 12)                      # <= 2048 points per pass: ~20 passes
    got, want = _check(nl, f, kfs, 0.3, 1 << 18)
    far = np.arange(40) % 3 == 0
    assert (want["shared"][far] == 0).all() and (want["shared"][~far] > 0).sum() > 5
    monkeypatch.setattr(kfm, "SLOT_BUDGET", 1 << 25)
    small = [_frame(nl, 100 + i, _cloud(rng, int(rng.integers(0, 4)), spread=4.0), base) for i in range(1100)]
    _check(nl, f, small, 0.3, 1 << 18)
    monkeypatch.setattr(kfm, "SLOT_BUDGET", 1 << 10)
    with pytest.raises(ValueError, match="does not fit"):
        kfm.keyframe_overlap(f, kfs[:1] + [_frame(nl, 9, _cloud(rng, 600), base)], 0.3)


# ---- the window on a drive that returns to its start ----------------------------------------------------------------------
N_LOOP, SPACING = 21, 1.0                                   # out to x = 10 m and back


def _loop_frame(nl, i, index=None):
    xyz, yaw = nl.synthetic.path_pose(i, N_LOOP, SPACING, "loop")
    pts, cos, pose = nl.synthetic.make_scan(seed=1000 + i, sensor_xyz=xyz, yaw=yaw)
    return nl.frame.LidarFrame(i if index is None else index, torch.from_numpy(pts), torch.from_numpy(cos),
                               nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose)), new_keyframe=True)


def test_revisit_selects_the_keyframes_of_the_same_place(nl):
    kg = nl.keyframes.KeyframeGraph(window_size=4, keyframe_gap=1.5, key_distance=30.0, n_rays=2048, voxel_size=0.3)
    for i in range(0, N_LOOP - 1, 2):                           # keyframes at x = 0, 2, .., 10, 8, .., 2
        kg.insert_keyframe(_loop_frame(nl, i))
    back = _loop_frame(nl, N_LOOP - 1)                          # x = 0 again, fresh noise
    g = kg.keyframe_graph
    ov = nl.keyframes.keyframe_overlap(back, g, 0.3)
    shared, kv, fv = ov.shared.cpu().tolist(), ov.kf_voxels.cpu().tolist(), int(ov.frame_voxels)
    iou = [s / (k + fv - s) for s, k in zip(shared, kv)]
    assert int(np.argmax(iou)) == 0, iou                       # the keyframe taken at the same place ranks first
    overlap = kg.select_optimize_targets(back, "overlap")
    previous = kg.select_optimize_targets(back, "previous")
    assert overlap[-1] is back and previous[-1] is back
    early = {g[0].index, g[1].index}                           # taken on the way out at x = 0 and 2
    assert early <= {f.index for f in overlap[:-1]}
    assert not early & {f.index for f in previous[:-1]}
    assert [f.index for f in overlap[:-1]] == sorted(f.index for f in overlap[:-1])     # graph order


class _Args:
    criteria = {"eiko_weight": 0.1, "sdf_weight": 10000.0, "fs_weight": 1.0, "sdf_truncation": 0.3}
    data_specs = {"max_depth": 40.0}


def test_overlap_window_feeds_the_captured_mapping_graph(nl):
    rh = nl.render_helpers
    mu = nl.mapping.MapUpdater(0.3, init_std=0.01, seed=3, reserve_nodes=200_000, reserve_rows=200_000)
    torch.manual_seed(5)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    crit = nl.criterion.Criterion(_Args())
    kg = nl.keyframes.KeyframeGraph(window_size=2, keyframe_gap=1.5, key_distance=30.0, n_rays=512, voxel_size=0.3)
    ms = None
    for i in range(0, 11, 2):                                   # keyframes at x = 0, 2, .., 10 (index i + 1: every pose is optimised)
        f = _loop_frame(nl, i, index=i + 1)
        ms = mu.create_voxels(f.points, f.get_pose().detach())
        kg.insert_keyframe(f)
    graphs, windows = [], []
    for i in (N_LOOP - 1, 10):                                  # back at x = 0, then at the far end x = 10
        tracked = _loop_frame(nl, i, index=100 + i)
        window = kg.select_optimize_targets(tracked, "overlap")
        assert len(window) == 3 and window[-1] is tracked
        before = [f.pose.data.clone() for f in kg.keyframe_graph]
        rh.bundle_adjust_frames(window, mu.embeddings, ms, dec, crit, 0.3, 0.15, N_rays=512, num_iterations=3, truncation=0.3,
                                max_voxel_hit=20, max_distance=40.0, learning_rate=[0.01, 0.005, 0.001])
        g = rh._MapGraph._cache["g"]
        graphs.append(g)
        assert np.isfinite(g.eng.read_stats().loss)
        for f, b in zip(kg.keyframe_graph, before):
            if any(f is w for w in window):
                assert not torch.equal(f.pose.data, b), f.index
            else:
                assert torch.equal(f.pose.data, b), f.index
        windows.append([f.index for f in window[:-1]])
    assert windows[0] != windows[1], windows
    assert graphs[1] is graphs[0]                               # the same captured graph replayed, no new capture
