"""slam.NeRFLOAM on the GPU: a whole synthetic sequence with the tracker and the mapper concurrent on two streams, against the true
poses, against the same lag-one order driven on one thread, mapping only (use_gt), the periodic mesh branch, a failing scan, and
scripts/run_slam.py."""
import importlib
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def nl():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    sys.path.insert(0, ROOT)
    return importlib.import_module("nerfloam_b200")


def drive(n, spacing=0.5):
    syn = importlib.import_module("nerf-loam_b200.synthetic")
    out = []
    for i in range(n):
        xyz, yaw = syn.path_pose(i, n, spacing)
        pts, cos, pose = syn.make_scan(seed=1000 + i, sensor_xyz=xyz, yaw=yaw)
        pose = pose.astype(np.float64)
        pose[:3, 3] -= syn.POSE_OFFSET                   # loaders return poses without the frame offset
        out.append((pts, cos, pose, xyz, yaw))
    return out


class MemoryStream:
    """A loader over scans held in memory (the interface of dataset.ScanLoader)."""

    def __init__(self, scans, use_gt):
        self.scans, self.use_gt = scans, use_gt

    def __len__(self):
        return len(self.scans)

    def __getitem__(self, i):
        pts, cos, pose = self.scans[i][:3]
        return i, torch.from_numpy(pts), torch.from_numpy(cos), (pose.copy() if self.use_gt else None)

    def get_init_pose(self, i):
        return self.scans[i][2].copy() if self.use_gt else np.eye(4)


def config(data_path="", use_gt=False, mesh_freq=0, final_iter=False, keyframe_gap=1.0, iters=25):
    # tracker rate 0.01: the first tracked scan runs at twice it (frame index < 2, render_helpers.py:448-450), the effective 0.02
    # that converges on this scene every time (DESIGN.md section 11, scripts/sweep_tracking_lr.py)
    return {"dataset": "kitti", "seeding": 777, "data_specs": {"data_path": data_path, "use_gt": use_gt, "max_depth": 40, "min_depth": 5},
            "criteria": {"sdf_weight": 10000.0, "fs_weight": 1, "eiko_weight": 0.1, "sdf_truncation": 0.3},
            "decoder_specs": {"depth": 2, "width": 256, "in_dim": 16, "skips": [], "embedder": "none", "multires": 0},
            "tracker_specs": {"N_rays": 2048, "learning_rate": 0.01, "step_size": 0.2, "max_voxel_hit": 20, "num_iterations": 25,
                              "start_frame": 0, "end_frame": -1, "read_offset": 1},
            "mapper_specs": {"N_rays_each": 2048, "use_local_coord": False, "voxel_size": 0.3, "step_size": 0.5, "window_size": 4,
                             "num_iterations": iters, "max_voxel_hit": 20, "final_iter": final_iter, "mesh_res": 2,
                             "learning_rate_emb": 0.01, "learning_rate_decorder": 0.005, "learning_rate_pose": 0.001, "freeze_frame": 5,
                             "keyframe_gap": keyframe_gap, "remove_back": False, "key_distance": 12},
            "debug_args": {"verbose": False, "mesh_freq": mesh_freq}}


def write_kitti(path, scans):
    os.makedirs(path / "velodyne", exist_ok=True)
    for i, (pts, *_rest) in enumerate(scans):
        rows = np.concatenate([pts, np.zeros((pts.shape[0], 1), np.float32)], 1).astype(np.float32)
        rows.tofile(str(path / "velodyne" / f"{i:06d}.bin"))
    np.savetxt(str(path / "poses_lidar.txt"), np.stack([s[2][:3, :4].reshape(-1) for s in scans]))


def read_poses(path):
    return np.loadtxt(path, ndmin=2).reshape(-1, 3, 4)


def our_threads():
    return [t for t in threading.enumerate() if t.name.startswith("nerfloam-")]


def test_sequence_from_kitti_files(nl, tmp_path):
    """Ten canyon scans 0.5 m apart, written as KITTI files, tracked and mapped concurrently.  Bound: every scan within 0.20 m of the
    true translation.  On an H100 80GB HBM3 at 700 W the error grew by about 1.2 cm per scan to 0.121 m at the last one: with the
    reference's 'current' window no keyframe is re-adjusted, and later scans track at a third of the rate (render_helpers.py:448-450)."""
    scans = drive(10)
    write_kitti(tmp_path / "seq", scans)
    import yaml
    (tmp_path / "cfg.yaml").write_text(yaml.safe_dump(config(str(tmp_path / "seq"))))
    s = nl.slam.NeRFLOAM(str(tmp_path / "cfg.yaml"), str(tmp_path / "out"))
    summary = s.run()
    est = read_poses(tmp_path / "out" / "misc" / "frame_poses.txt")
    assert est.shape == (10, 3, 4) and summary["scans"] == 10
    err = np.linalg.norm(est[:, :, 3] - np.stack([p[2][:3, 3] for p in scans]), axis=1)
    print("translation error per scan (m):", np.round(err, 4).tolist())
    assert err.max() < 0.20
    # both roles ran, each on its own non-default stream
    ts, ms = (st.cuda_stream for st in s.streams)
    assert s.tracker.streams == {ts} and s.mapper.streams == {ms} and ts != ms
    assert torch.cuda.default_stream().cuda_stream not in (ts, ms)
    assert os.path.exists(tmp_path / "out" / "mesh" / "final_mesh.ply")
    assert our_threads() == []


def run_serial(s):
    """The lag-one order on one thread, through the pipeline's step functions: BA(p), then track(p + 1) against the map of step p - 1,
    then the mapping step's update of p."""
    tr, mp = s.tracker, s.mapper
    versions = [mp.init(tr.first_frame())]
    ids = tr.frame_ids()
    frame = tr.track(ids[0], versions[0]) if ids else None
    for p in range(1, len(ids) + 1):
        state = mp.optimise(frame)
        if p < len(ids):
            frame = tr.track(ids[p], versions[p - 1])
        versions.append(mp.update(state))
    mp.finish()


def test_concurrent_matches_one_thread_order(nl, tmp_path):
    """The concurrent pipeline computes what the same lag-one order computes on one thread: the same keyframes, and poses whose mean
    absolute difference is within max(3 x that of two one-thread runs, 1 mm).  Only the order of the fp32 atomics' sums differs, and
    tracking amplifies it along the sequence, so the largest single entry is too noisy a statistic: on an H100 80GB HBM3 at 700 W two
    one-thread runs differed by up to 0.011-0.017, and the concurrent run from the first by 0.006 to 0.044; the means were 0.0013
    (one thread) and 0.0014 (concurrent)."""
    scans = drive(10)
    runs = []
    for k, mode in enumerate(["serial", "serial", "concurrent"]):
        s = nl.slam.NeRFLOAM(config(keyframe_gap=1.0), str(tmp_path / f"r{k}"), data_stream=MemoryStream(scans, False))
        s.run() if mode == "concurrent" else run_serial(s)
        torch.cuda.synchronize()
        runs.append((s.mapper.keyframe_indices, read_poses(tmp_path / f"r{k}" / "misc" / "frame_poses.txt")))
    (k0, p0), (k1, p1), (k2, p2) = runs
    assert k0 == k1 == k2 and len(k0) > 1
    base, diff = np.abs(p0 - p1), np.abs(p2 - p0)
    print(f"one-thread runs differ by {base.mean():.3g} mean, {base.max():.3g} max; concurrent against one-thread {diff.mean():.3g} "
          f"mean, {diff.max():.3g} max")
    assert diff.mean() <= max(3 * base.mean(), 1e-3)


def test_mapping_only_use_gt(nl, tmp_path):
    """use_gt: every scan comes with its pose and only the mapper works.  The final mesh against the scans' noise-free returns at the
    true poses: F-score (0.1 m) above 85; 93.2 on an H100 80GB HBM3 at 700 W (accuracy 0.051 m, completeness 0.027 m)."""
    syn = importlib.import_module("nerf-loam_b200.synthetic")
    scans = drive(8)
    s = nl.slam.NeRFLOAM(config(use_gt=True, final_iter=True), str(tmp_path), data_stream=MemoryStream(scans, True))
    s.run()
    est = read_poses(tmp_path / "misc" / "frame_poses.txt")
    assert est.shape == (8, 3, 4)
    assert np.abs(est[:, :, 3] - np.stack([p[2][:3, 3] for p in scans])).max() < 0.05
    from test_slam_cpu import _read_ply
    v, f = _read_ply(tmp_path / "mesh" / "final_mesh.ply")
    assert f.shape[0] > 1000
    clean = []
    for i, (_, _, _, xyz, yaw) in enumerate(scans):
        p, _, pose = syn.make_scan(seed=1000 + i, sensor_xyz=xyz, yaw=yaw, noise_std=0.0)
        pose = pose.astype(np.float64)
        clean.append(p.astype(np.float64) @ pose[:3, :3].T + pose[:3, 3] - syn.POSE_OFFSET)
    r = nl.evaluate.eval_mesh(torch.from_numpy(v.copy()).cuda(), torch.from_numpy(f.copy()).cuda(),
                              np.concatenate(clean).astype(np.float32), n_samples=1_000_000, res=0.05, threshold=0.1, truncation=0.5, seed=0)
    print("use_gt reconstruction:", r)
    assert r["fscore"] > 85.0


def test_periodic_mesh_and_graph_cut(nl, tmp_path):
    """More than 20 keyframes (every scan is one: keyframe_gap 0.1 m) and mesh_freq 22: at scan 22 the graph is refined, the mesh and
    the poses so far are written, and the graph is cut to the current keyframe.  The trajectory stays complete."""
    scans = drive(23, spacing=0.3)
    s = nl.slam.NeRFLOAM(config(use_gt=True, final_iter=True, mesh_freq=22, keyframe_gap=0.1, iters=10), str(tmp_path),
                         data_stream=MemoryStream(scans, True))
    summary = s.run()
    assert os.path.exists(tmp_path / "mesh" / "mesh_00022.ply") and os.path.exists(tmp_path / "mesh" / "mesh_00000.ply")
    assert len(s.mapper.keyframe_indices) == 23
    assert len(s.mapper.kg.keyframe_graph) == 1 and s.mapper.kg.keyframe_graph[0].index == 22
    assert read_poses(tmp_path / "misc" / "frame_poses_00022.txt").shape == (23, 3, 4)
    assert read_poses(tmp_path / "misc" / "frame_poses.txt").shape == (23, 3, 4)
    assert len(summary["refine_ms"]) == 2                     # at scan 22 and at the end
    for name in ("final_mesh_noreplay.ply", "final_mesh.ply"):
        assert os.path.exists(tmp_path / "mesh" / name)


def test_sparse_scan_raises_out_of_run(nl, tmp_path):
    """A scan with fewer than 2 x N_rays_each points is too sparse to become a keyframe: insert_keyframe's ValueError comes out of
    run() and neither thread survives it."""
    scans = drive(6)
    pts, cos, *rest = scans[3]
    keep = np.random.default_rng(0).choice(pts.shape[0], 3000, replace=False)
    scans[3] = (pts[np.sort(keep)], cos[np.sort(keep)], *rest)
    s = nl.slam.NeRFLOAM(config(keyframe_gap=0.1), str(tmp_path), data_stream=MemoryStream(scans, False))
    with pytest.raises(ValueError, match="valid_distance"):
        s.run()
    assert our_threads() == []


def test_run_slam_script(nl, tmp_path):
    scans = drive(4)
    write_kitti(tmp_path / "seq", scans)
    import yaml
    cfg = config("unused", mesh_freq=2)
    cfg.update(log_dir=str(tmp_path / "logs"), exp_name="tiny")
    (tmp_path / "cfg.yaml").write_text(yaml.safe_dump(cfg))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "run_slam.py"), str(tmp_path / "cfg.yaml"), "--data",
                          str(tmp_path / "seq"), "--out", str(tmp_path / "out")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    summary = json.loads(out.stdout.strip().splitlines()[-1])
    assert summary["scans"] == 4 and summary["keyframes"] >= 1
    for rel in ("mesh/mesh_00000.ply", "mesh/mesh_00002.ply", "mesh/final_mesh.ply", "mesh/final_mesh_noreplay.ply",
                "misc/frame_poses_00002.txt", "misc/frame_poses.txt"):
        assert os.path.exists(tmp_path / "out" / rel), rel
    assert read_poses(tmp_path / "out" / "misc" / "frame_poses.txt").shape == (4, 3, 4)


def test_shared_map_acquire_version(nl):
    """SharedMap.acquire(version) takes that publication while one of the two slots holds it, and raises once it has been overwritten
    or before it exists; acquire() still takes the latest."""
    syn = nl.synthetic
    pts, _, pose = syn.make_scan(n_beams=16, n_az=200, seed=3)
    mu = nl.mapping.MapUpdater(0.3, device="cuda")
    ms = mu.create_voxels(pts, pose)
    make = lambda: nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    dec, sm = make(), nl.share.SharedMap(make)
    v1 = sm.publish(ms, dec)
    v2 = sm.publish(ms, dec)
    _, _, slot = sm.acquire(v1)
    assert slot.version == v1
    sm.release(slot)
    _, _, slot = sm.acquire()
    assert slot.version == v2
    sm.release(slot)
    v3 = sm.publish(ms, dec)                                    # goes to v1's slot
    assert sm.acquire(v3)[2].version == v3 and sm.acquire(v2)[2].version == v2
    with pytest.raises(RuntimeError, match="not held"):
        sm.acquire(v1)
    with pytest.raises(RuntimeError, match="not held"):
        sm.acquire(v3 + 1)
