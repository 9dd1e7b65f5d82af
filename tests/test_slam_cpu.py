"""slam.py without a GPU: configuration, the keyframe-relative trajectory, the writers, the host-side rules against NumPy restatements,
and the lag-one scheduler driven by stub roles."""
import importlib
import math
import threading
import time

import numpy as np
import pytest
import torch

slam = importlib.import_module("nerf-loam_b200.slam")
frame_mod = importlib.import_module("nerf-loam_b200.frame")
se3 = importlib.import_module("nerf-loam_b200.se3pose")


def base_cfg():
    return {"dataset": "kitti", "data_specs": {"data_path": "x", "max_depth": 40},
            "criteria": {"sdf_weight": 1.0, "fs_weight": 1.0, "eiko_weight": 0.1, "sdf_truncation": 0.3},
            "decoder_specs": {"depth": 2, "width": 256, "in_dim": 16, "skips": [], "embedder": "none", "multires": 0},
            "tracker_specs": {"N_rays": 8, "learning_rate": 0.01, "step_size": 0.2, "max_voxel_hit": 20, "num_iterations": 5},
            "mapper_specs": {"N_rays_each": 8, "use_local_coord": False, "voxel_size": 0.3, "step_size": 0.5, "window_size": 4,
                             "num_iterations": 5, "max_voxel_hit": 20, "learning_rate_emb": 0.01, "learning_rate_decorder": 0.005,
                             "learning_rate_pose": 0.001, "freeze_frame": 5, "keyframe_gap": 8, "remove_back": False, "key_distance": 12},
            "debug_args": {"mesh_freq": 100}}


# ---------------------------------------------------------------------------------------------------------------------------- config
def test_base_config_merge(tmp_path):
    yaml = pytest.importorskip("yaml")
    base = base_cfg()
    (tmp_path / "base.yaml").write_text(yaml.safe_dump(base))
    (tmp_path / "seq.yaml").write_text(yaml.safe_dump({"base_config": "base.yaml", "exp_name": "seq",
                                                       "data_specs": {"data_path": "/seq", "use_gt": True},
                                                       "tracker_specs": {"start_frame": 2}, "seeding": 5}))
    a = slam.load_config(str(tmp_path / "seq.yaml"))
    assert a.data_specs == {"data_path": "/seq", "use_gt": True, "max_depth": 40, "min_depth": -1}
    assert a.tracker_specs["start_frame"] == 2 and a.tracker_specs["N_rays"] == 8 and a.tracker_specs["read_offset"] == 1
    assert a.mapper_specs["final_iter"] is False and a.mapper_specs["mesh_res"] == 8
    assert a.seeding == 5 and a.exp_name == "seq" and a.debug_args["mesh_freq"] == 100
    assert slam.load_config(base_cfg()).seeding == 777
    (tmp_path / "bad.yaml").write_text(yaml.safe_dump({"base_config": "missing.yaml"}))
    with pytest.raises(FileNotFoundError):
        slam.load_config(str(tmp_path / "bad.yaml"))


@pytest.mark.parametrize("patch,key", [
    ({"dataset": "ncd"}, "dataset: ncd"),
    ({"mapper_specs": {"use_local_coord": True}}, "use_local_coord"),
    ({"ckpt_freq": 10}, "ckpt_freq"),
    ({"debug_args": {"save_data_freq": 3}}, "save_data_freq"),
])
def test_rejected_keys(patch, key):
    cfg = base_cfg()
    for k, v in patch.items():
        if isinstance(v, dict):
            cfg[k] = {**cfg[k], **v}
        else:
            cfg[k] = v
    with pytest.raises(ValueError, match=key):
        slam.load_config(cfg)
    cfg = base_cfg()
    cfg["ckpt_freq"], cfg["debug_args"]["save_data_freq"] = -1, 0       # the reference's "off" values are accepted
    slam.load_config(cfg)


# ---------------------------------------------------------------------------------------------------------------------------- trajectory
class _Frame:
    def __init__(self, index, T):
        self.index = index
        self.pose = se3.OptimizablePose.from_matrix(torch.tensor(T, dtype=torch.float32))

    def get_pose(self):
        return self.pose.matrix()


class _Graph:
    def __init__(self):
        self.keyframe_graph, self.current_keyframe = [], None

    def insert(self, f):
        self.keyframe_graph.append(f)
        self.current_keyframe = f


def _T(x, yaw=0.0):
    T = np.eye(4)
    T[:2, :2] = [[math.cos(yaw), -math.sin(yaw)], [math.sin(yaw), math.cos(yaw)]]
    T[:3, 3] = [2000.0 + x, 2000.0, 2000.0]
    return T


def _shift(pose, dx):
    with torch.no_grad():
        pose.data[0] += dx


def test_updated_poses_follow_keyframes_then_stay_fixed():
    kg, tp = _Graph(), slam.KeyframePoses()
    k0 = _Frame(0, _T(0.0)); kg.insert(k0); tp.record(kg, k0)
    f1 = _Frame(1, _T(1.0, 0.1)); tp.record(kg, f1)
    k2 = _Frame(2, _T(2.0, 0.2)); kg.insert(k2); tp.record(kg, k2)
    f3 = _Frame(3, _T(3.0, 0.1)); tp.record(kg, f3)
    # a keyframe moved by bundle adjustment carries the scans recorded against it
    _shift(k0.pose, 0.5)
    _shift(k2.pose, -0.25)
    out = tp.get_updated_poses(kg)
    assert len(out) == 4 and tp.frame_poses == []
    want = [_T(0.5), _T(1.5, 0.1), _T(1.75, 0.2), _T(2.75, 0.1)]
    for got, w in zip(out, want):
        w = w.copy(); w[:3, 3] -= 2000.0                                  # the offset is removed
        np.testing.assert_allclose(got, w, atol=2e-4)
    # poses already written stay fixed when their keyframe moves again
    _shift(k0.pose, 1.0)
    f4 = _Frame(4, _T(4.0)); tp.record(kg, f4)
    out2 = tp.get_updated_poses(kg)
    assert len(out2) == 5
    np.testing.assert_array_equal(out2[0], out[0])
    np.testing.assert_allclose(out2[4][:3, 3], [4.0, 0.0, 0.0], atol=2e-4)
    # after the graph is cut back to the current keyframe, new scans index the new graph
    kg.keyframe_graph = [kg.current_keyframe]
    f5 = _Frame(5, _T(5.0)); tp.record(kg, f5)
    assert tp.frame_poses[0][0] == 0
    _shift(k2.pose, 0.1)
    out3 = tp.get_updated_poses(kg)
    np.testing.assert_allclose(out3[5][:3, 3], [5.1, 0.0, 0.0], atol=2e-4)
    np.testing.assert_array_equal(out3[3], out[3])


# ---------------------------------------------------------------------------------------------------------------------------- writers
def test_pose_file_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    poses = []
    for _ in range(5):
        T = np.eye(4, dtype=np.float32)
        T[:3, :4] = rng.normal(size=(3, 4)).astype(np.float32) * 100
        poses.append(T)
    slam.write_poses(tmp_path / "p.txt", poses)
    back = np.loadtxt(tmp_path / "p.txt").reshape(-1, 3, 4)
    assert back.shape == (5, 3, 4)
    np.testing.assert_array_equal(back.astype(np.float32), np.stack(poses)[:, :3, :4])


def _read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").splitlines()
    assert head[:2] == ["ply", "format binary_little_endian 1.0"]
    nv = int(next(l for l in head if l.startswith("element vertex")).split()[-1])
    nf = int(next(l for l in head if l.startswith("element face")).split()[-1])
    assert "property list uchar int vertex_indices" in head
    v = np.frombuffer(data, dtype="<f4", count=3 * nv, offset=end).reshape(nv, 3)
    rec = np.frombuffer(data, dtype=[("n", "u1"), ("v", "<i4", (3,))], count=nf, offset=end + 12 * nv)
    assert len(data) == end + 12 * nv + 13 * nf
    assert (rec["n"] == 3).all()
    return v, rec["v"]


def test_ply_round_trip(tmp_path):
    rng = np.random.default_rng(1)
    v = rng.normal(size=(100, 3)).astype(np.float32)
    f = rng.integers(0, 100, size=(57, 3)).astype(np.int32)
    slam.write_ply(tmp_path / "m.ply", v, f)
    v2, f2 = _read_ply(tmp_path / "m.ply")
    np.testing.assert_array_equal(v2, v)
    np.testing.assert_array_equal(f2, f)
    slam.write_ply(tmp_path / "e.ply", np.zeros((0, 3)), np.zeros((0, 3)))
    v3, f3 = _read_ply(tmp_path / "e.ply")
    assert v3.shape == (0, 3) and f3.shape == (0, 3)


# ---------------------------------------------------------------------------------------------------------------------------- rules
def _remove_back_np(points, rel, key_distance):
    """mapping.py:235-255 in float64: (keep mask, cosine)."""
    x, y = (1.0, 0.0) if rel is None else (float(rel[0, 3]), float(rel[1, 3]))
    xy = points[:, :2].astype(np.float64)
    c = (-xy[:, 0] * x - xy[:, 1] * y) / (np.linalg.norm(xy, axis=1) * math.hypot(x, y))
    return ~((c >= 0.7) & (np.linalg.norm(points.astype(np.float64), axis=1) > key_distance)), c


@pytest.mark.parametrize("rel", [None, "move"])
def test_remove_back_points(rel):
    rng = np.random.default_rng(2)
    pts = rng.uniform(-40, 40, size=(5000, 3)).astype(np.float32)
    cos = rng.uniform(0, 1, size=5000).astype(np.float32)
    f = frame_mod.LidarFrame(7, torch.from_numpy(pts), torch.from_numpy(cos), se3.OptimizablePose(torch.zeros(6)), new_keyframe=True)
    R = None
    if rel == "move":
        R = torch.eye(4); R[0, 3], R[1, 3] = 0.8, -0.3
        f.set_rel_pose(R)
    keep, c = _remove_back_np(pts, None if R is None else R.numpy(), 12.0)
    assert np.abs(c - 0.7).min() > 1e-5                  # no return within float32 rounding of the threshold
    assert 0 < keep.sum() < len(keep)
    out = slam.remove_back_points(f, 12.0)
    np.testing.assert_array_equal(out.points.numpy(), pts[keep])
    np.testing.assert_array_equal(out.pointsCos.numpy(), cos[keep])
    assert out.pose is f.pose and out.index == 7


def test_constant_velocity_guess_moves_translation_only():
    last = torch.from_numpy(_T(3.0, 0.3)).float()
    rel = torch.from_numpy(np.linalg.inv(_T(2.0, 0.1)) @ _T(3.0, 0.3)).float()
    g = slam.constant_velocity_guess(last, rel)
    want = last.double().numpy().copy()
    want[:3, 3] = (last.double().numpy() @ rel.double().numpy())[:3, 3]
    np.testing.assert_allclose(g.numpy(), want, atol=1e-3)
    np.testing.assert_array_equal(g[:3, :3].numpy(), last[:3, :3].numpy())     # the rotation is kept
    assert g.data_ptr() != last.data_ptr()
    np.testing.assert_array_equal(slam.constant_velocity_guess(last, None).numpy(), last.numpy())


# ---------------------------------------------------------------------------------------------------------------------------- scheduler
class StubTracker:
    def __init__(self, n, log, fail_at=None, delay=0.0):
        self.n, self.log, self.fail_at, self.delay = n, log, fail_at, delay

    def first_frame(self):
        return 0

    def frame_ids(self):
        return list(range(1, self.n))

    def track(self, fid, version):
        time.sleep(self.delay)
        if fid == self.fail_at:
            raise KeyError("tracker failed")
        self.log.append(("track", fid, version))
        return fid


class StubMapper:
    def __init__(self, log, fail_at=None, delay=0.0):
        self.log, self.fail_at, self.delay, self.version = log, fail_at, delay, 0
        self.finished = False

    def _publish(self, p):
        self.version += 1
        self.log.append(("publish", p, self.version))
        return self.version

    def init(self, f):
        return self._publish(f)

    def optimise(self, f):
        time.sleep(self.delay)
        self.log.append(("map", f, None))
        return f

    def update(self, f):
        if f == self.fail_at:
            raise ValueError("mapper failed")
        self.log.append(("update", f, None))
        return self._publish(f)

    def finish(self):
        self.finished = True


@pytest.mark.parametrize("td,md", [(0.0, 0.0), (0.003, 0.0), (0.0, 0.003)])
def test_lag_one_order(td, md):
    n = 12
    log = []
    lock = threading.Lock()

    class L(list):
        def append(self, x):
            with lock:
                list.append(self, x)
    log = L()
    mapper = StubMapper(log, delay=md)
    sched = slam.run_pipeline(StubTracker(n, log, delay=td), mapper)
    assert mapper.finished
    pos = {e: i for i, e in enumerate(log)}
    version_of = {p: v for what, p, v in log if what == "publish"}
    assert sorted(version_of) == list(range(n))
    for what, p, v in log:
        if what == "track":
            assert v == version_of[max(p - 2, 0)]                        # track(i+1) sees the map of step i-1
    rel = {p: i for i, (what, p, _) in enumerate(sched.log) if what == "release"}
    upd = {p: i for i, (what, p, _) in enumerate(sched.log) if what == "update"}
    for p in range(1, n - 1):
        assert rel[p + 1] < upd[p]                                         # update(i) after the release for track(i+1)
    for p in range(1, n):
        assert pos[("map", p, None)] < pos[("update", p, None)]
        assert pos[("track", p, version_of[max(p - 2, 0)])] < pos[("map", p, None)]


@pytest.mark.parametrize("who", ["tracker", "mapper"])
def test_failure_stops_both_threads(who):
    log = []
    tracker = StubTracker(50, log, fail_at=5 if who == "tracker" else None, delay=0.001)
    mapper = StubMapper(log, fail_at=4 if who == "mapper" else None)
    before = set(threading.enumerate())
    t0 = time.perf_counter()
    with pytest.raises(KeyError if who == "tracker" else ValueError):
        slam.run_pipeline(tracker, mapper)
    assert time.perf_counter() - t0 < 10.0
    assert not mapper.finished
    assert [t for t in threading.enumerate() if t not in before and t.name.startswith("nerfloam-")] == []
