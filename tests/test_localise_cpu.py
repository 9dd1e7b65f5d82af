"""Map files and the localiser's host side without a GPU: write_map / load_map round trip of a CPU MapUpdater and decoder, every
kind of malformed file rejected with its reason, the frozen map serving slam.Tracking one (map_state, decoder) for every version, and
the Localiser's configuration."""
import importlib

import numpy as np
import pytest
import torch

slam = importlib.import_module("nerf-loam_b200.slam")
localise = importlib.import_module("nerf-loam_b200.localise")
mapping = importlib.import_module("nerf-loam_b200.mapping")
lidar = importlib.import_module("nerf-loam_b200.lidar")
synthetic = importlib.import_module("nerf-loam_b200.synthetic")
share = importlib.import_module("nerf-loam_b200.share")
se3 = importlib.import_module("nerf-loam_b200.se3pose")
_capi = importlib.import_module("nerf-loam_b200._capi")

SPECS = {"depth": 2, "width": 64, "in_dim": 16, "skips": [], "embedder": "none", "multires": 0}
CONFIG = {"criteria": {"sdf_weight": 10000.0, "fs_weight": 1, "eiko_weight": 0.1, "sdf_truncation": 0.3},
          "tracker_specs": {"N_rays": 64, "learning_rate": 0.01, "step_size": 0.2, "max_voxel_hit": 20, "num_iterations": 25,
                            "start_frame": 0, "end_frame": -1, "read_offset": 1},
          "voxel_size": 0.3, "data_specs": {"data_path": "seq", "use_gt": False, "max_depth": 40, "min_depth": 5}, "dataset": "kitti"}


def _saved():
    """A CPU map of three small scans with trained-looking embeddings, a seeded decoder, and a trajectory of the scans' poses."""
    mu = mapping.MapUpdater(0.3, device="cpu", init_std=0.01, seed=4)
    poses = []
    for i in range(3):
        pts, _, pose = synthetic.make_scan(n_beams=16, n_az=200, seed=50 + i, sensor_xyz=(0.5 * i, 0.1 * i, 0.0), yaw=0.05 * i)
        mu.create_voxels(torch.from_numpy(pts), torch.from_numpy(pose).double())
        p = pose.astype(np.float64)
        p[:3, 3] -= synthetic.POSE_OFFSET
        poses.append(p)
    with torch.no_grad():
        mu.embeddings.copy_(torch.randn(mu.embeddings.shape, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16))
    torch.manual_seed(3)
    dec = lidar.Decoder(**SPECS)
    return slam.SavedMap(mu, dec, dict(SPECS), np.stack(poses), np.array([0, 1, 2], dtype=np.int64), dict(CONFIG))


def _bits(t):
    return t.detach().contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def test_round_trip(tmp_path):
    saved = _saved()
    path = tmp_path / "run.map"
    slam.write_map(path, saved)
    raw = torch.load(path, weights_only=True)
    assert raw["format"] == slam.MAP_FORMAT and set(raw) == set(slam.MAP_KEYS)
    back = slam.load_map(path, device="cpu")
    a, b = saved.map.state_dict(), back.map.state_dict()
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k
    assert torch.equal(_bits(share._flat_decoder_state(back.decoder)), _bits(share._flat_decoder_state(saved.decoder)))
    assert [k for k in back.decoder.state_dict()] == [k for k in saved.decoder.state_dict()]
    assert back.decoder_specs == SPECS and isinstance(back.decoder, lidar.Decoder)
    assert back.trajectory.dtype == torch.float64 and torch.equal(back.trajectory, torch.from_numpy(saved.trajectory))
    assert back.scan_ids.dtype == torch.int64 and back.scan_ids.tolist() == [0, 1, 2]
    assert back.config == CONFIG
    # the restored map is the saved one: same hot-path arrays
    ms_a, ms_b = saved.map.map_states["_mapstate"], back.map.map_states["_mapstate"]
    for f in ("centres", "structure", "vox2row", "emb"):
        assert torch.equal(getattr(ms_a, f), getattr(ms_b, f)), f
    assert not (tmp_path / "run.map.part").exists()


def _mutations():
    def drop(k):
        return lambda o: o.pop(k)

    def setv(path, v):
        def f(o):
            d = o
            for k in path[:-1]:
                d = d[k]
            d[path[-1]] = v(d[path[-1]]) if callable(v) else v
        return f

    nan = lambda t: t.clone().index_put_((torch.tensor([1]), torch.tensor([0]), torch.tensor([3])), torch.tensor(float("nan"), dtype=t.dtype))
    return [
        ("missing key", drop("decoder"), "keys decoder"),
        ("format", setv(["format"], "nerfloam_b200.map/0"), "format"),
        ("trajectory dtype", setv(["trajectory"], lambda t: t.float()), "trajectory a float64"),
        ("trajectory shape", setv(["trajectory"], lambda t: t[:, :3, :].contiguous()), r"trajectory of shape \[S,4,4\]"),
        ("non-finite pose", setv(["trajectory"], nan), "trajectory poses finite"),
        ("pose last row", setv(["trajectory"], lambda t: t.clone().index_fill_(1, torch.tensor([3]), 0.0)), "last row"),
        ("scan_ids dtype", setv(["scan_ids"], lambda t: t.int()), "scan_ids an int64"),
        ("scan_ids shape", setv(["scan_ids"], lambda t: t[:2].clone()), "one per pose"),
        ("decoder dtype", setv(["decoder", "params"], lambda t: t.double()), "flat float32"),
        ("decoder size", setv(["decoder", "params"], lambda t: t[:-1].clone()), "decoder params of"),
        ("decoder specs", setv(["decoder", "decoder_specs"], lambda s: {**s, "width": 100}), "decoder_specs a supported decoder"),
        ("non-finite decoder", setv(["decoder", "params"], lambda t: t.clone().fill_(float("inf"))), "decoder params finite"),
        ("config key", setv(["config"], lambda c: {k: v for k, v in c.items() if k != "criteria"}), "config keys criteria"),
        ("config voxel size", setv(["config", "voxel_size"], 0.2), "voxel_size equal to the map's"),
        ("config dataset", setv(["config", "dataset"], "ncd"), "dataset kitti or maicity"),
    ]


@pytest.mark.parametrize("name,mutate,reason", _mutations(), ids=[m[0] for m in _mutations()])
def test_malformed_file_rejected_with_reason(tmp_path, name, mutate, reason):
    path = tmp_path / "run.map"
    slam.write_map(path, _saved())
    obj = torch.load(path, weights_only=True)
    mutate(obj)
    torch.save(obj, path)
    with pytest.raises(ValueError, match=reason):
        slam.load_map(path, device="cpu")


def test_malformed_container_and_map(tmp_path):
    bad = tmp_path / "bad.map"
    bad.write_bytes(b"not a torch file")
    with pytest.raises(ValueError, match="not a map file"):
        slam.load_map(bad, device="cpu")
    with pytest.raises(ValueError, match="cannot read"):
        slam.load_map(tmp_path / "missing.map", device="cpu")
    torch.save([1, 2, 3], bad)
    with pytest.raises(ValueError, match="a dict"):
        slam.load_map(bad, device="cpu")
    slam.write_map(bad, _saved())
    obj = torch.load(bad, weights_only=True)
    obj["map"]["child"] = obj["map"]["child"].long()              # the map inside: from_state_dict's own checks
    torch.save(obj, bad)
    with pytest.raises(_capi.NerfLoamError, match="child a CPU torch.int32 tensor"):
        slam.load_map(bad, device="cpu")


def test_write_map_rejects_what_it_cannot_store(tmp_path):
    s = _saved()
    with pytest.raises(ValueError, match="config.tracker_specs.N_rays is a Tensor"):
        slam.write_map(tmp_path / "a.map", s._replace(config={**CONFIG, "tracker_specs": {**CONFIG["tracker_specs"], "N_rays": torch.tensor(5)}}))
    traj = s.trajectory.copy()
    traj[0, 0, 3] = np.inf
    with pytest.raises(ValueError, match="non-finite"):
        slam.write_map(tmp_path / "a.map", s._replace(trajectory=traj))
    with pytest.raises(ValueError, match="scan_ids"):
        slam.write_map(tmp_path / "a.map", s._replace(scan_ids=np.arange(2)))
    with pytest.raises(ValueError, match="voxel_size"):
        slam.write_map(tmp_path / "a.map", s._replace(config={**CONFIG, "voxel_size": 0.25}))
    assert not (tmp_path / "a.map").exists()
    cfg = {**CONFIG, "tracker_specs": {**CONFIG["tracker_specs"], "N_rays": np.int64(64)}, "criteria": {**CONFIG["criteria"], "fs_weight": np.float32(1)}}
    slam.write_map(tmp_path / "a.map", s._replace(config=cfg))      # numpy scalars are stored as Python numbers
    assert slam.load_map(tmp_path / "a.map", device="cpu").config == CONFIG


class _Stream:
    def __init__(self, n):
        self.scans = [synthetic.make_scan(n_beams=8, n_az=100, seed=i)[:2] for i in range(n)]

    def __len__(self):
        return len(self.scans)

    def __getitem__(self, i):
        return i, torch.from_numpy(self.scans[i][0]), torch.from_numpy(self.scans[i][1]), None

    def get_init_pose(self, i):
        return np.eye(4)


def test_frozen_map_serves_tracking_one_map(monkeypatch):
    """Tracking reads the frozen map through acquire / release: whatever version it asks for, it gets the same objects."""
    s = _saved()
    ms = s.map.map_states["_mapstate"]
    frozen = localise.FrozenMap(ms, s.decoder)
    for v in (None, 0, 1, 7, 10 ** 6):
        m, d, slot = frozen.acquire(v)
        assert m is ms and d is s.decoder
        frozen.release(slot)
    seen = []

    def fake_track_frame(pose, frame, map_state, decoder, *args, **kw):
        seen.append((map_state, decoder))
        return se3.OptimizablePose(pose.data.detach().clone()), torch.ones(4, dtype=torch.bool)

    monkeypatch.setattr(slam.rh, "track_frame", fake_track_frame)
    loc = localise.Localiser(s, _Stream(4))
    tr = loc.tracker
    tr.first_frame()
    for fid, version in zip(tr.frame_ids(), (0, 3, 99)):                        # Tracking.track without its stream bookkeeping
        index, points, pointcos, _ = tr.data_stream[fid]
        tr._do_tracking(slam.LidarFrame(index, points, pointcos), version)
    assert len(seen) == 3 and all(m is ms and d is s.decoder for m, d in seen)


def test_localiser_config():
    s = _saved()
    loc = localise.Localiser(s, _Stream(2), config={"tracker_specs": {"num_iterations": 7}, "global_specs": {"radius": 3.0}})
    assert loc.tracker.num_iterations == 7 and loc.tracker.N_rays == 64                 # overridden / kept from the file
    assert loc.tracker.voxel_size == 0.3 and loc.tracker.step_size == pytest.approx(0.06) and loc.tracker.max_distance == 40
    assert loc.global_specs["radius"] == 3.0 and loc.global_specs["yaw_steps"] == localise.GLOBAL_SPECS["yaw_steps"]
    assert s.config == CONFIG                                                          # the saved config is not modified
    want = torch.from_numpy(s.trajectory).clone()
    want[:, :3, 3] += synthetic.POSE_OFFSET
    assert torch.equal(loc.anchors, want)
    with pytest.raises(ValueError, match="voxel_size"):
        localise.Localiser(s, _Stream(2), config={"voxel_size": 0.2})
    with pytest.raises(ValueError, match="start_frame"):
        loc.run(start_frame=5)
