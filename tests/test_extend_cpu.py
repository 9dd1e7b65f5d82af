"""Growing a saved map with a later drive (slam.NeRFLOAM's base_map), without a GPU: the config agreement, frozen_rows' validation down
to the C entry point, the grown map file's trajectory, a failed placement, and a run without base_map building what it built before."""
import ctypes
import importlib
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

slam = importlib.import_module("nerf-loam_b200.slam")
localise = importlib.import_module("nerf-loam_b200.localise")
rh = importlib.import_module("nerf-loam_b200.render_helpers")
lidar = importlib.import_module("nerf-loam_b200.lidar")
capi = importlib.import_module("nerf-loam_b200._capi")
POSE_OFFSET = importlib.import_module("nerf-loam_b200.frame").POSE_OFFSET


def cfg():
    return {"dataset": "kitti", "seeding": 777, "data_specs": {"data_path": "x", "max_depth": 40},
            "criteria": {"sdf_weight": 10000.0, "fs_weight": 1, "eiko_weight": 0.1, "sdf_truncation": 0.3},
            "decoder_specs": {"depth": 2, "width": 256, "in_dim": 16, "skips": [], "embedder": "none", "multires": 0},
            "tracker_specs": {"N_rays": 8, "learning_rate": 0.01, "step_size": 0.2, "max_voxel_hit": 20, "num_iterations": 5},
            "mapper_specs": {"N_rays_each": 8, "use_local_coord": False, "voxel_size": 0.3, "step_size": 0.5, "window_size": 4,
                             "num_iterations": 5, "max_voxel_hit": 20, "learning_rate_emb": 0.01, "learning_rate_decorder": 0.005,
                             "learning_rate_pose": 0.001, "freeze_frame": 5, "keyframe_gap": 8, "remove_back": False, "key_distance": 12},
            "debug_args": {"mesh_freq": 0}}


class StubMap:
    """What NeRFLOAM and write_map touch of a MapUpdater."""

    def __init__(self, n_rows=40, voxel_size=0.3):
        self.n_rows, self.n_nodes, self.voxel_size, self.on_device, self.readers = n_rows, 9, voxel_size, False, None
        self.map_states = {"_mapstate": "the saved map's state"}
        self.reserved = None

    def reserve(self, nodes=0, rows=0):
        self.reserved = (nodes, rows)

    def state_dict(self):
        return {"voxel_size": self.voxel_size, "stub": torch.zeros(3)}


def saved(n=3, config=None, decoder_specs=None):
    c = cfg()
    traj = np.tile(np.eye(4), (n, 1, 1))
    traj[:, 0, 3] = np.arange(n) * 0.5
    return slam.SavedMap(StubMap(), lidar.Decoder(**c["decoder_specs"]), dict(decoder_specs or c["decoder_specs"]), traj,
                         np.arange(n, dtype=np.int64), config or slam.map_config(slam.load_config(c)))


class Stream:
    def __init__(self, n=3):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        pts = torch.tensor([[5.0, 0.0, 0.0], [0.0, 5.0, 0.0], [0.0, 0.0, -1.7]] * 4)
        return i, pts, torch.ones(pts.shape[0]), None

    def get_init_pose(self, i):
        return np.eye(4)


@pytest.fixture
def cpu_slam(monkeypatch):
    """NeRFLOAM constructible without a GPU: modules stay on the CPU, streams are placeholders, a new map is a record of its args."""
    made = []

    class NewMap(StubMap):
        def __init__(self, voxel_size, **kw):
            super().__init__(0, voxel_size)
            made.append(kw)
    monkeypatch.setattr(torch.nn.Module, "cuda", lambda self, *a, **k: self)
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: object())
    monkeypatch.setattr(slam, "MapUpdater", NewMap)
    return made


# ----------------------------------------------------------------------------------------------------------------------- config
@pytest.mark.parametrize("key", slam.BASE_KEYS)
def test_config_must_agree_with_the_map(cpu_slam, tmp_path, key):
    c = cfg()
    if key == "voxel_size":
        c["mapper_specs"]["voxel_size"] = 0.2
    elif key == "decoder_specs":
        c["decoder_specs"]["width"] = 128
    else:
        c["criteria"]["sdf_truncation"] = 0.2
    with pytest.raises(ValueError, match=key):
        slam.check_base_config(slam.load_config(c), saved())
    with pytest.raises(ValueError, match=key):
        slam.NeRFLOAM(c, str(tmp_path), data_stream=Stream(), base_map=saved())


def test_agreeing_config_passes_and_the_rest_comes_from_the_run(cpu_slam, tmp_path):
    c = cfg()
    c["tracker_specs"]["num_iterations"] = 11
    c["mapper_specs"]["window_size"] = 7
    c["criteria"]["fs_weight"] = 1.0                                    # 1 in the file: equal values of another type agree
    base = saved()
    s = slam.NeRFLOAM(c, str(tmp_path), data_stream=Stream(), base_map=base, reserve_nodes=5000, reserve_rows=3000)
    assert base.map.reserved == (5000, 3000)                            # the reserves reach the saved map
    assert s.tracker.num_iterations == 11 and s.mapper.window_size == 7
    assert s.mapper.map is base.map and s.mapper.decoder is base.decoder and cpu_slam == []
    assert s.mapper.frozen_rows == base.map.n_rows and s.mapper.train_decoder is False and s.tracker.place is not None
    base.map.on_device = True
    with pytest.raises(ValueError, match="host octree"):
        slam.NeRFLOAM(c, str(tmp_path), data_stream=Stream(), base_map=base)


# ------------------------------------------------------------------------------------------------------------------ frozen_rows
@pytest.mark.parametrize("bad", [-1, 101, 2.0, True])
def test_frozen_rows_out_of_range_is_rejected(bad):
    emb = torch.zeros((100, 16), dtype=torch.bfloat16)
    kw = dict(map_states={}, sdf_network=None, loss_criteria=None, voxel_size=0.3, step_size=0.15, frozen_rows=bad)
    with pytest.raises(ValueError, match="frozen_rows"):
        rh.bundle_adjust_frames([], emb, **kw)
    with pytest.raises(ValueError, match="frozen_rows"):
        rh.refine_map(SimpleNamespace(keyframe_graph=[]), emb, **kw)


def test_frozen_rows_limits_pass_the_check():
    emb = torch.zeros((100, 16), dtype=torch.bfloat16)
    for ok in (0, 57, 100, np.int64(100)):
        assert rh._frozen_rows(ok, emb, "t") == int(ok)


def test_mark_rows_floor_entry_point_rejects_a_bad_floor():
    L = capi.lib()
    assert "nl_mark_rows_floor" in capi.EXPORTED_SYMBOLS
    p = [ctypes.c_void_p(256 * k) for k in range(1, 6)]                 # never dereferenced: every call below fails its checks
    call = lambda floor, n_rows=1000: L.nl_mark_rows_floor(10, None, p[0], p[1], n_rows, floor, p[2], p[3], p[4], None)
    for bad in (-1, 1001, -(1 << 40)):
        assert call(bad) != 0 and "row_floor" in L.nl_last_error().decode(), bad
    assert call(0, n_rows=0) != 0 and "sizes" in L.nl_last_error().decode()
    assert L.nl_mark_rows_floor(0, None, p[0], p[1], 1000, 1000, p[2], p[3], p[4], None) == 0      # M = 0, floor = n_rows: nothing to do


# -------------------------------------------------------------------------------------------------------------- the grown file
def test_grown_trajectory_is_written_and_accepted(tmp_path):
    base = saved(n=3)
    new = np.tile(np.eye(4), (4, 1, 1))
    new[:, 1, 3] = 7.0 + np.arange(4)
    traj, ids = slam.grown_trajectory(base, new, [0, 1, 2, 5])
    assert traj.shape == (7, 4, 4) and np.array_equal(traj[:3], base.trajectory) and np.array_equal(traj[3:], new)
    assert ids.dtype == np.int64 and ids.tolist() == [0, 1, 2, 0, 1, 2, 5]          # ids repeat across drives
    path = tmp_path / "grown.map"
    slam.write_map(path, base._replace(trajectory=traj, scan_ids=ids))
    obj = torch.load(path, map_location="cpu", weights_only=True)
    assert slam._check_map_file(obj) == []
    assert torch.equal(obj["trajectory"], torch.from_numpy(traj)) and obj["scan_ids"].tolist() == ids.tolist()


# ------------------------------------------------------------------------------------------------------------ failed placement
def test_failed_placement_raises_and_writes_nothing(cpu_slam, tmp_path, monkeypatch):
    calls = []

    def place_scan(frame, map_state, decoder, tracker, anchors, specs, generator):
        calls.append((map_state, decoder, anchors.clone(), specs, generator))
        return SimpleNamespace(hit_mask=None), None, 12.0, None
    monkeypatch.setattr(localise, "place_scan", place_scan)
    c = cfg()
    c["global_specs"] = {"radius": 3.0}
    base = saved(n=3)
    s = slam.NeRFLOAM(c, str(tmp_path / "out"), data_stream=Stream(), base_map=base)
    with pytest.raises(capi.NerfLoamError, match="could not be placed"):
        slam.run_pipeline(s.tracker, s.mapper)
    assert [f for _, _, fs in os.walk(tmp_path) for f in fs] == []
    (map_state, decoder, anchors, specs, generator), = calls
    assert map_state == "the saved map's state" and decoder is base.decoder and generator is s.tracker.generator
    want = torch.from_numpy(base.trajectory).clone()
    want[:, :3, 3] += POSE_OFFSET
    assert torch.equal(anchors, want) and specs == {**localise.GLOBAL_SPECS, "radius": 3.0}
    assert s.place_ms == {"search": 12.0, "track": None}


# ------------------------------------------------------------------------------------------------------------- no base map
def test_without_base_map_nothing_changes(cpu_slam, tmp_path, monkeypatch):
    c = cfg()
    s = slam.NeRFLOAM(c, str(tmp_path), data_stream=Stream())
    after = (torch.get_rng_state(), np.random.get_state()[1].copy(), random.getstate())
    torch.manual_seed(777)
    np.random.seed(777)
    random.seed(777)
    lidar.Decoder(**c["decoder_specs"])                                  # the new decoder's initial weights: the only draw
    assert torch.equal(after[0], torch.get_rng_state())
    assert np.array_equal(after[1], np.random.get_state()[1]) and after[2] == random.getstate()
    assert torch.equal(s.tracker.generator.get_state(), torch.Generator().manual_seed(777).get_state())
    assert torch.equal(s.mapper.generator.get_state(), torch.Generator().manual_seed(778).get_state())
    assert s.base is None and s.tracker.place is None and s.mapper.frozen_rows == 0 and s.mapper.train_decoder is True
    assert cpu_slam == [{"reserve_nodes": 1 << 20, "reserve_rows": 1 << 20}]
    first = s.tracker.first_frame()                                     # get_init_pose, as before
    assert torch.allclose(first.get_pose().detach()[:3, 3], torch.full((3,), float(POSE_OFFSET)))
    monkeypatch.setattr(slam, "run_pipeline", lambda tracker, mapper, streams: None)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
    summary = s.run()
    assert "base" not in summary and set(summary) == {"scans", "keyframes", "wall_ms", "ms_per_scan_wall", "ms_per_scan", "init_ms",
                                                     "refine_ms", "out_dir"}
