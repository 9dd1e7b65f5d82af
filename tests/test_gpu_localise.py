"""localise.Localiser on the GPU: a street drive mapped by slam.NeRFLOAM and saved with save_map, then a second pass over the same
route (new scan noise, shifted 0.5 m and turned 10 degrees, no pose guess) localised in the file; the file restored onto both octrees
against the map it was saved from; the three sources localising alike; the map untouched by a run; a scan the map cannot explain; and
scripts/localise.py.

The drive is the street scene (synthetic.make_street_scan), not the canyon of test_gpu_slam.py: a half turn or a shift along x maps
the canyon onto itself, so no search could tell its placements apart.  The run maps with the true poses (use_gt), so the map frame is
the scene's frame and the localised poses can be held to the true ones."""
import importlib
import json
import math
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
share = importlib.import_module("nerf-loam_b200.share")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_MAP, SPACING = 12, 0.5
SHIFT, TURN = (0.3, 0.4, 0.0), math.radians(10.0)          # the second pass: 0.5 m and 10 degrees from the first run's start
N_PASS = 8
MAX_DT, MAX_DR = 0.10, 0.01                                  # metres; Frobenius norm of the rotation difference (demo_slam.py's)


@pytest.fixture(scope="module")
def nl():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    sys.path.insert(0, ROOT)
    return importlib.import_module("nerfloam_b200")


def street(nl, i, seed, shift=(0.0, 0.0, 0.0), turn=0.0):
    """Scan i of the route (x = SPACING i, a small weave in y and heading), moved by `shift` and turned by `turn`; the pose without
    POSE_OFFSET, as loaders return it."""
    syn = nl.synthetic
    xyz = (SPACING * i + shift[0], 0.05 * np.sin(0.7 * i) + shift[1], shift[2])
    pts, cos, pose = syn.make_street_scan(xyz, 0.01 * np.sin(0.5 * i) + turn, seed=seed)
    pose = pose.astype(np.float64)
    pose[:3, 3] -= syn.POSE_OFFSET
    return pts, cos, pose


class MemoryStream:
    def __init__(self, scans, use_gt):
        self.scans, self.use_gt = scans, use_gt

    def __len__(self):
        return len(self.scans)

    def __getitem__(self, i):
        pts, cos, pose = self.scans[i][:3]
        return i, torch.from_numpy(pts), torch.from_numpy(cos), (pose.copy() if self.use_gt else None)

    def get_init_pose(self, i):
        return self.scans[i][2].copy() if self.use_gt else np.eye(4)


def config():
    return {"dataset": "kitti", "seeding": 777, "data_specs": {"data_path": "", "use_gt": True, "max_depth": 40, "min_depth": 1.5},
            "criteria": {"sdf_weight": 10000.0, "fs_weight": 1, "eiko_weight": 0.1, "sdf_truncation": 0.3},
            "decoder_specs": {"depth": 2, "width": 256, "in_dim": 16, "skips": [], "embedder": "none", "multires": 0},
            "tracker_specs": {"N_rays": 2048, "learning_rate": 0.01, "step_size": 0.2, "max_voxel_hit": 20, "num_iterations": 25,
                              "start_frame": 0, "end_frame": -1, "read_offset": 1},
            "mapper_specs": {"N_rays_each": 2048, "use_local_coord": False, "voxel_size": 0.3, "step_size": 0.5, "window_size": 4,
                             "num_iterations": 25, "max_voxel_hit": 20, "final_iter": False, "mesh_res": 2,
                             "learning_rate_emb": 0.01, "learning_rate_decorder": 0.005, "learning_rate_pose": 0.001, "freeze_frame": 5,
                             "keyframe_gap": 1.0, "remove_back": False, "key_distance": 12},
            "debug_args": {"verbose": False, "mesh_freq": 0}}


@pytest.fixture(scope="module")
def run(nl, tmp_path_factory):
    tmp = tmp_path_factory.mktemp("localise")
    scans = [street(nl, i, seed=2000 + i) for i in range(N_MAP)]
    s = nl.slam.NeRFLOAM(config(), str(tmp / "run"), data_stream=MemoryStream(scans, True))
    s.run()
    torch.cuda.synchronize()
    path = tmp / "run.map"
    s.save_map(path)
    second = [street(nl, i, seed=5000 + i, shift=SHIFT, turn=TURN) for i in range(N_PASS)]
    return SimpleNamespace(slam=s, path=path, second=second, tmp=tmp)


def errors(poses, truth):
    """(translation error m, Frobenius norm of the rotation difference) per pose, both f64[S,4,4] without POSE_OFFSET."""
    T, G = torch.as_tensor(poses, dtype=torch.float64), torch.as_tensor(np.asarray(truth), dtype=torch.float64)
    return (T[:, :3, 3] - G[:, :3, 3]).norm(dim=-1), torch.linalg.matrix_norm(T[:, :3, :3] - G[:, :3, :3])


def test_second_pass_localised_without_a_guess(nl, run, monkeypatch):
    """Every scan of the second pass within 0.10 m and 0.01 of its true pose, the first scan's placement too; frame_poses.txt holds
    the poses; the captured tracking iteration is built once per tracking rate (scan 1 runs at twice the rate of the later scans)."""
    rh = nl.render_helpers
    builds = []
    init = rh._TrackGraph.__init__

    def counting(self, *a, **kw):
        builds.append(1)
        init(self, *a, **kw)
    monkeypatch.setattr(rh._TrackGraph, "__init__", counting)
    loc = nl.localise.Localiser(str(run.path), MemoryStream(run.second, False), generator=torch.Generator().manual_seed(1),
                                out_dir=str(run.tmp / "pass"))
    res = loc.run()
    truth = np.stack([p[2] for p in run.second])
    dt, dr = errors(res.poses, truth)
    summary = loc.summary(res)
    print("translation error (m):", np.round(dt.numpy(), 4).tolist())
    print("rotation error (Frobenius):", np.round(dr.numpy(), 5).tolist())
    print("loss:", np.round(res.loss.numpy(), 5).tolist(), "hit fraction:", np.round(res.hit_fraction.numpy(), 3).tolist())
    print("summary:", json.dumps(summary))
    assert res.scan_ids.tolist() == list(range(N_PASS))
    assert float(dt.max()) < MAX_DT and float(dr.max()) < MAX_DR
    P = nl.se3pose.OptimizablePose(res.placement.pose.data.detach().cpu().float().clone()).matrix().detach().double()
    P[:3, 3] -= nl.frame.POSE_OFFSET
    pdt, pdr = errors(P[None], truth[:1])
    assert float(pdt[0]) < MAX_DT and float(pdr[0]) < MAX_DR
    assert bool(torch.isfinite(res.loss).all()) and float(res.hit_fraction.min()) > 0.5
    written = np.loadtxt(run.tmp / "pass" / "frame_poses.txt", ndmin=2).reshape(-1, 3, 4)
    assert written.shape == (N_PASS, 3, 4) and np.abs(written - res.poses[:, :3, :].numpy()).max() < 1e-5
    assert len(builds) <= 2, len(builds)


def _bytes(t):
    return t.detach().contiguous().reshape(-1).view(torch.uint8)


def _buffers(ms, decoder):
    """Everything tracking reads of a map, as bytes: the hot-path arrays, the packed child image, the embedding rows, the decoder."""
    return {"centres": _bytes(ms.centres), "structure": _bytes(ms.structure), "vox2row": _bytes(ms.vox2row),
            "packed": _bytes(ms.packed_children()), "emb": _bytes(ms.emb), "decoder": _bytes(share._flat_decoder_state(decoder))}


def _same(a, b):
    for k in a:
        assert a[k].numel() == b[k].numel() and torch.equal(a[k], b[k]), k


def test_file_restores_what_tracking_reads_on_both_octrees(nl, run):
    mu = run.slam.mapper.map
    want = _buffers(mu.map_states["_mapstate"], run.slam.mapper.decoder)
    for octree in ("host", "device"):
        saved = nl.slam.load_map(run.path, octree=octree)
        assert saved.map.on_device == (octree == "device")
        _same(_buffers(saved.map.map_states["_mapstate"], saved.decoder), want)
        assert np.array_equal(saved.map.vertex2row, mu.vertex2row)
        assert saved.scan_ids.tolist() == list(range(N_MAP))
        frame_poses = np.loadtxt(run.tmp / "run" / "misc" / "frame_poses.txt", ndmin=2).reshape(-1, 3, 4)
        assert np.abs(saved.trajectory[:, :3, :].numpy() - frame_poses).max() < 1e-5


def test_three_sources_agree_and_leave_the_map_unchanged(nl, run):
    """The in-memory map, the file on the host tree and the file on the device tree, localised with the same generator seed: poses
    within 1 cm and 1e-3 of one another (fp32 atomics sum the pose gradient, so tracking is not bit-reproducible), and each map's
    buffers byte-identical before and after its run."""
    sources = {"memory": run.slam.saved_map(), "host": nl.slam.load_map(run.path, octree="host"),
               "device": nl.slam.load_map(run.path, octree="device")}
    poses = {}
    for name, saved in sources.items():
        before = {k: v.clone() for k, v in _buffers(saved.map.map_states["_mapstate"], saved.decoder).items()}
        loc = nl.localise.Localiser(saved, MemoryStream(run.second, False), generator=torch.Generator().manual_seed(7))
        poses[name] = loc.run().poses
        torch.cuda.synchronize()
        _same(_buffers(saved.map.map_states["_mapstate"], saved.decoder), before)
    for name in ("host", "device"):
        dt, dr = errors(poses[name], poses["memory"])
        print(f"{name} against memory: {float(dt.max()):.3g} m, {float(dr.max()):.3g}")
        assert float(dt.max()) < 0.01 and float(dr.max()) < 1e-3, name


def test_scan_the_map_cannot_explain_raises(nl, run):
    """A scan whose every return lies 20-30 m away at 70-85 degrees of elevation: from no placement near the trajectory does a ray
    reach the map (the street's walls end 7.3 m up), so run() raises on the first scan instead of keeping a constant pose."""
    rng = np.random.default_rng(0)
    n = 6000
    el, az, r = np.deg2rad(rng.uniform(70, 85, n)), rng.uniform(-np.pi, np.pi, n), rng.uniform(20, 30, n)
    pts = (np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1) * r[:, None]).astype(np.float32)
    loc = nl.localise.Localiser(str(run.path), MemoryStream([(pts, np.ones(n, np.float32), np.eye(4))], False))
    with pytest.raises(nl._capi.NerfLoamError, match="could not be placed"):
        loc.run()


def test_localise_script(nl, run):
    seq = run.tmp / "seq"
    os.makedirs(seq / "velodyne", exist_ok=True)
    for i, (pts, _, _) in enumerate(run.second[:6]):
        np.concatenate([pts, np.zeros((pts.shape[0], 1), np.float32)], 1).astype(np.float32).tofile(str(seq / "velodyne" / f"{i:06d}.bin"))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "localise.py"), str(run.path), "--data", str(seq), "--out",
                          str(run.tmp / "script")], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    summary = json.loads(out.stdout.strip().splitlines()[-1])
    print(summary)
    assert summary["scans"] == 6 and summary["placement"]["placements"] > 0
    assert {"load", "track", "score"} <= set(summary["ms_per_scan"]) and math.isfinite(summary["median_loss"])
    assert np.loadtxt(run.tmp / "script" / "frame_poses.txt", ndmin=2).shape == (6, 12)
