"""Ground segmentation on the GPU (csrc/ground.cu through ground.py) against the NumPy restatement (tests/ground_ref.py), value by value,
plus reproducibility, edge cases, and the SLAM loop end to end on KITTI-layout scans through dataset.kitti."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import ground_ref as GR
from test_ground_cpu import terrain_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-9


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


@pytest.fixture(scope="module")
def params(nl):
    return nl.ground.GroundParams()


def dense_scan(seed=5):
    """A scan with one patch of more than 20 000 points (a dense disc of ground near the sensor at theta ~ 0.2) plus sparse ground."""
    rng = np.random.default_rng(seed)
    r = rng.uniform(3.0, 6.0, 24_000)
    th = rng.uniform(0.05, 0.35, 24_000)
    dense = np.stack([r * np.cos(th), r * np.sin(th), -1.73 + rng.normal(0, 0.02, r.size)], 1)
    r2, th2 = rng.uniform(3.0, 60.0, 30_000), rng.uniform(0, 2 * np.pi, 30_000)
    sparse = np.stack([r2 * np.cos(th2), r2 * np.sin(th2), -1.73 + 0.01 * r2 * np.sin(th2) + rng.normal(0, 0.02, r2.size)], 1)
    return np.concatenate([dense, sparse]).astype(np.float32)


def run(nl, pts, params):
    g = nl.ground.segment_ground(pts, params)
    rec = {k: v.cpu().numpy() for k, v in g.patches._asdict().items()}
    return dict(label=g.label.cpu().numpy(), cos=g.cos.cpu().numpy(), patch=g.patch.cpu().numpy(), counts=g.counts.cpu().numpy(), rec=rec)


def compare(nl, pts, params):
    """Kernel against restatement with the exemptions of the definitions' knife edges; returns the report."""
    k = run(nl, pts, params)
    r = GR.segment(pts, params)
    R = r["patches"]
    edge = r["edge_margin"] < TOL
    assert np.array_equal(k["patch"][~edge], r["patch"][~edge])
    same_bins = np.array_equal(k["patch"], r["patch"])
    # patches whose points all binned alike, whose cuts are clear of every point by 1e-6 m and whose verdict is clear of its thresholds
    touched = np.unique(r["patch"][edge]) if edge.any() else np.array([], np.int64)
    exempt = (R["cut_margin"] < 1e-6) | (R["verdict_margin"] < TOL)
    exempt[touched[touched >= 0]] = True
    ok = ~exempt
    assert np.array_equal(k["rec"]["n_points"][ok], R["n_points"][ok])
    assert np.array_equal(k["rec"]["ring"], R["ring"])
    assert np.array_equal(k["rec"]["ground"][ok], R["ground"][ok])
    assert np.array_equal(k["rec"]["n_ground"][ok], R["n_ground"][ok])
    fit = ok & np.isfinite(R["d"])
    assert np.array_equal(np.isfinite(k["rec"]["d"][ok]), np.isfinite(R["d"][ok]))
    for f in ("mean", "d", "lambda_min"):
        assert np.abs(k["rec"][f][fit] - R[f][fit]).max(initial=0) < TOL, f
    nfit = fit & (R["eig_gap"] >= TOL)
    assert np.abs(k["rec"]["normal"][nfit] - R["normal"][nfit]).max(initial=0) < TOL
    pt_ok = ok[np.maximum(r["patch"], 0)] | (r["patch"] < 0)
    pt_ok &= ~edge
    assert np.array_equal(k["label"][pt_ok], r["label"][pt_ok])
    agree = pt_ok & (k["label"] == r["label"]) & (r["tie"] >= TOL)
    assert np.abs(k["cos"][agree].astype(np.float64) - r["cos"][agree]).max(initial=0) <= 1e-6
    assert k["counts"][2:].tolist() == r["counts"][2:].tolist()
    if same_bins and ok.all():
        assert k["counts"].tolist() == r["counts"].tolist()
    report = dict(points=len(pts), ground=int(k["counts"][0]), exempt_patches=int(exempt.sum()), edge_points=int(edge.sum()),
                  smallest_cut_margin_m=float(R["cut_margin"].min()), ground_patches=int(R["ground"].sum()),
                  largest_patch=int(R["n_points"].max()))
    print(report)
    return report


def test_canyon_scan_matches_the_restatement(nl, params):
    pts, _, _ = nl.synthetic.make_scan()
    rep = compare(nl, pts, params)
    assert rep["ground"] > 40_000


def test_terrain_scene_matches_the_restatement(nl, params):
    compare(nl, terrain_scene()[0], params)


def test_dense_patch_matches_the_restatement(nl, params):
    rep = compare(nl, dense_scan(), params)
    assert rep["largest_patch"] > 20_000


def test_two_calls_identical_and_stride4_equals_stride3(nl, params):
    pts, _, _ = nl.synthetic.make_scan(seed=11)
    a, b = run(nl, pts, params), run(nl, pts, params)
    p4 = np.concatenate([pts, np.random.default_rng(0).uniform(0, 1, (len(pts), 1)).astype(np.float32)], 1)
    c = run(nl, p4, params)
    for x in (b, c):
        for f in ("label", "cos", "patch", "counts"):
            assert x[f].tobytes() == a[f].tobytes(), f
        for f in a["rec"]:
            assert x["rec"][f].tobytes() == a["rec"][f].tobytes(), f
    P3, C3, I3 = (t.cpu().numpy() for t in nl.ground.points_and_cos(pts, params))
    P4, C4, I4 = (t.cpu().numpy() for t in nl.ground.points_and_cos(torch.from_numpy(p4).cuda(), params))
    assert P3.tobytes() == P4.tobytes() and C3.tobytes() == C4.tobytes() and I3.tobytes() == I4.tobytes()
    g = int(a["counts"][0])
    assert np.array_equal(P3, pts[I3]) and np.array_equal(C3, a["cos"][I3])
    assert np.all(np.diff(I3[:g]) > 0) and np.all(np.diff(I3[g:]) > 0) and (a["label"][I3[:g]] == 1).all() and (a["label"][I3[g:]] == 0).all()


def test_edge_cases(nl, params):
    g = run(nl, np.zeros((0, 3), np.float32), params)
    assert g["counts"].tolist() == [0, 0, 0, 0] and (g["rec"]["n_points"] == 0).all() and (g["rec"]["ground"] == 0).all()
    P, C, I = nl.ground.points_and_cos(np.zeros((0, 4), np.float32), params)
    assert P.shape == (0, 3) and C.shape == (0,) and I.shape == (0,)
    far = np.array([[0.5, 0.5, -1.7], [100.0, 0, -1.7], [0, 80.0, -1.7], [-1, 1, 0]], np.float32)
    g = run(nl, far, params)
    assert g["counts"].tolist() == [0, 4, 4, 0] and (g["patch"] == -1).all() and (g["cos"] == 1).all()
    rng = np.random.default_rng(2)
    few = np.stack([4.0 + rng.uniform(0, 0.5, 9), rng.uniform(0, 0.2, 9), -1.73 + rng.normal(0, 0.01, 9)], 1).astype(np.float32)
    ys, zs = np.meshgrid(np.linspace(0.05, 0.35, 30), np.linspace(-1.5, 1.5, 30))
    wall = np.stack([20.0 + rng.normal(0, 0.01, ys.size), ys.reshape(-1), zs.reshape(-1)], 1).astype(np.float32)   # a wall alone
    pts = np.concatenate([few, wall])
    g = run(nl, pts, params)
    r = GR.segment(pts, params)
    assert g["label"].sum() == 0 and (g["cos"] == 1).all()
    ids = np.unique(g["patch"])
    assert len(ids) == 2
    few_id, wall_id = g["patch"][0], g["patch"][-1]
    assert g["rec"]["n_points"][few_id] == 9 and np.isnan(g["rec"]["d"][few_id]) and g["rec"]["ground"][few_id] == 0
    assert g["rec"]["ground"][wall_id] == 0 and abs(g["rec"]["normal"][wall_id][2]) < 0.2
    assert np.array_equal(g["rec"]["ground"], r["patches"]["ground"]) and np.array_equal(g["label"], r["label"])
    assert abs(g["rec"]["normal"][wall_id] - r["patches"]["normal"][wall_id]).max() < TOL


def test_non_finite_row_raises(nl, params):
    pts, _, _ = nl.synthetic.make_scan(n_beams=16, n_az=200)
    for bad in (np.nan, np.inf):
        p = pts.copy()
        p[7, 1] = bad
        with pytest.raises(ValueError, match="non-finite"):
            nl.ground.segment_ground(p, params)
        with pytest.raises(ValueError, match="non-finite"):
            nl.ground.points_and_cos(p, params)


def test_slam_loop_on_kitti_layout_scans(nl, tmp_path):
    """Six canyon scans written as KITTI .bin files with poses_lidar.txt (without the frame offset), run through demo_slam.py --data:
    the bounds of the synthetic loop's end-to-end test hold with the loader's pointsCos."""
    syn = nl.synthetic
    os.makedirs(tmp_path / "velodyne")
    rows = []
    for i in range(6):
        xyz, yaw = syn.path_pose(i, 6, 0.5)
        pts, _, pose = syn.make_scan(seed=1000 + i, sensor_xyz=xyz, yaw=yaw)
        intensity = np.full((len(pts), 1), 0.5, np.float32)
        np.concatenate([pts, intensity], 1).astype(np.float32).tofile(str(tmp_path / "velodyne" / f"{i:06d}.bin"))
        pose = pose.astype(np.float64)
        pose[:3, 3] -= syn.POSE_OFFSET
        rows.append(pose[:3].reshape(12))
    np.savetxt(str(tmp_path / "poses_lidar.txt"), np.stack(rows))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "demo_slam.py"), "--data", str(tmp_path), "--dataset", "kitti",
                          "--init-calls", "8"], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    d = json.loads(out.stdout.strip().splitlines()[-1])
    print({k: d[k] for k in ("scans", "translation_error_m", "rotation_error_fro", "ground_points")})
    assert d["scans"] == 6 and "reconstruction" not in d
    assert d["translation_error_m"]["max"] < 0.10 and d["rotation_error_fro"]["max"] < 0.01, d
