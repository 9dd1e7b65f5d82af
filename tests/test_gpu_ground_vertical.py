"""The vertical-structure filter of the ground segmentation on the GPU (csrc/ground.cu through ground.py) against the NumPy restatement
(tests/ground_vertical_ref.py), value by value, plus reproducibility, stride 4, empty and all-vertical input, and the SLAM loop end to end
on KITTI-layout scans with the filter on."""
import dataclasses
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import ground_vertical_ref as GV
from test_ground_cpu import terrain_scene
from test_gpu_ground import dense_scan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-9


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


@pytest.fixture(scope="module")
def params(nl):
    return nl.ground.GroundParams(vertical_cell=0.2, vertical_height=0.3)


def run(nl, pts, params):
    g = nl.ground.segment_ground(pts, params)
    rec = {k: v.cpu().numpy() for k, v in g.patches._asdict().items()}
    return dict(label=g.label.cpu().numpy(), cos=g.cos.cpu().numpy(), patch=g.patch.cpu().numpy(), counts=g.counts.cpu().numpy(),
                vertical=g.vertical.cpu().numpy(), rec=rec)


def compare(nl, pts, params):
    """Kernel against restatement.  The vertical flags are exact (integer cell keys, fp64 extents of fp32 values) and must match
    everywhere; the rest takes tests/test_gpu_ground.py's tolerances and exemptions."""
    k = run(nl, pts, params)
    r = GV.segment(pts, params)
    R = r["patches"]
    assert np.array_equal(k["vertical"], r["vertical"])
    edge = r["edge_margin"] < TOL
    assert np.array_equal(k["patch"][~edge], r["patch"][~edge])
    same_bins = np.array_equal(k["patch"], r["patch"])
    touched = np.unique(r["patch"][edge]) if edge.any() else np.array([], np.int64)
    exempt = (R["cut_margin"] < 1e-6) | (R["verdict_margin"] < TOL)
    exempt[touched[touched >= 0]] = True
    ok = ~exempt
    for f in ("n_points", "n_vertical", "ground", "n_ground"):
        assert np.array_equal(k["rec"][f][ok], R[f][ok]), f
    assert np.array_equal(k["rec"]["ring"], R["ring"])
    fit = ok & np.isfinite(R["d"])
    assert np.array_equal(np.isfinite(k["rec"]["d"][ok]), np.isfinite(R["d"][ok]))
    for f in ("mean", "d", "lambda_min"):
        assert np.abs(k["rec"][f][fit] - R[f][fit]).max(initial=0) < TOL, f
    nfit = fit & (R["eig_gap"] >= TOL)
    assert np.abs(k["rec"]["normal"][nfit] - R["normal"][nfit]).max(initial=0) < TOL
    pt_ok = (ok[np.maximum(r["patch"], 0)] | (r["patch"] < 0)) & ~edge
    assert np.array_equal(k["label"][pt_ok], r["label"][pt_ok])
    assert (k["label"][k["vertical"] == 1] == 0).all() and (k["cos"][k["vertical"] == 1] == 1.0).all()
    agree = pt_ok & (k["label"] == r["label"]) & (r["tie"] >= TOL)
    assert np.abs(k["cos"][agree].astype(np.float64) - r["cos"][agree]).max(initial=0) <= 1e-6
    assert k["counts"][2:].tolist() == r["counts"][2:].tolist()
    if same_bins and ok.all():
        assert k["counts"].tolist() == r["counts"].tolist()
    report = dict(points=len(pts), vertical=int(k["vertical"].sum()), ground=int(k["counts"][0]), exempt_patches=int(exempt.sum()),
                  edge_points=int(edge.sum()), cell_edge_points=int((r["cell_margin"] < TOL).sum()),
                  smallest_cell_margin=float(r["cell_margin"].min()), smallest_cut_margin_m=float(R["cut_margin"].min()),
                  largest_patch=int(R["n_points"].max()))
    print(report)
    return report


def test_canyon_scan_matches_the_restatement(nl, params):
    pts, _, _ = nl.synthetic.make_scan()
    rep = compare(nl, pts, params)
    assert rep["vertical"] > 30_000 and rep["ground"] > 40_000


def test_terrain_scene_matches_the_restatement(nl, params):
    rep = compare(nl, terrain_scene()[0], params)
    assert rep["vertical"] > 20_000


def test_dense_patch_matches_the_restatement(nl, params):
    pts = dense_scan()
    rng = np.random.default_rng(8)                                       # a few poles inside the dense patch, so it holds vertical rows
    poles = np.concatenate([np.stack([np.full(40, x), np.full(40, y), np.linspace(-1.7, 0.5, 40)], 1)
                            for x, y in zip(rng.uniform(3.5, 5.5, 6), rng.uniform(0.5, 1.2, 6))]).astype(np.float32)
    rep = compare(nl, np.concatenate([pts, poles]), params)
    assert rep["largest_patch"] > 20_000 and rep["vertical"] >= 240


def test_rows_on_cell_edges(nl, params):
    """Rows snapped onto cell edges (a binary cell width, so the edges are exact in fp32) and one ulp either side of them."""
    p = dataclasses.replace(params, vertical_cell=0.25)
    pts, _, _ = nl.synthetic.make_scan(seed=21)
    rng = np.random.default_rng(9)
    rows = rng.choice(len(pts), 6000, replace=False)
    snapped = (np.round(pts[rows, :2] / np.float32(0.25)) * np.float32(0.25)).astype(np.float32)
    side = rng.integers(-1, 2, snapped.shape)
    snapped = np.where(side < 0, np.nextafter(snapped, np.float32(-np.inf)), np.where(side > 0, np.nextafter(snapped, np.float32(np.inf)), snapped))
    pts = pts.copy()
    pts[rows, :2] = snapped
    rep = compare(nl, pts, p)
    assert rep["cell_edge_points"] >= 2000 and rep["smallest_cell_margin"] == 0.0           # 5 / 9 of them keep x or y on an edge


def test_two_calls_identical_and_stride4_equals_stride3(nl, params):
    pts, _, _ = nl.synthetic.make_scan(seed=11)
    a, b = run(nl, pts, params), run(nl, pts, params)
    p4 = np.concatenate([pts, np.random.default_rng(0).uniform(0, 1, (len(pts), 1)).astype(np.float32)], 1)
    c = run(nl, p4, params)
    assert a["vertical"].sum() > 0
    for x in (b, c):
        for f in ("label", "cos", "patch", "counts", "vertical"):
            assert x[f].tobytes() == a[f].tobytes(), f
        for f in a["rec"]:
            assert x["rec"][f].tobytes() == a["rec"][f].tobytes(), f
    P3, C3, I3 = (t.cpu().numpy() for t in nl.ground.points_and_cos(pts, params))
    P4, C4, I4 = (t.cpu().numpy() for t in nl.ground.points_and_cos(torch.from_numpy(p4).cuda(), params))
    assert P3.tobytes() == P4.tobytes() and C3.tobytes() == C4.tobytes() and I3.tobytes() == I4.tobytes()
    g = int(a["counts"][0])
    assert np.array_equal(P3, pts[I3]) and np.array_equal(C3, a["cos"][I3]) and (a["label"][I3[:g]] == 1).all()
    # the filter off after a call with it on: the unfiltered bytes, and no vertical mask
    off = nl.ground.segment_ground(pts, dataclasses.replace(params, vertical_cell=0.0))
    ref = nl.ground.segment_ground(pts, nl.ground.GroundParams())
    assert off.vertical is None and (off.patches.n_vertical == 0).all()
    assert off.label.cpu().numpy().tobytes() == ref.label.cpu().numpy().tobytes()
    assert off.cos.cpu().numpy().tobytes() == ref.cos.cpu().numpy().tobytes()


def test_empty_and_all_vertical_input(nl, params):
    g = run(nl, np.zeros((0, 3), np.float32), params)
    assert g["counts"].tolist() == [0, 0, 0, 0] and g["vertical"].shape == (0,)
    assert (g["rec"]["n_points"] == 0).all() and (g["rec"]["n_vertical"] == 0).all() and (g["rec"]["ground"] == 0).all()
    P, C, I = nl.ground.points_and_cos(np.zeros((0, 4), np.float32), params)
    assert P.shape == (0, 3) and C.shape == (0,) and I.shape == (0,)
    rng = np.random.default_rng(12)                                      # 60 poles, 2.2 m tall, 30 returns each, plus two rows outside
    r, th = rng.uniform(3.0, 60.0, 60), rng.uniform(0, 2 * np.pi, 60)
    poles = np.concatenate([np.stack([np.full(30, a), np.full(30, b), np.linspace(-1.7, 0.5, 30)], 1)
                            for a, b in zip(r * np.cos(th), r * np.sin(th))])
    pts = np.concatenate([poles, [[0.5, 0.5, -1.7], [0.5, 0.5, 1.0]]]).astype(np.float32)
    g = run(nl, pts, params)
    n = len(pts)
    assert g["vertical"][:-2].all() and not g["vertical"][-2:].any()
    assert g["counts"].tolist() == [0, n, 2, 0] and (g["label"] == 0).all() and (g["cos"] == 1.0).all()
    rec = g["rec"]
    assert np.array_equal(rec["n_vertical"], rec["n_points"]) and rec["n_vertical"].sum() == n - 2
    assert (rec["ground"] == 0).all() and np.isnan(rec["d"]).all()
    ref = GV.segment(pts, params)
    assert np.array_equal(g["vertical"], ref["vertical"]) and np.array_equal(rec["n_vertical"], ref["patches"]["n_vertical"])


def test_slam_loop_on_kitti_layout_scans_with_the_filter(nl, tmp_path):
    """Six canyon scans written as KITTI .bin files, run through demo_slam.py --data --vertical-cell 0.2: the bounds of the unfiltered
    run (0.10 m, 0.01 Frobenius) hold."""
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
                          "--init-calls", "8", "--vertical-cell", "0.2"], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    d = json.loads(out.stdout.strip().splitlines()[-1])
    print({k: d[k] for k in ("scans", "vertical_cell", "translation_error_m", "rotation_error_fro", "ground_points")})
    assert d["scans"] == 6 and d["vertical_cell"] == 0.2
    assert d["translation_error_m"]["max"] < 0.10 and d["rotation_error_fro"]["max"] < 0.01, d
