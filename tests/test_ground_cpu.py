"""Ground segmentation without a GPU: the NumPy restatement (tests/ground_ref.py) at bin edges, its eigen-solve, its results on the
canyon scan and on a terrain scene, the scan loaders' parsing and filters, the C ABI's argument checks, and the `dataset` seam."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import ground_ref as GR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


@pytest.fixture(scope="module")
def params(nl):
    return nl.ground.GroundParams()


def polar(r, th, z=-1.7):
    return np.array([[r * np.cos(t), r * np.sin(t), z] for r, t in zip(np.broadcast_to(r, np.shape(th)), th)], np.float32)


def terrain_scene(seed=0, n=120_000):
    """A road along x rising at 4 % (z = -1.723 + 0.04 x), kerbs 0.12 m high at |y| = 6 with pavement beyond, two 1.6 m boxes on the
    road and a wall at y = 11, sampled like a spinning sensor (density ~ 1/r) with 0.02 m noise.  Returns the points, a mask of the
    true ground (road and pavement) and the height of every point above the surface under it."""
    rng = np.random.default_rng(seed)
    r = rng.uniform(2.8, 45.0, n)
    th = rng.uniform(-np.pi, np.pi, n)
    x, y = r * np.cos(th), r * np.sin(th)
    surf = lambda x, y: -1.723 + 0.04 * x + np.where(np.abs(y) > 6.0, 0.12, 0.0)
    z = surf(x, y)
    keep = np.abs(y) < 11.0
    x, y, z = x[keep], y[keep], z[keep]
    ground = np.ones(x.size, bool)
    parts = [(x, y, z)]
    for cx, cy in ((9.0, 2.5), (-14.0, -3.0)):                          # boxes 2 x 2 x 1.6 m: four sides and the top
        m = 6000
        u, h = rng.uniform(-1, 1, m), rng.uniform(0.0, 1.6, m)
        side = rng.integers(0, 5, m)
        bx = np.where(side == 0, -1.0, np.where(side == 1, 1.0, u))
        by = np.where(side == 2, -1.0, np.where(side == 3, 1.0, np.where(side == 4, rng.uniform(-1, 1, m), u)))
        bz = np.where(side == 4, 1.6, h)
        parts.append((cx + bx, cy + by, surf(cx + bx, cy + by) + bz))
    m = 15000                                                            # the wall
    wx, wz = rng.uniform(-40, 40, m), rng.uniform(0.0, 4.0, m)
    parts.append((wx, np.full(m, 11.0), surf(wx, np.full(m, 11.0)) + wz))
    X = np.concatenate([np.stack(p, 1) for p in parts])
    is_ground = np.concatenate([ground] + [np.zeros(p[0].size, bool) for p in parts[1:]])
    X = X + rng.normal(0.0, 0.02, X.shape)
    height = X[:, 2] - surf(X[:, 0], X[:, 1])
    return X.astype(np.float32), is_ground, height


# ---- restatement ------------------------------------------------------------------------------------------------------------
def test_binning_at_ring_and_sector_edges(params):
    b = GR.zone_edges(params)
    assert b == (2.7, (7 * 2.7 + 80) / 8, (3 * 2.7 + 80) / 4, (2.7 + 80) / 2, 80.0)
    assert GR.n_patches(params) == 504
    w0 = (b[1] - b[0]) / 2
    pts = np.array([[2.7, 0, -1.7], [np.nextafter(np.float32(2.7), np.float32(0)), 0, -1.7], [80.0, 0, -1.7],
                    [np.nextafter(np.float32(80), np.float32(0)), 0, -1.7], [0, 0, 0], [np.nan, 1, 1]], np.float32)
    pid, zone, ring, _ = GR.bin_points(pts, params)
    assert pid.tolist()[:2] == [0, -1]                                   # min_range is inside, just below it is outside
    assert pid[2] == -1 and zone[3] == 3 and ring[3] == 13                # max_range is outside, just below: the last ring
    assert pid[3] == 504 - 32                                            # theta = 0: sector 0 of zone 3's last ring
    assert pid[4] == -1 and pid[5] == -1
    # ring edges in zone 0 (the float32 row is what is binned: take points whose fp64 radius is exactly representable)
    r = np.float32(b[0] + w0 + 0.01)
    assert GR.bin_points(polar(r, [0.0]), params)[0][0] == 16           # ring 1 of zone 0
    r = np.float32(b[0] + w0 - 0.01)
    assert GR.bin_points(polar(r, [0.0]), params)[0][0] == 0
    # sector edges: 16 sectors in zone 0; theta just past pi / 8 is sector 1, negative angles wrap to the last sectors
    th = np.array([np.pi / 8 + 1e-6, np.pi / 8 - 1e-6, -1e-6, -np.pi + 1e-6, np.pi - 1e-6])
    assert GR.bin_points(polar(4.0, th), params)[0].tolist() == [1, 0, 15, 8, 7]
    # zone edges: b1 starts zone 1 (patch 32), whose ring 0 has 32 sectors
    assert GR.bin_points(polar(np.float32(b[1] + 1e-3), [0.0]), params)[0][0] == 32
    assert GR.bin_points(polar(np.float32(b[1] - 1e-3), [0.0]), params)[0][0] == 16
    assert GR.bin_points(polar(np.float32(b[3] + 1e-3), [np.pi / 2 + 1e-3]), params)[0][0] == 32 + 128 + 216 + 8
    assert GR.bin_points(polar(np.float32(b[3] + 1e-3), [np.pi / 2 + 1e-3]), params)[2][0] == 10


def test_eigen_solve_matches_eigh():
    rng = np.random.default_rng(3)
    cases = [np.diag([3.0, 1.0, 2.0]), np.zeros((3, 3)), np.eye(3), np.diag([1.0, 1.0, 1e-12])]
    for _ in range(200):
        A = rng.normal(size=(3, 3)) * rng.uniform(1e-3, 1e3)
        cases.append(A @ A.T)
    for C in cases:
        lam, V = GR.eig3(C)
        w = np.linalg.eigh(C)[0]
        scale = max(1.0, np.abs(w).max())
        assert np.allclose(np.sort(lam), w, rtol=0, atol=1e-12 * scale)
        assert np.allclose(V.T @ V, np.eye(3), atol=1e-12)
        assert np.allclose(C @ V, V * lam, atol=1e-10 * scale)


def test_canyon_scan(nl, params):
    """The canyon scan of synthetic.make_scan: 99.96 % of the true ground returns are labelled ground.  Their cosines are within 0.02
    of the analytic |d_z| for 85.5 % and within 0.14 for all: in the patches of zone 0's outer ring that hold a wall, the wall's
    lowest returns fall inside the th_dist band and tilt the plane towards the wall, by up to 0.14 in n after three fits, and the
    nearby ground points take that normal.  Patchwork++ removes such returns by region-wise vertical plane fitting, which is not built
    here (DESIGN.md section 12)."""
    pts, cos, _ = nl.synthetic.make_scan()
    r = GR.segment(pts, params)
    true = cos < 1.0
    lab = r["label"] == 1
    assert (lab & true).sum() >= 0.99 * true.sum()
    err = np.abs(r["cos"] - cos)[lab & true]
    assert (err < 0.02).mean() >= 0.83
    assert err.max() < 0.16
    assert (r["cos"][~lab] == 1.0).all()
    assert r["counts"].tolist() == [lab.sum(), (~lab).sum(), 0, 0]


def test_terrain_scene(params):
    """Road of 4 % grade, 0.12 m kerbs, 1.6 m boxes and a wall.  Measured with the restatement on this scene (80 749 points, 24 042 of
    them 0.3 m or more above the surface): ground recall 0.9995, and none of the high points labelled ground."""
    X, truth, height = terrain_scene()
    r = GR.segment(X, params)
    lab = r["label"] == 1
    recall = (lab & truth).sum() / truth.sum()
    high = height >= 0.3
    false_share = (lab & high).sum() / high.sum()
    assert recall >= 0.99, recall
    assert false_share <= 0.005, false_share


def test_points_and_cos_order(params):
    X, _, _ = terrain_scene(seed=1, n=20_000)
    r = GR.segment(X, params)
    P, c, idx = GR.points_and_cos(X, params)
    g = int(r["counts"][0])
    assert np.all(np.diff(idx[:g]) > 0) and np.all(np.diff(idx[g:]) > 0)
    assert (r["label"][idx[:g]] == 1).all() and (r["label"][idx[g:]] == 0).all()
    assert np.array_equal(P, X[idx]) and np.array_equal(c, r["cos"][idx])


# ---- loaders ----------------------------------------------------------------------------------------------------------------
def _write_sequence(root, name_fmt, pose_file, scans, poses):
    os.makedirs(os.path.join(root, "velodyne"))
    for i, s in enumerate(scans):
        s.astype(np.float32).tofile(os.path.join(root, "velodyne", name_fmt.format(i)))
    np.savetxt(os.path.join(root, pose_file), np.stack([p[:3].reshape(12) for p in poses]))


def _scan_rows():
    return np.array([[1, 0, 0, 0.5], [3, 4, 0, 0.1], [0, 0, -3.5, 0.2], [10, 0, 0, 0.3], [0, 0, -3.0, 0.0], [6, 8, 0, 0.9]], np.float32)


@pytest.mark.parametrize("name", ["kitti", "maicity"])
def test_loader_parsing_and_filters(nl, tmp_path, name):
    mod = getattr(nl.dataset, name)
    fmt, pose_file = ("{:06d}.bin", "poses_lidar.txt") if name == "kitti" else ("{:05d}.bin", "poses.txt")
    poses = [np.eye(4), np.eye(4)]
    poses[1][:3, 3] = (1.5, -2.0, 0.25)
    poses[1][:3, :3] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]
    _write_sequence(str(tmp_path), fmt, pose_file, [_scan_rows(), _scan_rows()[:2]], poses)
    assert os.path.exists(os.path.join(tmp_path, "velodyne", fmt.format(1)))
    d = mod.DataLoader(str(tmp_path))
    assert len(d) == 2 and d.gt_pose is None and np.array_equal(d.get_init_pose(1), np.eye(4))
    z_kept = [r for r in _scan_rows() if r[2] > -3.0] if name == "kitti" else list(_scan_rows())
    assert np.array_equal(d.read_points(0), np.array(z_kept, np.float32))
    d = mod.DataLoader(str(tmp_path), use_gt=True, max_depth=9.5, min_depth=2.0)
    assert d.gt_pose.shape == (2, 12)
    assert np.allclose(d.get_init_pose(1), poses[1]) and d.get_init_pose(1) is not d.get_init_pose(1)
    norms = np.linalg.norm(np.array(z_kept)[:, :3], axis=1)
    want = np.array(z_kept, np.float32)[(norms < 9.5) & (norms > 2.0)]
    assert np.array_equal(d.read_points(0), want)
    assert d.read_points(1).shape == (1, 4)                                # |(3, 4, 0)| = 5 passes, |(1, 0, 0)| = 1 does not


def test_c_abi_rejects_bad_arguments(nl):
    L = nl._capi.lib()
    err = lambda: L.nl_last_error().decode()
    ws, out, pts = (ctypes.c_void_p(256 * k) for k in (1, 2, 3))        # never dereferenced: every call below fails its checks
    good = nl.ground.GroundParams()

    def call(p=None, **kw):
        args = dict(n=5, pts=pts, stride=3, ws=ws, wsb=1 << 30, label=out, cos=out, patch=None, patches=None, counts=out)
        args.update(kw)
        return L.nl_ground_segment(args["n"], args["pts"], args["stride"], (p or good).to_c(), args["ws"], args["wsb"], args["label"],
                                   args["cos"], args["patch"], args["patches"], args["counts"], None)
    import dataclasses
    bad = lambda **kw: dataclasses.replace(good, **kw)
    assert call(n=-1) != 0 and "n must be" in err()
    for s in (0, 2, 5):
        assert call(stride=s) != 0 and "stride" in err()
    assert call(bad(num_rings_each_zone=(2, 0, 4, 4))) != 0 and "positive" in err()
    assert call(bad(num_sectors_each_zone=(16, 32, -1, 32))) != 0 and "positive" in err()
    assert call(bad(num_sectors_each_zone=(16, 32, 54, 200))) != 0 and "NL_GROUND_MAX_PATCHES" in err()
    for lo, hi in ((0.0, 80.0), (-1.0, 80.0), (10.0, 10.0), (20.0, 10.0), (2.7, float("inf")), (float("nan"), 80.0)):
        assert call(bad(min_range=lo, max_range=hi)) != 0 and "min_range" in err(), (lo, hi)
    for k in (0, -3, 1025):
        assert call(bad(num_lpr=k)) != 0 and "num_lpr" in err()
    assert call(bad(num_iter=0)) != 0 and "num_iter" in err()
    assert call(bad(th_dist=float("nan"))) != 0 and "finite" in err()
    for k in ("pts", "label", "cos", "counts"):
        assert call(**{k: None}) != 0 and "null" in err(), k
    assert call(wsb=100) != 0 and "workspace" in err()
    assert call(ws=ctypes.c_void_p(256 + 8)) != 0 and "aligned" in err()
    assert L.nl_ground_workspace_bytes(-1) < 0 and "n must be" in err()
    with pytest.raises(ValueError):
        bad(elevation_thr=(0.5, 0.7)).to_c()
    part = lambda **kw: L.nl_ground_partition(*[kw.get(k, v) for k, v in (("n", 5), ("pts", pts), ("stride", 4), ("label", out), ("cos", out),
                                                                          ("ws", ws), ("wsb", 1 << 30), ("op", out), ("oc", out),
                                                                          ("oi", out), ("st", None))])
    assert part(n=-1) != 0 and "n must be" in err()
    assert part(stride=2) != 0 and "stride" in err()
    for k in ("pts", "label", "cos", "op", "oc", "oi"):
        assert part(**{k: None}) != 0 and "null" in err(), k
    assert part(wsb=10) != 0 and "workspace" in err()


def test_dataset_seam_in_a_subprocess(tmp_path):
    _write_sequence(str(tmp_path), "{:06d}.bin", "poses_lidar.txt", [_scan_rows()], [np.eye(4)])
    code = f"""
import importlib, sys
sys.path.insert(0, {ROOT!r})
import nerfloam_b200
sys.modules["dataset"] = nerfloam_b200.dataset
mod = importlib.import_module("dataset.kitti")
d = mod.DataLoader({str(tmp_path)!r}, use_gt=True)
assert mod.__name__ == "dataset.kitti" and len(d) == 1
print(d.read_points(0).shape[0], d.get_init_pose(0).shape)
"""
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    assert out.stdout.split()[0] == "4"                                    # the rows at z = -3.5 and z = -3.0 are dropped
