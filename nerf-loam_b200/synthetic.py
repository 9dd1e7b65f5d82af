"""Deterministic synthetic LiDAR scans (no dataset / network needed).

The scene and sensor follow BASELINE.md section 3 / SURVEY.md section 8(d) config 4: a 64-beam
spinning LiDAR (elevation -24.8 .. +2.0 deg) x n_az azimuths inside a box-shaped street canyon:
ground plane z = -1.73 m, walls |y| = 8 m and |x| = 30 m, range noise N(0, 0.02^2) m, range gate
(min_depth, max_depth).  `points` are in the sensor frame like the reference data loaders return
them (src/dataset/kitti.py:75-81), `pointsCos` is |n.d| for ground returns and 1 elsewhere (the
reference computes it with patchwork++ ground segmentation, src/dataset/kitti.py:40-70; ground.points_and_cos computes it from
the points alone, as dataset.kitti / dataset.maicity do for recorded scans).
"""
import numpy as np

POSE_OFFSET = 2000.0  # src/lidarFrame.py:18


def make_scan(n_beams=64, n_az=1563, seed=777, min_depth=5.0, max_depth=40.0, sensor_xyz=(0.0, 0.0, 0.0),
              yaw=0.0, noise_std=0.02):
    rng = np.random.default_rng(seed)
    elev = np.deg2rad(np.linspace(-24.8, 2.0, n_beams))
    az = np.linspace(-np.pi, np.pi, n_az, endpoint=False)
    e, a = np.meshgrid(elev, az, indexing="ij")
    d = np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], -1).reshape(-1, 3)
    sx, sy, sz = sensor_xyz
    # world-axis-aligned scene, sensor rotated by yaw about z
    cy, syaw = np.cos(yaw), np.sin(yaw)
    Rw = np.array([[cy, -syaw, 0.0], [syaw, cy, 0.0], [0.0, 0.0, 1.0]])
    dw = d @ Rw.T
    big = 1e9
    with np.errstate(divide="ignore", invalid="ignore"):
        t_ground = np.where(dw[:, 2] < 0, (-1.73 - sz) / dw[:, 2], big)
        t_y = np.where(dw[:, 1] > 0, (8.0 - sy) / dw[:, 1], np.where(dw[:, 1] < 0, (-8.0 - sy) / dw[:, 1], big))
        t_x = np.where(dw[:, 0] > 0, (30.0 - sx) / dw[:, 0], np.where(dw[:, 0] < 0, (-30.0 - sx) / dw[:, 0], big))
    t = np.minimum(np.minimum(t_ground, t_y), t_x)
    is_ground = t_ground <= t
    t = t + rng.normal(0.0, noise_std, t.shape)
    keep = (t > min_depth) & (t < max_depth)
    pts = (d * t[:, None])[keep]
    cos = np.where(is_ground, np.abs(dw[:, 2]), 1.0)[keep]
    pose = np.eye(4)
    pose[:3, :3] = Rw
    pose[:3, 3] = np.array(sensor_xyz) + POSE_OFFSET
    return pts.astype(np.float32), cos.astype(np.float32), pose.astype(np.float32)


def path_pose(i, n_scans, spacing, path="line"):
    """(sensor_xyz, yaw) of scan i of scripts/demo_slam.py's drive.  "line": out along +x, spacing metres per scan.  "loop": out
    along +x for the first half and back over the same ground in the second, so the last scan is taken where the first was."""
    if path not in ("line", "loop"):
        raise ValueError(f"path must be 'line' or 'loop', got {path!r}")
    s = i if path == "line" else min(i, n_scans - 1 - i)
    return (spacing * s, 0.05 * np.sin(0.7 * i), 0.0), 0.01 * np.sin(0.5 * i)


def voxelize(points, pose, voxel_size):
    """src/mapping.py:283-290: sensor points -> world -> floor(/voxel_size) -> int32 voxel coords."""
    R = pose[:3, :3].astype(np.float32)
    t = pose[:3, 3].astype(np.float32)
    pw = (points.astype(np.float32) @ R.T + t).astype(np.float32)
    return np.floor(pw / np.float32(voxel_size)).astype(np.int32)


def street_boxes(seed=5, length=80.0, x0=-40.0):
    """Axis-aligned boxes f64[B, 6] (min xyz, max xyz) standing on the ground (z = -1.73) along both sides of a street on the x axis:
    buildings of varied length, depth and height with gaps between them, set back 6-10 m from y = 0, plus a few short kerbside
    objects at |y| 3.5-5 m.  Drawn from `seed`, so no two stretches of the street look alike and no half-turn maps it onto itself."""
    rng = np.random.default_rng(seed)
    boxes = []
    for side in (-1.0, 1.0):
        x = x0 + rng.uniform(0.0, 4.0)
        while x < x0 + length:
            L, D, H = rng.uniform(2.0, 12.0), rng.uniform(2.0, 7.0), rng.uniform(1.5, 9.0)
            y_in = rng.uniform(6.0, 10.0)
            y = (y_in, y_in + D) if side > 0 else (-y_in - D, -y_in)
            boxes.append([x, y[0], -1.73, x + L, y[1], -1.73 + H])
            x += L + rng.uniform(0.5, 6.0)
        x = x0 + rng.uniform(0.0, 10.0)
        while x < x0 + length:
            s, h = rng.uniform(0.3, 2.5), rng.uniform(0.8, 2.5)
            y_in = rng.uniform(3.5, 5.0)
            y = (y_in, y_in + s) if side > 0 else (-y_in - s, -y_in)
            boxes.append([x, y[0], -1.73, x + s, y[1], -1.73 + h])
            x += s + rng.uniform(4.0, 15.0)
    return np.asarray(boxes, dtype=np.float64)


def make_street_scan(sensor_xyz=(0.0, 0.0, 0.0), yaw=0.0, boxes=None, n_beams=64, n_az=1024, seed=777, min_depth=1.5, max_depth=40.0,
                     noise_std=0.02):
    """make_scan's 64-beam sensor ray-cast against the ground plane z = -1.73 and `boxes` (street_boxes() by default) instead of the
    canyon, which a half turn or a shift along x maps onto itself.  Returns (points f32[n,3] in the sensor frame, pointsCos f32[n]:
    |n.d| on the ground, 1 elsewhere, pose f32[4,4] with POSE_OFFSET added)."""
    boxes = street_boxes() if boxes is None else np.asarray(boxes, dtype=np.float64)
    rng = np.random.default_rng(seed)
    elev = np.deg2rad(np.linspace(-24.8, 2.0, n_beams))
    az = np.linspace(-np.pi, np.pi, n_az, endpoint=False)
    e, a = np.meshgrid(elev, az, indexing="ij")
    d = np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], -1).reshape(-1, 3)
    cy, syaw = np.cos(yaw), np.sin(yaw)
    Rw = np.array([[cy, -syaw, 0.0], [syaw, cy, 0.0], [0.0, 0.0, 1.0]])
    dw = d @ Rw.T
    o = np.asarray(sensor_xyz, dtype=np.float64)
    big = 1e9
    with np.errstate(divide="ignore", invalid="ignore"):
        t_ground = np.where(dw[:, 2] < 0, (-1.73 - o[2]) / dw[:, 2], big)
        t = t_ground.copy()
        inv = 1.0 / dw
        for b in boxes:                                # slab test, one box at a time over every ray
            t1, t2 = (b[None, :3] - o) * inv, (b[None, 3:] - o) * inv
            near = np.nanmax(np.minimum(t1, t2), axis=1)
            far = np.nanmin(np.maximum(t1, t2), axis=1)
            hit = (far >= np.maximum(near, 0.0)) & (near > 0.0)
            t = np.where(hit & (near < t), near, t)
    is_ground = t_ground <= t
    t = t + rng.normal(0.0, noise_std, t.shape)
    keep = (t > min_depth) & (t < max_depth)
    pts = (d * t[:, None])[keep]
    cos = np.where(is_ground, np.abs(dw[:, 2]), 1.0)[keep]
    pose = np.eye(4)
    pose[:3, :3] = Rw
    pose[:3, 3] = o + POSE_OFFSET
    return pts.astype(np.float32), cos.astype(np.float32), pose.astype(np.float32)
