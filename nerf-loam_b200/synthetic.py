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
