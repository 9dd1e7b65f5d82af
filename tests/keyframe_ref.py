"""NumPy restatement of the keyframe overlap counts (include/nerfloam_b200.h section 12, nerf-loam_b200/keyframes.py).

World point w_i = ((R_i0 x + R_i1 y) + R_i2 z) + t_i in float64 from the float32 matrix row Rt = (R row-major, t) and point; voxel
floor(w / voxel_size) in float64; a point whose voxel leaves [0, grid_dim)^3 is outside.  V = the set of distinct voxels."""
import numpy as np

AXIS_BITS = 18


def voxel_keys(points, Rt, voxel_size, grid_dim):
    """(keys int64[m] of the points inside the grid, in point order, with repeats; number of points outside)."""
    p = np.asarray(points, dtype=np.float32).reshape(-1, 3).astype(np.float64)
    Rt = np.asarray(Rt, dtype=np.float32).reshape(12).astype(np.float64)
    v = np.empty_like(p)
    with np.errstate(invalid="ignore"):                              # non-finite points: NaN voxels, counted as outside
        for i in range(3):
            w = ((Rt[3 * i] * p[:, 0] + Rt[3 * i + 1] * p[:, 1]) + Rt[3 * i + 2] * p[:, 2]) + Rt[9 + i]
            v[:, i] = np.floor(w / float(voxel_size))
        inside = np.all((v >= 0) & (v < grid_dim), axis=1)
    vi = v[inside].astype(np.int64)
    keys = (vi[:, 0] << (2 * AXIS_BITS)) | (vi[:, 1] << AXIS_BITS) | vi[:, 2]
    return keys, int((~inside).sum())


def overlap(frame_points, kf_points, Rt, voxel_size, grid_dim):
    """Rt f32[K+1,12]: row 0 the scan's pose, row k+1 keyframe k's.  Returns dict of shared, kf_voxels, outside (int64[K]) and
    frame_voxels (int)."""
    fk, _ = voxel_keys(frame_points, Rt[0], voxel_size, grid_dim)
    fset = np.unique(fk)
    shared, kfv, out = [], [], []
    for k, pts in enumerate(kf_points):
        keys, o = voxel_keys(pts, Rt[k + 1], voxel_size, grid_dim)
        u = np.unique(keys)
        shared.append(int(np.isin(u, fset).sum()))
        kfv.append(len(u))
        out.append(o)
    return dict(shared=np.array(shared, np.int64), kf_voxels=np.array(kfv, np.int64), outside=np.array(out, np.int64),
                frame_voxels=len(fset))
