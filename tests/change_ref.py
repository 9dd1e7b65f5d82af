"""NumPy restatement of change detection (nerf-loam_b200/changes.py, csrc/changes.cu; DESIGN.md §11.7), working from the same arrays
the kernels read: the engine's sample list, the scan points and their pose matrix, the map's leaves.  Everything is exact (fp32 for
d = g - depth, fp64 for the voxel key and the ratio test), so the GPU's counters must equal these integers."""
import numpy as np

EMPTY = (1 << 64) - 1


def votes(s_ray, s_vox, s_depth, sdf, gt, n_nodes, truncation, through_depth):
    """u32 counts [n_nodes, 2] (through, surface) from one render call's samples.  Per (ray, voxel) over the union of its samples
    with d = gt[ray] - depth in fp32: through when every d > through_depth and the smallest sdf <= 0 (NaN sdf ignored, as fminf),
    otherwise surface when some |d| <= truncation."""
    s_ray, s_vox = np.asarray(s_ray, np.int64), np.asarray(s_vox, np.int64)
    out = np.zeros((int(n_nodes), 2), np.int64)
    if s_ray.size == 0:
        return out
    d = np.asarray(gt, np.float32)[s_ray] - np.asarray(s_depth, np.float32)
    key = s_ray * int(n_nodes) + s_vox
    _, inv = np.unique(key, return_inverse=True)
    P = int(inv.max()) + 1
    front = np.ones(P, bool)
    np.logical_and.at(front, inv, d > np.float32(through_depth))
    surf = np.zeros(P, bool)
    np.logical_or.at(surf, inv, np.abs(d) <= np.float32(truncation))
    lo = np.full(P, np.inf, np.float32)
    np.fmin.at(lo, inv, np.asarray(sdf, np.float32))
    vox = np.zeros(P, np.int64)
    vox[inv] = s_vox
    through = front & (lo <= 0)
    surface = ~through & surf
    np.add.at(out[:, 0], vox[through], 1)
    np.add.at(out[:, 1], vox[surface], 1)
    return out


def voxel_keys(points, Rt12, voxel_size, grid_dim=1 << 18):
    """voxel.cuh's nl_voxel_key for points f32[n,3] posed by Rt12 f32[12]: (keys u64[n], valid bool[n])."""
    p = np.asarray(points, np.float32).astype(np.float64)
    Rt = np.asarray(Rt12, np.float32).astype(np.float64)
    k = np.zeros(p.shape[0], np.uint64)
    ok = np.ones(p.shape[0], bool)
    for i in range(3):
        w = ((Rt[3 * i] * p[:, 0] + Rt[3 * i + 1] * p[:, 1]) + Rt[3 * i + 2] * p[:, 2]) + Rt[9 + i]
        v = np.floor(w / float(voxel_size))
        ok &= (v >= 0) & (v < grid_dim)
        k = (k << np.uint64(18)) | np.where(ok, v, 0).astype(np.uint64)
    return k, ok


def leaf_keys(centres, structure, voxel_size, grid_dim=1 << 18):
    """The occupied set of globalloc.cu: floor(centre / voxel_size) of every leaf (side 1), as a set of ints."""
    c = np.asarray(centres, np.float32).astype(np.float64)[np.asarray(structure)[:, 8] == 1]
    v = np.floor(c / float(voxel_size))
    ok = ((v >= 0) & (v < grid_dim)).all(1)
    v = v[ok].astype(np.uint64)
    return set(((v[:, 0] << np.uint64(36)) | (v[:, 1] << np.uint64(18)) | v[:, 2]).tolist())


def added(scans, occupied, voxel_size, grid_dim=1 << 18):
    """{key: [points, distinct scans]} from scans = [(points f32[n,3], Rt12 f32[12]), ...] in order: the hits outside `occupied`."""
    table = {}
    for points, Rt12 in scans:
        k, ok = voxel_keys(points, Rt12, voxel_size, grid_dim)
        k = k[ok]
        k = k[~np.isin(k, np.fromiter(occupied, np.uint64, len(occupied)))] if occupied else k
        u, c = np.unique(k, return_counts=True)
        for key, n in zip(u.tolist(), c.tolist()):
            e = table.setdefault(key, [0, 0])
            e[0] += n
            e[1] += 1
    return table


def classify(counts, structure, min_votes, ratio):
    """(removed ids in node order, confirmed, removed, unobserved totals) over the leaves."""
    t, s = counts[:, 0].astype(np.int64), counts[:, 1].astype(np.int64)
    leaf = np.asarray(structure)[:, 8] == 1
    removed = leaf & (t >= min_votes) & (t.astype(np.float64) >= float(ratio) * (t.astype(np.float64) + s.astype(np.float64)))
    confirmed = leaf & (s > 0) & ~removed
    unobserved = leaf & (t == 0) & (s == 0)
    return np.nonzero(removed)[0], int(confirmed.sum()), int(removed.sum()), int(unobserved.sum())


def select_added(table, min_points, min_scans):
    """(keys u64[A] ascending, points, scans) of the added voxels."""
    keys = sorted(k for k, (p, s) in table.items() if p >= min_points and s >= min_scans)
    return (np.array(keys, np.uint64), np.array([table[k][0] for k in keys], np.int64), np.array([table[k][1] for k in keys], np.int64))
