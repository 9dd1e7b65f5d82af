"""NumPy restatement of the coarse stage of global localisation (include/nerfloam_b200.h section 15, DESIGN.md §3.4): the cell table,
the placement matrices, the occupied-voxel counts and the top-n selection.  Plain fp64 element-wise arithmetic in the kernels' order."""
import numpy as np

AXIS_BITS = 18


def box(x, r, step):
    """First lattice index and width of an anchor's box: one index of margin beyond [x - r, x + r] on each side."""
    return int(np.floor((x - r) / step)) - 1, int(np.ceil(2.0 * r / step)) + 4


def cells(anchors12, radius, xy_step):
    """int64[n, 3] = (i, j, anchor), ascending (i, j): lattice points within radius (fp64) of an anchor's xy, each with the anchor of
    least fp32 distance, the lower index on a tie."""
    best = {}
    for a, A in enumerate(np.asarray(anchors12, np.float64).reshape(-1, 12)):
        tx, ty = A[3], A[7]
        i0, W = box(tx, radius, xy_step)
        j0, _ = box(ty, radius, xy_step)
        i = np.arange(i0, i0 + W, dtype=np.int64)[:, None]
        j = np.arange(j0, j0 + W, dtype=np.int64)[None, :]
        dx = i.astype(np.float64) * xy_step - tx
        dy = j.astype(np.float64) * xy_step - ty
        d = np.sqrt(dx * dx + dy * dy)
        ii, jj = np.nonzero(d <= radius)
        for u, v in zip(ii, jj):
            key = (int(i[u, 0]), int(j[0, v]))
            cand = (int(np.float32(d[u, v]).view(np.uint32)), a)
            if key not in best or cand < best[key]:
                best[key] = cand
    return np.array([(k[0], k[1], best[k][1]) for k in sorted(best)], dtype=np.int64).reshape(-1, 3)


def matrices(cell_table, anchors12, yaw_steps, xy_step, ids):
    """f32[n, 12] (R row-major, then t) of placements `ids`: Rz(2 pi k / Y - psi_a) R_a, (i step, j step, t_a,z), fp64 then fp32."""
    ids = np.asarray(ids, np.int64)
    c, k = ids // yaw_steps, ids % yaw_steps
    cell = np.asarray(cell_table, np.int64)[c]
    A = np.asarray(anchors12, np.float64).reshape(-1, 12)[cell[:, 2]]
    psi = np.arctan2(A[:, 4], A[:, 0])
    phi = 2.0 * np.pi * k.astype(np.float64) / float(yaw_steps) - psi
    cs, sn = np.cos(phi)[:, None], np.sin(phi)[:, None]
    out = np.empty((ids.size, 12))
    out[:, 0:3] = cs * A[:, 0:3] - sn * A[:, 4:7]
    out[:, 3:6] = sn * A[:, 0:3] + cs * A[:, 4:7]
    out[:, 6:9] = A[:, 8:11]
    out[:, 9] = cell[:, 0].astype(np.float64) * xy_step
    out[:, 10] = cell[:, 1].astype(np.float64) * xy_step
    out[:, 11] = A[:, 11]
    return out.astype(np.float32)


def voxel_keys(Rt12, points, voxel_size, grid_dim):
    """(keys int64[P, M], valid bool[P, M]): the voxel of every point under every matrix, ((R0 x + R1 y) + R2 z) + t in fp64 from
    fp32, floor(w / voxel_size), packed as vx << 36 | vy << 18 | vz; invalid outside [0, grid_dim)^3 or not finite."""
    Rt = np.asarray(Rt12, np.float32).astype(np.float64).reshape(-1, 12)
    p = np.asarray(points, np.float32).astype(np.float64).reshape(-1, 3)
    keys = np.zeros((Rt.shape[0], p.shape[0]), np.int64)
    valid = np.ones(keys.shape, bool)
    for i in range(3):
        w = ((Rt[:, 3 * i, None] * p[None, :, 0] + Rt[:, 3 * i + 1, None] * p[None, :, 1]) + Rt[:, 3 * i + 2, None] * p[None, :, 2]) + Rt[:, 9 + i, None]
        with np.errstate(invalid="ignore"):
            v = np.floor(w / voxel_size)
            ok = (v >= 0.0) & (v < grid_dim)
        valid &= ok
        keys = (keys << AXIS_BITS) | np.where(ok, v, 0).astype(np.int64)
    return keys, valid


def leaf_keys(leaf_voxels):
    """Sorted int64 keys of integer voxel corners [n, 3] (Octree.get_leaf_voxels())."""
    v = np.asarray(leaf_voxels).astype(np.int64)
    return np.unique((v[:, 0] << (2 * AXIS_BITS)) | (v[:, 1] << AXIS_BITS) | v[:, 2])


def counts(Rt12, points, occupied_keys, voxel_size, grid_dim, block=256):
    """int64[P]: how many points land in an occupied voxel under each matrix."""
    occ = np.asarray(occupied_keys, np.int64)
    Rt12 = np.asarray(Rt12, np.float32).reshape(-1, 12)
    out = np.empty(Rt12.shape[0], np.int64)
    for b in range(0, Rt12.shape[0], block):
        k, ok = voxel_keys(Rt12[b:b + block], points, voxel_size, grid_dim)
        out[b:b + block] = (ok & np.isin(k, occ)).sum(1)
    return out


def select(count_array, n):
    """Ids of the n highest counts, ranked by (count desc, id asc), and their counts."""
    c = np.asarray(count_array, np.int64)
    order = np.lexsort((np.arange(c.size), -c))[:n]
    return order, c[order]
