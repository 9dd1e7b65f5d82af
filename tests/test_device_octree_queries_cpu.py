"""CPU-only: the device-octree query entry points (include/nerfloam_b200.h section 1b, queries) reject bad arguments before their
first CUDA call, and the two facts their kernels rest on hold on the host tree:
  * preorder (get_voxels / get_leaf_voxels) is the order of (Morton code of the min corner, level), and wherever codes tie the
    ancestor has the smaller id, so a stable sort of the codes in id order is the preorder;
  * try_insert is membership of the batch's distinct corner keys in the set of level-L node codes, counted after truncating the
    matching keys to int32.
"""
import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


def test_query_entry_points_reject_bad_arguments_without_touching_the_gpu(nl):
    L = nl._capi.lib()
    err = lambda: L.nl_last_error().decode()
    one = 16                                                              # a non-null stand-in pointer; never dereferenced
    big = 1 << 30
    assert L.nl_devoctree_query_workspace_bytes(-1, 0, 256) == -1 and "n_nodes" in err()
    assert L.nl_devoctree_query_workspace_bytes(10, -1, 256) == -1
    assert L.nl_devoctree_query_workspace_bytes(10, 0, 255) == -1
    assert L.nl_devoctree_query_workspace_bytes(10, 1 << 24, 256) == -1
    assert L.nl_devoctree_query_workspace_bytes(1 << 31, 0, 256) == -1
    ex = lambda gd, rows, child, vertex: L.nl_devoctree_export_nodes(gd, 0.3, rows, None, None, 0, child, one, one, one, one, one, None, None,
                                                                     vertex, None)
    assert ex(3, 4, one, one) != 0 and "grid_dim" in err()
    assert ex(256, -4, one, one) != 0 and "negative" in err()
    assert ex(256, 4, one, None) != 0 and "null" in err()
    assert ex(256, 4, None, one) != 0 and "null" in err()
    assert L.nl_devoctree_export_nodes(256, 0.3, 0, None, None, 0, None, None, None, None, None, None, None, None, None, None) == 0
    pre = lambda gd, n, code, leaves, out, count, ws, wsb: L.nl_devoctree_preorder(gd, n, code, one, one, leaves, out, count, ws, wsb, None)
    assert pre(255, 10, one, 0, one, one, one, big) != 0 and "grid_dim" in err()
    assert pre(1 << 21, 10, one, 0, one, one, one, big) != 0 and "grid_dim" in err()
    assert pre(256, 0, one, 0, one, one, one, big) != 0 and "sizes" in err()
    assert pre(256, -5, one, 0, one, one, one, big) != 0 and "sizes" in err()
    assert pre(256, 10, one, 2, one, one, one, big) != 0 and "sizes" in err()
    assert pre(256, 10, None, 0, one, one, one, big) != 0 and "null" in err()
    assert pre(256, 10, one, 0, None, one, one, big) != 0 and "null" in err()
    assert pre(256, 10, one, 1, one, None, one, big) != 0 and "null" in err()
    assert pre(256, 10, one, 0, one, one, None, big) != 0 and "null" in err()
    assert pre(256, 1000, one, 0, one, one, one, 16) != 0 and "workspace of 16 bytes" in err()
    tri = lambda gd, child, vox, n, ws, wsb, out: L.nl_devoctree_try_insert(gd, child, vox, n, ws, wsb, out, None)
    assert tri(6, one, one, 5, one, big, one) != 0 and "grid_dim" in err()
    assert tri(256, one, one, 0, one, big, one) != 0 and "n must" in err()
    assert tri(256, one, one, -3, one, big, one) != 0 and "n must" in err()
    assert tri(256, one, one, (1 << 23) + 1, one, big, one) != 0 and "n must" in err()
    for args in ((None, one, one, one), (one, None, one, one), (one, one, None, one), (one, one, one, None)):
        child, vox, ws, out = args
        assert tri(256, child, vox, 5, ws, big, out) != 0 and "null" in err()
    assert tri(256, one, one, 1000, one, 16, one) != 0 and "workspace of 16 bytes" in err()


def test_device_octree_queries_need_a_cuda_device(nl):
    o = nl.svo.DeviceOctree("cpu")
    for f in (o.get_voxels, o.get_leaf_voxels, o.get_centres_and_children, lambda: o.try_insert(np.zeros((1, 3), np.int32))):
        with pytest.raises(NotImplementedError):
            f()


# -- the host tree's equivalences -------------------------------------------------------------------------------------------
_INC = np.array([[(j >> 2) & 1, (j >> 1) & 1, j & 1] for j in range(8)], np.int64)   # octree.cpp:12-14


def _spread3(v):
    x = np.asarray(v, np.int64).astype(np.uint64) & np.uint64(0x1fffff)
    for s, m in ((32, 0x1f00000000ffff), (16, 0x1f0000ff0000ff), (8, 0x100f00f00f00f00f), (4, 0x10c30c30c30c30c3), (2, 0x1249249249249249)):
        x = (x | (x << np.uint64(s))) & np.uint64(m)
    return x


def _morton(xyz):
    xyz = np.asarray(xyz, np.int64)
    return _spread3(xyz[..., 0]) | (_spread3(xyz[..., 1]) << np.uint64(1)) | (_spread3(xyz[..., 2]) << np.uint64(2))


def _nodes(o, grid_dim):
    """Every node of a host tree by id: (min corner xyz, side, SURFACE flag), read from its public exports.  Non-FEATURE rows of
    get_centres_and_children carry their own xyz and side; every FEATURE leaf is a vertex of the SURFACE leaf of the point that
    created it, so the vertex rows give its coordinates."""
    v, _, f = (t.numpy() for t in o.get_centres_and_children())
    n = v.shape[0]
    xyz = np.full((n, 3), -1, np.int64)
    side = v[:, 3].astype(np.int64)
    seen = side > 0
    xyz[seen] = v[seen, :3].astype(np.int64)
    surface = seen & (side == 1)
    for i in np.nonzero(surface)[0]:
        for k in range(8):
            c = f[i, k]
            assert c >= 0
            want = xyz[i] + _INC[k]
            if side[c] == 0:
                assert (xyz[c] == -1).all() or (xyz[c] == want).all()
                xyz[c] = want
            else:
                assert (xyz[c] == want).all()
    feature = side == 0
    side[feature] = 1
    assert (xyz >= 0).all(), "a node not reached by the exports"
    level = np.log2(grid_dim).astype(int) - np.log2(side).astype(int)
    assert (side == grid_dim >> level).all() and (xyz % side[:, None] == 0).all()
    return xyz, side, level, surface


def _trees():
    import nerfloam_b200 as nl
    rng = np.random.default_rng(11)
    syn = nl.synthetic
    scan = syn.voxelize(*syn.make_scan(n_beams=16, n_az=400, seed=5)[::2], 0.3)
    hi = (1 << 20) - 2
    return {
        8: [rng.integers(0, 7, (n, 3)).astype(np.int32) for n in (40, 300, 5)],
        64: [rng.integers(0, 63, (n, 3)).astype(np.int32) for n in (1, 2000, 3000)],
        1 << 18: [scan[: len(scan) // 2], scan, scan + np.array([[3, -2, 1]], np.int32)],
        1 << 20: [rng.integers(hi - 40, hi + 1, (n, 3)).astype(np.int32) for n in (500, 4000)]
        # the same low 11 bits per axis, so equal low 32 bits of the leaf codes: try_insert's int32 truncation merges them
        + [np.concatenate([rng.integers(0, 30, (300, 3)), rng.integers(hi - 40, hi + 1, (300, 3)) - ((1 << 20) - (1 << 11))]).astype(np.int32)],
    }


def _try_insert_by_leaf_codes(leaf_codes, vox, truncate=True):
    keys = np.unique(_morton(vox.astype(np.int64)[:, None, :] + _INC[None]).reshape(-1))
    hit = keys[np.isin(keys, leaf_codes)]
    return 1.0 * len(np.unique(hit & np.uint64(0xffffffff) if truncate else hit)) / len(keys)


@pytest.mark.parametrize("grid_dim", [8, 64, 1 << 18, 1 << 20])
def test_host_preorder_is_the_stable_code_order_and_try_insert_is_leaf_code_membership(nl, grid_dim):
    rng = np.random.default_rng(grid_dim)
    some = rng.integers(-3000, 3000, (200, 3))
    assert np.array_equal(_morton(some), [nl.svo.encode(*p) for p in some])
    o = nl.svo.Octree()
    o.init(grid_dim, 16, 0.3)
    batches = _trees()[grid_dim]
    truncation_mattered = False
    for b, nxt in zip(batches, batches[1:] + [batches[0][::-1] + 1]):
        o.insert(torch.from_numpy(b))
        xyz, side, level, surface = _nodes(o, grid_dim)
        code = _morton(xyz)
        assert code[0] == 0 and level[0] == 0
        by_code = np.argsort(code, kind="stable")                        # node ids in id order, stably sorted by code
        assert np.array_equal(by_code, np.lexsort((level, code)))       # == by (code, level)
        tie = code[by_code][1:] == code[by_code][:-1]                   # equal codes: the ancestor holds the smaller id
        assert (np.diff(by_code)[tie] > 0).all() and (np.diff(level[by_code])[tie] > 0).all()
        rows = np.concatenate([xyz, side[:, None]], 1)[by_code].astype(np.float32)
        assert np.array_equal(o.get_voxels().numpy(), rows)
        assert np.array_equal(o.get_leaf_voxels().numpy(), rows[surface[by_code], :3])
        leaf_codes = code[level == level.max()]
        assert level.max() == int(np.log2(grid_dim))
        queries = [b, nxt, b + np.array([[1, 0, 0]]), b + np.array([[5, -3, 2]]), -b - 1, b - grid_dim, b + grid_dim, b + (1 << 21),
                   b * 3 + 7, rng.integers(-(1 << 22), 1 << 22, (300, 3)), np.concatenate([b, b + ((1 << 20) - (1 << 11))])]
        for q in queries:
            q = np.ascontiguousarray(q, dtype=np.int32)
            r = o.try_insert(torch.from_numpy(q))
            assert r == _try_insert_by_leaf_codes(leaf_codes, q)
            truncation_mattered |= r != _try_insert_by_leaf_codes(leaf_codes, q, truncate=False)
    assert truncation_mattered == (grid_dim == 1 << 20)
