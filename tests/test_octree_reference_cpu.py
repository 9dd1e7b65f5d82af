"""The host octree (svo.Octree, csrc/octree_host.cpp) against the compiled reference octree, run unmodified in child processes
(tests/octree_ref_child.py), on the cases of tests/octree_cases.py: every output after every batch, exactly, the map-update glue
on the reference's arrays, pickled trees that keep growing, and the inputs the product refuses on purpose."""
import copy
import io
import os
import pickle

import numpy as np
import pytest
import torch

import octree_cases as OC
import octree_ref_child as R

pytestmark = pytest.mark.skipif(not os.path.exists(R.SVO_REF), reason=f"the compiled reference octree {R.SVO_REF} is missing "
                                                                       "(oracle/build_ref.py svo builds it)")


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return R.run_cases({n: OC.case(n) for n in OC.names()}, str(tmp_path_factory.mktemp("octree_ref")))


def _dump(ref, name, restored=False):
    path, path2, err = ref[name]
    assert err is None, err
    return R.load(path2 if restored else path)


@pytest.mark.parametrize("name", OC.names())
def test_host_octree_equals_reference_after_every_batch(nl, ref, name):
    case, want = OC.case(name), _dump(ref, name)
    t = nl.svo.Octree()
    t.init(case.grid_dim, 16, case.voxel_size)
    for i, b in enumerate(case.batches):
        t.insert(torch.from_numpy(b))
        R.assert_equals_reference(t, want, i, case, name)
    if name == "drive_fine":
        assert t.count_nodes() > 60_000


@pytest.mark.parametrize("name", ["drive_demo", "drive_kitti", "drive_fine", "promotion_feature_to_surface", "random_17"])
def test_map_updater_rows_equal_the_reference_glue(nl, ref, name):
    """MapUpdater on the CPU (the full-export path): map_states equals mapping.py:320-337 run on the reference's arrays, with
    one embedding row per new vertex in the glue's order."""
    case, want = OC.case(name), _dump(ref, name)
    mu = nl.mapping.MapUpdater(case.voxel_size, grid_dim=case.grid_dim, device="cpu")
    v2r, n_rows = np.zeros(0, np.int32), 0
    for i, b in enumerate(case.batches):
        mu.insert_voxels(torch.from_numpy(b))
        v2r, n_rows = R.glue_rows(want[f"features{i}"], v2r, n_rows)
        centres, structure, vertex = R.glue(want, i, case.voxel_size)
        st = mu.map_states
        for k, y in (("voxel_center_xyz", centres), ("voxel_structure", structure), ("voxel_vertex_idx", vertex),
                     ("voxel_id2embedding_id", torch.from_numpy(v2r).view(-1, 1))):
            R._same(st[k].numpy(), y.numpy(), f"{name}, after batch {i}: map_states[{k!r}]")
        R._same(mu.vertex2row, v2r, f"{name}, after batch {i}: vertex2row")
        assert mu.n_rows == n_rows and mu.embeddings.shape[0] == n_rows


def _restore(tree, how):
    if how == "pickle":
        return pickle.loads(pickle.dumps(tree))
    if how == "deepcopy":
        return copy.deepcopy(tree)
    buf = io.BytesIO()
    torch.save(tree, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=False)


@pytest.mark.parametrize("how", ["pickle", "deepcopy", "torch.save"])
@pytest.mark.parametrize("name", [n for n in OC.names() if n.startswith("restore_")])
def test_restored_host_octree_grows_like_the_restored_reference(nl, ref, name, how):
    """Pickled after batch k, restored, then grown by the remaining batches: equal to the reference tree unpickled in a fresh process
    and grown by the same batches, at the restore point and after every later batch.  The tree that was pickled carries on too."""
    case = OC.case(name)
    full, restored = _dump(ref, name), _dump(ref, name, restored=True)
    k = case.restore_after
    for i in range(k, len(case.batches)):              # the reference's replay gives the ids of the uninterrupted tree
        for key in ("voxels", "children", "features", "gv", "lv", "counts", "try", "has"):
            R._same(restored[f"{key}{i}"], full[f"{key}{i}"], f"{name}: the restored reference's {key} after batch {i}")
    t = nl.svo.Octree()
    t.init(case.grid_dim, 16, case.voxel_size)
    for b in case.batches[:k + 1]:
        t.insert(torch.from_numpy(b))
    r = _restore(t, how)
    R.assert_equals_reference(r, restored, k, case, f"{name} restored by {how}")
    for i in range(k + 1, len(case.batches)):
        r.insert(torch.from_numpy(case.batches[i]))
        R.assert_equals_reference(r, restored, i, case, f"{name} restored by {how}")
    t.insert(torch.from_numpy(case.batches[k + 1]))
    R.assert_equals_reference(t, full, k + 1, case, f"{name}, the pickled tree")


@pytest.mark.parametrize("g", [1 << 11, 1 << 18])
def test_try_insert_truncation_cases_exercise_the_quirk(ref, g):
    """The reference gathers the intersection of 64-bit corner keys into a std::set<int> (octree.cpp:141-147), so keys that share
    their low 32 bits count once.  The truncation cases build probes where that changes the ratio, and controls where it does
    not; the reference's ratios after the last batch are the truncated ones.  (The product is compared with them in
    test_host_octree_equals_reference_after_every_batch.)"""
    name = f"truncated_keys_{g}"
    case, want = OC.case(name), _dump(ref, name)
    inserted = np.concatenate(case.batches)
    tree_keys = OC.corner_keys(inserted)
    last = len(case.batches) - 1
    collide = [OC.low_words_collide(p, inserted) for p in case.probes]
    assert collide == [True, True, False, False, False]
    for p, got, c in zip(case.probes, want[f"try{last}"], collide):
        keys = OC.corner_keys(p)
        hit = np.intersect1d(keys, tree_keys)
        truncated = np.unique(hit & np.uint64(0xFFFFFFFF)).shape[0] / keys.shape[0]
        assert got == truncated
        assert (got != hit.shape[0] / keys.shape[0]) == c


@pytest.mark.parametrize("g", [8, 1024, 1 << 18])
def test_out_of_grid_batch_is_refused_and_leaves_the_tree_unchanged(nl, g):
    """A deliberate difference: the reference wraps a corner outside [0, grid_dim) through `x & edge` into another cell; the product
    refuses the whole batch with NerfLoamError, before any of its points changes the tree (valid points come first here)."""
    rng = np.random.default_rng(g)
    t = nl.svo.Octree()
    t.init(g, 16, 0.3)
    good = rng.integers(0, g - 1, (50, 3)).astype(np.int32)
    t.insert(torch.from_numpy(good))
    t.export_dirty()
    before = [x.clone() for x in t.export_nodes()] + [t.get_voxels(), *t.export_map()]
    fresh = rng.integers(0, g - 1, (20, 3)).astype(np.int32)
    for axis in range(3):
        for bad_value in (g - 1, g, -1, 2 ** 31 - 1, -2 ** 31):
            bad = fresh.copy()
            bad[-1, axis] = bad_value
            with pytest.raises(nl._capi.NerfLoamError, match="rejected"):
                t.insert(torch.from_numpy(bad))
            after = [*t.export_nodes(), t.get_voxels(), *t.export_map()]
            assert all(torch.equal(a, b) for a, b in zip(before, after)) and not t.is_dirty()
    clean = nl.svo.Octree()                                           # the refusals leave nothing behind for later inserts either
    clean.init(g, 16, 0.3)
    for tree in (t, clean):
        if tree is clean:
            tree.insert(torch.from_numpy(good))
        tree.insert(torch.from_numpy(fresh))
    assert all(torch.equal(a, b) for a, b in zip((*t.export_nodes(), *t.export_map()), (*clean.export_nodes(), *clean.export_map())))
    assert t.try_insert(torch.from_numpy(bad)) == clean.try_insert(torch.from_numpy(bad))


@pytest.mark.parametrize("g", [0, 1, 3, 1000, 3 << 10, 1 << 21])
def test_grid_dim_outside_the_product_range_is_refused(nl, g):
    """A deliberate difference: the reference takes max_level_ = log2(size_) as a truncated double, so a grid_dim that is not a
    power of two builds a tree of the next smaller power's depth whose nodes still have side grid_dim / 2^d; the product accepts
    powers of two in [2, 2^20] only, on both trees."""
    with pytest.raises(nl._capi.NerfLoamError, match="power of two"):
        nl.svo.Octree().init(g, 16, 0.3)
