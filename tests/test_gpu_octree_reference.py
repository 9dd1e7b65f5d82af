"""The device octree (svo.DeviceOctree, csrc/octree_dev.cu) and MapUpdater(octree="device") against the compiled reference octree,
run unmodified in child processes (tests/octree_ref_child.py) on the cases of tests/octree_cases.py: every output after every
batch, exactly, with CPU and CUDA inputs; embedding rows against the reference glue; pickled trees that keep growing."""
import copy
import io
import os
import pickle

import numpy as np
import pytest
import torch

import octree_cases as OC
import octree_ref_child as R

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.path.exists(R.SVO_REF), reason=f"the compiled reference octree {R.SVO_REF} is missing "
                                                                        "(oracle/build_ref.py svo builds it)")]


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return R.run_cases({n: OC.case(n) for n in OC.names()}, str(tmp_path_factory.mktemp("octree_ref")))


def _dump(ref, name, restored=False):
    path, path2, err = ref[name]
    assert err is None, err
    return R.load(path2 if restored else path)


def _on(i):
    """Inputs of batch i: CPU tensors for even i, CUDA tensors for odd i."""
    return (lambda t: t.cuda()) if i % 2 else (lambda t: t)


@pytest.mark.parametrize("name", OC.names())
def test_device_octree_equals_reference_after_every_batch(nl, ref, name):
    case, want = OC.case(name), _dump(ref, name)
    t = nl.svo.DeviceOctree()
    t.init(case.grid_dim, 16, case.voxel_size)
    for i, b in enumerate(case.batches):
        t.insert(_on(i)(torch.from_numpy(b)))
        R.assert_equals_reference(t, want, i, case, name, probe_input=_on(i + 1))
    if name == "drive_fine":
        assert t.count_nodes() > 60_000


@pytest.mark.parametrize("name", ["drive_demo", "drive_kitti", "drive_fine", "promotion_feature_to_surface", "random_17"])
def test_device_map_updater_rows_equal_the_reference_glue(nl, ref, name):
    """MapUpdater(octree="device"): map_states and the device arrays equal mapping.py:320-337 run on the reference's arrays, with
    one embedding row per new vertex in the glue's order."""
    case, want = OC.case(name), _dump(ref, name)
    mu = nl.mapping.MapUpdater(case.voxel_size, grid_dim=case.grid_dim, octree="device")
    v2r, n_rows = np.zeros(0, np.int32), 0
    for i, b in enumerate(case.batches):
        ms = mu.insert_voxels(_on(i)(torch.from_numpy(b)))
        v2r, n_rows = R.glue_rows(want[f"features{i}"], v2r, n_rows)
        centres, structure, vertex = R.glue(want, i, case.voxel_size)
        at = f"{name}, after batch {i}"
        st = mu.map_states
        for k, y in (("voxel_center_xyz", centres), ("voxel_structure", structure), ("voxel_vertex_idx", vertex),
                     ("voxel_id2embedding_id", torch.from_numpy(v2r).view(-1, 1))):
            R._same(st[k].numpy(), y.numpy(), f"{at}: map_states[{k!r}]")
        R._same(mu.vertex2row, v2r, f"{at}: vertex2row")
        v = vertex.numpy()
        vox2row = np.where(v >= 0, v2r[np.clip(v, 0, None)], -1).astype(np.int32)
        for x, y, k in ((ms.centres, centres.numpy(), "centres"), (ms.structure, structure.numpy(), "structure"), (ms.vox2row, vox2row, "vox2row")):
            R._same(x.cpu().numpy(), y, f"{at}: MapState.{k}")
        assert mu.n_rows == n_rows and ms.emb.shape[0] == n_rows


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
def test_restored_device_octree_grows_like_the_restored_reference(nl, ref, name, how):
    """A DeviceOctree pickled after batch k (as its node arrays), restored and grown by the remaining batches equals the reference
    tree unpickled in a fresh process (a replay of its points) and grown by the same batches, after every batch."""
    case, restored = OC.case(name), _dump(ref, name, restored=True)
    k = case.restore_after
    t = nl.svo.DeviceOctree()
    t.init(case.grid_dim, 16, case.voxel_size)
    for b in case.batches[:k + 1]:
        t.insert(torch.from_numpy(b).cuda())
    r = _restore(t, how)
    R.assert_equals_reference(r, restored, k, case, f"{name} restored by {how}")
    for i in range(k + 1, len(case.batches)):
        r.insert(_on(i)(torch.from_numpy(case.batches[i])))
        R.assert_equals_reference(r, restored, i, case, f"{name} restored by {how}", probe_input=_on(i + 1))


@pytest.mark.parametrize("g", [8, 1 << 18])
def test_device_refuses_what_the_reference_wraps(nl, g):
    """The deliberate differences, on the device tree: a corner outside [0, grid_dim) (the reference wraps it through `x & edge`)
    rejects the whole batch and leaves the tree unchanged; a grid_dim that is not a power of two in [2, 2^20] is refused."""
    rng = np.random.default_rng(g)
    t = nl.svo.DeviceOctree()
    t.init(g, 16, 0.3)
    t.insert(torch.from_numpy(rng.integers(0, g - 1, (50, 3)).astype(np.int32)).cuda())
    before = [x.clone() for x in t.export_nodes()]
    fresh = rng.integers(0, g - 1, (20, 3)).astype(np.int32)
    for bad_value in (g - 1, -1, 2 ** 31 - 1):
        bad = fresh.copy()
        bad[-1, 2] = bad_value
        with pytest.raises(nl._capi.NerfLoamError, match="rejected"):
            t.insert(torch.from_numpy(bad).cuda())
        assert all(torch.equal(a, b) for a, b in zip(before, t.export_nodes()))
    for bad_dim in (3, 1000, 1 << 21):
        with pytest.raises(nl._capi.NerfLoamError, match="power of two"):
            nl.svo.DeviceOctree().init(bad_dim, 16, 0.3)


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_device_octree_rejects_int32_max_whose_far_corner_overflows(nl, axis):
    """Regression: k_corners bounded a point by `px + 1 >= size`, which overflows for px = INT32_MAX, so such a point passed the
    check and was inserted at the cell its bits alias to.  The batch must be rejected like any other out-of-grid one."""
    t = nl.svo.DeviceOctree()
    t.init(64, 16, 0.3)
    bad = np.array([[1, 2, 3], [4, 5, 6]], np.int32)
    bad[1, axis] = 2 ** 31 - 1
    with pytest.raises(nl._capi.NerfLoamError, match="rejected"):
        t.insert(torch.from_numpy(bad).cuda())
    assert t.count_nodes() == 1
