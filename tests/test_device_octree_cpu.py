"""CPU-only: the device-octree entry points of the C ABI (include/nerfloam_b200.h section 1b) reject bad arguments before their
first CUDA call, and the Python class validates its grid."""
import pytest


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


def test_device_octree_entry_points_reject_bad_arguments_without_touching_the_gpu(nl):
    L = nl._capi.lib()
    err = lambda: L.nl_last_error().decode()
    one = 16                                                              # a non-null stand-in pointer; never dereferenced
    assert L.nl_devoctree_workspace_bytes(-1, 256) == -1 and "n_points" in err()
    assert L.nl_devoctree_workspace_bytes(10, 255) == -1 and "grid_dim" in err()
    assert L.nl_devoctree_workspace_bytes(1 << 24, 256) == -1
    assert L.nl_devoctree_insert_count(255, one, one, 5, one, 1 << 20, one, None) != 0 and "grid_dim" in err()
    assert L.nl_devoctree_insert_count(256, one, one, -1, one, 1 << 20, one, None) != 0 and "n must" in err()
    assert L.nl_devoctree_insert_count(256, None, one, 5, one, 1 << 20, one, None) != 0 and "null" in err()
    assert L.nl_devoctree_insert_count(256, one, None, 5, one, 1 << 20, one, None) != 0 and "null" in err()
    assert L.nl_devoctree_insert_count(256, one, one, 5, one, 1 << 20, None, None) != 0 and "null" in err()
    assert L.nl_devoctree_insert_commit(0, 1, 0, 0, one, one, one, one, one, one, 5, one, 1 << 20, one, None) != 0 and "grid_dim" in err()
    assert L.nl_devoctree_insert_commit(256, 0, 0, 0, one, one, one, one, one, one, 5, one, 1 << 20, one, None) != 0 and "sizes" in err()
    assert L.nl_devoctree_insert_commit(256, 1, -3, 0, one, one, one, one, one, one, 5, one, 1 << 20, one, None) != 0 and "sizes" in err()
    assert L.nl_devoctree_insert_commit(256, 1, 0, 0, one, None, one, one, one, one, 5, one, 1 << 20, one, None) != 0 and "null" in err()
    assert L.nl_devoctree_insert_commit(256, 1, 4, 0, one, one, one, one, one, one, 0, one, 1 << 20, one, None) != 0 and "without points" in err()
    assert L.nl_devoctree_dirty_ids(256, 1, 2, 0, one, one, one, 0, one, 1 << 20, one, None) != 0 and "sizes" in err()
    assert L.nl_devoctree_dirty_ids(256, 1, 0, -1, one, one, one, 0, one, 1 << 20, one, None) != 0 and "sizes" in err()
    assert L.nl_devoctree_dirty_ids(256, 1, 0, 0, one, one, None, 0, one, 1 << 20, one, None) != 0 and "null" in err()
    assert L.nl_devoctree_export(3, 0.3, 4, None, None, 0, one, one, one, one, one, one, one, None) != 0 and "grid_dim" in err()
    assert L.nl_devoctree_export(256, 0.3, -4, None, None, 0, one, one, one, one, one, one, one, None) != 0 and "negative" in err()
    assert L.nl_devoctree_export(256, 0.3, 4, None, None, 0, one, one, one, one, None, one, one, None) != 0 and "null" in err()
    assert L.nl_devoctree_export(256, 0.3, 0, None, None, 0, None, None, None, None, None, None, None, None) == 0     # nothing to do
    assert L.nl_devoctree_assign_rows(256, -1, one, 1, one, one, one, one, 0, one, 1, one, 1 << 20, one, None) != 0 and "sizes" in err()
    assert L.nl_devoctree_assign_rows(256, 5, one, 1, one, one, one, one, -2, one, 1, one, 1 << 20, one, None) != 0 and "sizes" in err()
    assert L.nl_devoctree_assign_rows(256, 5, None, 1, one, one, one, one, 0, one, 1, one, 1 << 20, one, None) != 0 and "null" in err()
    assert L.nl_devoctree_find(6, one, one, 1, one, None) != 0 and "grid_dim" in err()
    assert L.nl_devoctree_find(256, one, one, -1, one, None) != 0 and "negative" in err()
    assert L.nl_devoctree_find(256, one, None, 1, one, None) != 0 and "null" in err()


def test_device_octree_validates_its_grid_and_scope(nl):
    o = nl.svo.DeviceOctree("cpu")
    with pytest.raises(RuntimeError, match="not initialized"):
        o.count_nodes()
    with pytest.raises(nl._capi.NerfLoamError, match="power of two"):
        o.init(100, 16, 0.3)
    with pytest.raises(NotImplementedError):
        o.get_voxels()
    with pytest.raises(ValueError):
        nl.mapping.MapUpdater(0.3, device="cpu", octree="device")
    with pytest.raises(ValueError):
        nl.mapping.MapUpdater(0.3, device="cpu", octree="gpu")
