"""svo.DeviceOctree's queries and pickling against the host octree: get_centres_and_children, get_voxels, get_leaf_voxels and
try_insert bit for bit after every insert, the reference's goldens, pickle / deepcopy / torch.save round trips that continue like
a restored host tree, and try_insert's transfers."""
import copy
import io
import json
import os
import pickle
import tempfile

import numpy as np
import pytest
import torch

from test_gpu_device_octree import _demo, _edge, _fine, _grid8, _kitti

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


def _top(nl):           # grid_dim 2^20, coordinates up to 2^20 - 2 (the top of the grid and of the 21-bit Morton range)
    rng = np.random.default_rng(3)
    hi = (1 << 20) - 2
    return 0.3, 1 << 20, [rng.integers(hi - 60, hi + 1, (n, 3)).astype(np.int32) for n in (3000, 20000)] + \
        [np.concatenate([rng.integers(0, 40, (2000, 3)), rng.integers(hi - 60, hi + 1, (2000, 3)) - ((1 << 20) - (1 << 11))]).astype(np.int32)]


SEQUENCES = {"demo": _demo, "kitti": _kitti, "fine": _fine, "grid8": _grid8, "edge": _edge, "top": _top}


def _queries(gd, b, nxt):
    """try_insert batches: the next and the same batch, shifted, negative and out-of-grid ones (keys alias through the 21-bit
    Morton mask as on the host), one whose matches share low 32 bits, and empty or malformed input."""
    q = [nxt, b, b + np.array([[1, 0, 0]]), b + np.array([[5, -3, 2]]), -b - 1, b - gd, b + gd, b + (1 << 21), b * 3 + 7,
         np.concatenate([b, b + ((1 << 20) - (1 << 11))]), np.zeros((0, 3)), b[:, :2], b[:1].reshape(-1), b[None]]
    return [np.ascontiguousarray(x, dtype=np.int32) for x in q]


def _assert_same_queries(host, dev, queries):
    for x, y in zip(dev.get_centres_and_children(), host.get_centres_and_children()):
        assert x.device.type == "cpu" and x.dtype == y.dtype and torch.equal(x, y)
    for f in ("get_voxels", "get_leaf_voxels"):
        x, y = getattr(dev, f)(), getattr(host, f)()
        assert x.device.type == "cpu" and x.dtype == y.dtype and torch.equal(x, y), f
    for i, q in enumerate(queries):
        t = torch.from_numpy(q)
        assert dev.try_insert(t.cuda() if i % 2 else t) == host.try_insert(t), i


@pytest.mark.parametrize("seq", list(SEQUENCES))
def test_device_queries_equal_host_after_every_insert(nl, seq):
    vs, gd, batches = SEQUENCES[seq](nl)
    host, dev = nl.svo.Octree(), nl.svo.DeviceOctree()
    host.init(gd, 16, vs)
    dev.init(gd, 16, vs)
    for i, v in enumerate(batches):
        nxt = batches[i + 1] if i + 1 < len(batches) else batches[0][::-1] + 1
        if i == 0:
            _assert_same_queries(host, dev, _queries(gd, nxt, nxt))          # the root alone
        host.insert(torch.from_numpy(v))
        dev.insert(torch.from_numpy(v).cuda())
        _assert_same_queries(host, dev, _queries(gd, v, nxt))
    for t in (host, dev):
        with pytest.raises(RuntimeError, match="int32"):
            t.try_insert(torch.zeros((4, 3), dtype=torch.int64))
    if seq == "fine":
        assert host.count_nodes() > 60_000


def test_get_centres_and_children_equals_the_reference_goldens(nl):
    z = np.load(os.path.join(GOLDEN, "octree.npz"))
    dev = nl.svo.DeviceOctree()
    dev.init(256 * 256 * 4, 16, 0.3)
    for k in ("1", "2"):
        dev.insert(torch.from_numpy(z["v" + k]).cuda())
        v, c, f = (t.numpy() for t in dev.get_centres_and_children())
        assert np.array_equal(v, z["voxels" + k]) and np.array_equal(c, z["children" + k]) and np.array_equal(f, z["features" + k])
        assert [dev.count_nodes(), dev.count_leaf_nodes()] == list(z["count" + k])
    z = np.load(os.path.join(GOLDEN, "octree_8.npz"))
    dev = nl.svo.DeviceOctree()
    dev.init(8, 16, 1.0)
    dev.insert(torch.from_numpy(z["v0"]))
    v, c, f = (t.numpy() for t in dev.get_centres_and_children())
    assert np.array_equal(v, z["voxels"]) and np.array_equal(c, z["children"]) and np.array_equal(f, z["features"])


def _everything(t, queries):
    """Every method's result: the query outputs, export_map, counts, has_voxel and try_insert."""
    tensors = [*t.get_centres_and_children(), t.get_voxels(), t.get_leaf_voxels(), *t.export_map()]
    scalars = [t.count_nodes(), t.count_leaf_nodes(), t.count_export_nodes()] + [t.has_voxel(q[0]) for q in queries[:3]] + \
        [t.try_insert(torch.from_numpy(q).cuda()) for q in queries]
    return tensors, scalars


def _assert_same_everything(a, b):
    assert a[1] == b[1]
    for x, y in zip(a[0], b[0]):
        assert x.dtype == y.dtype and torch.equal(x, y)


def test_pickle_deepcopy_and_torch_save_round_trips(nl):
    vs, gd, batches = _kitti(nl)
    dev = nl.svo.DeviceOctree()
    dev.init(gd, 16, vs)
    for v in batches[:3]:
        dev.insert(torch.from_numpy(v).cuda())
    queries = _queries(gd, batches[2], batches[3])[:10]
    ref = _everything(dev, queries)
    blob = pickle.dumps(dev)
    n = dev.count_nodes()
    assert len(blob) <= 42 * n + 2048, (len(blob), n)
    buf = io.BytesIO()
    torch.save({"svo": dev}, buf)
    buf.seek(0)
    for restored in (pickle.loads(blob), copy.deepcopy(dev), torch.load(buf, weights_only=False)["svo"]):
        assert restored._child.is_cuda
        _assert_same_everything(_everything(restored, queries), ref)
        ids, c, s, v = restored.export_dirty()                          # every row is dirty, as in a replayed host tree
        assert np.array_equal(ids, np.arange(n, dtype=np.int32))
        for x, y in zip((c, s, v), ref[0][5:]):
            assert np.array_equal(x, y.numpy())
    _assert_same_everything(_everything(dev, queries), ref)           # the original is untouched
    empty = pickle.loads(pickle.dumps(nl.svo.DeviceOctree()))
    with pytest.raises(RuntimeError, match="not initialized"):
        empty.count_nodes()


def _assert_same_exports(host, dev):
    assert dev.count_nodes() == host.count_nodes() and dev.count_leaf_nodes() == host.count_leaf_nodes()
    for x, y in zip(dev.export_map(), host.export_map()):
        assert x.dtype == y.dtype and torch.equal(x, y)
    for x, y in zip(dev.export_dirty(), host.export_dirty()):
        assert x.dtype == y.dtype and np.array_equal(x, y)


def test_restored_device_tree_continues_like_a_restored_host_tree(nl):
    vs, gd, batches = _demo(nl)
    host, dev = nl.svo.Octree(), nl.svo.DeviceOctree()
    host.init(gd, 16, vs)
    dev.init(gd, 16, vs)
    for i, v in enumerate(batches[:4]):
        host.insert(torch.from_numpy(v))
        dev.insert(torch.from_numpy(v).cuda())
        if i == 1:
            _assert_same_exports(host, dev)                             # pickled with two batches not yet exported
    host_r, dev_r = pickle.loads(pickle.dumps(host)), pickle.loads(pickle.dumps(dev))
    _assert_same_exports(host_r, dev_r)
    for v in batches[4:8]:
        host_r.insert(torch.from_numpy(v))
        dev_r.insert(torch.from_numpy(v).cuda())
        _assert_same_exports(host_r, dev_r)
    _assert_same_queries(host_r, dev_r, _queries(gd, batches[7], batches[8]))


def test_update_map_refuses_a_restored_tree(nl):
    mu = nl.mapping.MapUpdater(0.3, octree="device")
    pts, _, pose = nl.synthetic.make_scan(n_beams=16, n_az=160, seed=300)
    mu.create_voxels(torch.from_numpy(pts).cuda(), torch.from_numpy(pose).cuda())
    restored = copy.deepcopy(mu.svo)
    assert restored.count_nodes() == mu.svo.count_nodes()
    with pytest.raises(nl._capi.NerfLoamError, match="unpickled"):
        restored.update_map(mu._centres, mu._structure, mu._vertex, mu._v2r, mu._vox2row, mu.n_rows)
    mu.svo = restored
    pts, _, pose = nl.synthetic.make_scan(n_beams=16, n_az=160, seed=301, sensor_xyz=(0.8, 0.1, 0.0))
    with pytest.raises(nl._capi.NerfLoamError, match="unpickled"):
        mu.create_voxels(torch.from_numpy(pts).cuda(), torch.from_numpy(pose).cuda())


def test_share_data_round_trips_a_device_tree(nl):
    vs, gd, batches = _grid8(nl)
    dev = nl.svo.DeviceOctree()
    dev.init(gd, 16, vs)
    for v in batches:
        dev.insert(torch.from_numpy(v))
    queries = _queries(gd, batches[-1], batches[0])[:10]
    sd = nl.share.ShareData()
    sd.octree = dev
    _assert_same_everything(_everything(sd.octree, queries), _everything(dev, queries))


def test_try_insert_moves_no_bulk_data(nl):
    """A CUDA batch: no host-to-device copy and one device-to-host copy of <= 64 bytes (the two counts)."""
    vs, gd, batches = _demo(nl)
    dev = nl.svo.DeviceOctree()
    dev.init(gd, 16, vs)
    for v in batches[:3]:
        dev.insert(torch.from_numpy(v).cuda())
    q = torch.from_numpy(batches[3]).cuda()
    dev.try_insert(q)                                                   # warm-up: the workspace allocation
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        r = dev.try_insert(q)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "trace.json")
        prof.export_chrome_trace(f)
        ev = json.load(open(f))["traceEvents"]
    copies = [e for e in ev if e.get("cat") == "gpu_memcpy"]
    assert not [e for e in copies if "HtoD" in e["name"]], copies
    d2h = [e for e in copies if "DtoH" in e["name"]]
    assert len(d2h) == 1 and int(d2h[0]["args"]["bytes"]) <= 64, d2h
    assert 0.0 < r < 1.0


def test_queries_are_deterministic(nl):
    vs, gd, batches = _fine(nl)
    queries = _queries(gd, batches[1], batches[2])[:10]
    runs = []
    for _ in range(2):
        dev = nl.svo.DeviceOctree()
        dev.init(gd, 16, vs)
        for v in batches[:2]:
            dev.insert(torch.from_numpy(v).cuda())
        runs.append(_everything(dev, queries))
        runs.append(_everything(dev, queries))
    for r in runs[1:]:
        _assert_same_everything(r, runs[0])
