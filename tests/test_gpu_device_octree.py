"""svo.DeviceOctree and MapUpdater(octree="device") against the host octree: node ids, exports, dirty rows and embedding rows bit for
bit after every insert, a rejected batch leaves the tree unchanged, and a map update moves no bulk data between host and device."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from util import Args

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


def _vox(scan, vs):
    pts, _, pose = scan
    return nl_synthetic().voxelize(pts, pose, vs)


def nl_synthetic():
    import nerfloam_b200 as nl
    return nl.synthetic


def _demo(nl):          # scripts/demo_slam.py: 12 scans 0.5 m apart at 0.3 m
    syn = nl.synthetic
    return 0.3, 256 * 256 * 4, [_vox(syn.make_scan(seed=1000 + i, sensor_xyz=(0.5 * i, 0.05 * np.sin(0.7 * i), 0.0), yaw=0.01 * np.sin(0.5 * i)), 0.3)
                                for i in range(12)]


def _kitti(nl):         # test_config2_kitti_incremental_map: 6 scans 1 m apart
    syn = nl.synthetic
    return 0.3, 256 * 256 * 4, [_vox(syn.make_scan(n_beams=32, n_az=240, seed=100 + i, sensor_xyz=(1.0 * i, 0.0, 0.0)), 0.3) for i in range(6)]


def _fine(nl):          # MaiCity / NCD: 0.2 m voxels, scans 2 m apart; the first is a whole scan into an empty tree
    syn = nl.synthetic
    return 0.2, 256 * 256 * 4, [_vox(syn.make_scan(seed=2000 + i, sensor_xyz=(2.0 * i, 0.0, 0.0), min_depth=1.5, max_depth=50.0), 0.2)
                                for i in range(3)]


def _grid8(nl):         # BASELINE config 0: 8^3 grid
    rng = np.random.default_rng(7)
    return 1.0, 8, [rng.integers(0, 7, (n, 3)).astype(np.int32) for n in (40, 300, 5)]


def _edge(nl):          # shuffled scan, only repeated points, a re-inserted scan, an empty batch, one point
    syn = nl.synthetic
    a = _vox(syn.make_scan(n_beams=16, n_az=400, seed=5), 0.3)
    b = _vox(syn.make_scan(n_beams=16, n_az=400, seed=6, sensor_xyz=(3.0, 1.0, 0.0)), 0.3)
    rng = np.random.default_rng(1)
    rep = a[rng.integers(0, a.shape[0], 5000)]
    single = (b[:1] + np.array([[40, -30, 7]], np.int32)).astype(np.int32)
    return 0.3, 256 * 256 * 4, [a[rng.permutation(a.shape[0])], rep, b, a, np.zeros((0, 3), np.int32), single, np.repeat(b[7:8], 3, 0)]


def _check_same(host, dev):
    assert dev.count_nodes() == host.count_nodes() and dev.count_leaf_nodes() == host.count_leaf_nodes()
    for x, y in zip(dev.export_map(), host.export_map()):
        assert x.device.type == "cpu" and x.dtype == y.dtype and torch.equal(x, y)
    for x, y in zip(dev.export_dirty(), host.export_dirty()):
        assert x.dtype == y.dtype and np.array_equal(x, y)


@pytest.mark.parametrize("seq", ["demo", "kitti", "fine", "grid8", "edge"])
def test_device_octree_equals_host_after_every_insert(nl, seq):
    vs, gd, batches = {"demo": _demo, "kitti": _kitti, "fine": _fine, "grid8": _grid8, "edge": _edge}[seq](nl)
    host, dev = nl.svo.Octree(), nl.svo.DeviceOctree()
    host.init(gd, 16, vs)
    dev.init(gd, 16, vs)
    for i, v in enumerate(batches):
        host.insert(torch.from_numpy(v))
        dev.insert(torch.from_numpy(v).cuda() if i % 2 else torch.from_numpy(v))      # CUDA and CPU input
        _check_same(host, dev)
        assert dev.has_voxel(v[0]) if v.shape[0] else True
    if seq == "fine":
        assert host.count_nodes() > 60_000


def test_device_octree_accumulates_inserts_between_exports(nl):
    """Several inserts before one export (bench.py's `mu.svo.insert(...)` loop, then one update): the same dirty rows as the host."""
    vs, gd, batches = _kitti(nl)
    host, dev = nl.svo.Octree(), nl.svo.DeviceOctree()
    host.init(gd, 16, vs)
    dev.init(gd, 16, vs)
    for group in (batches[:1], batches[1:4], batches[4:]):
        for v in group:
            host.insert(torch.from_numpy(v))
            dev.insert(torch.from_numpy(v))
        _check_same(host, dev)


def test_device_octree_is_deterministic(nl):
    vs, gd, batches = _demo(nl)
    runs = []
    for _ in range(2):
        dev = nl.svo.DeviceOctree()
        dev.init(gd, 16, vs)
        for v in batches[:6]:
            dev.insert(torch.from_numpy(v).cuda())
        n = dev.count_nodes()
        runs.append([t[:n].clone() for t in (dev._child, dev._code, dev._type, dev._level)])
    assert all(torch.equal(a, b) for a, b in zip(*runs))


def test_rejected_batch_leaves_the_tree_unchanged(nl):
    vs, gd, batches = _kitti(nl)
    host, dev = nl.svo.Octree(), nl.svo.DeviceOctree()
    host.init(gd, 16, vs)
    dev.init(gd, 16, vs)
    host.insert(torch.from_numpy(batches[0]))
    dev.insert(torch.from_numpy(batches[0]))
    _check_same(host, dev)
    n = dev.count_nodes()
    before = [t[:n].clone() for t in (dev._child, dev._code, dev._type, dev._level, dev._scratch)]
    bad = batches[1].copy()
    bad[len(bad) // 2, 1] = gd - 1                                      # one coordinate outside [0, grid_dim-2]
    with pytest.raises(nl._capi.NerfLoamError, match="rejected"):
        dev.insert(torch.from_numpy(bad).cuda())
    assert dev.count_nodes() == n
    assert all(torch.equal(a, t[:n]) for a, t in zip(before, (dev._child, dev._code, dev._type, dev._level, dev._scratch)))
    host.insert(torch.from_numpy(batches[1]))
    dev.insert(torch.from_numpy(batches[1]))
    _check_same(host, dev)


def _scans(nl, k=4):
    syn = nl.synthetic
    return [syn.make_scan(n_beams=16, n_az=160, seed=300 + i, sensor_xyz=(0.8 * i, 0.1 * i, 0.0)) for i in range(k)]


def test_map_updater_device_equals_host_and_graphs_survive(nl):
    rh = nl.render_helpers
    kw = dict(init_std=0.01, seed=3, reserve_nodes=100_000, reserve_rows=100_000)
    hst = nl.mapping.MapUpdater(0.3, **kw)
    dev = nl.mapping.MapUpdater(0.3, octree="device", **kw)
    torch.manual_seed(5)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    crit = nl.criterion.Criterion(Args())
    scans = _scans(nl)
    N = min(s[0].shape[0] for s in scans)
    ptrs, graphs, frames = set(), [], []
    rows_before = 0
    for i, (pts, cos, pose) in enumerate(scans):
        a = dev.create_voxels(torch.from_numpy(pts).cuda(), torch.from_numpy(pose).cuda())
        b = hst.create_voxels(pts, pose)
        assert a.n_nodes == b.n_nodes
        for x, y in ((a.centres, b.centres), (a.structure, b.structure), (a.vox2row, b.vox2row), (a.packed_children(), b.packed_children()),
                     (a.emb[rows_before:], b.emb[rows_before:])):      # rows handed out by this update (older ones are trained below)
            assert torch.equal(x, y)
        assert a.emb.shape == b.emb.shape
        rows_before = a.emb.shape[0]
        assert np.array_equal(dev.vertex2row, hst.vertex2row) and dev.last_update == hst.last_update
        assert set(dev.map_states) == set(hst.map_states)
        for k in ("voxel_vertex_idx", "voxel_center_xyz", "voxel_structure", "voxel_id2embedding_id"):
            x, y = dev.map_states[k], hst.map_states[k]
            assert x.device == y.device and torch.equal(x, y), k
        ptrs.add((a.centres.data_ptr(), a.structure.data_ptr(), a.vox2row.data_ptr(), a.packed_children().data_ptr(), a.emb.data_ptr()))
        frames.append(nl.frame.LidarFrame(i + 1, torch.from_numpy(pts[:N]), torch.from_numpy(cos[:N]),
                                          nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose.copy())), new_keyframe=True))
        if i >= 1:
            rh.bundle_adjust_frames(frames[-2:], dev.embeddings, a, dec, crit, 0.3, 0.15, N_rays=512, num_iterations=2, truncation=0.3,
                                    max_voxel_hit=20, max_distance=40.0, learning_rate=[0.01, 0.005, 0.001])
            graphs.append(rh._MapGraph._cache["g"])
    assert len(ptrs) == 1 and all(g is graphs[0] for g in graphs)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(dev.embeddings.float()).all())


def test_bundle_adjust_on_device_map_equals_host_map(nl):
    """The device map feeds the optimisation exactly like the host map.  A deterministic render on both maps is bit-identical.
    bundle_adjust_frames itself is not reproducible bit for bit even on one map: the embedding, decoder and pose gradients are summed
    with fp32 atomics, and Adam turns last-bit differences of near-zero gradients into steps of up to the learning rate.  So three
    calls start from the same state -- two on the host map, one on the device map -- and the device run may differ from the first
    host run no more than the second host run does, plus a floor (mean absolute difference).  The pose floor covers what that
    mechanism does to the 18 pose components over the 15 Adam steps: two runs on the same map land ~7e-6 apart about as often as
    ~1e-7 apart.  A fourth call from embeddings moved by 1e-2 must land farther from the first run than every floor, so the floors
    still tell a different map state apart."""
    import copy
    rh = nl.render_helpers
    maps = {}
    scans = _scans(nl, 3)
    for octree in ("host", "device"):
        mu = nl.mapping.MapUpdater(0.3, init_std=0.01, seed=4, octree=octree)
        for pts, cos, pose in scans:
            ms = mu.create_voxels(torch.from_numpy(pts).cuda(), torch.from_numpy(pose).cuda())
        maps[octree] = (mu, ms)
    (mh, sh), (md, sd) = maps["host"], maps["device"]
    for x, y in ((sd.centres, sh.centres), (sd.structure, sh.structure), (sd.vox2row, sh.vox2row), (sd.emb, sh.emb)):
        assert torch.equal(x, y)
    torch.manual_seed(9)
    dec0 = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    # 1. a deterministic render of the last scan's rays: samples, depths and SDF bit for bit
    pts, _, pose = scans[-1]
    P = torch.from_numpy(pts[::4]).cuda()
    T = torch.from_numpy(pose).cuda()
    rd = (P / P.norm(dim=-1, keepdim=True)) @ T[:3, :3].T
    ro = T[:3, 3].expand_as(rd)
    r = {o: rh.render_rays(ro[None].contiguous(), rd[None].contiguous(), ms, dec0, 0.15, 0.3, 0.3, 20, 40.0, deterministic=True)
         for o, (mu, ms) in maps.items()}
    assert r["host"] is not None and set(r["host"]) == set(r["device"])
    for k in r["host"]:
        assert torch.equal(r["device"][k], r["host"][k]), k
    # 2. three bundle_adjust_frames runs from one starting state
    emb0 = mh.embeddings.clone()
    N = min(s[0].shape[0] for s in scans)
    out = []
    moved = (emb0.float() + 1e-2 * torch.randn(emb0.shape, generator=torch.Generator().manual_seed(5)).to(emb0.device)).to(emb0.dtype)
    for octree, start in (("host", emb0), ("host", emb0), ("device", emb0), ("host", moved)):
        mu, ms = maps[octree]
        mu.embeddings.copy_(start)
        dec = copy.deepcopy(dec0)
        torch.manual_seed(11)                             # the device ray selection draws its seed from torch's generator
        frames = [nl.frame.LidarFrame(i + 1, torch.from_numpy(p[:N]), torch.from_numpy(c[:N]), nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(T.copy())),
                                      new_keyframe=True) for i, (p, c, T) in enumerate(scans)]
        for _ in range(3):
            rh.bundle_adjust_frames(frames, mu.embeddings, ms, dec, nl.criterion.Criterion(Args()), 0.3, 0.15, N_rays=512, num_iterations=5,
                                    truncation=0.3, max_voxel_hit=20, max_distance=40.0, learning_rate=[0.01, 0.005, 0.001], deterministic=True)
        torch.cuda.synchronize()
        out.append((mu.embeddings.float().cpu(), torch.cat([p.detach().cpu().reshape(-1) for p in dec.parameters()]),
                    torch.cat([f.pose.data.detach().cpu().reshape(-1) for f in frames])))
    (a, b, c, d) = out
    for i, (k, floor) in enumerate(zip(("embeddings", "decoder", "poses"), (1e-5, 1e-6, 3e-5))):
        assert a[i].shape == c[i].shape and bool(torch.isfinite(c[i]).all()), k
        same_map = float((b[i] - a[i]).abs().mean())
        other_map = float((c[i] - a[i]).abs().mean())
        other_start = float((d[i] - a[i]).abs().mean())
        print(f"{k}: host vs host {same_map:.2e}, device vs host {other_map:.2e}, moved embeddings vs host {other_start:.2e}")
        assert other_map <= 4 * same_map + floor, (k, other_map, same_map)
        assert other_start > 4 * same_map + floor, (k, other_start, same_map)


def test_device_map_update_moves_no_bulk_data(nl):
    """init_std = 0, map_states never read: no host-to-device copy, at most two device-to-host copies of <= 64 bytes per update."""
    mu = nl.mapping.MapUpdater(0.3, octree="device", reserve_nodes=200_000, reserve_rows=200_000)
    scans = [(torch.from_numpy(p).cuda(), torch.from_numpy(T).cuda()) for p, _, T in _scans(nl, 6)]
    for p, T in scans[:2]:
        mu.create_voxels(p, T)                           # warm-up: workspace and dirty-list allocations
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        for p, T in scans[2:]:
            mu.create_voxels(p, T)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "trace.json")
        prof.export_chrome_trace(f)
        ev = json.load(open(f))["traceEvents"]
    copies = [e for e in ev if e.get("cat") == "gpu_memcpy"]
    h2d = [e for e in copies if "HtoD" in e["name"]]
    d2h = [e for e in copies if "DtoH" in e["name"]]
    assert not h2d, h2d
    assert 0 < len(d2h) <= 2 * (len(scans) - 2), d2h
    assert all(int(e["args"]["bytes"]) <= 64 for e in d2h), d2h
    assert mu.last_update["dirty_rows"] > 0
