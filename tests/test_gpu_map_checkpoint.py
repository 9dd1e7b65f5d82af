"""Map checkpoints on the GPU: MapUpdater.state_dict / from_state_dict across all four (saving tree, restoring tree) pairs continue
bit for bit like the uninterrupted map; a restored map renders, bundle-adjusts and tracks through the captured graphs; a device
restore copies each checkpoint array to the device once and reads back 16 bytes; nl_devoctree_validate sets the host's bits on
every mutation of the CPU tests; malformed DeviceOctree pickles and un-applied inserts raise."""
import copy
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from test_gpu_device_octree import _demo, _edge, _fine, _grid8, _kitti
from test_gpu_device_octree_queries import _top
from test_map_checkpoint_cpu import mutated_states
from util import Args

pytestmark = pytest.mark.gpu

SEQUENCES = {"demo": _demo, "kitti": _kitti, "fine": _fine, "grid8": _grid8, "edge": _edge, "top": _top}
PAIRS = [("host", "host"), ("host", "device"), ("device", "host"), ("device", "device")]


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


def _assert_same_state(a, b):
    assert set(a) == set(b)
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k
        else:
            assert type(a[k]) is type(b[k]) and a[k] == b[k], k


def _assert_same_map(a, b, updated=True):
    """a restored updater against the uninterrupted one on the same kind of tree (last_update: once both have updated since)"""
    n = b.n_nodes
    assert a.n_nodes == n and a.n_rows == b.n_rows and a.generation == b.generation
    assert a.last_update == (b.last_update if updated else {})
    for x, y in ((a._centres, b._centres), (a._structure, b._structure), (a._vox2row, b._vox2row)):
        assert torch.equal(x[:n], y[:n])
    assert torch.equal(a._packed[:n * 128], b._packed[:n * 128])
    assert np.array_equal(a.vertex2row, b.vertex2row) and torch.equal(a.embeddings, b.embeddings)
    if b.on_device:
        assert torch.equal(a._vertex[:n], b._vertex[:n])
    else:
        for x, y in zip((*a._host, a._vertex), (*b._host, b._vertex)):
            assert np.array_equal(x[:n], y[:n])
    assert set(a.map_states) == set(b.map_states)
    for k in a.map_states:
        x, y = a.map_states[k], b.map_states[k]
        if k == "_mapstate":
            for f in ("centres", "structure", "vox2row", "emb"):
                assert torch.equal(getattr(x, f), getattr(y, f)), f
            assert torch.equal(x.packed_children(), y.packed_children())
        else:
            assert x.device == y.device and torch.equal(x, y), k
    _assert_same_state(a.state_dict(), b.state_dict())


@pytest.mark.parametrize("seq", list(SEQUENCES))
def test_restored_map_continues_bit_for_bit_on_either_tree(nl, seq):
    vs, gd, batches = SEQUENCES[seq](nl)
    kw = dict(grid_dim=gd, init_std=0.01, seed=5)
    ref = {o: nl.mapping.MapUpdater(vs, octree=o, **kw) for o in ("host", "device")}
    k = max(1, len(batches) // 2)
    for v in batches[:k]:
        for mu in ref.values():
            mu.insert_voxels(torch.from_numpy(v))
    sd = {o: mu.state_dict() for o, mu in ref.items()}
    _assert_same_state(sd["host"], sd["device"])                     # one format, whichever tree saved it
    res = {(src, dst): nl.mapping.MapUpdater.from_state_dict(sd[src], octree=dst) for src, dst in PAIRS}
    for (src, dst), mu in res.items():
        assert not mu.svo.is_dirty()
        _assert_same_map(mu, ref[dst], updated=False)
    for v in batches[k:]:
        for mu in list(ref.values()) + list(res.values()):
            mu.insert_voxels(torch.from_numpy(v))
        for (src, dst), mu in res.items():
            _assert_same_map(mu, ref[dst])
    _assert_same_state(ref["host"].state_dict(), ref["device"].state_dict())


def _scans(nl, k=3):
    syn = nl.synthetic
    return [syn.make_scan(n_beams=16, n_az=160, seed=300 + i, sensor_xyz=(0.8 * i, 0.1 * i, 0.0)) for i in range(k)]


@pytest.mark.parametrize("octree", ["host", "device"])
def test_restored_map_renders_identically_and_runs_the_captured_graphs(nl, octree):
    rh = nl.render_helpers
    scans = _scans(nl)
    mu = nl.mapping.MapUpdater(0.3, init_std=0.01, seed=4, octree=octree)
    for pts, _, pose in scans:
        ms = mu.create_voxels(torch.from_numpy(pts).cuda(), torch.from_numpy(pose).cuda())
    torch.manual_seed(9)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    crit = nl.criterion.Criterion(Args())
    N = min(s[0].shape[0] for s in scans)
    frames = [nl.frame.LidarFrame(i + 1, torch.from_numpy(p[:N]), torch.from_numpy(c[:N]),
                                  nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(T.copy())), new_keyframe=True)
              for i, (p, c, T) in enumerate(scans)]
    for _ in range(3):
        rh.bundle_adjust_frames(frames, mu.embeddings, ms, dec, crit, 0.3, 0.15, N_rays=512, num_iterations=3, truncation=0.3,
                                max_voxel_hit=20, max_distance=40.0, learning_rate=[0.01, 0.005, 0.001])
    torch.cuda.synchronize()
    res = {o: nl.mapping.MapUpdater.from_state_dict(mu.state_dict(), octree=o) for o in ("host", "device")}
    pts, _, pose = scans[-1]
    P = torch.from_numpy(pts[::4]).cuda()
    T = torch.from_numpy(pose).cuda()
    rd = ((P / P.norm(dim=-1, keepdim=True)) @ T[:3, :3].T)[None].contiguous()
    ro = T[:3, 3].expand_as(rd).contiguous()
    want = rh.render_rays(ro, rd, mu.map_states["_mapstate"], dec, 0.15, 0.3, 0.3, 20, 40.0, deterministic=True)
    assert want is not None
    for o, r in res.items():
        got = rh.render_rays(ro, rd, r.map_states["_mapstate"], dec, 0.15, 0.3, 0.3, 20, 40.0, deterministic=True)
        assert set(got) == set(want)
        for key in ("z_vals", "sdf", "ray_mask", "valid_mask"):
            assert torch.equal(got[key], want[key]), (o, key)
    for o, r in res.items():                                          # the captured optimisation loops on the restored maps
        ms_r = r.map_states["_mapstate"]
        rh.bundle_adjust_frames(frames, r.embeddings, ms_r, copy.deepcopy(dec), crit, 0.3, 0.15, N_rays=512, num_iterations=2,
                                truncation=0.3, max_voxel_hit=20, max_distance=40.0, learning_rate=[0.01, 0.005, 0.001], cuda_graph=True)
        assert rh._MapGraph._cache.get("g") is not None
        fr = nl.frame.LidarFrame(9, torch.from_numpy(pts[:N]), torch.from_numpy(scans[-1][1][:N]),
                                 nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose.copy())), new_keyframe=True)
        out, hit = rh.track_frame(fr.pose, fr, ms_r, dec, crit, 0.3, N_rays=512, step_size=0.06, num_iterations=3, truncation=0.3,
                                  learning_rate=0.01, max_voxel_hit=20, max_distance=40.0, cuda_graph=True)
        assert rh._TrackGraph._cache
        torch.cuda.synchronize()
        assert hit is not None and int(hit.sum()) > 0 and bool(torch.isfinite(out.data).all())
        assert bool(torch.isfinite(r.embeddings.float()).all())


def _trace(fn):
    """(fn(), its host-to-device and device-to-host copies) from a profiler trace of one call.  The profiler runs a warm-up call
    of fn first and records the second: in a process that has already been profiled, the first GPU activity records of a new
    session can be missing (on an H100 80GB HBM3 after the preceding GPU test files, the trace lacked the first two host-to-device
    copies although the runtime trace showed every cudaMemcpyAsync), and a missing copy must not be mistaken for one not made."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA],
                                schedule=torch.profiler.schedule(wait=0, warmup=1, active=1, repeat=1)) as prof:
        for _ in range(2):
            out = fn()
            torch.cuda.synchronize()
            prof.step()
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "trace.json")
        prof.export_chrome_trace(f)
        ev = json.load(open(f))["traceEvents"]
    copies = [e for e in ev if e.get("cat") == "gpu_memcpy"]
    return out, [e for e in copies if "HtoD" in e["name"]], [e for e in copies if "DtoH" in e["name"]]


def test_device_restore_copies_each_array_once_and_reads_back_16_bytes(nl):
    vs, gd, batches = _kitti(nl)
    mu = nl.mapping.MapUpdater(vs, grid_dim=gd, octree="device")
    for v in batches[:3]:
        mu.insert_voxels(torch.from_numpy(v))
    sd = mu.state_dict()
    nl.mapping.MapUpdater.from_state_dict(sd, octree="device")        # warm-up: module loading
    res, h2d, d2h = _trace(lambda: nl.mapping.MapUpdater.from_state_dict(sd, octree="device"))
    assert len(h2d) == 6, h2d                                          # child, code, type, level, vertex2row, embeddings
    assert sum(int(e["args"]["bytes"]) for e in h2d) == sum(sd[k].numel() * sd[k].element_size()
                                                           for k in ("child", "code", "type", "level", "vertex2row", "embeddings"))
    assert len(d2h) == 1 and int(d2h[0]["args"]["bytes"]) == 16, d2h
    _assert_same_map(res, mu, updated=False)


def _device_bits(nl, s, rows=True):
    L = nl._capi.lib()
    n = s["type"].shape[0]
    d = [s[k].cuda() for k in ("child", "code", "type", "level", "vertex2row")]
    ws = torch.empty(max(12 * n + 1024, 256), dtype=torch.uint8, device="cuda")
    out = torch.full((2,), -1, dtype=torch.int64, device="cuda")
    p = nl._capi.ptr
    nl._capi.check(L.nl_devoctree_validate(s["grid_dim"], n, p(d[0]), p(d[1]), p(d[2]), p(d[3]), p(d[4]) if rows else None,
                                           s["embeddings"].shape[0], p(ws), ws.numel(), p(out), nl._capi.stream_ptr()), "nl_devoctree_validate")
    a, b = out.tolist()
    return a, b


def test_device_validator_sets_the_host_bits_on_every_mutation(nl):
    sd, cases = mutated_states(nl)
    for s in [sd] + [s for _, s in cases]:
        host = nl.svo.validate_nodes(s["grid_dim"], s["child"], s["code"], s["type"], s["level"], s["vertex2row"], s["embeddings"].shape[0])
        structural = nl.svo.validate_nodes(s["grid_dim"], s["child"], s["code"], s["type"], s["level"])
        a, b = _device_bits(nl, s)
        assert (a, b) == (structural, host & ~structural), (a, b, host, structural)
        assert _device_bits(nl, s) == (a, b)                             # deterministic
        assert _device_bits(nl, s, rows=False) == (structural, 0)
    for bit, _ in cases:
        assert bit in (1, 2, 4, 8, 16, 32, 64)


def test_malformed_device_octree_pickle_raises(nl):
    vs, gd, batches = _grid8(nl)
    dev = nl.svo.DeviceOctree()
    dev.init(gd, 16, vs)
    for v in batches:
        dev.insert(torch.from_numpy(v))
    state = dev.__getstate__()
    ok = nl.svo.DeviceOctree.__new__(nl.svo.DeviceOctree)
    ok.__setstate__(copy.deepcopy(state))
    assert ok.count_nodes() == dev.count_nodes() and ok._restored
    n = len(state["type"])
    gap = [i for i in range(n) if state["type"][i] == -1 and (state["child"][i] == -1).any()][0]
    for key, edit, name in (("child", lambda a: a.__setitem__((gap, int(np.nonzero(a[gap] == -1)[0][0])), n), "RANGE"),
                            ("type", lambda a: a.__setitem__(0, 0), "ROOT"),
                            ("level", lambda a: a.__setitem__(n - 1, 9), "RANGE")):
        bad = copy.deepcopy(state)
        edit(bad[key])
        t = nl.svo.DeviceOctree.__new__(nl.svo.DeviceOctree)
        with pytest.raises(nl._capi.NerfLoamError, match=name):
            t.__setstate__(bad)


def test_device_state_dict_refuses_inserts_not_applied_yet(nl):
    vs, gd, batches = _kitti(nl)
    mu = nl.mapping.MapUpdater(vs, grid_dim=gd, octree="device")
    with pytest.raises(nl._capi.NerfLoamError, match="not applied"):
        mu.state_dict()
    mu.insert_voxels(torch.from_numpy(batches[0]))
    mu.state_dict()
    mu.svo.insert(torch.from_numpy(batches[1]))
    with pytest.raises(nl._capi.NerfLoamError, match="not applied"):
        mu.state_dict()
    mu.update_grid_features()
    mu.state_dict()
