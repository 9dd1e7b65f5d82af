"""track_frames: K independent tracking problems in one launch chain must each compute what a solo call computes -- the front end bit
for bit per problem, the decoder's per-sample results bit for bit with per-problem loss constants and sums, and the optimised poses
of whole calls (eager and captured) against solo track_frame calls."""
import ctypes as C

import numpy as np
import pytest
import torch

from util import Args

pytestmark = pytest.mark.gpu

CFG = dict(step_size=0.15, voxel_size=0.3, max_distance=40.0, truncation=0.3, max_depth=40.0, fs_weight=1.0, sdf_weight=10000.0)


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


@pytest.fixture(scope="module")
def scene(nl):
    syn = nl.synthetic
    scans = [syn.make_scan(n_beams=32, n_az=240, seed=300 + i, sensor_xyz=(1.0 * i, 0.0, 0.0)) for i in range(3)]
    mu = nl.mapping.MapUpdater(0.3, init_std=0.02, seed=4)
    for pts, cos, pose in scans:
        ms = mu.insert_voxels(torch.from_numpy(syn.voxelize(pts, pose, 0.3)))
    return ms, scans


def _rays(scan, n, shift=(0.0, 0.0, 0.0), up=False):
    """n rays of a scan from its sensor (optionally moved), or n rays straight up that hit nothing; gt depth and cosines."""
    dev = torch.device("cuda")
    pts, cos, pose = scan
    idx = np.arange(n) % pts.shape[0]
    P = torch.from_numpy(pts[idx]).to(dev)
    d = P / P.norm(dim=-1, keepdim=True)
    rd = d @ torch.from_numpy(pose[:3, :3]).to(dev).T
    if up:
        rd = torch.tensor([[0.0, 0.0, 1.0]], device=dev).expand(n, 3)
    ro = (torch.from_numpy(pose[:3, 3]).to(dev) + torch.tensor(shift, device=dev)).expand(n, 3)
    c = torch.from_numpy(cos[idx]).to(dev)
    return ro.contiguous(), rd.contiguous(), (P.norm(dim=-1) * c).contiguous(), c.contiguous()


STAT_FIELDS = ("n_hit_rays", "max_hits", "max_samples", "n_samples", "max_steps_ceil", "cnt_fs_valid", "cnt_sdf_valid", "pad_fs_rays",
               "pad_fs_nsamp", "pad_sdf_rays", "pad_sdf_nsamp", "n_fs", "n_sdf", "w_fs", "w_sdf", "g_fs", "g_sdf")


def _problems(scene, K, chunked):
    ms, scans = scene
    N = 250000 if chunked else 3000
    probs = [_rays(scans[0], N)]
    if K >= 3:
        probs += [_rays(scans[1], N, up=True), _rays(scans[2], N, shift=(0.0, 0.5, 0.2))]
    if K >= 5:
        probs += [_rays(scans[1], N, shift=(-0.4, 0.0, 0.0)), _rays(scans[0], N, shift=(0.0, 0.0, 3.0))]
    return N, probs


@pytest.mark.parametrize("K,chunked", [(1, False), (3, False), (5, False), (3, True)])
@pytest.mark.parametrize("compat", [True, False])
@pytest.mark.parametrize("seeded", [False, True])
def test_front_end_equals_solo_per_problem(nl, scene, K, chunked, compat, seeded):
    """Per problem: hit ranks, R_hit, P, S_max, max_steps_ceil, error bits, raw counters, loss constants and the sample list (voxel
    ids, depths, positions, loss flags) equal nl_render_samples over that problem's rays alone -- including a problem that hits
    nothing, problems whose P differ and, chunked, a problem of more than 160 000 hit rays (the 800-ray chunking)."""
    ms = scene[0]
    dev = torch.device("cuda")
    N, probs = _problems(scene, K, chunked)
    seeds = [0x1234 + 77 * k for k in range(K)] if seeded else [0] * K
    tr = nl.track_batch.BatchTracker(K, N, K * N * 40, dev)
    cat = [torch.cat([p[i] for p in probs]).contiguous() for i in range(4)]
    tr.render(ms, CFG, cat[2], cat[3], ray_o=cat[0], ray_d=cat[1], reference_compat=compat,
              seeds_dev=torch.tensor(seeds, dtype=torch.int32, device=dev) if seeded else None)
    tot = tr.eng.read_stats()
    assert tot.error & 6 == 0
    bst = tr.problem_stats()
    off = 0
    Ps = set()
    for k, (ro, rd, gt, cos) in enumerate(probs):
        solo = nl.engine.SDFEngine(N, N * 40)
        solo.render_samples(ms, N, CFG, ro, rd, gt, cos, None, seeds[k], compat)
        st = solo.read_stats()
        b = bst[k]
        for f in STAT_FIELDS:       # (a problem without hits has NaN class weights, alone as in the batch)
            assert np.array_equal(getattr(b, f), getattr(st, f), equal_nan=True), (k, f, getattr(b, f), getattr(st, f))
        assert (b.error & 1) == (st.error & 1)
        assert b.pad_sdf_d2 == pytest.approx(st.pad_sdf_d2, rel=1e-12)
        assert torch.equal(tr.eng.hit_rank[k * N:(k + 1) * N], solo.hit_rank[:N])
        M = st.n_samples
        assert torch.equal(tr.eng.s_ray[off:off + M] - k * N, solo.s_ray[:M])
        for name in ("s_vox", "s_depth", "s_xyz", "s_flag"):
            assert torch.equal(getattr(tr.eng, name)[off:off + M], getattr(solo, name)[:M]), (k, name)
        off += M
        Ps.add(st.max_hits)
        if chunked and k == 0:
            assert st.n_hit_rays > 160000
    assert off == tot.n_samples
    if K >= 3:
        assert bst[1].n_hit_rays == 0 and len(Ps) >= 2
        assert tr.eng.hit_rank[N:2 * N].max().item() == -1


@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_decoder_loss_per_problem(nl, scene, monkeypatch, impl):
    """Per sample the batched decoder gives the solo sdf and d loss / d features bit for bit (its results do not depend on the tile
    a sample lands in); per problem the squared-error sums and the loss agree with the solo run (loss <= 1e-5 relative)."""
    monkeypatch.setenv("NL_MLP_IMPL", impl)
    ms = scene[0]
    dev = torch.device("cuda")
    torch.manual_seed(3)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).to(dev)
    bufs = nl.engine.DecoderBuffers(dec, dev)
    bufs.refresh_transposes()
    assert nl.engine.mlp_impl(bufs.width) == impl
    K = 3
    N, probs = _problems(scene, K, False)
    tr = nl.track_batch.BatchTracker(K, N, K * N * 40, dev)
    cat = [torch.cat([p[i] for p in probs]).contiguous() for i in range(4)]
    tr.render(ms, CFG, cat[2], cat[3], ray_o=cat[0], ray_d=cat[1])
    tr.eng._vs = CFG["voxel_size"]
    tr.eng.gather_forward(ms)
    tr.decoder(bufs, CFG, cat[2], cat[3])
    lib, st = nl._capi.lib(), nl._capi.stream_ptr()
    for k in range(K):
        nl._capi.check(lib.nl_loss_finalize(C.c_void_p(tr.pstats[k].data_ptr()), CFG["fs_weight"], CFG["sdf_weight"], st), "nl_loss_finalize")
    bst = tr.problem_stats()
    off = 0
    for k, (ro, rd, gt, cos) in enumerate(probs):
        solo = nl.engine.SDFEngine(N, N * 40)
        solo.render_samples(ms, N, CFG, ro, rd, gt, cos)
        solo._vs = CFG["voxel_size"]
        solo.gather_forward(ms)
        nl.engine.mlp_train(bufs, solo.max_samples, solo.n_samples_dev, solo.feats, solo.sdf, solo.dfeats, False, None, s_flag=solo.s_flag,
                            s_depth=solo.s_depth, s_ray=solo.s_ray, cos=cos, gt_depth=gt, stats_ptr=C.c_void_p(solo.stats.data_ptr()),
                            truncation=CFG["truncation"])
        nl._capi.check(lib.nl_loss_finalize(C.c_void_p(solo.stats.data_ptr()), CFG["fs_weight"], CFG["sdf_weight"], st), "nl_loss_finalize")
        s = solo.read_stats()
        M = s.n_samples
        assert torch.equal(tr.eng.feats[off:off + M], solo.feats[:M])
        assert torch.equal(tr.eng.sdf[off:off + M], solo.sdf[:M])
        assert torch.equal(tr.eng.dfeats[off:off + M], solo.dfeats[:M])
        b = bst[k]
        if M:
            assert b.fs_sum == pytest.approx(s.fs_sum, rel=1e-9) and b.sdf_sum == pytest.approx(s.sdf_sum, rel=1e-9)
            assert b.loss == pytest.approx(s.loss, rel=1e-5)
            assert b.loss > 0
        off += M


def _track_setup(nl):
    syn = nl.synthetic
    pts, cos, pose = syn.make_scan(n_beams=16, n_az=120, seed=9)
    mu = nl.mapping.MapUpdater(0.3, init_std=0.02, seed=4)
    ms = mu.insert_voxels(torch.from_numpy(syn.voxelize(pts, pose, 0.3)))
    torch.manual_seed(3)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    start = nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose)).data.detach().clone()
    starts = [start + torch.tensor(d) for d in ([0.05, -0.03, 0.02, 0, 0, 0], [-0.04, 0.02, 0.0, 0, 0, 0.01], [500.0, 0, 0, 0, 0, 0],
                                                  [0.0, 0.05, -0.03, 0.01, 0, 0])]
    return ms, dec, (pts, cos), starts


def _frame(nl, scan, start, index=5):
    pts, cos = scan
    return nl.frame.LidarFrame(index, torch.from_numpy(pts), torch.from_numpy(cos), nl.se3pose.OptimizablePose(start.clone()), new_keyframe=True)


KW = dict(step_size=0.06, num_iterations=3, truncation=0.3, learning_rate=0.03, max_voxel_hit=20, max_distance=40.0, deterministic=True)


@pytest.mark.parametrize("graph", [False, True])
def test_track_frames_equals_solo_track_frame(nl, graph):
    """Every ray selected (N_rays = points), deterministic sampling, 3 iterations: each problem's pose (atol 2e-4, as the solo
    eager/graph test) and hit mask equal a solo track_frame; a problem 500 m from the map returns (start pose, None) and leaves the
    others alone; one frame object appears twice with different starts and frame index 1 takes the 2 lr rate; a second call replays
    the cached graph."""
    ms, dec, scan, starts = _track_setup(nl)
    crit = nl.criterion.Criterion(Args())
    N = scan[0].shape[0]
    twice = _frame(nl, scan, starts[0])
    frames = [twice, _frame(nl, scan, starts[1], index=1), _frame(nl, scan, starts[2]), twice]
    poses = [twice.pose, frames[1].pose, frames[2].pose, nl.se3pose.OptimizablePose(starts[3].clone())]
    res = nl.track_frames(poses, frames, ms, dec, crit, 0.3, N_rays=N, cuda_graph=graph, ray_selection="device", **KW)
    assert len(res) == 4 and res.loss.shape == (4,)
    for k in range(4):
        fr = _frame(nl, scan, poses[k].data.detach(), index=frames[k].index)
        p_solo, h_solo = nl.render_helpers.track_frame(fr.pose, fr, ms, dec, crit, 0.3, N_rays=N, cuda_graph=False, ray_selection="device", **KW)
        p, h = res[k]
        if k == 2:
            assert h is None and h_solo is None and torch.isnan(res.loss[2])
            assert torch.equal(p.data.detach().cpu(), starts[2])
            continue
        assert h is not None and torch.equal(h, h_solo)
        torch.testing.assert_close(p.data.detach().cpu(), p_solo.data.detach().cpu(), rtol=0, atol=2e-4)
        assert float((p.data.detach().cpu() - poses[k].data.detach().cpu()).abs().max()) > 1e-3
        assert torch.isfinite(res.loss[k]) and res.loss[k] > 0
    assert torch.equal(twice.pose.data.detach(), starts[0]) and torch.equal(poses[3].data.detach(), starts[3])   # inputs untouched
    if graph:
        res2 = nl.track_frames(poses, frames, ms, dec, crit, 0.3, N_rays=N, cuda_graph=True, ray_selection="device", **KW)
        for (p, h), (q, g) in zip(res, res2):
            torch.testing.assert_close(q.data.detach().cpu(), p.data.detach().cpu(), rtol=0, atol=2e-5)
            assert (h is None) == (g is None) and (h is None or torch.equal(h, g))


def test_track_frames_sample_overflow_is_redone(nl, monkeypatch):
    """With one sample of capacity per ray every iteration overflows: the call is undone and redone with a larger engine and gives
    the unforced result."""
    ms, dec, scan, starts = _track_setup(nl)
    crit = nl.criterion.Criterion(Args())
    N = scan[0].shape[0]
    rh = nl.render_helpers

    def run(graph):
        frames = [_frame(nl, scan, s) for s in (starts[0], starts[1])]
        return nl.track_frames([f.pose for f in frames], frames, ms, dec, crit, 0.3, N_rays=N, cuda_graph=graph, **KW)
    for graph in (False, True):
        ok = run(graph)
        monkeypatch.setattr(rh, "SAMPLES_PER_RAY_TRACK", 1)
        nl.track_batch._TRACKERS.clear()
        forced = run(graph)
        monkeypatch.setattr(rh, "SAMPLES_PER_RAY_TRACK", 64)
        for (p, h), (q, g) in zip(ok, forced):
            torch.testing.assert_close(q.data.detach().cpu(), p.data.detach().cpu(), rtol=0, atol=2e-5)
            assert torch.equal(h, g)


def test_track_frames_graph_is_one_chain_and_one_read_back(nl):
    """The captured call: num_iterations replays of a chain whose launch count does not depend on K, and ONE host read-back."""
    ms, dec, scan, starts = _track_setup(nl)
    crit = nl.criterion.Criterion(Args())
    N = scan[0].shape[0]
    per_iter = []
    for K in (2, 4):
        frames = [_frame(nl, scan, starts[k % 2]) for k in range(K)]
        nl.track_frames([f.pose for f in frames], frames, ms, dec, crit, 0.3, N_rays=N, cuda_graph=True, **KW)   # capture
        g = next(reversed(nl.track_batch._TrackBatchGraph._cache.values()))
        assert g.K == K
        rb, l0 = g.tr.read_backs, nl._capi.LAUNCHES
        nl.track_frames([f.pose for f in frames], frames, ms, dec, crit, 0.3, N_rays=N, cuda_graph=True, **KW)
        assert g.tr.read_backs == rb + 1
        assert nl._capi.LAUNCHES - l0 == g.launches_per_iter * KW["num_iterations"] + 1      # + the decoder's weight images
        per_iter.append(g.launches_per_iter)
    assert per_iter[0] == per_iter[1]
    with pytest.raises(ValueError):
        frames = [_frame(nl, scan, starts[0])] * 32
        nl.track_frames([f.pose for f in frames], frames, ms, dec, crit, 0.3, N_rays=N, **KW)
