"""score_poses and relocalise on the GPU: the batched front end past 31 problems against solo nl_render_samples calls bit for bit, the
score decoder kernel against the forward and train_batch kernels, score_poses against render_rays + Criterion.forward, chunking and
capacity redos, and relocalise recovering a scan from a guess that track_frame cannot recover from."""
import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from util import Args

pytestmark = pytest.mark.gpu

CFG = dict(step_size=0.15, voxel_size=0.3, max_distance=40.0, truncation=0.3, max_depth=40.0, fs_weight=1.0, sdf_weight=10000.0)
STAT_FIELDS = ("n_hit_rays", "max_hits", "max_samples", "n_samples", "max_steps_ceil", "cnt_fs_valid", "cnt_sdf_valid", "pad_fs_rays",
               "pad_fs_nsamp", "pad_sdf_rays", "pad_sdf_nsamp", "n_fs", "n_sdf", "w_fs", "w_sdf", "g_fs", "g_sdf", "error")


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


@pytest.fixture(scope="module")
def scene(nl):
    syn = nl.synthetic
    pts, cos, pose = syn.make_scan(n_beams=32, n_az=240, seed=300)
    mu = nl.mapping.MapUpdater(0.3, init_std=0.02, seed=4)
    ms = mu.insert_voxels(torch.from_numpy(syn.voxelize(pts, pose, 0.3)))
    frame = nl.frame.LidarFrame(5, torch.from_numpy(pts), torch.from_numpy(cos),
                                nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose).float()), new_keyframe=True)
    return ms, frame, pose


def _hypotheses(nl, pose, K, far=()):
    """K poses around the scan's pose (deterministic spread in x, y and yaw); the indices in `far` are moved 500 m away."""
    t = np.linspace(0.0, 1.0, K)
    base = nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose).float()).data.detach()
    p = base.repeat(K, 1).clone()
    p[:, 0] += torch.from_numpy(0.4 * np.sin(7.0 * t)).float()
    p[:, 1] += torch.from_numpy(0.3 * np.cos(5.0 * t)).float()
    p[:, 5] += torch.from_numpy(0.1 * np.sin(3.0 * t)).float()
    for k in far:
        p[k, 0] += 500.0
    return p.contiguous()


def _batch(nl, ms, K, N, ro, rd, gt, cos, seed, cap_per_ray=40):
    """nl_render_samples_batch over K problems of N rays -> (engine, problem statistics (uint8 [K, STATS_BYTES]))."""
    dev = torch.device("cuda")
    eng = nl.engine.SDFEngine(K * N, K * N * cap_per_ray, dev)
    pst = torch.zeros((K, nl.engine.STATS_BYTES), dtype=torch.uint8, device=dev)
    base = torch.empty(K, dtype=torch.int32, device=dev)
    seeds = torch.full((K,), seed, dtype=torch.int32, device=dev)
    b = nl._capi.BatchArgs()
    b.n_problems, b.noise_rows, b.d_problem_stats, b.d_problem_base = K, 0, pst.data_ptr(), base.data_ptr()
    b.d_problem_seeds = seeds.data_ptr() if seed else None
    eng.render_samples(ms, K * N, CFG, ro, rd, gt.repeat(K).contiguous(), cos.repeat(K).contiguous(), None, 0, True, None, batch=b)
    return eng, pst


def _stats(nl, pst, k):
    return nl._capi.RenderStats.from_buffer_copy(pst[k].cpu().numpy().tobytes())


@pytest.mark.parametrize("K", [1, 31, 32, 1000, 4097])
def test_front_end_past_31_problems_equals_solo(nl, scene, K):
    """Problems at both ends, at 32-problem and 1024-problem edges and one 500 m from the map: hit ranks, R_hit, P, S_max, n_samples, raw
    counters, loss constants, error bits and the sample list equal nl_render_samples over that problem's rays alone, under one seed."""
    ms, frame, pose = scene
    dev = torch.device("cuda")
    N = 64
    dirs_all, cos_all, gt_all = nl.render_helpers._frame_arrays(frame, dev)
    ids = torch.arange(0, dirs_all.shape[0], dirs_all.shape[0] // N, device=dev)[:N]
    dirs, gt, cos = dirs_all[ids].contiguous(), gt_all[ids].contiguous(), cos_all[ids].contiguous()
    far = K // 2
    pose6 = _hypotheses(nl, pose, K, far=(far,) if K > 1 else ()).cuda()
    ro, rd = nl.score.rays_of_poses(pose6, dirs)
    seed = 0x5EED
    eng, pst = _batch(nl, ms, K, N, ro, rd, gt, cos, seed)
    tot = eng.read_stats()
    assert tot.error & 6 == 0
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), pst.view(torch.int32)[:, nl.score._NSAMP_WORD].long().cumsum(0)])
    assert int(offsets[-1]) == tot.n_samples
    check = sorted({k for k in (0, K - 1, 30, 31, 32, 1023, 1024, far) if k < K})
    for k in check:
        solo = nl.engine.SDFEngine(N, N * 40)
        solo.render_samples(ms, N, CFG, ro[k * N:(k + 1) * N].contiguous(), rd[k * N:(k + 1) * N].contiguous(), gt, cos, None, seed, True)
        st = solo.read_stats()
        b = _stats(nl, pst, k)
        for f in STAT_FIELDS:
            assert np.array_equal(getattr(b, f), getattr(st, f), equal_nan=True), (k, f, getattr(b, f), getattr(st, f))
        assert b.pad_sdf_d2 == pytest.approx(st.pad_sdf_d2, rel=1e-12)
        assert torch.equal(eng.hit_rank[k * N:(k + 1) * N], solo.hit_rank[:N])
        M, off = st.n_samples, int(offsets[k])
        assert torch.equal(eng.s_ray[off:off + M] - k * N, solo.s_ray[:M])
        for name in ("s_vox", "s_depth", "s_xyz", "s_flag"):
            assert torch.equal(getattr(eng, name)[off:off + M], getattr(solo, name)[:M]), (k, name)
        if k == far and K > 1:
            assert st.n_hit_rays == 0
        elif k == 0:
            assert st.n_hit_rays > 0 and M > 0


def test_score_decoder_kernel_equals_forward_and_train_batch(nl, scene):
    """Per sample the score kernel's sdf is nl_mlp_tc_forward's and nl_mlp_tc_train_batch's bit for bit; per problem its fs / sdf sums
    are train_batch's (fp64 atomics: 1e-12 relative)."""
    ms, frame, pose = scene
    dev = torch.device("cuda")
    torch.manual_seed(3)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).to(dev)
    bufs = nl.engine.DecoderBuffers(dec, dev)
    bufs.refresh_transposes()
    K, N = 40, 512
    dirs_all, cos_all, gt_all = nl.render_helpers._frame_arrays(frame, dev)
    ids = torch.arange(N, device=dev) * (dirs_all.shape[0] // N)
    dirs, gt, cos = dirs_all[ids].contiguous(), gt_all[ids].contiguous(), cos_all[ids].contiguous()
    ro, rd = nl.score.rays_of_poses(_hypotheses(nl, pose, K, far=(7,)).cuda(), dirs)
    eng, pst = _batch(nl, ms, K, N, ro, rd, gt, cos, 0)
    eng._vs = CFG["voxel_size"]
    eng.gather_forward(ms)
    gt_r, cos_r = gt.repeat(K).contiguous(), cos.repeat(K).contiguous()
    lib, st, ptr = nl._capi.lib(), nl._capi.stream_ptr(), nl._capi.ptr
    p = bufs.params
    M = eng.max_samples
    sdf_fwd, sdf_train, sdf_score = (torch.full((M,), float("nan"), device=dev) for _ in range(3))
    nl._capi.check(lib.nl_mlp_tc_forward(M, eng.n_samples_dev, ptr(eng.feats), ptr(bufs.tc_panels), ptr(p[1]), ptr(p[3]), ptr(p[4]), ptr(p[5]),
                                         ptr(sdf_fwd), st), "nl_mlp_tc_forward")
    pst_train, pst_score = pst.clone(), pst.clone()
    nl._capi.check(lib.nl_mlp_tc_train_batch(M, eng.n_samples_dev, ptr(eng.feats), ptr(bufs.tc_panels), ptr(p[1]), ptr(p[3]), ptr(p[4]), ptr(p[5]),
                                             ptr(eng.s_flag), ptr(eng.s_depth), ptr(eng.s_ray), ptr(cos_r), ptr(gt_r), ptr(pst_train), N,
                                             CFG["truncation"], ptr(sdf_train), ptr(eng.dfeats), st), "nl_mlp_tc_train_batch")
    nl._capi.check(lib.nl_mlp_tc_score_batch(M, eng.n_samples_dev, ptr(eng.feats), ptr(bufs.tc_panels), ptr(p[1]), ptr(p[3]), ptr(p[4]), ptr(p[5]),
                                             ptr(eng.s_flag), ptr(eng.s_depth), ptr(eng.s_ray), ptr(cos_r), ptr(gt_r), ptr(pst_score), N,
                                             CFG["truncation"], ptr(sdf_score), st), "nl_mlp_tc_score_batch")
    n = eng.read_stats().n_samples
    assert n > 10000
    assert torch.equal(sdf_score[:n], sdf_fwd[:n]) and torch.equal(sdf_score[:n], sdf_train[:n])
    assert torch.isnan(sdf_score[n:]).all()                # nothing written past the device-side count
    nonzero = 0
    for k in range(K):
        a, b = _stats(nl, pst_train, k), _stats(nl, pst_score, k)
        assert b.fs_sum == pytest.approx(a.fs_sum, rel=1e-12, abs=0) and b.sdf_sum == pytest.approx(a.sdf_sum, rel=1e-12, abs=0)
        nonzero += a.sdf_sum > 0
    assert nonzero >= K - 1 and _stats(nl, pst_score, 7).n_hit_rays == 0


def _decoder(nl, width):
    torch.manual_seed(3)
    return nl.lidar.Decoder(depth=2, width=width, in_dim=16, skips=[], embedder="none", multires=0).cuda()


@pytest.mark.parametrize("width", [256, 64])
@pytest.mark.parametrize("deterministic", [True, False])
def test_score_poses_equals_render_rays_and_criterion(nl, scene, width, deterministic):
    """Each hypothesis' loss is Criterion.forward(render_rays(...)) on the same rays and noise (1e-5 relative), NaN exactly where
    render_rays returns None; two identical poses score bit-identically."""
    ms, frame, pose = scene
    dec = _decoder(nl, width)
    crit = nl.criterion.Criterion(Args())
    K = 10
    pose6 = _hypotheses(nl, pose, K, far=(4,))
    pose6[9] = pose6[2]
    ids = torch.arange(512) * 7
    torch.manual_seed(11)
    res = nl.score_poses(pose6, frame, ms, dec, crit, 0.3, step_size=0.15, max_distance=40.0, deterministic=deterministic, ray_ids=ids)
    assert res.loss.shape == (K,) and res.hit_rays.shape == (K,) and res.n_samples.shape == (K,) and torch.equal(res.ray_ids.cpu(), ids.int())
    dirs_all = nl.render_helpers._frame_arrays(frame, torch.device("cuda"))[0]
    dirs = dirs_all[ids.cuda()].contiguous()
    obs, pcos = frame.points[ids].cuda().view(1, -1, 3), frame.pointsCos[ids].cuda().view(1, -1)
    loss = res.loss.cpu()
    for k in range(K):
        ro, rd = nl.score.rays_of_poses(pose6[k:k + 1].cuda(), dirs)
        torch.manual_seed(11)
        out = nl.render_helpers.render_rays(ro[None], rd[None], ms, dec, 0.15, 0.3, 0.3, 20, 40.0, deterministic=deterministic)
        if out is None:
            assert torch.isnan(loss[k]), k
            continue
        ref, _ = crit(out, obs, pcos)
        assert float(loss[k]) == pytest.approx(float(ref.detach()), rel=1e-5), k
        assert int(res.hit_rays[k]) == int(out["ray_mask"].sum())
        assert int(res.n_samples[k]) == int(out["valid_mask"].sum())
    assert torch.isnan(loss[4]) and int(res.hit_rays[4]) == 0
    assert int(torch.isfinite(loss).sum()) == K - 1
    assert torch.equal(loss[9], loss[2])


def test_chunking_and_capacity_redo_do_not_change_results(nl, scene, monkeypatch):
    """chunk_rays 2^14 (32 hypotheses per chunk) and 2^20 (all in one) give identical results, and so does a run whose chunks all exceed
    their sample capacity and are redone; every chunk reads the host once."""
    ms, frame, pose = scene
    dec = _decoder(nl, 256)
    crit = nl.criterion.Criterion(Args())
    pose6 = _hypotheses(nl, pose, 200, far=(50, 199))
    ids = torch.arange(512) * 5
    reads = []
    orig = nl.engine.SDFEngine.read_stats

    def counting(self):
        reads.append(1)
        return orig(self)
    monkeypatch.setattr(nl.engine.SDFEngine, "read_stats", counting)

    def run(chunk):
        reads.clear()
        torch.manual_seed(2)
        r = nl.score_poses(pose6, frame, ms, dec, crit, 0.3, step_size=0.15, max_distance=40.0, ray_ids=ids, chunk_rays=chunk)
        return r, len(reads)
    small, n_small = run(1 << 14)
    big, n_big = run(1 << 20)
    assert n_small == 7 and n_big == 1
    monkeypatch.setattr(nl.score, "SAMPLES_PER_RAY_SCORE", 1)
    nl.score._ENGINES.clear()
    forced, n_forced = run(1 << 14)
    monkeypatch.setattr(nl.score, "SAMPLES_PER_RAY_SCORE", 32)
    nl.score._ENGINES.clear()
    assert n_forced > 7
    for other in (big, forced):
        torch.testing.assert_close(other.loss, small.loss, rtol=0, atol=0, equal_nan=True)
        assert torch.equal(other.hit_rays, small.hit_rays) and torch.equal(other.n_samples, small.n_samples)
    assert torch.isnan(small.loss[50]) and torch.isnan(small.loss[199]) and int(torch.isfinite(small.loss).sum()) == 198


# ------------------------------------------------------------------------------------------------ relocalise
def _pose_error(nl, p, T_true):
    T = nl.se3pose.OptimizablePose(p.data.detach().cpu().float().clone()).matrix().detach().double()
    dt = float((T[:3, 3] - T_true[:3, 3]).norm())
    c = float(((T[:3, :3].T @ T_true[:3, :3]).trace() - 1.0) / 2.0)
    return dt, math.degrees(math.acos(max(-1.0, min(1.0, c))))


@pytest.fixture(scope="module")
def slam_map(nl):
    return build_slam_map(nl)


def build_slam_map(nl):
    """Four KITTI-shape synthetic scans mapped at their true poses (MapUpdater + bundle_adjust_frames, as scripts/demo_slam.py)."""
    dev = torch.device("cuda")
    syn, rh = nl.synthetic, nl.render_helpers
    vs, md, trunc = 0.3, 40.0, 0.3
    crit = nl.criterion.Criterion(SimpleNamespace(criteria={"eiko_weight": 0.1, "sdf_weight": 10000.0, "fs_weight": 1.0, "sdf_truncation": trunc},
                                                  data_specs={"max_depth": md}))
    torch.manual_seed(777)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).to(dev)
    mu = nl.mapping.MapUpdater(vs, device=dev, reserve_nodes=400_000, reserve_rows=400_000)
    scans = [syn.make_scan(seed=1000 + i, sensor_xyz=(0.5 * i, 0.05 * np.sin(0.7 * i), 0.0), yaw=0.01 * np.sin(0.5 * i)) for i in range(4)]
    gt = [torch.from_numpy(s[2]).float() for s in scans]
    frames = [nl.frame.LidarFrame(i, torch.from_numpy(scans[i][0]), torch.from_numpy(scans[i][1]),
                                  nl.se3pose.OptimizablePose.from_matrix(gt[i].clone()), new_keyframe=True) for i in range(4)]
    ms = None
    for i in range(4):
        ms = mu.create_voxels(scans[i][0], gt[i].double())
        for _ in range(6 if i else 12):
            rh.bundle_adjust_frames(frames[:i + 1], mu.embeddings, ms, dec, crit, vs, 0.5 * vs, N_rays=2048, num_iterations=25,
                                    truncation=trunc, max_voxel_hit=20, max_distance=md, learning_rate=[0.01, 0.005, 0.001],
                                    update_pose=False, update_decoder=True)
    return ms, dec, crit, scans, gt


TRACK = dict(step_size=0.06, truncation=0.3, max_voxel_hit=20, max_distance=40.0)
# 1024 rays and a rate of 0.01 (0.03 / 3 for scan index 2) over 150 iterations: with 512 rays at 0.02 the refined pose jitters by ~8 cm
RELOC = dict(N_rays=1024, refine_iterations=150, learning_rate=0.03, **TRACK)


def test_relocalise_recovers_a_lost_scan(nl, slam_map):
    """From a guess 15 degrees and 1.5 m off, track_frame ends far from the truth; relocalise returns within 5 cm and 0.5 degrees.  From
    the true pose relocalise stays within track_frame's own error (or 5 cm / 0.5 degrees, whichever is larger)."""
    ms, dec, crit, scans, gt = slam_map
    T_true = gt[2].double()
    yaw, off = math.radians(15.0), torch.tensor([1.2, -0.9, 0.0], dtype=torch.float64)
    Rz = torch.tensor([[math.cos(yaw), -math.sin(yaw), 0.0], [math.sin(yaw), math.cos(yaw), 0.0], [0.0, 0.0, 1.0]], dtype=torch.float64)
    T_guess = T_true.clone()
    T_guess[:3, :3] = Rz @ T_true[:3, :3]
    T_guess[:3, 3] = T_true[:3, 3] + off
    guess = nl.se3pose.OptimizablePose.from_matrix(T_guess.float())

    def frame(pose):
        return nl.frame.LidarFrame(2, torch.from_numpy(scans[2][0]), torch.from_numpy(scans[2][1]),
                                   nl.se3pose.OptimizablePose(pose.data.detach().cpu().float().clone()), new_keyframe=True)
    torch.manual_seed(1)
    p_track, _ = nl.render_helpers.track_frame(guess, frame(guess), ms, dec, crit, 0.3, N_rays=2048, num_iterations=25, learning_rate=0.06, **TRACK)
    dt, dr = _pose_error(nl, p_track, T_true)
    print(f"track_frame from the guess: {dt:.3f} m, {dr:.2f} deg")
    assert dt > 0.3 or dr > 3.0
    torch.manual_seed(1)
    p, hit, sc = nl.relocalise(frame(guess), guess, ms, dec, crit, 0.3, **RELOC)
    dt, dr = _pose_error(nl, p, T_true)
    print(f"relocalise from the guess: {dt:.3f} m, {dr:.2f} deg; {sc.loss.shape[0]} hypotheses")
    assert hit is not None and sc.loss.shape[0] == 31 * 81
    assert dt < 0.05 and dr < 0.5

    true = nl.se3pose.OptimizablePose.from_matrix(T_true.float())
    torch.manual_seed(1)
    p_t, _ = nl.render_helpers.track_frame(true, frame(true), ms, dec, crit, 0.3, N_rays=RELOC["N_rays"], num_iterations=RELOC["refine_iterations"],
                                           learning_rate=RELOC["learning_rate"], **TRACK)
    et = _pose_error(nl, p_t, T_true)
    torch.manual_seed(1)
    p_r, _, _ = nl.relocalise(frame(true), true, ms, dec, crit, 0.3, **RELOC)
    er = _pose_error(nl, p_r, T_true)
    print(f"from the true pose: track_frame {et[0]:.3f} m {et[1]:.2f} deg, relocalise {er[0]:.3f} m {er[1]:.2f} deg")
    assert er[0] <= max(et[0], 0.05) and er[1] <= max(et[1], 0.5)
