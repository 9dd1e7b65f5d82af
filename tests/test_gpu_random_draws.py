"""The device's random draws against their integer restatement (tests/draws_ref.py), bit for bit: the sampler's counter-based noise
(host seed, device seed, per-problem seeds of the batched front end), the batched ray selection at real subset sizes, and the seed
streams of every captured optimisation loop.

A draw is checked through what it produces: a seeded nl_render_samples call must give the same sample list, bit for bit, as the
same call fed the restated noise as a tensor; a selection must be the top-N of the restated keys; iteration t of a captured call
must select and sample exactly what one engine-level iteration does under the seeds s0 + t inc (mod 2^32)."""

import numpy as np
import pytest
import torch

import draws_ref as D
from util import Args, product_map

pytestmark = pytest.mark.gpu

INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
STAT_FIELDS = ("n_hit_rays", "max_hits", "max_samples", "n_samples", "max_steps_ceil", "error", "cnt_fs_valid", "cnt_sdf_valid",
               "pad_fs_rays", "pad_fs_nsamp", "pad_sdf_rays", "pad_sdf_nsamp", "n_fs", "n_sdf", "w_fs", "w_sdf", "g_fs", "g_sdf")
SAMPLE_ARRAYS = ("s_ray", "s_vox", "s_depth", "s_xyz", "s_flag")
PER_RAY = ("hit_rank", "ray_nsamp", "ray_offset")


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


def _i32(x):
    return int(D.i32(x))


def _seed_tensor(x, dev="cuda"):
    return torch.tensor([_i32(x)], dtype=torch.int32, device=dev)


def _assert_same_stats(a, b, what):
    for f in STAT_FIELDS:
        assert np.array_equal(getattr(a, f), getattr(b, f), equal_nan=True), (what, f, getattr(a, f), getattr(b, f))


def _sample_list(eng, st, r0, R):
    M = st.n_samples
    out = {k: getattr(eng, k)[:M].cpu() for k in SAMPLE_ARRAYS}
    out.update({k: getattr(eng, k)[r0:r0 + R].cpu() for k in PER_RAY})
    return out


def _assert_same_list(a, b, what):
    for k in SAMPLE_ARRAYS + PER_RAY:
        x, y = a[k], b[k]
        if x.dtype == torch.float32:
            x, y = x.view(torch.int32), y.view(torch.int32)
        assert torch.equal(x, y), (what, k)


# ------------------------------------------------------------------------------------------------------------------ A. sampler noise
BLOCK_CFG = dict(step_size=0.25, voxel_size=1.0, max_distance=100.0, truncation=0.3, max_depth=60.0, fs_weight=1.0, sdf_weight=1.0)


@pytest.fixture(scope="module")
def block(nl):
    """A solid 8^3 block of 1 m voxels: a ray across it crosses up to 22 voxels, so the hit lists fill all NL_MAX_HITS = 20 slots."""
    vox = np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.int32)
    m = product_map(vox, 1.0, grid_dim=16)
    n = m["centres"].shape[0]
    return nl.engine.MapState(torch.as_tensor(m["centres"]), torch.as_tensor(m["structure"]), torch.full((n, 8), -1, dtype=torch.int32),
                              torch.zeros((1, 16), dtype=torch.bfloat16), "cuda")


def _block_rays(R, seed):
    """Rays aimed at random points of the block from 20-30 m away, about half of them turned away (misses between hits, so that a
    ray's hit rank differs from its index); gt depth around the block, cosines in [0.5, 1]."""
    rng = np.random.default_rng(seed)
    u = rng.normal(size=(R, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    target = rng.uniform(0.0, 8.0, (R, 3))
    ro = (target + rng.uniform(20.0, 30.0, (R, 1)) * u).astype(np.float32)
    rd = np.where(rng.random((R, 1)) < 0.5, -u, u).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t(ro), t(rd), t(rng.uniform(15.0, 35.0, R).astype(np.float32)), t(rng.uniform(0.5, 1.0, R).astype(np.float32))


def _render(nl, ms, rays, **kw):
    ro, rd, gt, cos = rays
    R = ro.shape[0]
    eng = nl.engine.SDFEngine(R, R * 64)
    eng.render_samples(ms, R, BLOCK_CFG, ro, rd, gt, cos, **kw)
    st = eng.read_stats()
    assert st.error == 0, st.error
    return eng, st


@pytest.mark.parametrize("R", [20_000, 700_001])
def test_sampler_noise_equals_the_restated_hash(nl, block, R):
    """A seeded call against the same call fed the restated hash_uniform table (rows by hit rank, keyed by ray index): every output
    bit for bit.  Host seeds, device seeds (0 behaves as 1, INT32_MIN and -1 as their uint32 values), host seed 0 = the midpoints,
    with the reference's chunk quirks on and off.  700 001 rays give ~350 000 hit rays: Kp = R_hit / 200 > 2 x 800, three sampler
    chunks per batch."""
    rays = _block_rays(R, R)
    big = R > 100_000
    if big:
        cases = [(dict(rng_seed=0x9E3779B9), 0x9E3779B9, True), (dict(rng_seed_dev=_seed_tensor(-7)), D.u32(-7), False)]
    else:
        cases = [(dict(rng_seed=s), s, c) for s in (1, 0x1234567, 2 ** 32 - 1) for c in (True, False)]
        cases += [(dict(rng_seed_dev=_seed_tensor(s)), D.sampler_seed(rng_seed_dev=s), c) for s in (0, 5, INT32_MIN, -1, INT32_MAX)
                  for c in (True, False)]
        cases += [(dict(rng_seed=0), 0, c) for c in (True, False)]
        # the device seed 0 is seed 1 (k_sample: seed ? seed : 1u), the same draw as host seed 1
        e0, s0 = _render(nl, block, rays, rng_seed_dev=_seed_tensor(0))
        e1, s1 = _render(nl, block, rays, rng_seed=1)
        _assert_same_stats(s0, s1, "device seed 0 vs host seed 1")
        _assert_same_list(_sample_list(e0, s0, 0, R), _sample_list(e1, s1, 0, R), "device seed 0 vs host seed 1")
        del e0, e1
    for kw, seed, compat in cases:
        what = (sorted(kw), int(seed), compat)
        eng, st = _render(nl, block, rays, reference_compat=compat, **kw)
        got = _sample_list(eng, st, 0, R)
        if not big:
            assert st.max_hits == 20 and st.n_hit_rays < R
        else:
            assert -(-st.n_hit_rays // 200) > 2 * 800, st.n_hit_rays
        del eng
        table = torch.from_numpy(D.noise_table(int(seed), got["hit_rank"].numpy(), st.max_steps_ceil)).cuda()
        eng, st2 = _render(nl, block, rays, noise=table, reference_compat=compat)
        _assert_same_stats(st, st2, what)
        _assert_same_list(got, _sample_list(eng, st2, 0, R), what)
        assert st.pad_sdf_d2 == pytest.approx(st2.pad_sdf_d2, rel=1e-12)     # fp64 atomics: the order of the sum is free
        del eng, table
        torch.cuda.empty_cache()
    print(f"\n[noise] R={R}: R_hit={st.n_hit_rays} P={st.max_hits} samples={st.n_samples} cases={len(cases)}")


# ------------------------------------------------------------------------------------------------------------------ scenes
VS = 0.3
CFG = dict(step_size=0.15, voxel_size=VS, max_distance=40.0, truncation=0.3, max_depth=40.0, fs_weight=1.0, sdf_weight=10000.0)


@pytest.fixture(scope="module")
def scene(nl):
    """Three synthetic scans on a MapUpdater map (stable addresses: the captured loops run on it), a seeded decoder."""
    syn = nl.synthetic
    mu = nl.mapping.MapUpdater(VS, init_std=0.02, seed=4, reserve_nodes=200_000, reserve_rows=200_000)
    frames, ms = [], None
    for i in range(3):
        pts, cos, pose = syn.make_scan(n_beams=32, n_az=600, seed=300 + i, sensor_xyz=(1.0 * i, 0.0, 0.0))
        f = nl.frame.LidarFrame(i, torch.from_numpy(pts), torch.from_numpy(cos), nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose).float()),
                                new_keyframe=True)
        ms = mu.create_voxels(f.points, f.get_pose().detach())
        frames.append(f)
    torch.manual_seed(3)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    return mu, ms, frames, dec


def _pose6(nl, frame, far=False):
    p = frame.pose.data.detach().reshape(6).float().clone()
    if far:
        p[0] += 500.0
    return p


# ------------------------------------------------------------------------------------------------------------------ B. batched front end
@pytest.mark.parametrize("K", [1, 2, 31, 40])
def test_batched_front_end_draws_each_problem_from_its_own_seed(nl, scene, K):
    """nl_render_samples_batch with per-problem seeds (0, -1, INT32_MIN, INT32_MAX and others; one problem 500 m from the map): problem k
    equals a solo call with rng_seed_dev = seeds[k], and a solo call fed the restated table keyed by ray counter r - kN."""
    mu, ms, frames, dec = scene
    dev = torch.device("cuda")
    N = 512
    dirs_all, cos_all, gt_all = nl.render_helpers._frame_arrays(frames[0], dev)
    ids = torch.arange(N, device=dev) * (dirs_all.shape[0] // N)
    dirs, gt, cos = dirs_all[ids].contiguous(), gt_all[ids].contiguous(), cos_all[ids].contiguous()
    base = _pose6(nl, frames[0])
    pose6 = base.repeat(K, 1).clone()
    t = torch.linspace(0.0, 1.0, K)
    pose6[:, 0] += 0.4 * torch.sin(7.0 * t)
    pose6[:, 5] += 0.1 * torch.sin(3.0 * t)
    far = K // 2 if K > 1 else None
    if far is not None:
        pose6[far, 0] += 500.0
    ro, rd = nl.score.rays_of_poses(pose6.cuda().contiguous(), dirs)
    special = [0, -1, INT32_MIN, INT32_MAX, 0x5EED]
    seeds = [special[k] if k < len(special) else 0x1000 + 7919 * k for k in range(K)]
    eng = nl.engine.SDFEngine(K * N, K * N * 40, dev)
    pst = torch.zeros((K, nl.engine.STATS_BYTES), dtype=torch.uint8, device=dev)
    bbase = torch.empty(K, dtype=torch.int32, device=dev)
    sd = torch.tensor(seeds, dtype=torch.int32, device=dev)
    b = nl._capi.BatchArgs()
    b.n_problems, b.noise_rows, b.d_problem_stats, b.d_problem_base, b.d_problem_seeds = K, 0, pst.data_ptr(), bbase.data_ptr(), sd.data_ptr()
    eng.render_samples(ms, K * N, CFG, ro, rd, gt.repeat(K).contiguous(), cos.repeat(K).contiguous(), None, 0, True, None, batch=b)
    tot = eng.read_stats()
    assert tot.error & 6 == 0
    host = pst.cpu().numpy()
    off = 0
    for k in range(K):
        bs = nl._capi.RenderStats.from_buffer_copy(host[k].tobytes())
        M = bs.n_samples
        batch_list = {n: getattr(eng, n)[off:off + M].cpu() for n in SAMPLE_ARRAYS}
        batch_list["s_ray"] = batch_list["s_ray"] - k * N
        batch_list.update({n: getattr(eng, n)[k * N:(k + 1) * N].cpu() for n in ("hit_rank", "ray_nsamp")})
        ro_k, rd_k = ro[k * N:(k + 1) * N].contiguous(), rd[k * N:(k + 1) * N].contiguous()
        solo = nl.engine.SDFEngine(N, N * 40, dev)
        solo.render_samples(ms, N, CFG, ro_k, rd_k, gt, cos, rng_seed_dev=_seed_tensor(seeds[k]))
        st = solo.read_stats()
        _assert_same_stats(bs, st, (K, k, "solo"))
        sl = _sample_list(solo, st, 0, N)
        for n in SAMPLE_ARRAYS + ("hit_rank", "ray_nsamp"):
            x, y = batch_list[n], sl[n]
            if x.dtype == torch.float32:
                x, y = x.view(torch.int32), y.view(torch.int32)
            assert torch.equal(x, y), (K, k, n)
        if st.n_hit_rays > 0:
            table = torch.from_numpy(D.noise_table(D.sampler_seed(seg_seed=seeds[k]), sl["hit_rank"].numpy(), st.max_steps_ceil)).cuda()
            solo.render_samples(ms, N, CFG, ro_k, rd_k, gt, cos, noise=table)
            st2 = solo.read_stats()
            _assert_same_stats(st, st2, (K, k, "table"))
            _assert_same_list(sl, _sample_list(solo, st2, 0, N), (K, k, "table"))
        else:
            assert k == far
        if k == 0:
            assert st.n_hit_rays > 0
        off += M
    assert off == tot.n_samples


# ------------------------------------------------------------------------------------------------------------------ C. batched selection
SEL_N = 2048
SEL_CAP = 262_144
SEL_LENGTHS = [SEL_N - 1, SEL_N, SEL_N + 1, 131_072, 131_073, SEL_CAP, 70_001]
SENTINEL = -7


@pytest.mark.parametrize("K", [1, 2, 31, 100])
def test_select_rays_batch_draws_each_problem_like_a_solo_call(nl, K):
    """Problem k of nl_select_rays_batch = nl_select_rays over scan k alone under seeds[k] = the N smallest restated keys (frame 0, ties
    to the lower index) in point order; the gathered dirs / gt / cos are those points'; slots past a scan shorter than N keep their
    sentinel.  Scan lengths N - 1, N, N + 1, 131 072 (the last length whose keys stay in registers) and 131 073 (re-hashed), up to cap."""
    dev = torch.device("cuda")
    lib, ptr = nl._capi.lib(), nl._capi.ptr
    special = [0, -1, INT32_MIN, INT32_MAX]
    seeds = [special[k] if k < 4 else int(D.i32(0x2545F491 * (k + 1))) for k in range(K)]
    lengths = [SEL_LENGTHS[(k * 3) % len(SEL_LENGTHS)] if K > 1 else 131_073 for k in range(K)]
    if K >= len(SEL_LENGTHS):
        lengths[:len(SEL_LENGTHS)] = SEL_LENGTHS
    gen = torch.Generator(device=dev).manual_seed(K)
    dirs_all = torch.randn((K, SEL_CAP, 3), device=dev, generator=gen)
    gt_all = torch.arange(SEL_CAP, dtype=torch.float32, device=dev).repeat(K, 1).contiguous()     # exact: every index below 2^24
    cos_all = torch.rand((K, SEL_CAP), device=dev, generator=gen)
    n_dev = torch.tensor(lengths, dtype=torch.int64, device=dev)
    sd = torch.tensor(seeds, dtype=torch.int32, device=dev)

    def outs(k):
        return (torch.full((k * SEL_N, 3), float(SENTINEL), device=dev), torch.full((k * SEL_N,), float(SENTINEL), device=dev),
                torch.full((k * SEL_N,), float(SENTINEL), device=dev), torch.full((k * SEL_N,), SENTINEL, dtype=torch.int32, device=dev))

    o = outs(K)
    nl._capi.check(lib.nl_select_rays_batch(K, SEL_CAP, SEL_N, ptr(n_dev), ptr(sd), ptr(dirs_all), ptr(gt_all), ptr(cos_all), ptr(o[0]), ptr(o[1]),
                                            ptr(o[2]), ptr(o[3]), nl._capi.stream_ptr()), "nl_select_rays_batch")
    idx = o[3].view(K, SEL_N).cpu().numpy()
    for k in range(K):
        n = lengths[k]
        take = min(SEL_N, n)
        want = D.top_n(D.point_key(seeds[k], k, np.arange(n), batched=True), SEL_N)
        assert np.array_equal(idx[k, :take], want), (K, k, seeds[k], n)
        assert (idx[k, take:] == SENTINEL).all(), (K, k)
        w = torch.from_numpy(want).to(dev)
        rows = slice(k * SEL_N, k * SEL_N + take)
        assert torch.equal(o[0][rows], dirs_all[k, w]) and torch.equal(o[1][rows], gt_all[k, w]) and torch.equal(o[2][rows], cos_all[k, w])
        tail = slice(k * SEL_N + take, (k + 1) * SEL_N)
        assert (o[0][tail] == SENTINEL).all() and (o[1][tail] == SENTINEL).all() and (o[2][tail] == SENTINEL).all()
        if k < 8 or k == K - 1:       # the solo kernel call under the same seed
            s = outs(1)
            nl._capi.check(lib.nl_select_rays(1, SEL_CAP, SEL_N, ptr(n_dev[k:k + 1]), ptr(sd[k:k + 1]), 0, ptr(dirs_all[k]), ptr(gt_all[k]),
                                              ptr(cos_all[k]), ptr(s[0]), ptr(s[1]), ptr(s[2]), ptr(s[3]), nl._capi.stream_ptr()), "nl_select_rays")
            assert torch.equal(s[3], o[3][k * SEL_N:(k + 1) * SEL_N])
            for a, b in zip(s[:3], o[:3]):
                assert torch.equal(a, b[k * SEL_N:(k + 1) * SEL_N])


# ------------------------------------------------------------------------------------------------------------------ D. seed streams
# Every loop runs with all learning rates 0: Adam then moves nothing (lr * m / (sqrt(v) + eps) = 0), so the parameters stay at their
# starting values and each iteration's statistics depend on its draw alone.  Its last iteration is replayed on a fresh engine with
# nl_select_rays under seed_at(sel0, 0x632BE5, T - 1) and the sampler under seed_at(noise0, 0x3779B1, T - 1).  Counts, the sample
# list and the loss constants must be equal bit for bit; fs_sum / sdf_sum are fp64 atomic sums whose order is free (1e-12 relative),
# and the fp32 loss read from them may differ by one rounding (2 ulp).
NOISE0_WRAP = 2 ** 31 - 2 * D.SEED_INC_NOISE + 5        # a positive int32 that passes 2^31 in the third iteration
SEL0_WRAP = 2 ** 32 - D.SEED_INC_SELECT + 3              # a negative int32 that passes 2^32 in the second iteration


def _patch_seeds(monkeypatch, nl, noise, sel):
    """The loops' seed draws (render_helpers._seed_from_torch for the sampler, _seed_from_cuda for the selection) return these
    values in order, so that s0 is known and may sit next to a wrap."""
    rh = nl.render_helpers
    noise, sel = iter(noise), iter(sel)
    monkeypatch.setattr(rh, "_seed_from_torch", lambda generator=None: next(noise))
    monkeypatch.setattr(rh, "_seed_from_cuda", lambda dev, generator=None: _seed_tensor(next(sel), dev))


def _replica(nl, ms, dec, frames, pose6, N, sel_seed, noise_seed, update_decoder, update_emb, update_pose, one_frame=False):
    """One engine-level iteration: per-scan selection under sel_seed, rays from pose6, sampler under noise_seed."""
    dev = torch.device("cuda")
    arrays = [nl.render_helpers._frame_arrays(f, dev) for f in frames]
    F = len(frames)
    cap = max(a[0].shape[0] for a in arrays)
    dirs_all, cos_all, gt_all = torch.zeros((F, cap, 3), device=dev), torch.zeros((F, cap), device=dev), torch.zeros((F, cap), device=dev)
    n_dev = torch.zeros(F, dtype=torch.int64, device=dev)
    for i, (d, c, g) in enumerate(arrays):
        n = d.shape[0]
        dirs_all[i, :n], cos_all[i, :n], gt_all[i, :n] = d, c, g
        n_dev[i] = n
    dirs, gt, cos = nl.render_helpers.select_rays_device(dirs_all, gt_all, cos_all, N, n_dev=n_dev, seed=_seed_tensor(sel_seed))
    fid = torch.arange(F, dtype=torch.int32, device=dev).repeat_interleave(N).contiguous()
    eng = nl.engine.SDFEngine(F * N, F * N * 64, dev)
    bufs = nl.engine.DecoderBuffers(dec, dev)
    p6 = pose6.to(dev).reshape(F, 6).contiguous().clone()
    eng.rays_from_poses(p6, dirs, None if one_frame else fid)
    eng.forward_backward(ms, bufs, F * N, CFG, gt, cos, dir_local=dirs, ray_frame=None if one_frame else fid, n_frames=F,
                         update_decoder=update_decoder, update_emb=update_emb, update_pose=update_pose, pose6=p6,
                         rng_seed_dev=_seed_tensor(noise_seed))
    st = eng.read_stats()
    assert st.error & 6 == 0
    return eng, st


def _assert_same_iteration(a_st, a_list, b_st, b_list, what):
    _assert_same_stats(a_st, b_st, what)
    _assert_same_list(a_list, b_list, what)
    assert a_st.fs_sum == pytest.approx(b_st.fs_sum, rel=1e-12, abs=0) and a_st.sdf_sum == pytest.approx(b_st.sdf_sum, rel=1e-12, abs=0), what
    assert abs(a_st.loss - b_st.loss) <= 2 * np.spacing(np.float32(abs(b_st.loss))), (what, a_st.loss, b_st.loss)


def _device_seeds(sel, noise):
    return int(D.u32(int(sel.view(-1)[0]))), int(D.u32(int(noise.view(-1)[0])))


CRIT_ARGS = Args(max_depth=CFG["max_depth"], trunc=CFG["truncation"])
LOOP_KW = dict(step_size=CFG["step_size"], truncation=CFG["truncation"], max_voxel_hit=20, max_distance=CFG["max_distance"])


@pytest.mark.parametrize("pose_rows", [True, False])
def test_bundle_adjust_seed_streams(nl, scene, monkeypatch, pose_rows):
    """bundle_adjust_frames' captured loop (_MapGraph) over two scans: with a pose row (F <= 31: the seeds advance inside the fused pose
    step, nl_pose_step) and without (the torch add_ tail).  After T = 1..4 iterations the device seeds are s0 + T inc; iteration T
    draws what an engine-level iteration draws under s0 + (T - 1) inc.  Then a call with both scans 500 m from the map: every
    iteration is skipped (nothing hit), and the seeds still advance T times, because both tails advance them unconditionally."""
    mu, ms, frames, dec = scene
    rh = nl.render_helpers
    crit = nl.criterion.Criterion(CRIT_ARGS)
    fr = [frames[0], frames[2]]                  # frame index 0 keeps its pose; index 2 is a pose row when update_pose
    N = 512
    pose0 = torch.stack([_pose6(nl, f) for f in fr])
    cases = [(T, 0x1234567 + T, 0x7654321 + 3 * T, False) for T in (1, 2, 3)] + [(4, NOISE0_WRAP, SEL0_WRAP, False), (3, 0xBEEF, 0xF00D, True)]
    for T, noise0, sel0, far in cases:
        keep = [f.pose.data.clone() for f in fr]
        if far:
            with torch.no_grad():        # bundle_adjust_frames leaves the pose parameters requiring grad
                for f in fr:
                    f.pose.data.view(-1)[0] += 500.0
        try:
            _patch_seeds(monkeypatch, nl, [noise0], [sel0])
            rh.bundle_adjust_frames(fr, mu.embeddings, ms, dec, crit, VS, N_rays=N, num_iterations=T, learning_rate=[0.0, 0.0, 0.0],
                                    update_pose=pose_rows, update_decoder=True, deterministic=False, cuda_graph=True, **LOOP_KW)
        finally:
            with torch.no_grad():
                for f, k in zip(fr, keep):
                    f.pose.data.copy_(k)
        g = rh._MapGraph._cache["g"]
        assert (len(g.key[4]) > 0) == pose_rows            # pose_rows: the fused tail ran
        sel_dev, noise_dev = _device_seeds(g.sel_seed, g.seed_dev)
        assert sel_dev == int(D.seed_at(sel0, D.SEED_INC_SELECT, T)), (T, hex(sel_dev))
        assert noise_dev == int(D.seed_at(noise0, D.SEED_INC_NOISE, T)), (T, hex(noise_dev))
        st = g.eng.read_stats()
        if far:
            assert st.n_hit_rays == 0 and g.eng.read_ctl()[nl._capi.CTL_SKIPPED] == T
            continue
        assert torch.equal(torch.stack([_pose6(nl, f) for f in fr]), pose0)       # lr 0: nothing moved
        lst = _sample_list(g.eng, st, 0, 2 * N)
        eng, rst = _replica(nl, ms, dec, fr, pose0, N, D.seed_at(sel0, D.SEED_INC_SELECT, T - 1), D.seed_at(noise0, D.SEED_INC_NOISE, T - 1),
                            True, True, pose_rows)
        assert rst.n_hit_rays > 0
        _assert_same_iteration(st, lst, rst, _sample_list(eng, rst, 0, 2 * N), ("bundle_adjust", pose_rows, T))


def test_track_frame_seed_streams(nl, scene, monkeypatch):
    """track_frame's captured loop (_TrackGraph, seeds advanced in nl_pose_step): device seeds after T = 1..4 iterations and the last
    iteration's draw; a pose 500 m from the map skips every iteration and still advances both seeds T times."""
    mu, ms, frames, dec = scene
    rh = nl.render_helpers
    crit = nl.criterion.Criterion(CRIT_ARGS)
    fr = frames[1]
    N = 1024
    pose0 = _pose6(nl, fr)
    cases = [(T, 0x2345678 + T, 0x3456789 + T, False) for T in (1, 2, 3)] + [(4, NOISE0_WRAP, SEL0_WRAP, False), (2, 0xABC, 0xDEF, True)]
    for T, noise0, sel0, far in cases:
        start = nl.se3pose.OptimizablePose(_pose6(nl, fr, far).reshape(fr.pose.data.shape).clone())
        _patch_seeds(monkeypatch, nl, [noise0], [sel0])
        pose, hit = rh.track_frame(start, fr, ms, dec, crit, VS, N_rays=N, num_iterations=T, learning_rate=0.0, deterministic=False,
                                   cuda_graph=True, ray_selection="device", **LOOP_KW)
        g = list(rh._TrackGraph._cache.values())[-1]
        sel_dev, noise_dev = _device_seeds(g.sel_seed, g.seed_dev)
        assert sel_dev == int(D.seed_at(sel0, D.SEED_INC_SELECT, T)) and noise_dev == int(D.seed_at(noise0, D.SEED_INC_NOISE, T)), (T, far)
        st = g.eng.read_stats()
        if far:
            assert hit is None and st.n_hit_rays == 0 and g.eng.read_ctl()[nl._capi.CTL_SKIPPED] == T
            continue
        assert torch.equal(pose.data.detach().reshape(6).cpu(), pose0)
        eng, rst = _replica(nl, ms, dec, [fr], pose0[None], N, D.seed_at(sel0, D.SEED_INC_SELECT, T - 1),
                            D.seed_at(noise0, D.SEED_INC_NOISE, T - 1), False, False, True, one_frame=True)
        assert rst.n_hit_rays > 0
        _assert_same_iteration(st, _sample_list(g.eng, st, 0, N), rst, _sample_list(eng, rst, 0, N), ("track_frame", T))


def test_track_frames_seed_streams(nl, scene, monkeypatch):
    """track_frames' captured loop (_TrackBatchGraph, seeds advanced per problem in nl_pose_step_batch): three problems with different
    seeds (one about to wrap) and one 500 m from the map.  After T = 1..4 iterations problem k's seeds are its s0 + T inc -- the
    skipped problem's too -- and each live problem's last iteration is the solo engine-level iteration under its own seeds."""
    mu, ms, frames, dec = scene
    crit = nl.criterion.Criterion(CRIT_ARGS)
    dev = torch.device("cuda")
    N = 512
    fr = [frames[0], frames[1], frames[2], frames[1]]
    far = 3
    poses0 = [_pose6(nl, f, far=(k == far)) for k, f in enumerate(fr)]
    for T in (1, 2, 3, 4):
        noise0 = [0x11111 + T, NOISE0_WRAP, 0x33333, 0x44444 + T]
        _patch_seeds(monkeypatch, nl, noise0, [])
        state = torch.cuda.get_rng_state(dev)
        sel0 = [int(D.u32(int(s))) for s in torch.randint(1, 2 ** 31 - 1, (4,), device=dev, dtype=torch.int32).cpu()]   # the call's draw
        torch.cuda.set_rng_state(state, dev)
        starts = [nl.se3pose.OptimizablePose(p.reshape(fr[0].pose.data.shape).clone()) for p in poses0]
        res = nl.track_frames(starts, fr, ms, dec, crit, VS, N_rays=N, num_iterations=T, learning_rate=0.0, deterministic=False,
                              cuda_graph=True, ray_selection="device", **LOOP_KW)
        g = list(nl.track_batch._TrackBatchGraph._cache.values())[-1]
        sel_dev = [int(D.u32(int(s))) for s in g.sel_seeds.cpu()]
        noise_dev = [int(D.u32(int(s))) for s in g.seeds_dev.cpu()]
        assert len(set(sel0)) == 4 and len(set(noise0)) == 4
        for k in range(4):
            assert sel_dev[k] == int(D.seed_at(sel0[k], D.SEED_INC_SELECT, T)), (T, k)
            assert noise_dev[k] == int(D.seed_at(noise0[k], D.SEED_INC_NOISE, T)), (T, k)
        assert res[far][1] is None
        pst = g.tr.problem_stats()
        off = 0
        for k in range(4):
            st = pst[k]
            if k == far:
                assert st.n_hit_rays == 0
                continue
            assert torch.equal(res[k][0].data.detach().reshape(6).cpu(), poses0[k])
            lst = {n: getattr(g.tr.eng, n)[off:off + st.n_samples].cpu() for n in SAMPLE_ARRAYS}
            lst["s_ray"] = lst["s_ray"] - k * N
            lst.update({n: getattr(g.tr.eng, n)[k * N:(k + 1) * N].cpu() for n in ("hit_rank", "ray_nsamp")})
            off += st.n_samples
            eng, rst = _replica(nl, ms, dec, [fr[k]], poses0[k][None], N, D.seed_at(sel0[k], D.SEED_INC_SELECT, T - 1),
                                D.seed_at(noise0[k], D.SEED_INC_NOISE, T - 1), False, False, True, one_frame=True)
            assert rst.n_hit_rays > 0
            rl = _sample_list(eng, rst, 0, N)
            rl = {n: rl[n] for n in lst}
            _assert_same_stats(st, rst, ("track_frames", T, k))
            for n in lst:
                x, y = lst[n], rl[n]
                if x.dtype == torch.float32:
                    x, y = x.view(torch.int32), y.view(torch.int32)
                assert torch.equal(x, y), ("track_frames", T, k, n)
            assert st.fs_sum == pytest.approx(rst.fs_sum, rel=1e-12, abs=0) and st.sdf_sum == pytest.approx(rst.sdf_sum, rel=1e-12, abs=0)
            assert abs(st.loss - rst.loss) <= 2 * np.spacing(np.float32(abs(rst.loss))), (T, k)


def test_refine_map_seed_streams(nl, scene, monkeypatch):
    """refine_map's captured loop (_RefineGraph).  nl_refine_pass_begin sets the selection and noise seeds to the pass's own draws
    (refine_schedule: sel_seeds[p], noise_seeds[p]) on the first iteration of every pass -- a pass does not continue the previous
    pass's stream -- and nl_refine_iter_end advances both after every iteration.  So after P passes of T iterations the device seeds
    are s0[P - 1] + T inc, and the last iteration draws under s0[P - 1] + (T - 1) inc over the last pass's window."""
    mu, ms, frames, dec = scene
    rh = nl.render_helpers
    crit = nl.criterion.Criterion(CRIT_ARGS)
    kg = nl.keyframes.KeyframeGraph(window_size=2, keyframe_gap=0.5, key_distance=CFG["max_distance"], n_rays=512, voxel_size=VS)
    for f in frames:
        kg.insert_keyframe(f)
    N, P = 512, 2
    for T in (1, 2, 3, 4):
        noise0 = [0x5151 + T, NOISE0_WRAP if T == 4 else 0x6161]
        sel0 = [0x7171 + T, SEL0_WRAP if T == 4 else 0x8181]
        _patch_seeds(monkeypatch, nl, noise0, sel0)
        rh.refine_map(kg, mu.embeddings, ms, dec, crit, VS, CFG["step_size"], N_rays=N, num_iterations=T, truncation=CFG["truncation"],
                      max_voxel_hit=20, max_distance=CFG["max_distance"], learning_rate=0.0, passes=P, deterministic=False)
        g = rh._RefineGraph._cache["g"]
        sel_dev, noise_dev = _device_seeds(g.sel_seed, g.seed_dev)
        assert sel_dev == int(D.seed_at(sel0[-1], D.SEED_INC_SELECT, T)) and noise_dev == int(D.seed_at(noise0[-1], D.SEED_INC_NOISE, T)), T
        window = [kg.keyframe_graph[i] for i in g.windows[P - 1].tolist()]
        pose6 = torch.stack([_pose6(nl, f) for f in window])
        st = g.eng.read_stats()
        F = len(window)
        eng, rst = _replica(nl, ms, dec, window, pose6, N, D.seed_at(sel0[-1], D.SEED_INC_SELECT, T - 1), D.seed_at(noise0[-1], D.SEED_INC_NOISE, T - 1),
                            False, True, False)
        assert rst.n_hit_rays > 0
        _assert_same_iteration(st, _sample_list(g.eng, st, 0, F * N), rst, _sample_list(eng, rst, 0, F * N), ("refine_map", T))


def test_capture_is_not_invalidated_by_garbage_holding_pinned_buffers(nl):
    """Regression: refine_map's capture failed ("operation failed due to a previous error during capture") when the cyclic garbage
    collector ran inside it and freed a dropped _RefineGraph -- freeing its engine's pinned read-back buffers records an event on the
    legacy default stream, which invalidates the capture.  _graph_capture now collects such garbage first and keeps the collector off
    while the capture runs."""
    import gc
    import weakref
    rh = nl.render_helpers

    class Holder:
        pass

    h = Holder()
    h.me = h                                             # only the cyclic collector frees it
    h.buf = torch.empty(64, dtype=torch.uint8).pin_memory()
    h.buf.copy_(torch.arange(64, dtype=torch.uint8, device="cuda"), non_blocking=True)      # a stream use of the pinned block
    torch.cuda.synchronize()
    alive = weakref.ref(h)
    del h
    x = torch.zeros(8, device="cuda")
    g = torch.cuda.CUDAGraph()
    with rh._graph_capture(g):
        assert alive() is None and not gc.isenabled()
        x.add_(1.0)
    assert gc.isenabled()
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(x, torch.full((8,), 2.0, device="cuda"))
