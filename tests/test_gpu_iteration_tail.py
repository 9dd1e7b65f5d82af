"""The tail of an optimisation iteration against float64 (tests/pose_ref.py): pose matrices, rays and the pose Jacobian within
their derived bars; the fused and batched pose steps, the loss read-out and the iteration control bit for bit against their
restatements; and the multi-rank kernels (statistics exchange, fused reduce + Adam) at W = 2, 3 and 8 ranks emulated on one GPU
through their device pointer tables (no kernel waits on another rank, so launching rank 0 .. W-1 in turn is a valid schedule).
The worst ratio of error to bar of each bar-based test is printed (pytest -s)."""
import ctypes as C

import numpy as np
import pytest
import torch

import pose_ref as P

pytestmark = pytest.mark.gpu

F32 = np.float32
WORST = {}


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


def _note(name, r):
    WORST[name] = max(WORST.get(name, 0.0), float(r))
    print(f"\n{name}: worst {WORST[name]:.3g} of the bar")


# Tensors staged for a launch stay referenced until the test ends: a temporary passed as `cap.ptr(dev(x))` would go back to the
# caching allocator before the kernel runs, and the next argument of the same call could be staged into the same block.
_KEEP = []


@pytest.fixture(autouse=True)
def _release_staged():
    yield
    _KEEP.clear()


def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype=dtype).contiguous()
    _KEEP.append(t)
    return t


def stats_dev(nl, items):
    """Device bytes of one RenderStats per dict in `items`."""
    out = bytearray()
    for fields in items:
        st = nl._capi.RenderStats()
        for k, v in fields.items():
            setattr(st, k, v)
        out += bytes(st)
    t = torch.frombuffer(out, dtype=torch.uint8).cuda()
    _KEEP.append(t)
    return t


def stats_host(nl, t, K=1):
    b = t.cpu().numpy().tobytes()
    n = C.sizeof(nl._capi.RenderStats)
    return [nl._capi.RenderStats.from_buffer_copy(b[k * n:(k + 1) * n]) for k in range(K)]


def f32_bits(x):
    return np.asarray(x, F32).view(np.uint32)


POSES = P.pose_set()


# ------------------------------------------------------------------------------------------------ a. matrices and rays
def _matrices(nl, pose6):
    F = len(pose6)
    Rt = torch.full((F, 12), float("nan"), device="cuda")
    nl._capi.check(nl._capi.lib().nl_pose_matrices(F, nl._capi.ptr(dev(pose6)), nl._capi.ptr(Rt), nl._capi.stream_ptr()))
    return Rt.cpu().numpy()


def test_pose_matrices_within_the_bar(nl):
    for F in (1, 3, 4, 5, 31, 32, 33, len(POSES)):
        for s in range(0, len(POSES), max(F, 17)):
            pose6 = POSES[s:s + F] if s + F <= len(POSES) else np.roll(POSES, -s, 0)[:F]
            Rt = _matrices(nl, pose6)
            R, _ = P.rotation(pose6[:, 3:].astype(np.float64))
            bar = P.rotation_bar(pose6[:, 3:])
            r = np.abs(Rt[:, :9].reshape(-1, 3, 3) - R) / bar
            assert r.max() <= 1, (F, s, np.unravel_index(r.argmax(), r.shape))
            _note("nl_pose_matrices R", r.max())
            assert np.array_equal(f32_bits(Rt[:, 9:]), f32_bits(pose6[:, :3]))
    # theta = 0 and theta^ = 0 with w != 0 (the squares underflow): R = I + [w]x + [w]x^2 / 2, exactly I + [w]x in fp32
    pose6 = np.zeros((2, 6), F32)
    pose6[1, 3:] = F32([1e-23, -2e-23, 3e-23])
    Rt = _matrices(nl, pose6)
    assert np.array_equal(Rt[0, :9], np.eye(3, dtype=F32).reshape(9))
    assert np.array_equal(Rt[1, :9], (np.eye(3) + P.skew(pose6[1, 3:].astype(np.float64))).astype(F32).reshape(9))


RAY_COUNTS = (0, 1, 255, 256, 257, 2048, 10 ** 6 + 3)


@pytest.mark.parametrize("R", RAY_COUNTS)
def test_rays_within_the_bar_and_fused_equals_separate(nl, R):
    cap, lib = nl._capi, nl._capi.lib()
    rng = np.random.default_rng(R)
    st = cap.stream_ptr()
    dirs = rng.standard_normal((R, 3)).astype(F32)
    dirs[: R // 7] = np.eye(3, dtype=F32)[rng.integers(0, 3, R // 7)] * F32(-1) ** rng.integers(0, 2, (R // 7, 1))   # axis-aligned
    dirs_d = dev(dirs.reshape(R, 3)) if R else torch.zeros((1, 3), device="cuda")          # R = 0: valid pointers, nothing read
    for F in (1, 3, 4, 5, 31, 32):
        pose6 = np.roll(POSES, -5 * F, 0)[:F]
        p6 = dev(pose6)
        for with_frame in (False, True):
            if with_frame and F == 1:
                continue
            frame = rng.integers(0, F, R).astype(np.int32) if with_frame else None
            fr = dev(frame) if with_frame and R else None
            Rt_a = torch.empty((F, 12), device="cuda")
            cap.check(lib.nl_pose_matrices(F, cap.ptr(p6), cap.ptr(Rt_a), st))
            o_a, d_a, o_b, d_b, o_c, d_c = (torch.full((max(R, 1), 3), float("nan"), device="cuda") for _ in range(6))
            Rt_b = torch.full((F, 12), float("nan"), device="cuda")
            cap.check(lib.nl_rays_from_poses(R, cap.ptr(dirs_d), cap.ptr(fr), cap.ptr(Rt_a), cap.ptr(o_a), cap.ptr(d_a), st))
            cap.check(lib.nl_rays_from_pose6(R, F, cap.ptr(dirs_d), cap.ptr(fr), cap.ptr(p6), cap.ptr(Rt_b), cap.ptr(o_b), cap.ptr(d_b), st))
            cap.check(lib.nl_rays_from_pose6(R, F, cap.ptr(dirs_d), cap.ptr(fr), cap.ptr(p6), None, cap.ptr(o_c), cap.ptr(d_c), st))
            torch.cuda.synchronize()
            if R == 0:                       # nothing written, nothing launched
                assert torch.isnan(o_a).all() and torch.isnan(o_b).all() and torch.isnan(Rt_b).all()
                continue
            assert torch.equal(Rt_a, Rt_b)
            for o, d in ((o_b, d_b), (o_c, d_c)):
                assert torch.equal(o_a, o) and torch.equal(d_a, d), (F, with_frame)
            Rt = Rt_a.cpu().numpy()
            ro, rd, bar = P.rays(dirs, frame, Rt)
            got = d_a.cpu().numpy()
            r = np.abs(got - rd) / np.maximum(bar, 1e-300)
            assert np.all((r <= 1) | (got == rd)), (F, with_frame, r.max())
            _note("ray directions", np.where(bar > 0, r, 0).max())
            assert np.array_equal(f32_bits(o_a.cpu().numpy()), f32_bits(ro.astype(F32)))


def test_rays_from_pose6_rejects_33_frames(nl):
    cap = nl._capi
    z = torch.zeros((33, 6), device="cuda")
    d = torch.zeros((4, 3), device="cuda")
    assert cap.lib().nl_rays_from_pose6(4, 33, cap.ptr(d), None, cap.ptr(z), None, cap.ptr(d), cap.ptr(d), cap.stream_ptr()) != 0
    assert cap.lib().nl_pose_step(32, cap.ptr(z), cap.ptr(z), cap.ptr(z), 0, None, None, 1e-3, 0.9, 0.999, 1e-8, cap.ptr(z), None, 1.0, 1.0,
                                  None, 0, None, 0, cap.stream_ptr()) != 0


# ------------------------------------------------------------------------------------------------ b. nl_pose_grad
def _pose_grad(nl, pose6, acc):
    F = len(pose6)
    g = torch.full((F, 6), float("nan"), device="cuda")
    nl._capi.check(nl._capi.lib().nl_pose_grad(F, nl._capi.ptr(dev(pose6)), nl._capi.ptr(dev(acc)), nl._capi.ptr(g), nl._capi.stream_ptr()))
    return g.cpu().numpy()


def test_pose_grad_reads_out_the_full_jacobian(nl):
    """Nine one-hot G per pose read dR/dw entry by entry; every entry within its bar; at theta = 0 dR/dw_i = E_i exactly."""
    n = len(POSES)
    worst = 0.0
    for j in range(9):
        acc = np.zeros((n, 12), F32)
        acc[:, 3 + j] = 1
        got = _pose_grad(nl, POSES, acc)
        ref, _ = P.pose_grad(POSES[:, 3:].astype(np.float64), acc.astype(np.float64))
        bar = P.pose_grad_bar(POSES[:, 3:], acc)
        r = np.abs(got[:, 3:] - ref[:, 3:]) / bar
        assert r.max() <= 1, (j, np.unravel_index(r.argmax(), r.shape))
        worst = max(worst, r.max())
        assert np.all(got[:, :3] == 0)
        zero = np.all(POSES[:, 3:] == 0, axis=1)
        assert np.array_equal(got[zero, 3:], np.broadcast_to(P.GEN.reshape(3, 9)[:, j], (zero.sum(), 3)).astype(F32))
    _note("nl_pose_grad one-hot G", worst)


@pytest.mark.parametrize("F", [1, 3, 4, 5, 31, 32, 33])
def test_pose_grad_random_g_and_translation_rows(nl, F):
    rng = np.random.default_rng(F)
    pose6 = np.roll(POSES, -3 * F, 0)[:F]
    acc = (rng.standard_normal((F, 12)) * 10.0 ** rng.integers(-3, 4, (F, 1))).astype(F32)
    got = _pose_grad(nl, pose6, acc)
    ref, _ = P.pose_grad(pose6[:, 3:].astype(np.float64), acc.astype(np.float64))
    bar = P.pose_grad_bar(pose6[:, 3:], acc)
    r = np.abs(got[:, 3:] - ref[:, 3:]) / bar
    assert r.max() <= 1, np.unravel_index(r.argmax(), r.shape)
    _note("nl_pose_grad random G", r.max())
    assert np.array_equal(f32_bits(got[:, :3]), f32_bits(acc[:, :3]))          # dL/dt of every frame passes through


# ------------------------------------------------------------------------------------------------ c. nl_pose_step
LOSS_STATS = dict(n_hit_rays=1000, max_samples=37, n_samples=20000, fs_sum=123.456789, sdf_sum=7.891011, w_fs=0.3, w_sdf=0.7, pad_fs_sum=11.0,
                  pad_sdf_sum=5.5)


def _check_loss_fields(s, fields, fs_w, sdf_w):
    fs, sdf, losses = P.loss_finalize_f32(fields["n_hit_rays"], fields["max_samples"], fields["fs_sum"], fields["sdf_sum"], fields["pad_fs_sum"],
                                          fields["pad_sdf_sum"], fields["w_fs"], fields["w_sdf"], fs_w, sdf_w)
    assert f32_bits(s.fs_loss) == f32_bits(fs) and f32_bits(s.sdf_loss) == f32_bits(sdf)
    assert int(f32_bits(s.loss)) in {int(f32_bits(x)) for x in losses}, (s.loss, losses)


def _adam_rows(pose6, grad6, m, v, mask, lr, step, F):
    p, mm, vv = pose6.copy(), m.copy(), v.copy()
    for f in range(F):
        if (mask >> f) & 1:
            p[f], mm[f], vv[f] = P.adam_step(pose6[f], grad6[f], m[f], v[f], lr, 0.9, 0.999, 1e-8, step, False)
    return p, mm, vv


@pytest.mark.parametrize("F", [1, 7, 31])
def test_pose_step_equals_adam_on_its_own_gradient(nl, F):
    cap, lib = nl._capi, nl._capi.lib()
    st = cap.stream_ptr()
    rng = np.random.default_rng(100 + F)
    pose6 = np.roll(POSES, -F, 0)[:F].copy()
    acc = (rng.standard_normal((F, 12)) * 10.0 ** rng.integers(-2, 3, (F, 1))).astype(F32)
    m0 = (rng.standard_normal((F, 6)) * 1e-2).astype(F32)
    v0 = (rng.random((F, 6)) * 1e-4).astype(F32)
    alt = sum(1 << f for f in range(0, F, 2))
    lr = 1e-3 / 3
    fs_w, sdf_w = 1.0, 10000.0
    for mask in (0, (1 << F) - 1, alt, 1 << (F - 1)):
        for step in (1, 2, 1000):
            for skip in (0, 1):
                ctl = torch.zeros(cap.CTL_WORDS, dtype=torch.int32, device="cuda")
                ctl[cap.CTL_ADAM_STEP], ctl[cap.CTL_SKIP_NOW] = step, skip
                p6, m, v, g6 = dev(pose6), dev(m0), dev(v0), torch.full((F, 6), float("nan"), device="cuda")
                stats = stats_dev(nl, [LOSS_STATS])
                seeds = torch.tensor([2 ** 31 - 5, -7], dtype=torch.int32, device="cuda")
                inc_a, inc_b = 0x632BE5 + step, 2 ** 31 - 1
                cap.check(lib.nl_pose_step(F, cap.ptr(p6), cap.ptr(dev(acc)), cap.ptr(g6), mask, cap.ptr(m), cap.ptr(v), lr, 0.9, 0.999, 1e-8,
                                           cap.ptr(ctl), cap.ptr(stats), fs_w, sdf_w, cap.ptr(seeds[0:1]), inc_a, cap.ptr(seeds[1:2]), inc_b, st))
                g = g6.cpu().numpy()
                assert np.array_equal(f32_bits(g), f32_bits(_pose_grad(nl, pose6, acc)))
                eff = 0 if skip else mask
                p_ref, m_ref, v_ref = _adam_rows(pose6, g, m0, v0, eff, lr, step, F)
                for got, want in ((p6, p_ref), (m, m_ref), (v, v_ref)):
                    assert np.array_equal(f32_bits(got.cpu().numpy()), f32_bits(want)), (mask, step, skip)
                _check_loss_fields(stats_host(nl, stats)[0], LOSS_STATS, fs_w, sdf_w)
                wrap = lambda s, i: (s + i + 2 ** 31) % 2 ** 32 - 2 ** 31
                assert seeds.tolist() == [wrap(2 ** 31 - 5, inc_a), wrap(-7, inc_b)]


# ------------------------------------------------------------------------------------------------ d. nl_pose_step_batch
@pytest.mark.parametrize("K", [1, 2, 17, 31])
def test_pose_step_batch_equals_solo_steps(nl, K):
    cap, lib = nl._capi, nl._capi.lib()
    st = cap.stream_ptr()
    rng = np.random.default_rng(200 + K)
    pose6 = np.roll(POSES, -7 * K, 0)[:K].copy()
    acc = (rng.standard_normal((K, 12)) * 10.0 ** rng.integers(-2, 3, (K, 1))).astype(F32)
    m0 = (rng.standard_normal((K, 6)) * 1e-2).astype(F32)
    v0 = (rng.random((K, 6)) * 1e-4).astype(F32)
    lr = 1e-3 * (1 + np.arange(K) / 7.0) / 3                      # f64 rates fp32 cannot hold
    assert np.all(lr.astype(F32).astype(np.float64) != lr)
    steps = np.array([1, 2, 5, 1000, 3][:1] + list(rng.choice([1, 2, 5, 1000], K - 1)), np.int32)
    skip = (np.arange(K) % 3 == 1).astype(np.int32)
    ctl = np.zeros((K, 8), np.int32)
    ctl[:, P.CTL_ADAM_STEP], ctl[:, P.CTL_SKIP_NOW] = steps, skip
    pstats = [dict(LOSS_STATS, n_hit_rays=int(rng.integers(1, 5000)), max_samples=int(rng.integers(1, 300)), fs_sum=float(rng.random() * 100),
                   sdf_sum=float(rng.random()), w_fs=float(F32(rng.random())), w_sdf=float(F32(rng.random()))) for _ in range(K)]
    seeds_a0 = rng.integers(-2 ** 31, 2 ** 31, K).astype(np.int32)
    seeds_b0 = rng.integers(-2 ** 31, 2 ** 31, K).astype(np.int32)
    seeds_a0[0] = 2 ** 31 - 3
    inc_a, inc_b = 0x632BE5, 0x7FFF0001
    fs_w, sdf_w = 1.0, 10000.0

    def run(with_extras):
        p6, m, v, g6 = dev(pose6), dev(m0), dev(v0), torch.full((K, 6), float("nan"), device="cuda")
        stats = stats_dev(nl, pstats) if with_extras else None
        last = torch.full((K,), float("nan"), device="cuda") if with_extras else None
        sa, sb = (dev(seeds_a0), dev(seeds_b0)) if with_extras else (None, None)
        cap.check(lib.nl_pose_step_batch(K, cap.ptr(p6), cap.ptr(dev(acc)), cap.ptr(g6), cap.ptr(m), cap.ptr(v), cap.ptr(dev(lr)), 0.9, 0.999, 1e-8,
                                         cap.ptr(dev(ctl)), cap.ptr(stats), fs_w, sdf_w, cap.ptr(last), cap.ptr(sa), inc_a, cap.ptr(sb), inc_b, st))
        return p6, m, v, g6, stats, last, sa, sb

    p6, m, v, g6, stats, last, sa, sb = run(True)
    q6, qm, qv, qg, *_ = run(False)
    assert all(torch.equal(a, b) for a, b in ((p6, q6), (m, qm), (v, qv), (g6, qg)))
    got_stats = stats_host(nl, stats, K)
    last = last.cpu().numpy()
    for k in range(K):
        s6, sm, sv, sg = dev(pose6[k:k + 1]), dev(m0[k:k + 1]), dev(v0[k:k + 1]), torch.empty((1, 6), device="cuda")
        sst = stats_dev(nl, [pstats[k]])
        seeds = torch.tensor([seeds_a0[k], seeds_b0[k]], dtype=torch.int32, device="cuda")
        cap.check(lib.nl_pose_step(1, cap.ptr(s6), cap.ptr(dev(acc[k:k + 1])), cap.ptr(sg), 1, cap.ptr(sm), cap.ptr(sv), float(lr[k]), 0.9, 0.999,
                                   1e-8, cap.ptr(dev(ctl[k])), cap.ptr(sst), fs_w, sdf_w, cap.ptr(seeds[0:1]), inc_a, cap.ptr(seeds[1:2]), inc_b, st))
        for a, b in ((p6[k], s6[0]), (m[k], sm[0]), (v[k], sv[0]), (g6[k], sg[0])):
            assert torch.equal(a, b), k
        assert bytes(got_stats[k]) == bytes(stats_host(nl, sst)[0]), k
        assert [int(sa[k]), int(sb[k])] == seeds.tolist(), k
        if skip[k]:
            assert np.isnan(last[k]) and f32_bits(last[k]) == 0x7fc00000, k                 # the NaN sentinel survives
            assert torch.equal(p6[k], dev(pose6[k])) and torch.equal(m[k], dev(m0[k])), k
        else:
            assert f32_bits(last[k]) == f32_bits(got_stats[k].loss), k


# ------------------------------------------------------------------------------------------------ e. loss read-out
def counter_cases():
    base = dict(n_hit_rays=2048, max_samples=37, cnt_fs_valid=30000, cnt_sdf_valid=9000, pad_fs_rays=300, pad_fs_nsamp=4000, pad_sdf_rays=40,
                pad_sdf_nsamp=700, pad_sdf_d2=40 * 612.25 + 0.1, pad_sdf_d2_nsamp=700 * 611.3 + 1e-7)
    big = dict(base, n_hit_rays=2 ** 31 - 1, max_samples=3, cnt_fs_valid=10 ** 10 + 1, cnt_sdf_valid=2 ** 24 + 1, pad_fs_rays=2 ** 31 + 5,
               pad_fs_nsamp=2 ** 32 + 3, pad_sdf_rays=2 ** 25 + 1, pad_sdf_nsamp=2 ** 26 + 7, pad_sdf_d2=1.2345678901e12, pad_sdf_d2_nsamp=3.3e12 + 0.5)
    fs_only = dict(base, cnt_sdf_valid=0, pad_sdf_rays=0, pad_sdf_nsamp=0, pad_sdf_d2=0.0, pad_sdf_d2_nsamp=0.0)
    sdf_only = dict(base, cnt_fs_valid=0, pad_fs_rays=0, pad_fs_nsamp=0)
    pad_only = dict(base, cnt_fs_valid=0, cnt_sdf_valid=0)
    no_hit = dict(base, n_hit_rays=0, max_samples=0, cnt_fs_valid=0, cnt_sdf_valid=0, pad_fs_rays=0, pad_fs_nsamp=0, pad_sdf_rays=0, pad_sdf_nsamp=0,
                  pad_sdf_d2=0.0, pad_sdf_d2_nsamp=0.0)
    return dict(base=base, past_2_31=big, fs_only=fs_only, sdf_only=sdf_only, padding_only=pad_only, no_hit=no_hit)


@pytest.mark.parametrize("case", list(counter_cases()))
def test_loss_prepare_and_finalize(nl, case):
    cap, lib = nl._capi, nl._capi.lib()
    c = counter_cases()[case]
    fs_w, sdf_w = 1.0, 10000.0
    s = stats_dev(nl, [dict(c, fs_sum=5.0, sdf_sum=-1.0, loss=9.0)])
    cap.check(lib.nl_loss_prepare(cap.ptr(s), fs_w, sdf_w, cap.stream_ptr()))
    got = stats_host(nl, s)[0]
    want = P.loss_prepare_f32(c, fs_w, sdf_w)
    for f in ("n_fs", "n_sdf", "w_fs", "w_sdf", "g_fs", "g_sdf", "pad_fs_sum"):
        g, w = F32(getattr(got, f)), want[f]
        assert f32_bits(g) == f32_bits(w) or (np.isnan(g) and np.isnan(w)), (case, f, g, w)
    assert int(f32_bits(got.pad_sdf_sum)) in {int(f32_bits(x)) for x in want["pad_sdf_sum"]}
    assert got.fs_sum == 0 and got.sdf_sum == 0 and got.loss == 0 and got.fs_loss == 0 and got.sdf_loss == 0
    if case == "no_hit":                                          # 0 / 0 class weights; the gradient scales stay finite and zero
        assert got.g_fs == 0 and got.g_sdf == 0 and np.isnan(got.w_fs) and np.isnan(got.w_sdf)
        return
    k64 = P.loss_prepare(c, fs_w, sdf_w)
    worst = 0.0
    N = c["n_hit_rays"] * c["max_samples"]
    for f, a in (("w_fs", abs(k64["w_fs"]) + 2), ("w_sdf", abs(k64["w_sdf"]) + 2), ("g_fs", fs_w * (abs(k64["w_fs"]) + 2) / N),
                 ("g_sdf", sdf_w * (abs(k64["w_sdf"]) + 2) / N)):
        bar = 6 * P.U * a                                           # w = 1 - x with x <= 1: its terms sum to at most |w| + 2
        worst = max(worst, abs(float(getattr(got, f)) - k64[f]) / bar)
        assert abs(float(getattr(got, f)) - k64[f]) <= bar, (case, f)
    # the read-out on sums the decoder would have added
    s2 = stats_dev(nl, [dict(c, **{f: float(getattr(got, f)) for f in ("n_fs", "n_sdf", "w_fs", "w_sdf", "g_fs", "g_sdf", "pad_fs_sum", "pad_sdf_sum")},
                             fs_sum=1234.56789, sdf_sum=0.0123456789)])
    cap.check(lib.nl_loss_finalize(cap.ptr(s2), fs_w, sdf_w, cap.stream_ptr()))
    g2 = stats_host(nl, s2)[0]
    fields = dict(n_hit_rays=c["n_hit_rays"], max_samples=c["max_samples"], fs_sum=1234.56789, sdf_sum=0.0123456789, pad_fs_sum=got.pad_fs_sum,
                  pad_sdf_sum=got.pad_sdf_sum, w_fs=got.w_fs, w_sdf=got.w_sdf)
    _check_loss_fields(g2, fields, fs_w, sdf_w)
    fs, sdf, lo = P.loss_finalize(c["n_hit_rays"], c["max_samples"], 1234.56789, 0.0123456789, k64["pad_fs_sum"], k64["pad_sdf_sum"], k64["w_fs"],
                                  k64["w_sdf"], fs_w, sdf_w)
    for name, g, w, a in (("fs", g2.fs_loss, fs, (1234.56789 + k64["pad_fs_sum"]) / N * (abs(k64["w_fs"]) + 2)),
                          ("sdf", g2.sdf_loss, sdf, (0.0123456789 + k64["pad_sdf_sum"]) / N * (abs(k64["w_sdf"]) + 2))):
        bar = 12 * P.U * a + 1e-300
        worst = max(worst, abs(g - w) / bar)
        assert abs(g - w) <= bar, (case, name, g, w)
    _note("loss constants and read-out vs float64", worst)


def test_loss_finalize_batch_nan_conditions(nl):
    cap, lib = nl._capi, nl._capi.lib()
    fs_w, sdf_w = 1.0, 10000.0
    base = dict(LOSS_STATS)
    items = [base, dict(base, n_hit_rays=0), dict(base, error=1), dict(base, n_samples=0), dict(base, error=2), dict(base, error=4),
             dict(base, error=6, n_samples=5), dict(base, max_samples=3, fs_sum=0.5)]
    K = len(items)
    s = stats_dev(nl, items)
    out = torch.full((K,), -1.0, device="cuda")
    cap.check(lib.nl_loss_finalize_batch(K, cap.ptr(s), fs_w, sdf_w, cap.ptr(out), cap.stream_ptr()))
    got = out.cpu().numpy()
    hs = stats_host(nl, s, K)
    for k, it in enumerate(items):
        f = dict(it)
        _check_loss_fields(hs[k], f, fs_w, sdf_w)            # every block is finalised, NaN or not
        if k in (1, 2, 3):
            assert np.isnan(got[k]), k
        else:
            assert f32_bits(got[k]) == f32_bits(hs[k].loss), k


# ------------------------------------------------------------------------------------------------ f. control
def test_iter_status_in_place_and_alternating(nl):
    cap, lib = nl._capi, nl._capi.lib()
    rng = np.random.default_rng(9)
    seq = [ps[0] for _, ps in P.scripted_stats(rng, 12, 1)]
    inplace = torch.tensor(P.ctl_init(), dtype=torch.int32, device="cuda")
    blocks = torch.zeros((2, 8), dtype=torch.int32, device="cuda")
    blocks[0] = inplace
    want = P.ctl_init()
    for i, s in enumerate(seq):
        d = stats_dev(nl, [s])
        cap.check(lib.nl_iter_status(cap.ptr(d), cap.ptr(inplace), cap.ptr(inplace), cap.stream_ptr()))
        cap.check(lib.nl_iter_status(cap.ptr(d), cap.ptr(blocks[i & 1]), cap.ptr(blocks[(i + 1) & 1]), cap.stream_ptr()))
        prev = want
        want = P.iter_status(want, s)
        assert inplace.tolist() == want and blocks[(i + 1) & 1].tolist() == want, i
        assert blocks[i & 1].tolist() == prev, i                        # the previous iteration's block is left as it was


def test_iter_status_batch_over_a_scripted_call(nl):
    cap, lib = nl._capi, nl._capi.lib()
    K = 31
    rng = np.random.default_rng(10)
    ctl = torch.tensor([P.ctl_init()] * K, dtype=torch.int32, device="cuda")
    want = [P.ctl_init()] * K
    for it, (tot, ps) in enumerate(P.scripted_stats(rng, 9, K)):
        cap.check(lib.nl_iter_status_batch(K, cap.ptr(stats_dev(nl, [tot])), cap.ptr(stats_dev(nl, ps)), cap.ptr(ctl), cap.stream_ptr()))
        want = P.iter_status_batch(want, tot, ps)
        assert ctl.tolist() == want, it
    assert any(c[P.CTL_STOPPED] for c in want) and not all(c[P.CTL_STOPPED] for c in want)


# ------------------------------------------------------------------------------------------------ g. multi-rank on one GPU
def rank_stats(rng, W):
    out = []
    for r in range(W):
        out.append(dict(n_hit_rays=int(rng.integers(0, 10 ** 6)), max_samples=int(rng.integers(0, 400)), error=int(rng.integers(0, 8)) if r % 2 else 0,
                        cnt_fs_valid=int(rng.integers(0, 10 ** 10)), cnt_sdf_valid=int(rng.integers(0, 10 ** 8)), pad_fs_rays=int(rng.integers(0, 10 ** 5)),
                        pad_fs_nsamp=int(rng.integers(0, 10 ** 6)), pad_sdf_rays=int(rng.integers(0, 10 ** 5)), pad_sdf_nsamp=int(rng.integers(0, 10 ** 6)),
                        pad_sdf_d2=float(rng.random() * 1e6), pad_sdf_d2_nsamp=float(rng.random() * 1e8), fs_sum=float(rng.random() * 1e3) / 3,
                        sdf_sum=float(rng.random()) / 7))
    return out


def ptr_table(ts):
    t = torch.tensor([t.data_ptr() for t in ts], dtype=torch.int64, device="cuda")
    _KEEP.append(t)
    return t


@pytest.mark.parametrize("W", [2, 3, 8])
def test_stats_exchange_across_emulated_ranks(nl, W):
    cap, lib = nl._capi, nl._capi.lib()
    st = cap.stream_ptr()
    rng = np.random.default_rng(W)
    fs_w, sdf_w = 1.0, 10000.0
    ranks = rank_stats(rng, W)
    words = cap.STATS_PACK_FIXED + 2 * W
    bufs = [torch.full((words,), float("nan"), dtype=torch.float64, device="cuda") for _ in range(W)]
    for r in range(W):
        cap.check(lib.nl_stats_pack(cap.ptr(stats_dev(nl, [ranks[r]])), cap.ptr(bufs[r]), r, W, 0, st))
    host = [b.cpu().numpy() for b in bufs]
    total = np.zeros(words)
    for h in host:                                         # the SUM all-reduce, in rank order
        total = total + h
    a = stats_dev(nl, [ranks[0]])
    b = stats_dev(nl, [ranks[0]])
    cap.check(lib.nl_stats_unpack(cap.ptr(a), cap.ptr(dev(total)), W, 0, fs_w, sdf_w, st))
    table = ptr_table(bufs)
    cap.check(lib.nl_stats_unpack_peers(cap.ptr(b), cap.ptr(table), W, fs_w, sdf_w, st))
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    g = stats_host(nl, a)[0]
    for f in ("n_hit_rays", "cnt_fs_valid", "cnt_sdf_valid", "pad_fs_rays", "pad_fs_nsamp", "pad_sdf_rays", "pad_sdf_nsamp"):
        assert getattr(g, f) == sum(x[f] for x in ranks), f
    for f in ("pad_sdf_d2", "pad_sdf_d2_nsamp"):
        acc = 0.0
        for x in ranks:
            acc += x[f]
        assert getattr(g, f) == acc, f
    assert g.max_samples == max(x["max_samples"] for x in ranks)
    assert g.error == np.bitwise_or.reduce([x["error"] for x in ranks])
    glob = {f: getattr(g, f) for f in P.COUNTERS}
    want = P.loss_prepare_f32(glob, fs_w, sdf_w)
    for f in ("n_fs", "n_sdf", "w_fs", "w_sdf", "g_fs", "g_sdf", "pad_fs_sum"):
        assert f32_bits(getattr(g, f)) == f32_bits(want[f]), f
    # phase 1: every rank's squared-error sums travel as (hi, lo) float pairs and come back to ~2^-48
    for r in range(W):
        buf = torch.zeros(4, dtype=torch.float32, device="cuda")
        s = stats_dev(nl, [ranks[r]])
        cap.check(lib.nl_stats_pack(cap.ptr(s), cap.ptr(buf), r, W, 1, st))
        back = stats_dev(nl, [{}])
        cap.check(lib.nl_stats_unpack(cap.ptr(back), cap.ptr(buf), W, 1, fs_w, sdf_w, st))
        h = stats_host(nl, back)[0]
        for f in ("fs_sum", "sdf_sum"):
            assert abs(getattr(h, f) - ranks[r][f]) <= 2.0 ** -48 * abs(ranks[r][f]), (r, f)


@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("rows", ["W-1", 3001, 2 ** 16 + 5])
def test_peer_reduce_adam_across_emulated_ranks(nl, W, rows):
    cap, lib = nl._capi, nl._capi.lib()
    st = cap.stream_ptr()
    rows = W - 1 if rows == "W-1" else rows
    n = rows * 16
    hdr_n = 28
    rng = np.random.default_rng(rows + W)
    grads = [(rng.standard_normal(n) * 10.0 ** rng.integers(-3, 1)).astype(F32) for _ in range(W)]
    for g in grads:
        g[rng.random(n) < 0.2] = 0
    hdrs = [rng.standard_normal(hdr_n).astype(F32) for _ in range(W)]
    p0 = P.bf16_bits((rng.standard_normal(n) * 0.01).astype(F32))
    m0 = P.bf16_bits((rng.standard_normal(n) * 1e-3).astype(F32))
    v0 = P.bf16_bits((rng.random(n) * 1e-5).astype(F32))
    lr, step = 0.01, 3
    gsum = np.zeros(n, F32)
    for g in grads:                                          # ((0 + G_0) + G_1) + ... in fp32
        gsum = gsum + g
    hsum = np.zeros(hdr_n, F32)
    for h in hdrs:
        hsum = hsum + h
    pa, ma, va = P.adam_step(P.bf16_to_f32(p0), gsum, P.bf16_to_f32(m0), P.bf16_to_f32(v0), lr, 0.9, 0.999, 1e-8, step, True)
    want_p, want_m, want_v = P.bf16_bits(pa), P.bf16_bits(ma), P.bf16_bits(va)
    u16 = lambda a: dev(a.view(np.int16))
    for skip in (0, 1):
        g_t = [dev(g) for g in grads]
        h_t = [dev(h) for h in hdrs]
        p_t = [u16(p0) for _ in range(W)]
        m_t = [u16(m0) for _ in range(W)]
        v_t = [u16(v0) for _ in range(W)]
        out = [torch.full((hdr_n,), float("nan"), device="cuda") for _ in range(W)]
        ctl = torch.zeros(cap.CTL_WORDS, dtype=torch.int32, device="cuda")
        ctl[cap.CTL_ADAM_STEP], ctl[cap.CTL_SKIP_NOW] = step, skip
        gt, pt, ht = ptr_table(g_t), ptr_table(p_t), ptr_table(h_t)
        for r in range(W):
            cap.check(lib.nl_peer_reduce_adam_bf16(n, r, W, cap.ptr(gt), None, cap.ptr(pt), None, cap.ptr(m_t[r]), cap.ptr(v_t[r]), lr, 0.9, 0.999,
                                                   1e-8, cap.ptr(ctl), hdr_n, cap.ptr(ht), None, cap.ptr(out[r]), st))
        torch.cuda.synchronize()
        bits = lambda t: t.cpu().numpy().view(np.uint16)
        for r in range(W):
            assert np.array_equal(bits(p_t[r]), p0 if skip else want_p), (r, skip)
            lo, hi = rows * r // W * 16, rows * (r + 1) // W * 16
            em, ev = m0.copy(), v0.copy()
            if not skip:
                em[lo:hi], ev[lo:hi] = want_m[lo:hi], want_v[lo:hi]
            assert np.array_equal(bits(m_t[r]), em) and np.array_equal(bits(v_t[r]), ev), (r, skip)
            assert np.array_equal(f32_bits(out[r].cpu().numpy()), f32_bits(hsum)), r
