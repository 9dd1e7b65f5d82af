"""The yardstick of the iteration tail (tests/pose_ref.py) checked on the CPU.

* rotation() and pose_grad() against torch float64 autograd through se3pose.OptimizablePose.rotation(), and against central
  differences, at every pose of the GPU test's pose set.
* The loss constants and read-out against criterion.Criterion on explicit padded [R_hit, S] float64 tensors.
* The control folds against literal loops of the reference's `continue` (mapping) and `break` (tracking).
* The bars: the fp32 emulation of the kernels stays inside them, and every Jacobian mutant exceeds its bar by at least 4x."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import pose_ref as P

MARGIN = 4.0
POSES = P.pose_set()


def one_hot_accs():
    """The nine one-hot G (acc = (0, e_j)): they read dR/dw out entry by entry."""
    out = np.zeros((9, 12))
    out[np.arange(9), 3 + np.arange(9)] = 1
    return out


def torch_pose(pose6):
    import nerfloam_b200 as nl
    p = nl.se3pose.OptimizablePose(torch.zeros(6)).double()
    with torch.no_grad():
        p.data.copy_(torch.from_numpy(np.asarray(pose6, np.float64)))
    return p


def test_rotation_and_jacobian_equal_float64_autograd():
    rng = np.random.default_rng(0)
    for pose in POSES:
        w = pose[3:].astype(np.float64)
        R, a = P.rotation(w)
        for acc in list(one_hot_accs()) + [rng.standard_normal(12)]:
            tp = torch_pose(pose)
            Rt = tp.rotation()
            L = (Rt * torch.from_numpy(acc[3:].reshape(3, 3))).sum() + (tp.translation() * torch.from_numpy(acc[:3])).sum()
            L.backward()
            assert np.abs(Rt.detach().numpy() - R).max() <= 1e-12 * a.max(), pose
            g, ga = P.pose_grad(w, acc)
            assert np.all(np.abs(tp.data.grad.numpy() - g) <= 1e-12 * (ga + 1e-300)), (pose, tp.data.grad.numpy(), g)


def test_jacobian_equals_central_differences():
    h = 1e-6
    for pose in POSES:
        w = pose[3:].astype(np.float64)
        _, a = P.rotation(w)
        for i in range(3):
            e = np.zeros(3)
            e[i] = h
            fd = (P.rotation(w + e)[0] - P.rotation(w - e)[0]) / (2 * h)
            for j, acc in enumerate(one_hot_accs()):
                g, _ = P.pose_grad(w, acc)
                assert abs(g[3 + i] - fd.reshape(9)[j]) <= 1e-7 * (1 + a.max()), (pose, i, j)


def test_jacobian_at_theta_zero_is_the_generators():
    for acc in one_hot_accs():
        g, _ = P.pose_grad(np.zeros(3), acc)
        assert np.array_equal(g[3:], P.GEN[:, :, :].reshape(3, 9)[:, np.argmax(acc[3:])])


def test_taylor_polynomials_match_se3pose():
    import nerfloam_b200 as nl
    th = torch.tensor(P.THETAS, dtype=torch.float64, requires_grad=True)
    A, B = nl.se3pose.OptimizablePose.taylor_A(th), nl.se3pose.OptimizablePose.taylor_B(th)
    p = P.taylor_AB(np.asarray(P.THETAS))
    assert np.allclose(A.detach().numpy(), p["A"], rtol=0, atol=1e-13 * p["aA"].max())
    assert np.allclose(B.detach().numpy(), p["B"], rtol=0, atol=1e-13 * p["aB"].max())
    dA, = torch.autograd.grad(A.sum(), th)
    assert np.allclose(dA.numpy(), p["dA"], rtol=0, atol=1e-13 * p["adA"].max())


# ------------------------------------------------------------------------------------------------ the bars
def _ratios(mutant=None):
    worst = 0.0
    for pose in POSES:
        w = pose[3:]
        for acc in one_hot_accs():
            ref, _ = P.pose_grad(w.astype(np.float64), acc)
            bar = P.pose_grad_bar(w, acc)
            got = P.emulate_pose_grad(w, acc[3:].astype(np.float32), mutant)
            worst = max(worst, float((np.abs(got.astype(np.float64) - ref[3:]) / bar).max()))
    return worst


def test_emulated_kernels_within_the_bars():
    w = POSES[:, 3:]
    R, _ = P.rotation(w.astype(np.float64))
    em = np.stack([P.emulate_rotation(x) for x in w])
    rot = float((np.abs(em - R) / P.rotation_bar(w)).max())
    jac = _ratios()
    print(f"\nemulated design: rotation {rot:.3f}, Jacobian {jac:.3f} of the bar")
    assert rot <= 1 and jac <= 1


@pytest.mark.parametrize("mutant", P.MUTANTS)
def test_every_jacobian_mutant_exceeds_the_bar(mutant):
    r = _ratios(mutant)
    print(f"\n{mutant}: {r:.3g} x the bar")
    assert r >= MARGIN, r


def test_theta_candidates_cover_every_evaluation_order():
    """Each candidate is a real evaluation: the unfused order is the first, an exactly representable sum gives one value."""
    w = np.float32([3, 4, 12])
    assert np.all(P.theta_candidates(w) == 13.0)
    w = np.float32([0.1, -0.2, 0.3])
    with np.errstate(under="ignore"):
        unfused = np.sqrt(np.float32(np.float32(w[0] * w[0]) + np.float32(w[1] * w[1])) + np.float32(w[2] * w[2]), dtype=np.float32)
    assert P.theta_candidates(w)[0] == unfused
    assert np.all(P.theta_candidates(np.float32([1e-23, 0, 0])) == 0)          # the squares underflow: theta^ = 0 with w != 0


def test_f32_round_and_fma_round_once():
    from fractions import Fraction
    one = Fraction(1)
    # 1 + 2^-24 + 2^-60: a double holds 1 + 2^-24 (a tie for fp32, which would go to 1), the exact value goes up
    x = one + Fraction(1, 2 ** 24) + Fraction(1, 2 ** 60)
    assert P.f32_round(x) == np.float32(1 + 2.0 ** -23)
    assert P.f32_round(one + Fraction(1, 2 ** 24)) == np.float32(1)
    a = np.float32(1 + 2.0 ** -12)
    assert P.fma32(a, a, np.float32(-1)) == np.float32(2.0 ** -11 + 2.0 ** -24)


# ------------------------------------------------------------------------------------------------ loss
def padded_problem(rng, trunc=0.3, max_depth=60.0):
    """Explicit padded [R_hit, S] float64 tensors (the render_rays output the reference's criterion reads) that contain front,
    sdf and back cells among the valid ones, padded cells (valid = 0, z_vals = 80, so z = 80 cos) that are front, sdf or
    neither, and rays of unequal sample counts; one ray misses (ray_mask False)."""
    R, S = 40, 12
    nsamp = rng.integers(1, S + 1, R)
    nsamp[:3] = S
    cos = rng.uniform(0.4, 1.0, R)
    depth = rng.uniform(3, 30, R)
    kind = np.arange(R) % 4                           # padded cells: 1 front, 2 sdf, 0 / 3 back
    depth[kind == 1] = 80 * cos[kind == 1] + trunc + rng.uniform(0.5, 5, (kind == 1).sum())
    depth[kind == 2] = 80 * cos[kind == 2] + rng.uniform(-0.8, 0.8, (kind == 2).sum()) * trunc
    depth = np.minimum(depth, max_depth - 1)
    z_vals = np.full((R, S), 80.0)
    for r in range(R):
        z = depth[r] / cos[r] + rng.uniform(-3, 3, nsamp[r]) * trunc / cos[r]
        z_vals[r, :nsamp[r]] = np.sort(z)
    valid = (np.arange(S)[None, :] < nsamp[:, None]).astype(np.float64)
    sdf = rng.standard_normal((R, S))
    dirs = rng.standard_normal((R + 1, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    cos_all = np.concatenate([cos, [0.7]])
    obs = dirs * (np.concatenate([depth, [5.0]]) / cos_all)[:, None]
    ray_mask = np.ones(R + 1, bool)
    ray_mask[-1] = False
    return dict(z_vals=z_vals, valid=valid, sdf=sdf, obs=obs, cos=cos_all, ray_mask=ray_mask, trunc=trunc, max_depth=max_depth)


def counters_of(pp):
    """The render kernels' loss counters and squared-error sums of a padded problem, in float64 / int."""
    m = pp["ray_mask"]
    cos = pp["cos"][m]
    depth = np.linalg.norm(pp["obs"][m], axis=-1) * cos
    z = pp["z_vals"] * cos[:, None]
    d = depth[:, None]
    t = pp["trunc"]
    front = z < d - t
    back = z > d + t
    sdfm = ~front & ~back & ((d > 0) & (d < pp["max_depth"]))
    v = pp["valid"] > 0
    S = z.shape[1]
    nsamp = v.sum(1)
    zp = 80.0 * cos
    pf = zp < depth - t
    ps = ~pf & ~(zp > depth + t) & (depth > 0) & (depth < pp["max_depth"])
    c = dict(n_hit_rays=int(m.sum()), max_samples=S, cnt_fs_valid=int((front & v).sum()), cnt_sdf_valid=int((sdfm & v).sum()),
             pad_fs_rays=int(pf.sum()), pad_fs_nsamp=int(nsamp[pf].sum()), pad_sdf_rays=int(ps.sum()), pad_sdf_nsamp=int(nsamp[ps].sum()),
             pad_sdf_d2=float((depth[ps] ** 2).sum()), pad_sdf_d2_nsamp=float((depth[ps] ** 2 * nsamp[ps]).sum()))
    sdf = pp["sdf"]
    fs_sum = float(((sdf * front - front) ** 2 * v).sum())
    sdf_sum = float((((z + sdf * t) * sdfm - d * sdfm) ** 2 * v).sum())
    kinds = dict(front=int((front & v).sum()), sdf=int((sdfm & v).sum()), back=int((back & v).sum()), pad_front=int((pf & (nsamp < S)).sum()),
                 pad_sdf=int((ps & (nsamp < S)).sum()), pad_back=int((~pf & ~ps & (nsamp < S)).sum()))
    return c, fs_sum, sdf_sum, kinds


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_loss_restatement_equals_criterion(seed):
    import nerfloam_b200 as nl
    pp = padded_problem(np.random.default_rng(seed))
    fs_w, sdf_w = 1.0, 10000.0
    args = SimpleNamespace(criteria=dict(eiko_weight=0.0, sdf_weight=sdf_w, fs_weight=fs_w, sdf_truncation=pp["trunc"]),
                           data_specs=dict(max_depth=pp["max_depth"]))
    crit = nl.criterion.Criterion(args)
    t = lambda x: torch.from_numpy(np.asarray(x))
    out = dict(ray_mask=t(pp["ray_mask"]), z_vals=t(pp["z_vals"]), sdf=t(pp["sdf"]), valid_mask=t(pp["valid"]))
    loss, parts = crit(out, t(pp["obs"]), t(pp["cos"][:, None]))
    c, fs_sum, sdf_sum, kinds = counters_of(pp)
    assert min(kinds.values()) > 0, kinds                              # every kind of cell is present
    k = P.loss_prepare(c, fs_w, sdf_w)
    k32 = P.loss_prepare_f32(c, fs_w, sdf_w)
    # criterion.py counts with .float(): its class weights are fp32 values whatever the tensors' type, so they come from the
    # fp32 restatement here; the rest is float64
    fs, sdf, lo = P.loss_finalize(c["n_hit_rays"], c["max_samples"], fs_sum, sdf_sum, k["pad_fs_sum"], k["pad_sdf_sum"], k32["w_fs"],
                                  k32["w_sdf"], fs_w, sdf_w)
    assert abs(lo - float(loss)) <= 1e-12 * abs(float(loss))
    assert abs(fs - parts["fs_loss"]) <= 1e-12 * abs(fs) and abs(sdf - parts["sdf_loss"]) <= 1e-12 * abs(sdf)
    fs, sdf, lo = P.loss_finalize(c["n_hit_rays"], c["max_samples"], fs_sum, sdf_sum, k["pad_fs_sum"], k["pad_sdf_sum"], k["w_fs"], k["w_sdf"],
                                  fs_w, sdf_w)
    # the fp32 emulation stays within a few u of float64 on the same counters
    for f in ("w_fs", "w_sdf", "g_fs", "g_sdf", "pad_fs_sum"):
        assert abs(float(k32[f]) - k[f]) <= 8 * P.U * abs(k[f]), f
    fs32, sdf32, l32 = P.loss_finalize_f32(c["n_hit_rays"], c["max_samples"], fs_sum, sdf_sum, k32["pad_fs_sum"], k32["pad_sdf_sum"][0],
                                           k32["w_fs"], k32["w_sdf"], fs_w, sdf_w)
    assert all(abs(float(x) - lo) <= 8 * P.U * (fs_w * abs(fs) + sdf_w * abs(sdf)) for x in l32)


def test_loss_prepare_f32_rounds_counts_past_2_to_the_24():
    c = dict(n_hit_rays=1, max_samples=1, cnt_fs_valid=2 ** 24 + 1, cnt_sdf_valid=3, pad_fs_rays=0, pad_fs_nsamp=0, pad_sdf_rays=0,
             pad_sdf_nsamp=0, pad_sdf_d2=0.0, pad_sdf_d2_nsamp=0.0)
    k = P.loss_prepare_f32(c, 1.0, 1.0)
    assert k["n_fs"] == np.float32(2 ** 24) and k["n_sdf"] == np.float32(3)
    z = dict(c, n_hit_rays=0, cnt_fs_valid=0, cnt_sdf_valid=0)
    k = P.loss_prepare_f32(z, 1.0, 1.0)
    assert k["g_fs"] == 0 and k["g_sdf"] == 0 and np.isnan(k["w_fs"])          # no hit ray: g finite and zero (w is 0/0)


# ------------------------------------------------------------------------------------------------ control
def test_iter_status_equals_the_mapping_loop():
    """render_helpers.py:405-409: an iteration whose render_rays returns None is skipped (`continue`), no optimiser step."""
    rng = np.random.default_rng(5)
    for trial in range(50):
        seq = [ps[0] for _, ps in P.scripted_stats(rng, int(rng.integers(1, 12)), 1)]
        ctl = P.ctl_init()
        steps = skipped = err = 0
        mn, mx = P.INT32_MAX, 0
        last_none = 0
        for s in seq:
            ctl = P.iter_status(ctl, s)
            err |= s["error"]
            mn, mx = min(mn, s["n_hit_rays"]), max(mx, s["n_samples"])
            last_none = int(s["n_hit_rays"] <= 0 or s["error"] & 1)
            if last_none:
                skipped += 1
                continue
            steps += 1
        assert ctl == [err, skipped, last_none, steps, mn, len(seq), mx, 0], (trial, seq)


def test_iter_status_batch_equals_the_tracking_loops():
    """render_helpers.py:488-491: a tracking problem whose render_rays returns None stops (`break`); the batch keeps iterating
    for the others, and counts the stopped problem's remaining iterations as skipped ones."""
    rng = np.random.default_rng(6)
    K = 31
    for trial in range(20):
        seq = P.scripted_stats(rng, int(rng.integers(1, 10)), K)
        ctl = [P.ctl_init() for _ in range(K)]
        for tot, ps in seq:
            ctl = P.iter_status_batch(ctl, tot, ps)
        for k in range(K):
            steps, stopped = 0, False
            for tot, ps in seq:                                    # the reference's loop for problem k alone
                s = ps[k]
                if s["n_hit_rays"] <= 0 or s["error"] & 1 or s["n_samples"] <= 0:
                    stopped = True
                    break
                steps += 1
            err = 0
            for tot, ps in seq:
                err |= (ps[k]["error"] & 1) | (tot["error"] & 6)
            n = len(seq)
            want = [err, n - steps, int(stopped), steps, min(ps[k]["n_hit_rays"] for _, ps in seq), n, max(t["n_samples"] for t, _ in seq),
                    int(stopped)]
            assert ctl[k] == want, (trial, k)
