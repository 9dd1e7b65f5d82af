"""Pins the numpy references of tests/embedding_ref.py (used by test_gpu_embedding_path.py against the kernels) on the CPU: bf16
rounding against torch, the gather / scatter / d xyz / pose references against float64 autograd through oracle/chain.py, the
exactness of the dyadic inputs, and the Adam step against torch.optim.Adam."""
import numpy as np
import pytest
import torch

import embedding_ref as ER
from oracle import chain as OC

F32 = np.float32


def test_bf16_rne_matches_torch():
    special = np.array([
        0x3f808000, 0x3f818000, 0xbf808000, 0xbf818000,            # exact ties: even below (stays), odd below (rounds up); both signs
        0x3f807fff, 0x3f808001, 0x00000000, 0x80000000,            # just below / above a tie, +-0
        0x00000001, 0x00008000, 0x00018000, 0x007fffff, 0x807f8000,  # subnormals, ties among them, the largest subnormal
        0x7f7f0000, 0x7f7f7fff, 0x7f7f8000, 0x7f7fffff, 0xff7fffff,  # the largest bf16, the largest below its tie, overflows to +-inf
        0x7f800000, 0xff800000,                                      # +-inf
    ], np.uint32)
    rng = np.random.default_rng(0)
    rand = rng.integers(0, 2 ** 32, 200_000, dtype=np.uint64).astype(np.uint32)
    u = np.concatenate([special, rand])
    u = u[(u & 0x7fffffff) <= 0x7f800000]                          # NaN separately below
    x = u.view(F32)
    want = torch.from_numpy(x.copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    got = ER.bf16_bits(x)
    assert np.array_equal(got, want), int((got != want).sum())
    nan = np.array([0x7fc00000, 0x7f800001, 0xffa00000, 0x7fffffff], np.uint32).view(F32)
    r = ER.bf16_rne(nan)
    assert np.all(np.isnan(r)) and np.all(ER.bf16_bits(nan) & 0x40)      # quiet NaN, also from a signalling one


def _runs(rng, n_vox, M, p=0.25):
    out = []
    while len(out) < M:
        out += [int(rng.integers(0, n_vox))] * int(rng.geometric(p))
    return np.array(out[:M], np.int32)


def _problem(seed, M=3000, **kw):
    rng = np.random.default_rng(seed)
    P = ER.dyadic_problem(rng, _runs(rng, 200, M), 200, 300, empty_vox=(5,), **kw)
    return P


def _autograd(P, ray_frame, F, dtype=torch.float64):
    """float64 autograd: feats = get_features(...), L = sum(feats * dfeats), xyz = t_f + depth * R_f d (straight-through onto the
    given sample positions; R_f = I, t_f = 0 at the evaluation point).  Rows of -1 read a zero row appended to the table."""
    M = len(P["vox"])
    V = P["emb"].shape[0]
    emb = torch.zeros(V + 1, 16, dtype=dtype)
    emb[:V] = torch.from_numpy(P["emb"]).to(dtype)
    emb.requires_grad_()
    rows = torch.from_numpy(P["vox2row"]).long()
    rows = torch.where(rows < 0, torch.full_like(rows, V), rows)
    t = torch.zeros(F, 3, dtype=dtype, requires_grad=True)
    R = torch.eye(3, dtype=dtype).repeat(F, 1, 1).requires_grad_()
    fr = torch.from_numpy(ray_frame[P["s_ray"]]).long() if ray_frame is not None else torch.zeros(M, dtype=torch.long)
    d = torch.from_numpy(P["dir_local"]).to(dtype)[torch.from_numpy(P["s_ray"]).long()]
    dep = torch.from_numpy(P["s_depth"]).to(dtype)
    chain = t[fr] + dep[:, None] * torch.einsum("mab,mb->ma", R[fr], d)
    x0 = torch.from_numpy(P["xyz"]).to(dtype)
    xyz_leaf = x0.clone().requires_grad_()
    xyz = xyz_leaf + (chain - chain.detach())
    feats = OC.get_features(torch.from_numpy(P["vox"]).long(), xyz, torch.from_numpy(P["centres"]).to(dtype), rows, emb,
                            P["voxel_size"])
    g = torch.from_numpy(P["dfeats"]).to(dtype)
    (feats * g).sum().backward()
    acc = torch.cat([t.grad, R.grad.reshape(F, 9)], 1)
    return feats.detach().numpy(), emb.grad[:V].numpy(), xyz_leaf.grad.numpy(), acc.numpy()


@pytest.mark.parametrize("F", [1, 3])
def test_references_equal_float64_autograd_on_dyadic_inputs(F):
    """On dyadic inputs every product and sum is exact in both, so the references equal autograd exactly."""
    P = _problem(1)
    M = len(P["vox"])
    rf = None if F == 1 else (np.arange(M) // 7 % F).astype(np.int32)
    feats, gemb, gxyz, acc = _autograd(P, rf, F)
    args = (P["xyz"], P["vox"], P["centres"], P["vox2row"], P["emb"], P["voxel_size"])
    assert np.array_equal(ER.gather_fwd_f32(*args).astype(np.float64), feats)
    _, w = ER.corner_factors(P["xyz"], P["vox"], P["centres"], P["voxel_size"])
    assert np.array_equal(ER.scatter_ref(P["vox"], P["vox2row"], w, P["dfeats"], P["n_rows"], round_bf16=False)[0], gemb)
    d, da = ER.dxyz_ref(*args, P["dfeats"])
    assert np.array_equal(d, gxyz) and np.all(da >= np.abs(d))
    a, aab = ER.pose_acc_ref(d, da, P["s_ray"], P["s_depth"], P["dir_local"], rf, F)
    assert np.array_equal(a, acc) and np.all(aab >= np.abs(a))
    assert np.any(gemb != 0) and np.any(d != 0) and np.any(acc[:, 3:] != 0)


def test_references_match_float64_autograd_on_random_inputs():
    """General inputs (0.3 m voxel, normal embeddings and gradients): the fp32 forward within a few ulp of float64, the float64
    references within the difference that the fp32 trilinear factors make."""
    rng = np.random.default_rng(2)
    P = _problem(2)
    M = len(P["vox"])
    P["voxel_size"] = 0.3
    P["centres"] = rng.uniform(-5, 5, P["centres"].shape).astype(F32)
    P["xyz"] = (P["centres"][P["vox"]] + rng.uniform(-0.15, 0.15, (M, 3))).astype(F32)
    P["emb"] = ER.bf16_rne(rng.standard_normal(P["emb"].shape).astype(F32))
    P["dfeats"] = rng.standard_normal((M, 16)).astype(F32)
    P["dir_local"] = rng.standard_normal((M, 3)).astype(F32)
    P["s_depth"] = rng.uniform(1, 30, M).astype(F32)
    feats, gemb, gxyz, acc = _autograd(P, None, 1)
    args = (P["xyz"], P["vox"], P["centres"], P["vox2row"], P["emb"], P["voxel_size"])
    np.testing.assert_allclose(ER.gather_fwd_f32(*args), feats, rtol=1e-5, atol=1e-5)
    _, w = ER.corner_factors(P["xyz"], P["vox"], P["centres"], P["voxel_size"])
    np.testing.assert_allclose(ER.scatter_ref(P["vox"], P["vox2row"], w, P["dfeats"], P["n_rows"], round_bf16=False)[0], gemb,
                               rtol=1e-5, atol=1e-5)
    d, da = ER.dxyz_ref(*args, P["dfeats"])
    np.testing.assert_allclose(d, gxyz, rtol=1e-4, atol=1e-4 * np.abs(gxyz).max())
    a, _ = ER.pose_acc_ref(d, da, P["s_ray"], P["s_depth"], P["dir_local"], None, 1)
    np.testing.assert_allclose(a, acc, rtol=1e-4, atol=1e-4 * np.abs(acc).max())


def _orders_exact(terms, key, n_keys):
    """fp32 sums of `terms` grouped by `key`, taken forward, reversed, pairwise (numpy) and in a random order, all equal the
    float64 sum.  terms: float64 values that must be fp32 numbers."""
    t32 = terms.astype(F32)
    assert np.array_equal(t32.astype(np.float64), terms)
    order = np.argsort(key, kind="stable")
    ks, t = key[order], t32[order]
    bounds = np.searchsorted(ks, np.arange(n_keys + 1))
    rng = np.random.default_rng(0)
    busiest = np.argsort(np.diff(bounds))[::-1][:64]
    for k in busiest:
        seg = t[bounds[k]:bounds[k + 1]]
        if not len(seg):
            continue
        want = seg.astype(np.float64).sum(0)
        for s in (np.cumsum(seg, 0, dtype=F32)[-1], np.cumsum(seg[::-1], 0, dtype=F32)[-1], np.sum(seg, 0, dtype=F32),
                  np.cumsum(seg[rng.permutation(len(seg))], 0, dtype=F32)[-1]):
            assert np.array_equal(s.astype(np.float64), want)


@pytest.mark.parametrize("hot", [False, True])
def test_dyadic_inputs_sum_exactly_in_any_order(hot):
    """The premise of the GPU test's exact comparisons, on the same kind of inputs: runs of voxel ids, or one hot voxel shared by
    10^5 samples."""
    if hot:
        rng = np.random.default_rng(3)
        P = ER.dyadic_problem(rng, np.full(100_000, 7, np.int32), 16, 64, g_levels=1, f_levels=1)
    else:
        P = _problem(3, M=20_000, g_levels=1, f_levels=1)
    m = ER.dyadic_margins(P, () if hot else ((None, 1),))
    assert max(m.values()) < 1, m
    _, w = ER.corner_factors(P["xyz"], P["vox"], P["centres"], P["voxel_size"])
    c, rows = ER.contributions(P["vox"], P["vox2row"], w, P["dfeats"])
    keep = rows.reshape(-1) >= 0
    _orders_exact(c.reshape(-1, 16)[keep].astype(np.float64), rows.reshape(-1)[keep], P["n_rows"])
    if not hot:
        d, _ = ER.dxyz_ref(P["xyz"], P["vox"], P["centres"], P["vox2row"], P["emb"], P["voxel_size"], P["dfeats"])
        v, _ = ER.pose_terms(d, P["s_ray"], P["s_depth"], P["dir_local"])
        _orders_exact(v, np.zeros(len(v), np.int64), 1)


def test_adam_step_f32_matches_torch_adam():
    """adam_step (fp32) against torch.optim.Adam on the CPU over a few steps, each from torch's state of the step before.  m and v
    within 1 ulp; p within 4 ulp of the largest operand of its last addition (old p, increment): torch's CPU addcdiv forms
    value * m / denom in another order and divides by the bias correction through a reciprocal, and p + increment may cancel."""
    rng = np.random.default_rng(4)
    n = 10_000
    p = (rng.standard_normal(n) * 0.05).astype(F32)
    m, v = np.zeros(n, F32), np.zeros(n, F32)
    tp = torch.from_numpy(p.copy()).requires_grad_()
    opt = torch.optim.Adam([tp], lr=0.01, foreach=False)
    for t in range(1, 6):
        g = (rng.standard_normal(n) * 10.0 ** -t).astype(F32)
        g[::5] = 0
        tp.grad = torch.from_numpy(g.copy())
        opt.step()
        st = opt.state[tp]
        want = (tp.detach().numpy(), st["exp_avg"].numpy(), st["exp_avg_sq"].numpy())
        got = ER.adam_step(p, g, m, v, 0.01, 0.9, 0.999, 1e-8, t, False)
        for x0, a, b, k in zip((p, m, v), got, want, (4, 1, 1)):
            ulp = np.spacing(np.maximum(np.maximum(np.abs(x0), np.abs(b)), np.abs(b - x0)))
            assert np.all(np.abs(a.astype(np.float64) - b) <= k * ulp), t
        p, m, v = (x.copy() for x in want)
