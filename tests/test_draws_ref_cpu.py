"""tests/draws_ref.py -- the integer restatement of the device generators (sampler noise, ray-selection keys, seed streams) -- against a
plain Python-int restatement and the torch one of test_gpu_ops, and the statistical properties the generators are meant to have.

Every statistical check uses fixed seeds, so its outcome is deterministic; each bar is stated with its derivation next to it, and
the observed value is printed beside the bar (pytest -s)."""
import math

import numpy as np
import pytest
import torch

import draws_ref as D

M = 0xFFFFFFFF
EXTREMES = [0, 1, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1]


# ------------------------------------------------------------------------------------------------------------------ plain Python
def py_mix32(x):
    x &= M
    x ^= x >> 16; x = (x * 0x7FEB352D) & M; x ^= x >> 15; x = (x * 0x846CA68B) & M; x ^= x >> 16
    return x


def py_point_key(seed, f, i):
    s = py_mix32((seed & M) ^ ((0x9E3779B9 * (f + 1)) & M))
    return py_mix32(s ^ py_mix32((i * 0x9E3779B1 + 0x7F4A7C15) & M))


def py_hash_uniform(seed, ray, step):
    x = py_mix32((seed & M) ^ ((ray * 0x9E3779B1) & M) ^ ((step * 0x85EBCA77) & M))
    u = np.float32(x >> 8) * np.float32(1.0 / 16777216.0)
    return min(max(u, np.float32(0.001)), np.float32(0.999))


def _inputs():
    rng = np.random.default_rng(1)
    return EXTREMES + [int(v) for v in rng.integers(0, 2 ** 32, 60, dtype=np.uint64)]


def test_mix32_and_seed_views_match_python_ints():
    xs = _inputs()
    got = D.mix32(np.array(xs, np.uint64))
    assert got.dtype == np.uint32
    assert [int(v) for v in got] == [py_mix32(x) for x in xs]
    # int32 <-> uint32: the device word of a seed and back
    for x in xs:
        w = D.i32(x)
        assert w.dtype == np.int32 and int(w) == (x if x < 2 ** 31 else x - 2 ** 32)
        assert int(D.u32(w)) == x
    assert int(D.u32(-1)) == M and int(D.u32(np.int32(-2 ** 31))) == 2 ** 31


def test_point_keys_match_python_ints_and_the_torch_restatement():
    from test_gpu_ops import _select_keys_torch
    n = 3000
    idx = list(range(50)) + [2 ** 17 - 1, 2 ** 17, 2 ** 31 - 1, 2 ** 31, M]
    for seed in _inputs()[:12]:
        for f in (0, 1, 4, 30):
            got = D.point_key(seed, f, np.array(idx, np.uint64))
            assert [int(v) for v in got] == [py_point_key(seed, f, i) for i in idx], (seed, f)
            t = _select_keys_torch(seed, f, n, torch.device("cpu")).numpy()
            assert np.array_equal(D.point_key(seed, f, np.arange(n)).astype(np.int64), t), (seed, f)
        # batched problems are drawn as frame 0 whatever their index
        assert np.array_equal(D.point_key(seed, 7, np.arange(64), batched=True), D.point_key(seed, 0, np.arange(64)))


def test_hash_uniform_matches_python_ints_and_the_seed_conventions():
    seeds = _inputs()[:20]
    rays = [0, 1, 799, 800, 2 ** 31 - 1, M]
    steps = [0, 1, 19, 127, 4095]
    for s in seeds:
        for r in rays:
            got = D.hash_uniform(s, np.array(r, np.uint64), np.array(steps, np.uint64))
            assert got.dtype == np.float32
            want = np.array([py_hash_uniform(s, r, i) for i in steps], np.float32)
            assert np.array_equal(got.view(np.int32), want.view(np.int32)), (s, r)
    # host seed 0 -> midpoints; device / batch seed 0 -> 1; int32 views of the same seed are the same seed
    assert D.sampler_seed(rng_seed=0) == 0 and D.noise_by_ray(0, 3, 4).tolist() == [[0.5] * 4] * 3
    assert D.sampler_seed(rng_seed_dev=0) == 1 and D.sampler_seed(seg_seed=0) == 1
    assert D.sampler_seed(rng_seed_dev=np.int32(-1)) == M and D.sampler_seed(rng_seed=2 ** 31) == 2 ** 31
    assert D.sampler_seed(rng_seed_dev=np.int32(-2 ** 31), seg_seed=np.int32(5)) == 5


def test_seed_streams_wrap_modulo_2_32():
    for s0 in EXTREMES + [2 ** 31 - 0x632BE5, 2 ** 32 - 3]:
        for inc in (D.SEED_INC_SELECT, D.SEED_INC_NOISE):
            for t in range(6):
                assert int(D.seed_at(s0, inc, t)) == (s0 + inc * t) % 2 ** 32
    assert int(D.seed_at(np.int32(-1), D.SEED_INC_NOISE, 1)) == D.SEED_INC_NOISE - 1


def test_top_n_takes_the_smallest_keys_ties_to_the_lower_index_in_point_order():
    rng = np.random.default_rng(2)
    for n, N in ((1, 1), (7, 3), (1000, 999), (1000, 1000), (1000, 1500), (5000, 64)):
        keys = rng.integers(0, 40, n).astype(np.uint32)              # many ties
        got = D.top_n(keys, N)
        want = sorted(sorted(range(n), key=lambda i: (int(keys[i]), i))[:min(N, n)])
        assert got.tolist() == want


def test_noise_table_is_laid_out_by_hit_rank_and_keyed_by_ray():
    hit_rank = np.array([-1, 0, -1, 1, 2, -1, 3], np.int32)
    t = D.noise_table(0xABC, hit_rank, 5)
    by_ray = D.noise_by_ray(0xABC, 7, 5)
    assert t.shape == (4, 5)
    for r, q in enumerate(hit_rank):
        if q >= 0:
            assert np.array_equal(t[q], by_ray[r])
    assert not np.array_equal(t[1], D.noise_by_ray(0xABC, 2, 5)[1])       # rank 1 is ray 3, not ray 1
    assert D.noise_table(5, np.full(4, -1, np.int32), 3).shape == (1, 3)


# ------------------------------------------------------------------------------------------------------------------ statistics
N_RAYS, N_STEPS = 512, 256                     # n = 131 072 draws per seed
SEEDS = [0x1234567, 0x7FFFFFF0, 0xDEADBEEF]


def _noise(seed):
    r = np.arange(N_RAYS, dtype=np.uint64)[:, None]
    i = np.arange(N_STEPS, dtype=np.uint64)[None, :]
    return D.hash_uniform(seed, r, i), D.hash_word(seed, r, i)


def test_noise_marginal_is_uniform_with_the_clamp_mass_at_both_ends():
    """KS distance to the clamped uniform (CDF 0 below 0.001, x on [0.001, 0.999), 1 from 0.999): under the null sqrt(n) D follows the
    Kolmogorov law, P(sqrt(n) D > 1.95) = 0.001, so the bar is D < 1.95 / sqrt(n).  The clamp masses: the float32 values (x >> 8) / 2^24
    below 0.001f (k <= k_lo) and above 0.999f are counted exactly over all 2^24 words; the number of draws equal to 0.001f (and to
    0.999f) is then Binomial(n, p), held to n p +- 5 sqrt(n p (1 - p))."""
    from scipy import stats
    k = np.arange(1 << 24, dtype=np.float32) * np.float32(1.0 / 16777216.0)
    p_lo, p_hi = float((k < D.U_LO).mean()), float((k > D.U_HI).mean())
    for seed in SEEDS:
        u, _ = _noise(seed)
        u = u.ravel().astype(np.float64)
        n = u.size
        cdf = lambda x: np.where(x < 0.001, 0.0, np.where(x < 0.999, x, 1.0))
        d = stats.kstest(u, cdf).statistic
        bar = 1.95 / math.sqrt(n)
        print(f"\n[marginal] seed {seed:#x}: KS D = {d:.5f} (bar {bar:.5f}); min {u.min()}, max {u.max()}")
        assert d < bar
        assert u.min() == np.float32(0.001) and u.max() == np.float32(0.999)
        for val, p in ((D.U_LO, p_lo), (D.U_HI, p_hi)):
            c = int((u == np.float64(val)).sum())
            sd = math.sqrt(n * p * (1 - p))
            print(f"[marginal] seed {seed:#x}: {c} draws at {float(val):.3f} (expected {n * p:.1f} +- {5 * sd:.1f})")
            assert abs(c - n * p) <= 5 * sd


def test_consecutive_iterations_are_uncorrelated_and_do_not_repeat():
    """For the same (ray, step), the noise of iteration t (seed s) and of t + 1 (seed s + 0x3779B1): under independence the sample
    correlation of n pairs is about N(0, 1/n), so |r| < 5 / sqrt(n) fails by chance with probability 6e-7.  Equal 32-bit words occur
    by chance at rate 2^-32 per pair (lambda = n / 2^32 = 3e-5 expected), equal noise values at about 2^-24 (plus the clamp mass
    p^2 at each end): the count must stay within lambda + 5 sqrt(lambda) + 1 (a Poisson tail of ~1e-9 at these lambda).  The same
    between neighbouring rays at the same step and seed."""
    k = np.arange(1 << 24, dtype=np.float32) * np.float32(1.0 / 16777216.0)
    p_lo, p_hi = float((k < D.U_LO).mean()), float((k > D.U_HI).mean())
    p_val = 2.0 ** -24 + p_lo ** 2 + p_hi ** 2
    for seed in SEEDS:
        for t in range(4):
            a, wa = _noise(int(D.seed_at(seed, D.SEED_INC_NOISE, t)))
            b, wb = _noise(int(D.seed_at(seed, D.SEED_INC_NOISE, t + 1)))
            n = a.size
            r = float(np.corrcoef(a.ravel(), b.ravel())[0, 1])
            assert abs(r) < 5 / math.sqrt(n), (seed, t, r)
            for what, same, rate in (("words", int((wa == wb).sum()), 2.0 ** -32), ("values", int((a == b).sum()), p_val)):
                lam = n * rate
                assert same <= lam + 5 * math.sqrt(lam) + 1, (seed, t, what, same, lam)
            if t == 0:
                print(f"\n[lag-1] seed {seed:#x}: r = {r:+.5f} (bar {5 / math.sqrt(n):.5f}), equal words {int((wa == wb).sum())}, "
                      f"equal values {int((a == b).sum())} (expected {n * p_val:.3f})")
        a, wa = _noise(seed)
        n = a[1:].size
        for what, same, rate in (("words", int((wa[1:] == wa[:-1]).sum()), 2.0 ** -32), ("values", int((a[1:] == a[:-1]).sum()), p_val)):
            lam = n * rate
            assert same <= lam + 5 * math.sqrt(lam) + 1, (seed, "rays", what, same, lam)
        r = float(np.corrcoef(a[1:].ravel(), a[:-1].ravel())[0, 1])
        assert abs(r) < 5 / math.sqrt(n), (seed, "rays", r)


def _hypergeom(n, N):
    """Overlap of two independent uniform N-subsets of n points: hypergeometric, mean N^2 / n, variance
    N^2/n (n - N)/n (n - N)/(n - 1)."""
    mu = N * N / n
    var = mu * (n - N) / n * (n - N) / (n - 1)
    return mu, var


@pytest.mark.parametrize("n,N", [(20_000, 2048), (131_073, 512)])
def test_selection_overlaps_match_the_hypergeometric_mean(n, N):
    """Consecutive iterations draw with seeds s and s + 0x632BE5; batched problems k and k + 1 with seeds s and s + 1 (each as frame
    0).  If the subsets are independent uniform N-subsets, their overlap is hypergeometric; summed over T pairs its mean is
    T N^2/n and its variance T var (the pairs share one subset with their neighbours, but overlaps of disjoint pairs are
    independent and adjacent ones uncorrelated under the null), so the bar is |sum - T mu| <= 5 sqrt(T var)."""
    T = 12
    mu, var = _hypergeom(n, N)
    bar = 5 * math.sqrt(T * var)
    for s0, label, step, batched in ((0x2468ACE, "iterations", D.SEED_INC_SELECT, False), (0x7FFFFFFA, "problems", 1, True)):
        subsets = [set(D.top_n(D.point_key(int(D.seed_at(s0, step, t)), 0, np.arange(n), batched=batched), N).tolist())
                   for t in range(T + 1)]
        assert all(len(s) == N for s in subsets)
        total = sum(len(subsets[t] & subsets[t + 1]) for t in range(T))
        print(f"\n[overlap] n={n} N={N} {label}: total {total} over {T} pairs, expected {T * mu:.1f} +- {bar:.1f}")
        assert abs(total - T * mu) <= bar, (label, total, T * mu, bar)
