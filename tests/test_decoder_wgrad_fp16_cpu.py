"""The fp16 split that k_wgrad_tc forms G from, emulated in NumPy.

Per 64-sample chunk and per row k of v = dsdf * h1 (one h1 unit), the kernel scales the row by the power of two 2^s that puts its
largest |v| in [2^14, 2^15) (s = 0 for an all-zero row, s <= 126), splits v 2^s into fp16 hi = rn(v 2^s) and lo = rn(v 2^s - hi),
multiplies both by the exact 0/1 mask on the tensor cores and scales the chunk's sums back by 2^-s.  These tests pin the split's
error bound, and show that the same split without the scaling fails the 2e-5 norm-wise gate of the weight gradients on the
inputs tests/test_gpu_decoder_wgrad_fp16.py runs, so that test would see a lost scaling."""
import numpy as np
import pytest

KC = 64                 # samples per chunk
BAR = 2e-5              # norm-wise relative error of a weight gradient against fp64


def shift(mx):
    """The kernel's f16_shift: s with mx 2^s in [2^14, 2^15), 0 for mx = 0, at most 126."""
    e = np.frexp(mx.astype(np.float64))[1]          # mx = f 2^e, f in [0.5, 1)
    return np.where(mx == 0, 0, np.minimum(15 - e, 126)).astype(np.int64)


def split(v, scaled=True):
    """v [rows, KC] fp32 -> (hi, lo) fp16 and the row shifts s; hi + lo approximates v 2^s."""
    s = shift(np.abs(v).max(axis=1)) if scaled else np.zeros(v.shape[0], np.int64)
    vs = np.ldexp(v, s[:, None].astype(np.int32)).astype(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        hi = vs.astype(np.float16)
        r = vs - hi.astype(np.float32)
    if scaled:
        assert np.array_equal(r.astype(np.float64), vs.astype(np.float64) - hi.astype(np.float64)), "v 2^s - hi is not exact in fp32"
    with np.errstate(over="ignore", invalid="ignore"):
        return hi, r.astype(np.float16), s, vs


def g_transposed(v, m, scaled=True):
    """G^T [rows, J] = sum over chunks of 2^-s (hi + lo) m, with the tensor-core sums exact (fp64): only the split's error."""
    out = np.zeros((v.shape[0], m.shape[1]))
    for c in range(0, v.shape[1], KC):
        hi, lo, s, _ = split(v[:, c:c + KC], scaled)
        with np.errstate(invalid="ignore", over="ignore"):
            part = (hi.astype(np.float64) + lo.astype(np.float64)) @ m[c:c + KC].astype(np.float64)
        out += np.ldexp(part, -s[:, None])
    return out


def stress(kind, rows=64, S=8 * KC, seed=0):
    """v = dsdf h1 [rows, S] in fp32 and a 0/1 mask [S, 128] for the cases the GPU test runs."""
    rng = np.random.default_rng(seed)
    h1 = np.maximum(rng.standard_normal((rows, S)) * 0.3, 0)
    h1[: rows // 8] = 0                                                        # all-zero rows (dead layer-1 units)
    if kind == "span":         # dsdf over 1e-12 .. 1e6 inside every chunk
        d = np.sign(rng.standard_normal(S)) * 10.0 ** rng.uniform(-12, 6, S)
    elif kind == "single":     # one non-zero dsdf per chunk
        d = np.zeros(S)
        d[np.arange(0, S, KC) + rng.integers(0, KC, S // KC)] = rng.standard_normal(S // KC) * 1e-3
    elif kind == "mapping":    # the scale of a mapping step: the loss is a mean over ~1e6 samples
        d = rng.standard_normal(S) * 1e-6
    else:                      # features at 1e-3 .. 10: h1 spans four decades
        d = rng.standard_normal(S) * 0.1
        h1 *= np.asarray([1e-3, 0.05, 1.0, 10.0])[np.arange(S) % 4]
    v = (d[None, :].astype(np.float32) * h1.astype(np.float32)).astype(np.float32)
    m = (rng.random((S, 128)) < 0.5).astype(np.float32)
    return v, m


@pytest.mark.parametrize("kind", ["span", "single", "mapping", "scales"])
def test_scaled_split_error_bound(kind):
    v, _ = stress(kind)
    for c in range(0, v.shape[1], KC):
        hi, lo, s, vs = split(v[:, c:c + KC])
        mx = np.abs(vs).max(axis=1)
        live = mx > 0
        assert ((mx[live] >= 2.0 ** 14) & (mx[live] < 2.0 ** 15)).all()
        assert np.isfinite(hi.astype(np.float32)).all() and np.isfinite(lo.astype(np.float32)).all()
        res = np.abs(vs.astype(np.float64) - hi.astype(np.float64) - lo.astype(np.float64))
        normal = np.abs(lo.astype(np.float64)) >= 2.0 ** -14
        assert (res[normal] <= 2.0 ** -22 * np.abs(vs.astype(np.float64))[normal]).all()
        assert (res <= np.maximum(2.0 ** -22 * np.abs(vs.astype(np.float64)), 2.0 ** -25)).all()
        # in terms of the row's largest |v|: at most 2^-39 of it wherever lo is subnormal
        assert (res[~normal] <= 2.0 ** -39 * np.broadcast_to(mx[:, None], res.shape)[~normal]).all()


def test_shift_limits():
    mx = np.array([0.0, 1.0, 1.9999999, 2.0 ** -130, 3e38, 2.0 ** 14, 2.0 ** 15 - 1], np.float32)
    assert shift(mx).tolist() == [0, 14, 14, 126, -113, 0, 0]


@pytest.mark.parametrize("kind", ["span", "single", "mapping", "scales"])
def test_scaled_split_meets_the_gate_and_unscaled_fails_it(kind):
    """The scaled split stays 100x inside the gate.  Unscaled, dsdf over 1e-12 .. 1e6 overflows fp16, and the sizes a mapping step
    or a lone dsdf produce fall where fp16 is subnormal; only with dsdf ~ 0.1 (scales) does the unscaled split pass as well."""
    v, m = stress(kind)
    ref = v.astype(np.float64) @ m.astype(np.float64)
    err = float(np.linalg.norm(g_transposed(v, m) - ref) / np.linalg.norm(ref))
    bad = g_transposed(v, m, scaled=False)
    err_unscaled = float(np.linalg.norm(bad - ref) / np.linalg.norm(ref)) if np.isfinite(bad).all() else float("inf")
    print(f"{kind}: scaled {err:.2e}  unscaled {err_unscaled:.2e}")
    assert err < BAR / 100
    assert (not err_unscaled < BAR) if kind != "scales" else err_unscaled < BAR
