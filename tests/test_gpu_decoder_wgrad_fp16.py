"""Decoder weight gradients on inputs that stress k_wgrad_tc's fp16 G (a power-of-two scale per 64-sample chunk and h1 row, then an
fp16 hi + lo split; tests/test_decoder_wgrad_fp16_cpu.py emulates it), against fp64.

Cases: dsdf spanning 1e-12 .. 1e6 inside every chunk; chunks with a single non-zero dsdf; the golden decoder with every layer-1
bias negative (h1 rows that are all zero); features at the scales 1e-3 .. 10; the trained-scale decoder with dsdf at the size a
mapping step produces (~1e-6, where an unscaled fp16 split would fall into fp16's subnormals).  Sample counts: less than one chunk
(45), a partial chunk past most CTAs (77), one tile per SM and either side of it (128 S +- 1) and 776 000.

Every gradient must stay inside the 2e-5 norm-wise gate of test_gpu_decoder_wgrad.py.  The worst element-wise error relative to
the fp64 evaluation of the absolute terms is printed beside it."""
import numpy as np
import pytest
import torch

import decoder_tc_ref as T
from test_gpu_decoder_tc import _decoder, params_np
from test_gpu_decoder_wgrad import BAR, NAMES, _params64, fp64_grads, kernel_grads

pytestmark = pytest.mark.gpu

KC = 64
CASES = ("span", "single", "dead", "scales", "trained")
COUNTS = [(0, 45), (0, 77), (1, -1), (1, 1), (0, 776_000)]


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


def zero_near(dec, x, g):
    """g = 0 on samples with a pre-activation within 1e-4 (relative) of zero, as in test_gpu_decoder_wgrad.inputs."""
    W0, b0, W1, b1 = _params64(dec)[:4]
    for s in range(0, x.shape[0], 1 << 17):
        xs = x[s:s + (1 << 17)].double()
        z1 = xs @ W0.T + b0
        h1 = z1.clamp_min(0)
        z2 = h1 @ W1.T + b1
        near = ((z1.abs() <= 1e-4 * (xs.abs() @ W0.abs().T + b0.abs())).any(dim=1)) | \
               ((z2.abs() <= 1e-4 * (h1 @ W1.abs().T + b1.abs())).any(dim=1))
        g[s:s + (1 << 17)][near] = 0.0
    return g


def case_inputs(nl, case, M, seed=11):
    rng = np.random.default_rng(seed)
    name = {"dead": "dead", "trained": "trained"}.get(case, "golden")
    dec = _decoder(nl, name)
    if case in ("span", "single"):
        x = (rng.standard_normal((M, 16)) * 0.05).astype(np.float32)
    else:
        x = T.features(M, seed, params_np(name))
    if case == "span":
        g = np.sign(rng.standard_normal(M)) * 10.0 ** rng.uniform(-12, 6, M)
    elif case == "single":
        g = np.zeros(M)
        for c in range(0, M, KC):
            g[c + rng.integers(0, min(KC, M - c))] = rng.standard_normal() * 10.0 ** rng.uniform(-6, 2)
    elif case == "trained":
        g = rng.standard_normal(M) * 1e-6
    else:
        g = rng.standard_normal(M) * 0.1
    x = torch.from_numpy(x).cuda().contiguous()
    g = zero_near(dec, x, torch.from_numpy(g.astype(np.float32)).cuda().contiguous())
    return dec, x, g


def fp64_abs_grads(dec, x, g):
    """Every gradient's sum with each term replaced by its absolute value; gW2 as the kernel forms it,
    sum_k W1[j, k] G[j, k] + b1[j] c[j] with G = m2^T (g h1) and c = m2^T g."""
    W0, b0, W1, b1, w2, b2 = _params64(dec)
    out = [torch.zeros_like(p) for p in (W0, b0, W1, b1, w2, b2)]
    for s in range(0, x.shape[0], 1 << 17):
        xs, gs = x[s:s + (1 << 17)].double(), g[s:s + (1 << 17)].double().abs()
        z1 = xs @ W0.T + b0
        h1 = z1.clamp_min(0)
        z2 = h1 @ W1.T + b1
        dz2 = gs[:, None] * w2[0].abs() * (z2 > 0)
        dz1 = (dz2 @ W1.abs()) * (z1 > 0)
        out[0] += dz1.T @ xs.abs()
        out[1] += dz1.sum(0)
        out[2] += dz2.T @ h1
        out[3] += dz2.sum(0)
        m2g = gs[:, None] * (z2 > 0)
        out[4] += ((W1.abs() * (m2g.T @ h1)).sum(1) + b1.abs() * m2g.sum(0)).reshape(1, -1)
        out[5] += gs.sum().reshape(1)
    return out


@pytest.mark.parametrize("count", COUNTS, ids=lambda c: str(c[1]) if c[0] == 0 else f"128S{c[1]:+d}")
@pytest.mark.parametrize("case", CASES)
def test_decoder_weight_gradients_on_fp16_stress_inputs_match_fp64(nl, case, count):
    M = count[0] * 128 * torch.cuda.get_device_properties(0).multi_processor_count + count[1]
    dec, x, g = case_inputs(nl, case, M)
    got = kernel_grads(nl.engine, dec, x, g, M)
    ref, absum = fp64_grads(dec, x, g), fp64_abs_grads(dec, x, g)
    err, worst = {}, {}
    for n, a, b, s in zip(NAMES, got, ref, absum):
        d = (a.double() - b).abs()
        err[n] = float(d.norm() / b.norm()) if float(b.norm()) > 0 else float(a.double().norm())
        worst[n] = float((d[s > 0] / s[s > 0]).max()) if bool((s > 0).any()) else 0.0
    print(f"{case} M={M} nonzero g: {int((g != 0).sum())}  norm-wise: " + " ".join(f"{n}={e:.2e}" for n, e in err.items()) +
          "  worst / abs sum: " + " ".join(f"{n}={e:.2e}" for n, e in worst.items()))
    assert all(bool(t.isfinite().all()) for t in got)
    assert all(e < BAR for e in err.values()), err
