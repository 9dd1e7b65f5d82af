"""Tensor-core decoder weight gradients at full size against an fp64 evaluation, and the device-side sample count.

The decoder (16 -> 256 -> 256 -> 1, ReLU) is trained through engine.mlp_train with an external d loss / d sdf g, so every weight
gradient is a sum over samples of products of g, x and the activations.  The yardstick evaluates those sums in fp64 from x, the
weights and g alone.  A sample whose layer-1 or layer-2 pre-activation lies within 1e-4 (relative to the absolute sum of its
terms) of zero gets g = 0: two valid fp32 evaluations may disagree on its relu', and with g = 0 it contributes nothing to any
weight gradient."""
import ctypes as C

import pytest
import torch

import decoder_wgrad_ref as W
from util import golden, load_decoder

pytestmark = pytest.mark.gpu

BAR = 2e-5             # norm-wise relative error of every gradient against fp64
NAMES = ("gW0", "gb0", "gW1", "gb1", "gW2", "gb2")


@pytest.fixture(scope="module")
def setup():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    z = golden("render.npz")
    dec = load_decoder(z, "dec_")
    return nl.engine, dec


def inputs(dec, M, seed):
    """Seeded x and g; g = 0 where a pre-activation is within rounding of zero (see the module docstring)."""
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(seed)
    x = (torch.randn(M, 16, device=dev, generator=gen) * 0.05).contiguous()
    g = (torch.randn(M, device=dev, generator=gen) * 0.1).contiguous()
    W0, b0, W1, b1 = _params64(dec)[:4]
    for s in range(0, M, 1 << 17):
        xs = x[s:s + (1 << 17)].double()
        z1 = xs @ W0.T + b0
        a1 = xs.abs() @ W0.abs().T + b0.abs()
        h1 = z1.clamp_min(0)
        z2 = h1 @ W1.T + b1
        a2 = h1 @ W1.abs().T + b1.abs()
        near = ((z1.abs() <= 1e-4 * a1).any(dim=1)) | ((z2.abs() <= 1e-4 * a2).any(dim=1))
        g[s:s + (1 << 17)][near] = 0.0
    return x, g


def _params64(dec):
    """W0, b0, W1, b1, w2, b2 in fp64 (the order of DecoderBuffers.params and .grads)."""
    lin = list(dec.pts_linears)
    return [p.detach().double() for p in (lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias, dec.sdf_out.weight, dec.sdf_out.bias)]


def fp64_grads(dec, x, g):
    """decoder_wgrad_ref.grads64 over chunks of samples, on the device."""
    p = _params64(dec)
    out = [torch.zeros_like(q) for q in p]
    for s in range(0, x.shape[0], 1 << 17):
        for o, d in zip(out, W.grads64(x[s:s + (1 << 17)].double(), p, g[s:s + (1 << 17)].double())):
            o += d
    return out


def kernel_grads(E, dec, x, g, M_cap, count=None):
    """engine.mlp_train on the tensor-core path; count: the device-side sample count (None: all M_cap rows)."""
    dev = torch.device("cuda")
    bufs = E.DecoderBuffers(dec, dev)
    assert E.mlp_impl(bufs.width) == "tc"
    bufs.refresh_transposes()
    bufs.gradflat.zero_()
    sdf = torch.empty(M_cap, device=dev)
    dx = torch.empty(M_cap, 16, device=dev)
    act = E.alloc_act(256, M_cap, dev)
    mdev = torch.tensor([count], dtype=torch.int32, device=dev) if count is not None else None
    E.mlp_train(bufs, M_cap, C.c_void_p(mdev.data_ptr()) if mdev is not None else None, x, sdf, dx, True, act, dsdf_ext=g)
    torch.cuda.synchronize()
    return [t.clone() for t in bufs.grads]


def rel_errors(got, ref):
    return {n: float((a.double() - b).norm() / b.norm()) for n, a, b in zip(NAMES, got, ref)}


@pytest.mark.parametrize("M", [776_000, 132 * 128 * 3 + 77])
def test_decoder_weight_gradients_match_fp64(setup, M):
    E, dec = setup
    x, g = inputs(dec, M, seed=5)
    err = rel_errors(kernel_grads(E, dec, x, g, M), fp64_grads(dec, x, g))
    print(f"M={M} zeroed g: {int((g == 0).sum())}  errors vs fp64: " + " ".join(f"{n}={e:.2e}" for n, e in err.items()))
    assert all(e < BAR for e in err.values()), err


def test_samples_past_the_device_count_contribute_nothing(setup):
    E, dec = setup
    cap, count = 40_000, 40_000 - 3 * 128 - 45
    x, g = inputs(dec, cap, seed=9)
    x[count:] = float("nan")
    g[count:] = float("nan")
    got = kernel_grads(E, dec, x, g, cap, count=count)
    assert all(bool(t.isfinite().all()) for t in got)
    alone = kernel_grads(E, dec, x[:count].contiguous(), g[:count].contiguous(), count)
    ref = fp64_grads(dec, x[:count], g[:count])
    err_alone = {n: float((a - b).double().norm() / b.double().norm()) for n, a, b in zip(NAMES, got, alone)}
    err_ref = rel_errors(got, ref)
    print("count run vs first-rows run: " + " ".join(f"{n}={e:.2e}" for n, e in err_alone.items()))
    assert all(e < BAR for e in err_alone.values()), err_alone
    assert all(e < BAR for e in err_ref.values()), err_ref
