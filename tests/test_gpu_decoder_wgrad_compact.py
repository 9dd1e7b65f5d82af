"""The compact weight-gradient scratch (engine.alloc_act(..., dh1=False)): the tensor-core training kernel then writes no dh1
plane, only the relu'(h2) words and d loss / d sdf, and forms gW0 / gb0 itself.  Against the default layout on the same inputs the
per-sample outputs are bit-equal, the gradients stay within the fp64 bar of test_gpu_decoder_wgrad.py, rows past a device-side
count contribute nothing, nothing is written past the compact buffer, and SDFEngine allocates the compact layout."""
import ctypes as C
import sys

import pytest
import torch

from test_gpu_decoder_wgrad import BAR, NAMES, fp64_grads, inputs, rel_errors
from util import G, golden, load_decoder

pytestmark = pytest.mark.gpu

sys.path.insert(0, G)
import make_decoder_train_bits as R  # noqa: E402

GUARD = 4096           # sentinel floats behind the compact buffer


@pytest.fixture(scope="module")
def setup():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    z = golden("render.npz")
    return nl, load_decoder(z, "dec_"), z


def run(nl, dec, x, M_cap, dh1, g=None, loss=None, count=None):
    """engine.mlp_train with weight gradients; returns sdf, d feats, the words + d sdf part of the scratch, the gradients and the
    compact buffer's guard (None with dh1)."""
    E, dev = nl.engine, torch.device("cuda")
    bufs = E.DecoderBuffers(dec, dev)
    assert E.mlp_impl(bufs.width) == "tc"
    bufs.refresh_transposes()
    bufs.gradflat.zero_()
    sdf = torch.full((M_cap,), float("nan"), device=dev)
    dx = torch.full((M_cap, 16), float("nan"), device=dev)
    act = E.alloc_act(256, M_cap, dev, dh1=dh1)
    guard = None
    if not dh1:   # the same layout, with sentinels behind it
        assert act["dh1"] is None and act["buf"].numel() == int(nl._capi.lib().nl_mlp_tc_act_floats(M_cap))
        n = act["buf"].numel()
        big = torch.full((n + GUARD,), -7.25, device=dev)
        act = {"buf": big[:n], "dh1": None, "act": big[:n]}
        guard = big[n:]
    act["buf"].fill_(float("nan"))
    mdev = torch.tensor([count], dtype=torch.int32, device=dev) if count is not None else None
    kw = dict(dsdf_ext=g)
    if loss is not None:
        flag, depth, ray, cos, gt, _ = loss
        st = torch.frombuffer(bytearray(R._stats(nl, 1.0 / M_cap, 1e4 / M_cap)), dtype=torch.uint8).to(dev)
        kw.update(s_flag=flag.to(dev), s_depth=depth.to(dev), s_ray=ray.to(dev), cos=cos.to(dev), gt_depth=gt.to(dev),
                  stats_ptr=nl._capi.ptr(st), truncation=R.TRUNC)
    E.mlp_train(bufs, M_cap, C.c_void_p(mdev.data_ptr()) if mdev is not None else None, x, sdf, dx, True, act, **kw)
    torch.cuda.synchronize()
    return sdf, dx, act["act"].clone(), [t.clone() for t in bufs.grads], guard


def bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("own_loss", [False, True])
def test_compact_and_default_outputs_are_bit_equal(setup, own_loss):
    nl, dec, z = setup
    M = 132 * 128 + 77
    gen = torch.Generator().manual_seed(21)
    x = (torch.randn(M, 16, generator=gen) * 0.1).cuda()
    kw = dict(loss=R._loss_inputs(z, M, gen)) if own_loss else dict(g=(torch.randn(M, generator=gen) * 0.1).cuda())
    full = run(nl, dec, x, M, True, **kw)
    comp = run(nl, dec, x, M, False, **kw)
    for name, a, b in zip(("sdf", "dfeats", "words+dsdf"), full[:3], comp[:3]):
        assert bits_equal(a, b), name
    err = {n: float((a - b).double().norm() / b.double().norm()) for n, a, b in zip(NAMES, comp[3], full[3])}
    assert all(e < BAR for e in err.values()), err


@pytest.mark.parametrize("M", [776_000, 132 * 128 * 3 + 77, 77, 45])
def test_compact_gradients_match_fp64(setup, M):
    nl, dec, _ = setup
    x, g = inputs(dec, M, seed=5)
    got = run(nl, dec, x, M, False, g=g)[3]
    err = rel_errors(got, fp64_grads(dec, x, g))
    print(f"M={M} errors vs fp64: " + " ".join(f"{n}={e:.2e}" for n, e in err.items()))
    assert all(e < BAR for e in err.values()), err


def test_compact_rows_past_the_device_count_contribute_nothing(setup):
    nl, dec, _ = setup
    cap, count = 40_000, 40_000 - 3 * 128 - 45
    x, g = inputs(dec, cap, seed=9)
    x[count:] = float("nan")
    g[count:] = float("nan")
    got = run(nl, dec, x, cap, False, g=g, count=count)[3]
    assert all(bool(t.isfinite().all()) for t in got)
    alone = run(nl, dec, x[:count].contiguous(), count, False, g=g[:count].contiguous())[3]
    err = {n: float((a - b).double().norm() / b.double().norm()) for n, a, b in zip(NAMES, got, alone)}
    assert all(e < BAR for e in err.values()), err


def test_compact_buffer_gets_no_writes_past_its_end(setup):
    nl, dec, _ = setup
    for M, count in ((16_384, None), (132 * 128 + 77, None), (132 * 128 + 77, 16_000)):
        gen = torch.Generator().manual_seed(M)
        x = (torch.randn(M, 16, generator=gen) * 0.1).cuda()
        g = (torch.randn(M, generator=gen) * 0.1).cuda()
        guard = run(nl, dec, x, M, False, g=g, count=count)[4]
        assert bool((guard == -7.25).all()), (M, count)


def test_engine_allocates_the_compact_layout(setup):
    nl, dec, _ = setup
    dev = torch.device("cuda")
    eng = nl.engine.SDFEngine(1000, 1_654_400, dev)
    eng._ensure_act(256)
    assert eng.act["dh1"] is None
    assert eng.act["buf"].numel() == int(nl._capi.lib().nl_mlp_tc_act_floats(1_654_400))
    assert eng.act["buf"].numel() * 4 < 1_654_528 * 37
