"""The tensor-core decoder (mlp_tc.cu: k_mlp_wg, k_wgrad_tc) against the fp64 yardstick, with the bars of tests/decoder_tc_ref.py.

Per sample: the forward pass (nl_mlp_tc_forward), training from an external d loss / d sdf with weight gradients off and on
(nl_mlp_tc_train), the activation planes the weight gradients read (relu'(h2) words, d loss / d sdf, and the optional dh1 plane),
the device-side sample count and the in-kernel loss.  Every per-sample output must stay inside the hard per-row bound (HARD u a,
derived from the k-step model) and inside the discriminating bar (DISC: max err / (u a) over the run), which the emulator shows
every near miss of the 3xTF32 design (a dropped lo term, single-pass tf32) exceeds by at least 4x.  sdf must also stay within the
project's 1e-5 parity bar wherever the scale allows it: on rows whose absolute evaluation a_sdf is at most 100 (the features a map
produces are |x| ~ 0.05 and an untrained decoder has a_sdf ~ 1); larger rows are held to the relative bars only.

Decoders: the golden one, three seeded lidar.Decoder initialisations, one at trained scale (weights x 8, biases so that half of
every layer's units are active), and the golden one with every layer-1 bias negative (so that it has rows whose layer-1 units are
all dead).  Features: rows cycling through the scales 1e-3, 0.05, 1 and 10, an all-zero row, a tf32-exact row, and the dead row
where the decoder has one.  Sample counts: tile edges (1 .. 129), one tile per SM and past it (128 S +- 1, 2 x 128 S + 77, S the
SM count) and 776 000 (about 46 tiles per CTA: 18 and 42 ring items per tile are not multiples of the 4 slots, so the ring's
parity crosses tile boundaries in every phase).

Rows with a pre-activation within the near-zero margin get d loss / d sdf = 0; their relu' may go either way.

Weight gradients keep the 2e-5 norm-wise gate against fp64 (tests/test_gpu_decoder_wgrad.py).  The emulator puts the training
kernel's gW0 (three mma.sync terms, accumulators restarted every 32 samples) at about 1e-6 with all terms and at 2e-4 with any
one lo term dropped, so that gate already sees a dropped term; gb0 is a plain fp32 sum, with no split."""
import ctypes as C

import numpy as np
import pytest
import torch

import decoder_ref as R
import decoder_tc_ref as T
from util import golden, load_decoder

pytestmark = pytest.mark.gpu

U = T.U
SENT = -7.25
SENT_BITS = int(np.float32(SENT).view(np.int32))      # the sentinel as the int32 words of the relu'(h2) plane
GRAD_BAR = 2e-5
LOSS_BAR = 1e-9
SDF_ABS, SDF_ABS_SCALE = 1e-5, 100.0
TRUNC = 0.3
NAMES = ("gW0", "gb0", "gW1", "gb1", "gW2", "gb2")
DECODERS = ("golden", "seed0", "seed1", "seed2", "trained", "dead")
# sample counts as (a, b): a x 128 S + b
COUNTS = [(0, m) for m in (1, 8, 9, 16, 63, 64, 65, 127, 128, 129)] + [(1, -1), (1, 0), (1, 1), (2, 77), (0, 776_000)]
WGRAD_M = (1, 64, 65, 128, 129)
WORST = {}     # (kind, decoder, output) -> worst ratio over the run, printed at the end of the module


def _count_id(c):
    a, b = c
    return str(b) if a == 0 else f"{a}x128S{b:+d}"


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    yield nl
    print("\nworst err / (u a) per output and decoder:")
    for k in sorted(WORST):
        print(f"  {k[0]:8s} {k[1]:8s} {k[2]:4s} {WORST[k]:8.3f}   (bar {T.DISC[k[2]]})")


def _M(c):
    S = torch.cuda.get_device_properties(0).multi_processor_count
    return c[0] * 128 * S + c[1]


def _golden_np():
    z = golden("render.npz")
    return [z["dec_" + k].astype(np.float32) for k in ("pts_linears.0.weight", "pts_linears.0.bias", "pts_linears.1.weight",
                                                       "pts_linears.1.bias", "sdf_out.weight", "sdf_out.bias")]


_PARAMS = {}


def params_np(name):
    if name not in _PARAMS:
        if name == "golden":
            P = _golden_np()
        elif name.startswith("seed"):
            P = T.seeded_params(T.SEEDS[int(name[4:])])
        elif name == "trained":
            P = T.trained_scale(T.seeded_params(T.SEEDS[0]))
        else:
            P = T.dead_layer1(_golden_np())
        _PARAMS[name] = P
    return _PARAMS[name]


def _decoder(nl, name):
    if name == "golden":
        return load_decoder(golden("render.npz"), "dec_")
    if name.startswith("seed"):
        torch.manual_seed(T.SEEDS[int(name[4:])])
        return nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0)
    keys = ("pts_linears.0.weight", "pts_linears.0.bias", "pts_linears.1.weight", "pts_linears.1.bias", "sdf_out.weight", "sdf_out.bias")
    dec.load_state_dict({k: torch.from_numpy(v) for k, v in zip(keys, params_np(name))})
    return dec.cuda()


def _bufs(nl, dec):
    bufs = nl.engine.DecoderBuffers(dec, torch.device("cuda"))
    assert nl.engine.mlp_impl(bufs.width) == "tc"
    bufs.refresh_transposes()
    return bufs


def _full(shape, v=SENT):
    return torch.full(shape, v, dtype=torch.float32, device="cuda")


def _mdev(n):
    t = torch.tensor([n], dtype=torch.int32, device="cuda")
    return t, C.c_void_p(t.data_ptr())


CHUNK = 1 << 16


def _near(x, p):
    """bool [M]: this file's near-zero margin (decoder_tc_ref: twice the hard pre-activation bound)."""
    W0, b0, W1, b1 = p[:4]
    out = torch.empty(x.shape[0], dtype=torch.bool, device=x.device)
    for s in range(0, x.shape[0], CHUNK):
        xs = x[s:s + CHUNK].double()
        z1 = xs @ W0.T + b0
        a1 = xs.abs() @ W0.abs().T + b0.abs()
        z2 = z1.clamp_min(0) @ W1.T + b1
        a2 = a1 @ W1.abs().T + b1.abs()
        out[s:s + CHUNK] = (z1.abs() <= T.NEAR_Z1 * a1).any(1) | (z2.abs() <= T.NEAR_Z2 * a2).any(1)
    return out


def _inputs(nl, name, M, seed):
    """(decoder, bufs, fp64 params, x, g, near) for M rows."""
    dec = _decoder(nl, name)
    p = R.params64(dec)
    x = torch.from_numpy(T.features(M, seed, params_np(name))).cuda()
    g = torch.from_numpy((np.random.default_rng(seed + 1).standard_normal(M) * 0.1).astype(np.float32)).cuda()
    near = _near(x, p)
    g[near] = 0.0
    return dec, _bufs(nl, dec), p, x, g, near


def _m2_bits(words):
    """relu'(h2) [M, 256] from the kernel's words [M, 8] (mlp_tc.cu m2_word / m2_bit)."""
    c = torch.arange(256, device=words.device)
    word = 2 * ((c >> 1) & 3) + (c >> 7)
    bit = (2 * (c >> 3) + (c & 1)) & 31
    return ((words.long()[:, word] >> bit) & 1) != 0


def _check(kind, name, x, p, sdf=None, g=None, dh1=None, dx=None, m2=None, near=None):
    """Every given per-sample output against fp64, chunk by chunk: the hard per-row bound (asserted per entry), the 1e-5 bar
    where a_sdf <= 100, and the discriminating bar on the worst ratio of the run.  Returns {output: worst ratio}."""
    W0, b0, W1, b1, w2, b2 = p
    worst = {}
    wabs = 0.0

    def bar(key, got, ref, a, rows):
        err = (got.double() - ref).abs()
        bad = err > T.HARD[key] * U * a
        assert not bool(bad.any()), f"{kind} {name}: {key} outside the hard bound at chunk row {rows} + {bad.nonzero()[:4].tolist()}"
        live = a > 0
        r = float((err[live] / (U * a[live])).max()) if bool(live.any()) else 0.0
        worst[key] = max(worst.get(key, 0.0), r)
        return err

    for s in range(0, x.shape[0], CHUNK):
        e = min(x.shape[0], s + CHUNK)
        xs = x[s:e].double()
        z1 = xs @ W0.T + b0
        h1 = z1.clamp_min(0)
        z2 = h1 @ W1.T + b1
        a1 = xs.abs() @ W0.abs().T + b0.abs()
        a2 = a1 @ W1.abs().T + b1.abs()
        if sdf is not None:
            ref = (z2.clamp_min(0) @ w2.T + b2).reshape(-1)
            a_sdf = (a2 @ w2.abs().T + b2.abs()).reshape(-1)
            err = bar("sdf", sdf[s:e], ref, a_sdf, s)
            small = a_sdf <= SDF_ABS_SCALE
            if bool(small.any()):
                wabs = max(wabs, float(err[small].max()))
        if m2 is not None:
            keep = ~near[s:e]
            got = _m2_bits(m2[s:e])
            assert torch.equal(got[keep], (z2 > 0)[keep]), f"{kind} {name}: relu'(h2) words differ from fp64 z2 > 0"
        if g is not None:
            gs = g[s:e].double()
            m1, m2r = z1 > 0, z2 > 0
            dz1 = ((gs[:, None] * w2[0] * m2r) @ W1) * m1
            a_dh1 = ((gs.abs()[:, None] * w2[0].abs() * m2r) @ W1.abs()) * m1
            if dh1 is not None:
                bar("dh1", dh1[s:e], dz1, a_dh1, s)
            if dx is not None:
                bar("dx", dx[s:e], dz1 @ W0, a_dh1 @ W0.abs(), s)
    assert wabs <= SDF_ABS, f"{kind} {name}: sdf {wabs:.2e} from fp64 on a row with a_sdf <= {SDF_ABS_SCALE}"
    for k, r in worst.items():
        WORST[(kind, name, k)] = max(WORST.get((kind, name, k), 0.0), r)
        assert r <= T.DISC[k], f"{kind} {name}: {k} reaches {r:.3f} u a, above the discriminating bar {T.DISC[k]}"
    return worst, wabs


def _fmt(worst):
    return " ".join(f"{k} {v:.3f}" for k, v in worst.items())


# ------------------------------------------------------------------------------------------------------------- a. forward
@pytest.mark.parametrize("count", COUNTS, ids=_count_id)
@pytest.mark.parametrize("name", DECODERS)
def test_forward(nl, name, count):
    M = _M(count)
    dec, bufs, p, x, _, near = _inputs(nl, name, M, seed=M)
    sdf = _full((M + 37,))
    nl.engine.mlp_forward(bufs, M, None, x, sdf)
    torch.cuda.synchronize()
    assert bool((sdf[M:] == SENT).all()), "sdf written past M"
    worst, wabs = _check("forward", name, x, p, sdf=sdf[:M])
    print(f"forward {name} M={M}: {_fmt(worst)} u a_sdf, max |sdf - fp64| {wabs:.2e} where a_sdf <= {SDF_ABS_SCALE}")


# ------------------------------------------------------------------------------------------------------------- b. training, external d sdf
def _train(nl, bufs, M_cap, x, sdf, dx, wgrad, mdev=None, act=None, **kw):
    bufs.gradflat.zero_()
    nl.engine.mlp_train(bufs, M_cap, mdev, x, sdf, dx, wgrad, act, **kw)
    torch.cuda.synchronize()
    return [t.clone() for t in bufs.grads] if wgrad else None


def _act(nl, M):
    """alloc_act(..., dh1=True) filled with the sentinel, and its planes: (act, dh1 [cap, 256], m2 words [cap, 8], dsdf [cap])."""
    act = nl.engine.alloc_act(256, M, torch.device("cuda"), dh1=True)
    act["buf"].fill_(SENT)
    cap = act["dh1"].numel() // 256
    assert act["act"].numel() == cap * 9 and cap == (M + 127) // 128 * 128
    return act, act["dh1"].view(cap, 256), act["act"][:cap * 8].view(torch.int32).view(cap, 8), act["act"][cap * 8:]


def _grad_errors(got, ref, g):
    """Norm-wise relative errors; gb2 = sum of d loss / d sdf g, which cancels to a few % of sum |g|, is measured against sum |g|
    (its condition: the fp32 atomics that reduce it round at the size of their partial sums, whatever the total)."""
    out = {}
    for n, a, b in zip(NAMES, got, ref):
        nb = float(g.double().abs().sum()) if n == "gb2" else float(b.norm())
        out[n] = float((a.double() - b).norm()) / nb if nb > 0 else float(a.abs().max())
    return out


@pytest.mark.parametrize("count", COUNTS, ids=_count_id)
@pytest.mark.parametrize("name", DECODERS)
def test_training(nl, name, count):
    M = _M(count)
    dec, bufs, p, x, g, near = _inputs(nl, name, M, seed=3 * M + 1)
    sdf0, dx0 = _full((M + 3,)), _full((M + 3, 16))
    _train(nl, bufs, M, x, sdf0, dx0, False, dsdf_ext=g)
    act, dh1, m2, dpl = _act(nl, M)
    sdf, dx = _full((M + 3,)), _full((M + 3, 16))
    grads = _train(nl, bufs, M, x, sdf, dx, True, act=act, dsdf_ext=g)
    assert bool((sdf[M:] == SENT).all() and (dx[M:] == SENT).all() and (sdf0[M:] == SENT).all() and (dx0[M:] == SENT).all())
    # both instantiations do the same per-sample arithmetic, and it is the forward kernel's: the training kernel runs the same
    # layer-1, layer-2 and output-layer code on the same ring items
    assert torch.equal(sdf0, sdf) and torch.equal(dx0, dx), "weight gradients on / off changed sdf or d features"
    fwd = _full((M,))
    nl.engine.mlp_forward(bufs, M, None, x, fwd)
    torch.cuda.synchronize()
    assert torch.equal(fwd, sdf[:M]), "the training kernel's sdf differs from the forward kernel's"
    zero = g == 0
    assert bool((dx[:M][zero] == 0).all() and (dh1[:M][zero] == 0).all()), "d features or dh1 nonzero on a row with d loss / d sdf = 0"
    # the activation planes: dsdf is g bit for bit; rows in [M, cap) are not written (the copies cover live rows only)
    assert torch.equal(dpl[:M], g), "the dsdf plane is not d loss / d sdf"
    assert bool((dh1[M:] == SENT).all() and (m2[M:] == SENT_BITS).all() and (dpl[M:] == SENT).all()), "an activation row past M was written"
    worst, wabs = _check("train", name, x, p, sdf=sdf[:M], g=g, dh1=dh1[:M], dx=dx[:M], m2=m2[:M], near=near)
    line = f"train {name} M={M} (g = 0 on {int(near.sum())} near-zero rows): {_fmt(worst)} u a"
    if M in WGRAD_M or name == "trained":
        ref = R.backward(x, g, p)[1]
        err = _grad_errors(grads, ref, g)
        line += " | grads " + " ".join(f"{n}={e:.1e}" for n, e in err.items())
        assert all(e <= GRAD_BAR for e in err.values()), err
    print(line)


# ------------------------------------------------------------------------------------------------------------- c. device-side count
@pytest.mark.parametrize("name", ["golden", "trained"])
def test_forward_rows_past_the_device_count(nl, name):
    cap, count = 40_000, 40_000 - 3 * 128 - 45
    dec, bufs, p, x, _, _ = _inputs(nl, name, cap, seed=9)
    xn = x.clone()
    xn[count:] = float("nan")
    _, mdev = _mdev(count)
    sdf = _full((cap,))
    nl.engine.mlp_forward(bufs, cap, mdev, xn, sdf)
    alone = _full((count,))
    nl.engine.mlp_forward(bufs, count, None, x[:count].contiguous(), alone)
    torch.cuda.synchronize()
    assert bool((sdf[count:] == SENT).all()), "a row past the device count was written"
    assert torch.equal(sdf[:count], alone)
    _, mdev0 = _mdev(0)
    sdf = _full((cap,))
    nl.engine.mlp_forward(bufs, cap, mdev0, xn, sdf)
    _, mdev2 = _mdev(cap + 1000)
    over, host = _full((cap + 5,)), _full((cap + 5,))
    nl.engine.mlp_forward(bufs, cap, mdev2, x, over)
    nl.engine.mlp_forward(bufs, cap, None, x, host)
    torch.cuda.synchronize()
    assert bool((sdf == SENT).all()), "count 0 wrote sdf"
    assert torch.equal(over, host) and bool((over[cap:] == SENT).all())


@pytest.mark.parametrize("name", ["golden", "trained"])
def test_training_rows_past_the_device_count(nl, name):
    cap, count = 40_000, 40_000 - 3 * 128 - 45
    dec, bufs, p, x, g, _ = _inputs(nl, name, cap, seed=19)
    xn, gn = x.clone(), g.clone()
    xn[count:], gn[count:] = float("nan"), float("nan")
    _, mdev = _mdev(count)
    act, dh1, m2, dpl = _act(nl, cap)
    sdf, dx = _full((cap,)), _full((cap, 16))
    got = _train(nl, bufs, cap, xn, sdf, dx, True, mdev, act=act, dsdf_ext=gn)
    assert all(bool(t.isfinite().all()) for t in got)
    assert bool((sdf[count:] == SENT).all() and (dx[count:] == SENT).all()), "a row past the device count was written"
    assert bool((dh1[count:] == SENT).all() and (m2[count:] == SENT_BITS).all() and (dpl[count:] == SENT).all())
    act1, dh1a, m2a, dpla = _act(nl, count)
    sdf1, dx1 = _full((count,)), _full((count, 16))
    alone = _train(nl, bufs, count, x[:count].contiguous(), sdf1, dx1, True, act=act1, dsdf_ext=g[:count].contiguous())
    assert torch.equal(sdf[:count], sdf1) and torch.equal(dx[:count], dx1)
    assert torch.equal(dh1[:count], dh1a[:count]) and torch.equal(m2[:count], m2a[:count]) and torch.equal(dpl[:count], dpla[:count])
    e_alone = _grad_errors(got, [t.double() for t in alone], g[:count])
    e_ref = _grad_errors(got, R.backward(x[:count], g[:count], p)[1], g[:count])
    print(f"count {name}: vs first-rows run " + " ".join(f"{n}={e:.1e}" for n, e in e_alone.items())
          + " | vs fp64 " + " ".join(f"{n}={e:.1e}" for n, e in e_ref.items()))
    # the gradients of two runs differ by the order of their fp32 atomics, which gb2 (a sum of d loss / d sdf that cancels to a
    # few % of its absolute sum) magnifies; each run is held to fp64 instead of to the other
    assert all(e <= GRAD_BAR for e in e_ref.values()), e_ref
    # a count of 0 writes nothing and adds nothing
    _, mdev0 = _mdev(0)
    act0, dh10, m20, dpl0 = _act(nl, cap)
    sdf, dx = _full((cap,)), _full((cap, 16))
    zero = _train(nl, bufs, cap, xn, sdf, dx, True, mdev0, act=act0, dsdf_ext=gn)
    assert bool((sdf == SENT).all() and (dx == SENT).all() and (act0["buf"] == SENT).all()), "count 0 wrote something"
    assert all(bool((t == 0).all()) for t in zero), "count 0 added to the gradients"
    # a count above the capacity is the capacity
    _, mdev2 = _mdev(cap + 1000)
    sdf, dx = _full((cap + 5,)), _full((cap + 5, 16))
    over = _train(nl, bufs, cap, x, sdf, dx, True, mdev2, act=_act(nl, cap)[0], dsdf_ext=g)
    sdf2, dx2 = _full((cap + 5,)), _full((cap + 5, 16))
    host = _train(nl, bufs, cap, x, sdf2, dx2, True, act=_act(nl, cap)[0], dsdf_ext=g)
    assert torch.equal(sdf, sdf2) and torch.equal(dx, dx2) and bool((sdf[cap:] == SENT).all())
    e_over = _grad_errors(over, R.backward(x, g, p)[1], g)
    assert all(e <= GRAD_BAR for e in e_over.values()), e_over
    print(f"count {name} above the capacity: vs the host-count run " + " ".join(
        f"{n}={e:.1e}" for n, e in _grad_errors(over, [t.double() for t in host], g).items()) + " | vs fp64 " + " ".join(f"{n}={e:.1e}" for n, e in e_over.items()))


# ------------------------------------------------------------------------------------------------------------- d. in-kernel loss
def _stats(nl, g_fs, g_sdf):
    s = nl._capi.RenderStats()
    s.g_fs, s.g_sdf = g_fs, g_sdf
    return torch.frombuffer(bytearray(bytes(s)), dtype=torch.uint8).cuda()


def _samples(M, n_rays, seed, with_cos):
    """Samples in ray order, several per ray, flags 0 / 1 / 2 mixed; per-ray gt depth and cosine; depths around the surface."""
    gen = torch.Generator().manual_seed(seed)
    ray = torch.sort(torch.randint(0, n_rays, (M,), generator=gen)).values.to(torch.int32)
    flag = torch.randint(0, 3, (M,), generator=gen).to(torch.uint8)
    gt = (2.0 + 28.0 * torch.rand(n_rays, generator=gen)).float()
    cos = (0.5 + 0.5 * torch.rand(n_rays, generator=gen)).float()
    c = cos[ray.long()] if with_cos else 1.0
    depth = (gt[ray.long()] / c + 0.8 * (torch.rand(M, generator=gen) - 0.5)).float()
    return [t.cuda().contiguous() for t in (flag, depth, ray, gt)] + [cos.cuda().contiguous() if with_cos else None]


@pytest.mark.parametrize("wgrad", [False, True], ids=["nograd", "wgrad"])
@pytest.mark.parametrize("with_cos", [True, False], ids=["cos", "nocos"])
def test_in_kernel_loss(nl, with_cos, wgrad):
    S = torch.cuda.get_device_properties(0).multi_processor_count
    M = 128 * S + 1100
    dec, bufs, p, x, _, near = _inputs(nl, "seed1", M, seed=41 + with_cos)
    flag, depth, ray, gt, cos = _samples(M, 3000, seed=7 + with_cos, with_cos=with_cos)
    flag[near] = 0
    g_fs, g_sdf = 0.7 / M, 1e4 / M
    st = _stats(nl, g_fs, g_sdf)
    sdf, dx = _full((M,)), _full((M, 16))
    act = _act(nl, M)[0] if wgrad else None
    grads = _train(nl, bufs, M, x, sdf, dx, wgrad, act=act, s_flag=flag, s_depth=depth, s_ray=ray, cos=cos, gt_depth=gt,
                   stats_ptr=C.c_void_p(st.data_ptr()), truncation=TRUNC)
    s = nl._capi.RenderStats.from_buffer_copy(st.cpu().numpy().tobytes())
    fs, sd, _ = R.loss(sdf, flag, depth, ray, gt, cos, TRUNC, g_fs, g_sdf)
    e_fs, e_sd = abs(s.fs_sum - fs) / fs, abs(s.sdf_sum - sd) / sd
    assert e_fs <= LOSS_BAR and e_sd <= LOSS_BAR, (s.fs_sum, fs, s.sdf_sum, sd)
    worst, _ = _check("loss", "seed1", x, p, sdf=sdf)
    # the fp64 chain: fp64 sdf -> fp64 d loss / d sdf -> fp64 backward.  The kernel's d loss / d sdf carries its sdf error and the
    # fp32 roundings of e: a bound dg per row, carried through |W| (as in test_gpu_decoder_simt.py::test_in_kernel_loss)
    sdf64 = R.forward(x, p)["sdf"]
    _, _, g64 = R.loss(sdf64, flag, depth, ray, gt, cos, TRUNC, g_fs, g_sdf)
    dx_ref, ref, a_dx = R.backward(x, g64, p, with_abs=True)
    a_sdf = torch.cat([R.absolute(x[a:b], p)[2] for a, b in R._chunks(M)])
    dsdf = T.HARD["sdf"] * U * a_sdf
    zr = depth.double() * (cos.double()[ray.long()] if cos is not None else 1.0)
    t, f = float(torch.tensor(TRUNC, dtype=torch.float32)), flag.long()
    mag = zr.abs() + sdf64.abs() * t + gt.double()[ray.long()].abs()
    dg = torch.where((f & 1) != 0, 2 * g_fs * (dsdf + 4 * U * (sdf64 - 1).abs()), 0.0) + \
        torch.where((f & 2) != 0, 2 * g_sdf * t * (t * dsdf + 6 * U * mag), 0.0)
    _, _, a_dg = R.backward(x, dg, p, with_abs=True)
    zero = flag == 0
    assert bool((dx[zero] == 0).all()), "d features written on a row without a loss term"
    err = (dx.double() - dx_ref).abs()
    bound = T.HARD["dx"] * U * (a_dx + a_dg) + a_dg
    bad = (err > bound) & ~zero[:, None]
    assert not bool(bad.any()), f"d features outside the bound at {bad.nonzero()[:5].tolist()}"
    frac = float((err / bound).masked_fill(~(bound > 0) | zero[:, None], 0).max())
    line = f"loss cos={with_cos} wgrad={wgrad} M={M}: fs_sum {e_fs:.1e} sdf_sum {e_sd:.1e}, {_fmt(worst)} u a_sdf, dx at {frac:.3f} of its bound"
    if wgrad:
        err = _grad_errors(grads, ref, g64)
        line += " | grads " + " ".join(f"{n}={e:.1e}" for n, e in err.items())
        assert all(e <= GRAD_BAR for e in err.values()), err
    print(line)
