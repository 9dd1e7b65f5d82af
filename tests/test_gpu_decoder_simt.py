"""The fp32 CUDA-core decoder (mlp.cu: k_mlp, k_dw1) against the fp64 yardstick of tests/decoder_ref.py at every width.

It is the only decoder at widths 32, 64 and 128, and the exact-gradient choice at width 256 (NL_MLP_IMPL=simt).  Covered here:
the forward pass (nl_mlp_forward), training from an external d loss / d sdf with and without weight gradients (nl_mlp_train), the
device-side sample count, the in-kernel loss, and the per-problem loss of the batched kernels (nl_mlp_train_batch, and at width 256
the tensor-core nl_mlp_tc_train_batch / nl_mlp_tc_score_batch, which share nl_seg_loss_add).

Bars (u = 2^-24):
  * sdf per row within (2W + 20) u a_sdf (the dot-product bound carried through the absolute evaluation), and never above 1e-5;
  * d features per element within (2W + 40) u a_dx, exactly 0 on rows whose d loss / d sdf is 0;
  * every weight gradient within 1e-4 norm-wise of fp64 (the one-step gradient gate, DESIGN section 5);
  * loss sums within 1e-9 of the restatement on the kernel's own sdf (fp64 sums of the same fp32 errors, in another order).
Rows with a pre-activation within rounding of zero (decoder_ref.near_zero) get d loss / d sdf = 0 (or flag 0): two valid fp32
evaluations may disagree on their relu'."""
import ctypes as C

import pytest
import torch

import decoder_ref as R
from util import golden, load_decoder

pytestmark = pytest.mark.gpu

WIDTHS = (32, 64, 128, 256)
DECODERS = [(W, "seed") for W in WIDTHS] + [(256, "golden")]
U = R.U
SDF_BAR = 1e-5
GRAD_BAR = 1e-4
LOSS_BAR = 1e-9
TRUNC = 0.3
SENT = -7.25                       # sentinel in the output rows a call must not write
NAMES = ("gW0", "gb0", "gW1", "gb1", "gW2", "gb2")
FULL = 132 * 128                   # one tile per SM of an H100 SXM


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


@pytest.fixture
def simt(monkeypatch):
    monkeypatch.setenv("NL_MLP_IMPL", "simt")


def _ids(c):
    return f"W{c[0]}-{c[1]}"


def _decoder(nl, W, src):
    if src == "golden":
        return load_decoder(golden("render.npz"), "dec_")
    torch.manual_seed(1000 + W)
    return nl.lidar.Decoder(depth=2, width=W, in_dim=16, skips=[], embedder="none", multires=0).cuda()


def _bufs(nl, dec, impl="simt"):
    bufs = nl.engine.DecoderBuffers(dec, torch.device("cuda"))
    assert nl.engine.mlp_impl(bufs.width) == impl
    bufs.refresh_transposes()
    return bufs


def _features(M, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(M, 16, device="cuda", generator=gen) * 0.05).contiguous()
    g = (torch.randn(M, device="cuda", generator=gen) * 0.1).contiguous()
    return x, g


def _full(shape, v=SENT):
    return torch.full(shape, v, dtype=torch.float32, device="cuda")


def _mdev(n):
    t = torch.tensor([n], dtype=torch.int32, device="cuda")
    return t, C.c_void_p(t.data_ptr())


def _rel(got, ref):
    return float((got.double() - ref).norm() / ref.norm())


def _check_forward(x, p, W, sdf, h1=None):
    """Per-row sdf bound (and the h1 scratch against the layer-1 bound); returns the worst |err| and the worst err / (u a_sdf)."""
    worst, ratio = 0.0, 0.0
    for s, e in R._chunks(x.shape[0]):
        f = R.forward(x[s:e], p, keep=("h1", "sdf") if h1 is not None else ("sdf",))
        a1, _, a_sdf = R.absolute(x[s:e], p)
        err = (sdf[s:e].double() - f["sdf"]).abs()
        assert bool((err <= (2 * W + 20) * U * a_sdf).all()), f"sdf outside the bound at rows {s}+{(err > (2 * W + 20) * U * a_sdf).nonzero()[:5].tolist()}"
        worst, ratio = max(worst, float(err.max())), max(ratio, float((err / (U * a_sdf)).max()))
        if h1 is not None:     # layer 1: 16 products and the bias
            eh = (h1[s:e].double() - f["h1"]).abs()
            assert bool((eh <= 20 * U * a1).all()), "act_h1 outside the layer-1 bound"
    assert worst <= SDF_BAR, worst
    return worst, ratio


def _check_dx(dx, ref, a_dx, W, zero_rows, extra=None):
    """d features: exactly 0 on zero_rows; elsewhere within (2W + 40) u a_dx (+ extra).  Returns the worst err / (u a_dx) and the
    largest fraction of the bound used."""
    assert bool((dx[zero_rows] == 0).all()), "d features written on a row whose d loss / d sdf is 0"
    err = (dx.double() - ref).abs()
    bound = (2 * W + 40) * U * a_dx + (extra if extra is not None else 0.0)
    bad = (err > bound) & ~zero_rows[:, None]
    assert not bool(bad.any()), f"d features outside the bound at {bad.nonzero()[:5].tolist()}"
    live = ~zero_rows[:, None] & (a_dx > 0)
    return float((err / (U * a_dx)).masked_fill(~live, 0).max()), float((err / bound).masked_fill(~live, 0).max())


def _train(nl, bufs, M_cap, x, sdf, dx, wgrad, mdev=None, **kw):
    E = nl.engine
    act = E.alloc_act(bufs.width, M_cap, torch.device("cuda")) if wgrad else None
    bufs.gradflat.zero_()
    E.mlp_train(bufs, M_cap, mdev, x, sdf, dx, wgrad, act, **kw)
    torch.cuda.synchronize()
    return [t.clone() for t in bufs.grads] if wgrad else None, act


# ------------------------------------------------------------------------------------------------------------- a. forward
@pytest.mark.parametrize("M", [1, 15, 16, 17, 127, 128, 129, FULL - 1, FULL + 1, 3 * FULL + 77])
@pytest.mark.parametrize("case", DECODERS, ids=_ids)
def test_forward_within_the_dot_product_bound(nl, simt, case, M):
    W, src = case
    dec = _decoder(nl, W, src)
    bufs = _bufs(nl, dec)
    p = R.params64(dec)
    x, _ = _features(M, seed=M + W)
    sdf = _full((M + 37,))
    nl.engine.mlp_forward(bufs, M, None, x, sdf)
    torch.cuda.synchronize()
    assert bool((sdf[M:] == SENT).all()), "sdf written past M"
    worst, ratio = _check_forward(x, p, W, sdf[:M])
    print(f"forward W={W} {src} M={M}: max |sdf - fp64| = {worst:.2e} = {ratio:.1f} u a_sdf (bound {2 * W + 20})")


# ------------------------------------------------------------------------------------------------------------- b. training, external d sdf
TRAIN_CASES = [(c, M) for c in DECODERS for M in (45, 77, 128, 129, FULL + 77)] + \
              [(c, 776_000) for c in DECODERS if c[0] in (64, 256)]


@pytest.mark.parametrize("case,M", TRAIN_CASES, ids=[f"{_ids(c)}-M{M}" for c, M in TRAIN_CASES])
def test_training_matches_fp64(nl, simt, case, M):
    W, src = case
    dec = _decoder(nl, W, src)
    bufs = _bufs(nl, dec)
    p = R.params64(dec)
    x, g = _features(M, seed=5 * M + W)
    near = R.near_zero(x, p)
    g[near] = 0.0
    sdf, dx = _full((M + 3,)), _full((M + 3, 16))
    grads, act = _train(nl, bufs, M, x, sdf, dx, True, dsdf_ext=g)
    sdf0, dx0 = _full((M + 3,)), _full((M + 3, 16))
    _train(nl, bufs, M, x, sdf0, dx0, False, dsdf_ext=g)
    assert bool((sdf[M:] == SENT).all() and (dx[M:] == SENT).all() and (sdf0[M:] == SENT).all() and (dx0[M:] == SENT).all())
    # both instantiations (weight gradients on / off) do the same per-sample arithmetic
    assert torch.equal(sdf0, sdf) and torch.equal(dx0, dx)
    worst, ratio = _check_forward(x, p, W, sdf[:M], h1=act["h1"])
    dx_ref, ref, a_dx = R.backward(x, g, p, with_abs=True)
    dratio, _ = _check_dx(dx[:M], dx_ref, a_dx, W, g == 0)
    err = {n: _rel(a, b) for n, a, b in zip(NAMES, grads, ref)}
    print(f"train W={W} {src} M={M} (g=0 on {int(near.sum())} rows): sdf {worst:.2e} ({ratio:.1f} u a_sdf), dx {dratio:.1f} u a_dx, "
          + " ".join(f"{n}={e:.2e}" for n, e in err.items()))
    assert all(e <= GRAD_BAR for e in err.values()), err


# ------------------------------------------------------------------------------------------------------------- c. device-side count
@pytest.mark.parametrize("W", WIDTHS)
def test_rows_past_the_device_count(nl, simt, W):
    dec = _decoder(nl, W, "seed")
    bufs = _bufs(nl, dec)
    p = R.params64(dec)
    cap, count = 40_000, 40_000 - 3 * 128 - 45
    x, g = _features(cap, seed=9 + W)
    g[R.near_zero(x, p)] = 0.0
    xn, gn = x.clone(), g.clone()
    xn[count:], gn[count:] = float("nan"), float("nan")
    n_keep, mdev = _mdev(count)
    sdf, dx = _full((cap,)), _full((cap, 16))
    got, _ = _train(nl, bufs, cap, xn, sdf, dx, True, mdev, dsdf_ext=gn)
    assert all(bool(t.isfinite().all()) for t in got)
    assert bool((sdf[count:] == SENT).all() and (dx[count:] == SENT).all()), "a row past the device count was written"
    sdf1, dx1 = _full((count,)), _full((count, 16))
    alone, _ = _train(nl, bufs, count, x[:count].contiguous(), sdf1, dx1, True, dsdf_ext=g[:count].contiguous())
    assert torch.equal(sdf[:count], sdf1) and torch.equal(dx[:count], dx1)
    ref = R.backward(x[:count], g[:count], p)[1]
    e_alone = {n: float((a - b).double().norm() / b.double().norm()) for n, a, b in zip(NAMES, got, alone)}
    e_ref = {n: _rel(a, b) for n, a, b in zip(NAMES, got, ref)}
    print(f"count W={W}: vs first-rows run " + " ".join(f"{n}={e:.1e}" for n, e in e_alone.items())
          + " | vs fp64 " + " ".join(f"{n}={e:.1e}" for n, e in e_ref.items()))
    assert all(e <= GRAD_BAR for e in e_alone.values()), e_alone
    assert all(e <= GRAD_BAR for e in e_ref.values()), e_ref
    # a count of 0 writes nothing and adds nothing
    n_zero, mdev0 = _mdev(0)
    sdf, dx = _full((cap,)), _full((cap, 16))
    zero, _ = _train(nl, bufs, cap, xn, sdf, dx, True, mdev0, dsdf_ext=gn)
    assert bool((sdf == SENT).all() and (dx == SENT).all()) and all(bool((t == 0).all()) for t in zero)
    # a count above the capacity is the capacity
    n_over, mdev2 = _mdev(cap + 1000)
    sdf, dx = _full((cap + 5,)), _full((cap + 5, 16))
    over, _ = _train(nl, bufs, cap, x, sdf, dx, True, mdev2, dsdf_ext=g)
    sdf2, dx2 = _full((cap + 5,)), _full((cap + 5, 16))
    host, _ = _train(nl, bufs, cap, x, sdf2, dx2, True, dsdf_ext=g)
    assert torch.equal(sdf, sdf2) and torch.equal(dx, dx2) and bool((sdf[cap:] == SENT).all())
    assert all(float((a - b).double().norm() / b.double().norm()) <= GRAD_BAR for a, b in zip(over, host))


# ------------------------------------------------------------------------------------------------------------- d. in-kernel loss
def _stats(nl, g_fs, g_sdf):
    s = nl._capi.RenderStats()
    s.g_fs, s.g_sdf = g_fs, g_sdf
    return bytes(s)


def _read_stats(nl, st, k=0):
    n = C.sizeof(nl._capi.RenderStats)
    return nl._capi.RenderStats.from_buffer_copy(st.cpu().numpy().tobytes()[k * n:(k + 1) * n])


def _samples(counts, rays_per_problem, seed, with_cos=True):
    """Samples sorted by problem (counts[k] of problem k), several per ray, flags 0 / 1 / 2 in mixed order; per-ray gt depth and
    cosine; depths around the surface.  Returns device tensors (flag, depth, ray, gt, cos)."""
    gen = torch.Generator().manual_seed(seed)
    K = len(counts)
    rays = [k * rays_per_problem + torch.sort(torch.randint(0, rays_per_problem, (n,), generator=gen)).values for k, n in enumerate(counts)]
    ray = torch.cat(rays).to(torch.int32)
    M = ray.shape[0]
    flag = torch.randint(0, 3, (M,), generator=gen).to(torch.uint8)
    gt = (2.0 + 28.0 * torch.rand(K * rays_per_problem, generator=gen)).float()
    cos = (0.5 + 0.5 * torch.rand(K * rays_per_problem, generator=gen)).float()
    c = cos[ray.long()] if with_cos else 1.0
    depth = (gt[ray.long()] / c + 0.8 * (torch.rand(M, generator=gen) - 0.5)).float()
    return [t.cuda().contiguous() for t in (flag, depth, ray, gt)] + [cos.cuda().contiguous() if with_cos else None]


@pytest.mark.parametrize("with_cos", [True, False], ids=["cos", "nocos"])
@pytest.mark.parametrize("W", WIDTHS)
def test_in_kernel_loss(nl, simt, W, with_cos):
    dec = _decoder(nl, W, "seed")
    bufs = _bufs(nl, dec)
    p = R.params64(dec)
    n_rays = 3000
    flag, depth, ray, gt, cos = _samples([FULL + 1100], n_rays, seed=W + with_cos, with_cos=with_cos)
    M = flag.shape[0]
    x, _ = _features(M, seed=31 * W)
    flag[R.near_zero(x, p)] = 0
    g_fs, g_sdf = 0.7 / M, 1e4 / M
    st = torch.frombuffer(bytearray(_stats(nl, g_fs, g_sdf)), dtype=torch.uint8).cuda()
    sdf, dx = _full((M,)), _full((M, 16))
    grads, _ = _train(nl, bufs, M, x, sdf, dx, True, s_flag=flag, s_depth=depth, s_ray=ray, cos=cos, gt_depth=gt,
                      stats_ptr=C.c_void_p(st.data_ptr()), truncation=TRUNC)
    s = _read_stats(nl, st)
    fs, sd, _ = R.loss(sdf, flag, depth, ray, gt, cos, TRUNC, g_fs, g_sdf)
    e_fs, e_sd = abs(s.fs_sum - fs) / fs, abs(s.sdf_sum - sd) / sd
    assert e_fs <= LOSS_BAR and e_sd <= LOSS_BAR, (s.fs_sum, fs, s.sdf_sum, sd)
    # the fp64 chain: fp64 sdf -> fp64 d loss / d sdf -> fp64 backward
    worst, _ = _check_forward(x, p, W, sdf)
    sdf64 = R.forward(x, p)["sdf"]
    _, _, g64 = R.loss(sdf64, flag, depth, ray, gt, cos, TRUNC, g_fs, g_sdf)
    dx_ref, ref, a_dx = R.backward(x, g64, p, with_abs=True)
    # the kernel's d loss / d sdf carries its sdf error and the fp32 roundings of e: a bound dg per row, carried through |W|
    a_sdf = torch.cat([R.absolute(x[s_:e_], p)[2] for s_, e_ in R._chunks(M)])
    dsdf = (2 * W + 20) * U * a_sdf
    zr = depth.double() * (cos.double()[ray.long()] if cos is not None else 1.0)
    t, f = float(torch.tensor(TRUNC, dtype=torch.float32)), flag.long()
    mag = zr.abs() + sdf64.abs() * t + gt.double()[ray.long()].abs()
    dg = torch.where((f & 1) != 0, 2 * g_fs * (dsdf + 4 * U * (sdf64 - 1).abs()), 0.0) + \
        torch.where((f & 2) != 0, 2 * g_sdf * t * (t * dsdf + 6 * U * mag), 0.0)
    _, _, a_dg = R.backward(x, dg, p, with_abs=True)
    _, dfrac = _check_dx(dx, dx_ref, a_dx + a_dg, W, flag == 0, extra=a_dg)
    err = {n: _rel(a, b) for n, a, b in zip(NAMES, grads, ref)}
    print(f"loss W={W} cos={with_cos} M={M}: fs_sum {e_fs:.1e} sdf_sum {e_sd:.1e}, sdf {worst:.2e}, dx at {dfrac:.2f} of its bound, "
          + " ".join(f"{n}={e:.2e}" for n, e in err.items()))
    assert all(e <= GRAD_BAR for e in err.values()), err


# ------------------------------------------------------------------------------------------------------------- e. batched per-problem loss
BATCH_COUNTS = (0, 5, 16, 17, 33, 1, 4000)
BATCH_CASES = [("simt", W, "train") for W in WIDTHS] + [("tc", 256, "train"), ("tc", 256, "score")]


@pytest.mark.parametrize("impl,W,kind", BATCH_CASES, ids=[f"{i}-W{W}-{k}" for i, W, k in BATCH_CASES])
def test_batched_loss_per_problem(nl, monkeypatch, impl, W, kind):
    monkeypatch.setenv("NL_MLP_IMPL", impl)
    lib, ptr, E = nl._capi.lib(), nl._capi.ptr, nl.engine
    dec = _decoder(nl, W, "seed")
    bufs = _bufs(nl, dec, impl)
    K, RP = len(BATCH_COUNTS), 64
    flag, depth, ray, gt, cos = _samples(BATCH_COUNTS, RP, seed=77 + W)
    M = flag.shape[0]
    x, _ = _features(M, seed=55 + W)
    g_fs = [0.37 * (k + 1) / M for k in range(K)]
    g_sdf = [1e4 / (k + 1) / M for k in range(K)]
    pst = torch.frombuffer(bytearray(b"".join(_stats(nl, a, b) for a, b in zip(g_fs, g_sdf))), dtype=torch.uint8).cuda()
    sdf, dx = _full((M + 3,)), _full((M + 3, 16))
    st = nl._capi.stream_ptr()
    p = bufs.params
    if impl == "simt":
        w = bufs.weights_struct()
        nl._capi.check(lib.nl_mlp_train_batch(M, None, ptr(x), C.byref(w), ptr(flag), ptr(depth), ptr(ray), ptr(cos), ptr(gt), ptr(pst), RP,
                                              TRUNC, ptr(sdf), ptr(dx), st), "nl_mlp_train_batch")
    elif kind == "train":
        nl._capi.check(lib.nl_mlp_tc_train_batch(M, None, ptr(x), ptr(bufs.tc_panels), ptr(p[1]), ptr(p[3]), ptr(p[4]), ptr(p[5]), ptr(flag),
                                                 ptr(depth), ptr(ray), ptr(cos), ptr(gt), ptr(pst), RP, TRUNC, ptr(sdf), ptr(dx), st),
                       "nl_mlp_tc_train_batch")
    else:
        nl._capi.check(lib.nl_mlp_tc_score_batch(M, None, ptr(x), ptr(bufs.tc_panels), ptr(p[1]), ptr(p[3]), ptr(p[4]), ptr(p[5]), ptr(flag),
                                                 ptr(depth), ptr(ray), ptr(cos), ptr(gt), ptr(pst), RP, TRUNC, ptr(sdf), st),
                       "nl_mlp_tc_score_batch")
    torch.cuda.synchronize()
    assert bool((sdf[M:] == SENT).all() and (dx[M:] == SENT).all())
    fs, sd, _ = R.problem_loss(sdf[:M], flag, depth, ray, gt, cos, TRUNC, RP, g_fs, g_sdf)
    worst = 0.0
    for k in range(K):
        s = _read_stats(nl, pst, k)
        for got, ref in ((s.fs_sum, float(fs[k])), (s.sdf_sum, float(sd[k]))):
            if ref == 0.0:
                assert got == 0.0, (k, got)
            else:
                worst = max(worst, abs(got - ref) / ref)
                assert abs(got - ref) <= LOSS_BAR * ref, (k, got, ref)
    # per sample, the single-problem kernel with that problem's constants, bit for bit
    off = 0
    for k, n in enumerate(BATCH_COUNTS):
        if n == 0:
            continue
        sl = slice(off, off + n)
        st1 = torch.frombuffer(bytearray(_stats(nl, g_fs[k], g_sdf[k])), dtype=torch.uint8).cuda()
        sdf1, dx1 = _full((n,)), _full((n, 16))
        _train(nl, bufs, n, x[sl].contiguous(), sdf1, dx1, False, s_flag=flag[sl].contiguous(), s_depth=depth[sl].contiguous(),
               s_ray=ray[sl].contiguous(), cos=cos, gt_depth=gt, stats_ptr=C.c_void_p(st1.data_ptr()), truncation=TRUNC)
        assert torch.equal(sdf[sl], sdf1), k
        if kind == "train":
            assert torch.equal(dx[sl], dx1), k
        off += n
    print(f"batch {impl} W={W} {kind}: K={K} M={M}, worst per-problem sum error {worst:.1e}")
