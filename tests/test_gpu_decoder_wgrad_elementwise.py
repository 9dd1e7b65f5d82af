"""The decoder weight gradients, element by element, against fp64 (tests/decoder_wgrad_ref.py).

A norm-wise gate cannot see a fault confined to small elements, which is where the fp16 scaling of G, dead layer-1 units and the
tile and chunk edges live.  So every element of gW0, gb0, gW1, gb1, gW2 and gb2 is held to the hard bound u (HARD(M, S) A + F)
derived from the kernels' arithmetic (S the SM count), and at the sample count the emulator calibrated, the worst err / (u A) of
each gradient (err / (u (A + F)), F the fp16 floor of gW1 and gW2) to the discriminating bar DISC, which every emulated near miss of the design exceeds by at least 4x.

Tensor-core path (engine.mlp_train with an external d loss / d sdf, weight gradients on), in both activation layouts (with and
without the dh1 plane): the decoders and d loss / d sdf kinds of the CPU test, at tile and chunk edges (1 .. 129, 64 nsplit +- 1,
128 S +- 1, 3 x 128 S + 77), the calibrated count and 776 000; the device-side count (rows past it hold NaN; a count of 0 adds
nothing); and accumulation into gradients that already hold a sum.  The fp32 CUDA-core path (NL_MLP_IMPL=simt) at widths 32 .. 256,
held to a classical fp32 bound over each gradient's summation (derivation at hard_simt).

Rows whose pre-activation is within decoder_tc_ref's near-zero margin get d loss / d sdf = 0, as in the other decoder tests."""
import ctypes as C

import pytest
import torch

import decoder_ref as R
import decoder_tc_ref as T
import decoder_wgrad_ref as W
from test_gpu_decoder_tc import _golden_np, _near

pytestmark = pytest.mark.gpu

U = T.U
NAMES = W.NAMES
DECODERS = ("golden", "seed0", "seed1", "seed2", "trained", "dead", "graded")
CPU_M = 2 * 128 * W.SMS + 77        # the sample count test_decoder_wgrad_ref_cpu.py emulates
WORST = {}                           # (path, gradient) -> (worst err / (u A), HARD at that M)


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    yield nl
    print("\nworst err / (u (A + F)) per gradient (HARD at the worst run's M; DISC where the CPU test calibrated it):")
    for k in sorted(WORST):
        r, h = WORST[k]
        print(f"  {k[0]:10s} {k[1]:4s} {r:10.4f}   HARD {h:6.0f}   DISC {W.DISC[k[1]] if k[0].startswith('tc') else '-'}")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


_PARAMS, _BUFS = {}, {}


def params_np(name):
    if name not in _PARAMS:
        if name == "golden":
            P = _golden_np()
        elif name.startswith("seed"):
            P = T.seeded_params(T.SEEDS[int(name[4:])])
        elif name == "trained":
            P = T.trained_scale(T.seeded_params(T.SEEDS[0]))
        elif name == "dead":
            P = T.dead_layer1(_golden_np())
        else:
            P = W.graded(T.seeded_params(T.SEEDS[0]))
        _PARAMS[name] = P
    return _PARAMS[name]


def _bufs(nl, name):
    """DecoderBuffers of the decoder with the numpy parameters params_np(name), and its fp64 parameters."""
    if name not in _BUFS:
        dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0)
        keys = ("pts_linears.0.weight", "pts_linears.0.bias", "pts_linears.1.weight", "pts_linears.1.bias", "sdf_out.weight", "sdf_out.bias")
        dec.load_state_dict({k: torch.from_numpy(v) for k, v in zip(keys, params_np(name))})
        dec = dec.cuda()
        bufs = nl.engine.DecoderBuffers(dec, torch.device("cuda"))
        assert nl.engine.mlp_impl(bufs.width) == "tc"
        bufs.refresh_transposes()
        _BUFS[name] = (bufs, R.params64(dec))
    return _BUFS[name]


_DEAD = {}


def _features(name, M, seed):
    """decoder_tc_ref.features(M, seed, P) with the decoder's dead row found once."""
    if name not in _DEAD:
        _DEAD[name] = T.dead_row(params_np(name))
    x = T.features(M, seed)
    if M > 3 and _DEAD[name] is not None:
        x[3] = _DEAD[name]
    return x


def _inputs(name, kind, M, seed, p64):
    x = torch.from_numpy(_features(name, M, seed)).cuda()
    g = torch.from_numpy(W.raw_dsdf(kind, M, seed + 1)).cuda()
    g[_near(x, p64)] = 0.0
    return x, g


def _mdev(n):
    t = torch.tensor([n], dtype=torch.int32, device="cuda")
    return t, C.c_void_p(t.data_ptr())


def _train(nl, bufs, M_cap, x, g, dh1=True, count=None, zero=True):
    """Weight gradients of one engine.mlp_train call (into zeroed gradients unless zero=False)."""
    dev = torch.device("cuda")
    if zero:
        bufs.gradflat.zero_()
    act = nl.engine.alloc_act(bufs.width, M_cap, dev, dh1=dh1) if nl.engine.mlp_impl(bufs.width) == "tc" else \
        nl.engine.alloc_act(bufs.width, M_cap, dev)
    sdf, dx = torch.empty(M_cap, device=dev), torch.empty(M_cap, 16, device=dev)
    keep = _mdev(count) if count is not None else (None, None)
    nl.engine.mlp_train(bufs, M_cap, keep[1], x, sdf, dx, True, act, dsdf_ext=g)
    torch.cuda.synchronize()
    return [t.clone() for t in bufs.grads]


def _check(path, label, got, x, g, p64, hard, disc=False, A=None, F=None, ref=None):
    """Every element of every gradient within u (hard A + F); with disc, the worst err / (u (A + F)) under DISC.  Returns the ratios."""
    if ref is None:
        ref = W.grads64(x.double(), p64, g.double())
    if A is None:
        A, F = W.absolute64(x.double(), p64, g.double())
    out = {}
    for n, a, r, aa in zip(NAMES, got, ref, A):
        err = (a.double() - r).abs()
        bound = U * (hard[n] * aa + F.get(n, 0.0))
        bad = ~(err <= bound)
        assert not bool(bad.any()), (f"{path} {label}: {n} outside the hard bound ({hard[n]} u A) at "
                                     f"{bad.nonzero()[:4].tolist()}: err {err[bad][:4].tolist()} bound {bound[bad][:4].tolist()}")
        ae = aa + F.get(n, 0.0)
        live = ae > 0
        out[n] = float((err[live] / (U * ae[live])).max()) if bool(live.any()) else 0.0
        if out[n] >= WORST.get((path, n), (-1.0, 0))[0]:
            WORST[(path, n)] = (out[n], hard[n])
        if disc:
            assert out[n] <= W.DISC[n], f"{path} {label}: {n} reaches {out[n]:.3f} u A, above the discriminating bar {W.DISC[n]}"
    return out


def _fmt(r):
    return " ".join(f"{k} {v:.3f}" for k, v in r.items())


# ------------------------------------------------------------------------------------------------------------- tensor cores
def _counts():
    S = _sms()
    ns = max(S // 4, 1)
    c = [1, 45, 63, 64, 65, 77, 127, 128, 129, 64 * ns - 1, 64 * ns + 1, 128 * S - 1, 128 * S + 1, 3 * 128 * S + 77, CPU_M, 776_000]
    return sorted(set(c))


@pytest.mark.parametrize("dh1", [True, False], ids=["dh1", "compact"])
@pytest.mark.parametrize("which", range(16))
def test_tensor_core_gradients_per_element(nl, which, dh1):
    counts = _counts()
    if which >= len(counts):
        pytest.skip("fewer distinct sample counts on this device")
    M = counts[which]
    S = _sms()
    hard = W.hard(M, S)
    calibrated = M == CPU_M and S == W.SMS
    lines = []
    for name in DECODERS:
        bufs, p64 = _bufs(nl, name)
        for kind in W.KINDS:
            x, g = _inputs(name, kind, M, seed=M + DECODERS.index(name), p64=p64)
            got = _train(nl, bufs, M, x, g, dh1=dh1)
            r = _check("tc", f"{name} {kind} M={M}", got, x, g, p64, hard, disc=calibrated)
            lines.append(f"  {name:8s} {kind:8s} {_fmt(r)}")
    print(f"\ntc {'dh1' if dh1 else 'compact'} M={M} (HARD {hard}{', DISC checked' if calibrated else ''}):\n" + "\n".join(lines))


@pytest.mark.parametrize("name", ["golden", "graded"])
def test_rows_past_the_device_count(nl, name):
    bufs, p64 = _bufs(nl, name)
    cap, count = 40_000, 40_000 - 3 * 128 - 45
    x, g = _inputs(name, "span", cap, seed=9, p64=p64)
    xn, gn = x.clone(), g.clone()
    xn[count:], gn[count:] = float("nan"), float("nan")
    got = _train(nl, bufs, cap, xn, gn, count=count)
    assert all(bool(t.isfinite().all()) for t in got), "a row past the device count reached the gradients"
    r = _check("tc-count", f"{name} count={count} of {cap}", got, x[:count], g[:count], p64, W.hard(cap, _sms()))
    print(f"count {name}: {_fmt(r)}")
    zero = _train(nl, bufs, cap, xn, gn, count=0)
    assert all(bool((t == 0).all()) for t in zero), "a device count of 0 added to the gradients"


def test_gradients_accumulate(nl):
    """The gradient outputs are accumulated: a second call adds its sums to the first's."""
    bufs, p64 = _bufs(nl, "graded")
    S = _sms()
    M1, M2 = CPU_M, 777
    x1, g1 = _inputs("graded", "mapping", M1, seed=31, p64=p64)
    x2, g2 = _inputs("graded", "span", M2, seed=32, p64=p64)
    _train(nl, bufs, M1, x1, g1)
    got = _train(nl, bufs, M2, x2, g2, zero=False)
    r1, r2 = W.grads64(x1.double(), p64, g1.double()), W.grads64(x2.double(), p64, g2.double())
    (A1, F1), (A2, F2) = W.absolute64(x1.double(), p64, g1.double()), W.absolute64(x2.double(), p64, g2.double())
    h1, h2 = W.hard(M1, S), W.hard(M2, S)
    hard = {n: h1[n] + h2[n] for n in NAMES}
    r = _check("tc-accum", f"{M1} + {M2}", got, None, None, p64, hard, ref=[a + b for a, b in zip(r1, r2)],
               A=[a + b for a, b in zip(A1, A2)], F={n: F1[n] + F2[n] for n in F1})
    print(f"accumulated {M1} + {M2}: {_fmt(r)}")


# ------------------------------------------------------------------------------------------------------------- CUDA cores
def hard_simt(M, Wd, sms):
    """The fp32 CUDA-core kernels' bound, in u times the same absolute evaluations (decoder_wgrad_ref), first order plus 1.
    k_mlp: grid = min(tiles, S) CTAs over 128-sample tiles, T tiles per CTA; 8 warps of 16 samples per tile.  The activations carry
    h1 20 (16 fma + bias, test_gpu_decoder_simt's layer-1 bound), h2 20 + W + 2 (W fma, bias), dh2 = fl(dsdf w2) 1, dh1 W + 2
    (W fma after dh2).  Each gradient is a 16-sample chain per warp (16 roundings), a shared-memory atomic per warp and tile
    (8T) and a global atomic per CTA (grid).  k_dw1 (gW1): per split an fma chain over its 16-sample chunks, 16 C (C = chunks
    per split, nsplit = S / (W / min(W, 128))^2 splits), then an atomic per live split."""
    tiles = -(-M // 128)
    grid = max(min(tiles, sms), 1)
    Tn = -(-tiles // grid)
    red = 16 + 8 * Tn + grid
    nsplit = max(sms // (Wd // min(Wd, 128)) ** 2, 1)
    chunks = -(-M // 16)
    return {"gW0": Wd + 2 + red + 1, "gb0": Wd + 2 + red + 1, "gW1": 20 + 1 + 16 * -(-chunks // nsplit) + min(nsplit, chunks) + 1,
            "gb1": 1 + red + 1, "gW2": 20 + Wd + 2 + red + 1, "gb2": red + 1}


@pytest.mark.parametrize("Wd", [32, 64, 128, 256])
def test_cuda_core_gradients_per_element(nl, monkeypatch, Wd):
    monkeypatch.setenv("NL_MLP_IMPL", "simt")
    S = _sms()
    torch.manual_seed(1000 + Wd)
    dec = nl.lidar.Decoder(depth=2, width=Wd, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    bufs = nl.engine.DecoderBuffers(dec, torch.device("cuda"))
    assert nl.engine.mlp_impl(bufs.width) == "simt"
    bufs.refresh_transposes()
    p64 = R.params64(dec)
    lines = []
    for M in (1, 129, 128 * S + 1, 3 * 128 * S + 77):
        hard = hard_simt(M, Wd, S)
        for kind in W.KINDS:
            x = torch.from_numpy(T.features(M, M + Wd, None)).cuda()
            g = torch.from_numpy(W.raw_dsdf(kind, M, M + Wd + 1)).cuda()
            g[_near(x, p64)] = 0.0
            got = _train(nl, bufs, M, x, g)
            r = _check(f"simt-W{Wd}", f"{kind} M={M}", got, x, g, p64, hard)
            lines.append(f"  M={M:6d} {kind:8s} {_fmt(r)}")
    print(f"\nsimt W={Wd}:\n" + "\n".join(lines))
