"""The emulator of the tensor-core decoder's arithmetic (tests/decoder_tc_ref.py) and the bars it sets for the GPU test.

* The tf32 split: the kernel's bit trick against an independent round-half-away-from-zero, and what the split leaves.
* The design (3, 3, 2, 3 terms) stays inside the hard bound and the discriminating bar on every decoder the GPU test uses.
* Every near miss -- a layer with one lo term dropped, single-pass tf32 in layer 1 -- exceeds the discriminating bar of an output
  it feeds by at least 4x, so the GPU test can tell it from the design.  The ratios are printed (pytest -s)."""
import numpy as np
import pytest

import decoder_tc_ref as T
from util import golden

U = T.U
ROWS = 1024
MARGIN = 4.0
# mutant -> the outputs whose discriminating bar must see it (the forward mutants leave the backward inputs as they are: the
# backward pass reads only the relu' masks and d loss / d sdf)
MUTANTS = {
    "layer 1 without al*bh": ((2, 3, 2, 3), ("sdf",)),
    "layer 1 single-pass tf32": ((1, 3, 2, 3), ("sdf",)),
    "layer 2 without al*bh": ((3, 2, 2, 3), ("sdf",)),
    "backward 2 without a*bl": ((3, 3, 1, 3), ("dh1", "dx")),
    "backward 1 without al*bh": ((3, 3, 2, 2), ("dx",)),
}
DECODERS = ("golden", "seed0", "seed1", "seed2", "trained", "dead")


def golden_params():
    z = golden("render.npz")
    return [z["dec_" + k].astype(np.float32) for k in ("pts_linears.0.weight", "pts_linears.0.bias", "pts_linears.1.weight",
                                                       "pts_linears.1.bias", "sdf_out.weight", "sdf_out.bias")]


# ------------------------------------------------------------------------------------------------ the split
def _f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def test_bit_trick_rounds_half_away_from_zero():
    rng = np.random.default_rng(0)
    ties = (rng.integers(0, 1 << 19, 4096, dtype=np.uint32) << 13) | 0x1000          # exactly half a tf32 ulp below the next
    ties &= 0x7f7fffff                                                                 # finite, below the exponent of FLT_MAX
    near_ties = np.concatenate([ties - 1, ties + 1])
    subnormal = np.concatenate([np.arange(1, 1 << 14, dtype=np.uint32), rng.integers(1, 1 << 23, 4096, dtype=np.uint32),
                                np.uint32([0x007fffff, 0x007ff000, 0x00001000])])
    powers = (np.arange(1, 254, dtype=np.uint32) << 23)
    rand = rng.integers(0, 0x7f7fe000, 1 << 16, dtype=np.uint32)
    bits = np.concatenate([ties, near_ties, subnormal, powers, powers - 1, powers + 1, rand, np.uint32([0, 0x3f800fff, 0x3f801000])])
    a = _f32(bits)
    for v in (a, -a):
        got, want = T.rna(v), T.rna_ref(v)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), v[got.view(np.uint32) != want.view(np.uint32)][:5]
    assert T.rna(np.float32(0.0)).view(np.uint32) == 0 and T.rna(np.float32(-0.0)).view(np.uint32) == 0x80000000
    # ties go away from zero: 1 + 2^-11 -> 1 + 2^-10, and the same below zero
    assert T.rna(np.float32(1 + 2.0 ** -11)) == np.float32(1 + 2.0 ** -10) and T.rna(np.float32(-1 - 2.0 ** -11)) == np.float32(-1 - 2.0 ** -10)


def test_split_leaves_at_most_2_to_the_minus_22():
    rng = np.random.default_rng(1)
    a = (rng.standard_normal(1 << 18) * np.exp2(rng.integers(-100, 100, 1 << 18))).astype(np.float32)
    hi, lo = T.split(a)
    r = np.abs(a.astype(np.float64) - hi.astype(np.float64) - lo.astype(np.float64))
    assert bool((r <= 2.0 ** -22 * np.abs(a.astype(np.float64))).all()), float((r / np.abs(a.astype(np.float64))).max())


def test_finite_inputs_near_flt_max_round_to_inf():
    """Outside the kernels' contract: the carry of the rounding reaches the exponent, as cvt.rna.tf32.f32 does."""
    big = _f32(np.uint32([0x7f7ff000, 0x7f7fffff]))
    assert np.isinf(T.rna(big)).all() and np.isinf(T.rna(-big)).all()
    assert T.rna(_f32(np.uint32(0x7f7fefff))) == _f32(np.uint32(0x7f7fe000))


# ------------------------------------------------------------------------------------------------ the bars
def params(name):
    if name == "golden":
        return golden_params()
    if name.startswith("seed"):
        return T.seeded_params(T.SEEDS[int(name[4:])])
    if name == "trained":
        return T.trained_scale(T.seeded_params(T.SEEDS[0]))
    return T.dead_layer1(golden_params())


@pytest.fixture(scope="module", params=DECODERS)
def emulated(request):
    """Per decoder: the fp64 yardstick, and the worst ratios of the design and of every mutant."""
    P = params(request.param)
    x = T.features(ROWS, 11, P)
    g = T.dsdf(ROWS, 11, x, P)
    ref = T.reference(x, P, g)
    out = {}
    fwd = {}
    for name, terms in [("design", T.DESIGN)] + [(n, t) for n, (t, _) in MUTANTS.items()]:
        if terms[:2] not in fwd:
            fwd[terms[:2]] = T.forward(x, P, terms)
        z1, z2, sdf = fwd[terms[:2]]
        dh1, dx = T.backward(z1, z2, g, P, terms)
        out[name] = dict(sdf=(sdf, ref["a_sdf"]), dh1=(dh1, ref["a_dh1"]), dx=(dx, ref["a_dx"]))
    return request.param, x, g, ref, out


def test_design_within_the_bars(emulated):
    name, x, g, ref, out = emulated
    W0, b0 = params(name)[:2]
    worst = {}
    for k, (got, a) in out["design"].items():
        err = np.abs(got.astype(np.float64) - ref[k])
        assert bool((err <= T.HARD[k] * U * a).all()), f"{name} {k} outside the hard bound"
        worst[k] = T.ratio(got, ref[k], a)
        assert worst[k] * MARGIN <= T.DISC[k], (name, k, worst[k])
    assert bool((out["design"]["dx"][0][g == 0] == 0).all())
    print(f"\n{name}: design worst " + " ".join(f"{k} {v:.3f}" for k, v in worst.items()) + f" u a (bars {T.DISC}); "
          f"near-zero rows {int(ref['near'].sum())} of {ROWS}; dead row {'yes' if T.dead_row(params(name)) is not None else 'no'}")


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_every_mutant_fails_the_discriminating_bar(emulated, mutant):
    name, x, g, ref, out = emulated
    seen = {k: T.ratio(out[mutant][k][0], ref[k], out[mutant][k][1]) for k in MUTANTS[mutant][1]}
    print(f"\n{name} {mutant}: " + " ".join(f"{k} {v:.1f} u a ({v / T.DISC[k]:.0f}x its bar)" for k, v in seen.items()))
    assert max(v / T.DISC[k] for k, v in seen.items()) >= MARGIN, seen


def test_seeded_params_are_lidar_decoders():
    import torch
    import nerfloam_b200 as nl
    for s in T.SEEDS:
        torch.manual_seed(s)
        dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0)
        lin = list(dec.pts_linears)
        got = [t.detach().numpy() for t in (lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias, dec.sdf_out.weight, dec.sdf_out.bias)]
        assert all(np.array_equal(a, b) for a, b in zip(got, T.seeded_params(s)))


def test_trained_scale_and_dead_decoders():
    P = T.trained_scale(T.seeded_params(T.SEEDS[0]))
    x = (np.random.default_rng(3).standard_normal((4096, 16)) * 0.05).astype(np.float32)
    r = T.reference(x, P)
    for z in (r["z1"], r["z2"]):
        assert 0.4 <= float((z > 0).mean()) <= 0.6
    D = T.dead_layer1(golden_params())
    d = T.dead_row(D)
    assert d is not None and bool((T.reference(d[None], D)["z1"] < 0).all())
    assert bool((T.features(8, 0, D)[3] == d).all())
