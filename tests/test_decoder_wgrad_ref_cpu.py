"""The emulator of the decoder's weight-gradient arithmetic (tests/decoder_wgrad_ref.py) and the per-element bars it sets for
tests/test_gpu_decoder_wgrad_elementwise.py.

* The design stays inside the hard bound u (HARD A + F) on every element, and its worst err / (u (A + F)) stays 4x under DISC, on
  every decoder and d loss / d sdf kind the GPU test runs.
* Every near miss (a dropped tf32 term in gW0 or in the recomputed h1, G without lo, without the power-of-two scaling, or with
  one shift per chunk instead of one per row, gW2 without b1 c) exceeds DISC on a gradient it feeds by at least 4x.
* One shift per chunk passes the old 2e-5 norm-wise gate of the weight gradients on graded units while failing DISC: the fault
  the element-wise bars exist to see.
The ratios are printed (pytest -s).  M covers three tiles per CTA of the training kernel and 17 chunks per split of k_wgrad_tc
at 132 SMs."""
import numpy as np
import pytest

import decoder_tc_ref as T
import decoder_wgrad_ref as W
from test_decoder_tc_ref_cpu import params as tc_params

U = T.U
M = 2 * 128 * W.SMS + 77
MARGIN = 4.0
GATE = 2e-5            # the norm-wise gate of tests/test_gpu_decoder_wgrad.py
DECODERS = ("golden", "seed0", "trained", "dead", "graded")
# the inputs each mutant runs on (the emulator takes seconds per run); its worst ratio over them must clear the bar
MUTANT_INPUTS = (("graded", "mapping"), ("golden", "span"))


def params(name):
    return W.graded(T.seeded_params(T.SEEDS[0])) if name == "graded" else tc_params(name)


class Case:
    """One decoder: features, fp64 masks, and dh1 for d loss / d sdf = 1 (decoder_tc_ref.backward; dh1 = fl(g D) for any g)."""

    def __init__(self, name):
        self.name, self.P = name, params(name)
        self.P64 = [p.astype(np.float64) for p in self.P]
        self.x = T.features(M, 11, self.P)
        self.ref = T.reference(self.x, self.P)
        self.m2 = self.ref["z2"] > 0
        self.D = T.backward(self.ref["z1"], self.ref["z2"], np.ones(M, np.float32), self.P)[0]
        self.runs = {}

    def inputs(self, kind):
        """(g, fp64 gradients, A, F, dh1) for a d loss / d sdf kind."""
        if kind not in self.runs:
            g = W.raw_dsdf(kind, M, 7)
            g[self.ref["near"]] = 0
            x64, g64 = self.x.astype(np.float64), g.astype(np.float64)
            A, F = W.absolute64(x64, self.P64, g64)
            self.runs[kind] = dict(g=g, ref=W.grads64(x64, self.P64, g64), A=A, F=F, dh1=(g[:, None] * self.D).astype(np.float32))
        return self.runs[kind]

    def emulate(self, kind, **mut):
        r = self.inputs(kind)
        key = ("out",) + tuple(sorted(mut.items()))
        if key not in r:
            if "gw0_terms" in mut:
                r[key] = list(W.emulate_gw0(self.x, r["dh1"], terms=mut["gw0_terms"])) + [None] * 4
            elif "b1c" in mut:
                self.emulate(kind)                       # the design's G sums, which the epilogue reruns from
                r[key] = [None, None] + W.emulate_g(self.x, r["g"], self.m2, self.P, b1c=False, tot=r["tot"])[0]
            else:
                gs, tot = W.emulate_g(self.x, r["g"], self.m2, self.P, **mut)
                if not mut:
                    r["tot"] = tot
                    gs = list(W.emulate_gw0(self.x, r["dh1"])) + gs
                else:
                    gs = [None, None] + gs
                r[key] = gs
        return r[key]


_CASES = {}


def case(name):
    if name not in _CASES:
        _CASES[name] = Case(name)
    return _CASES[name]


@pytest.mark.parametrize("name", DECODERS)
def test_design_within_the_bars(name):
    c = case(name)
    hard = W.hard(M)
    lines = []
    for kind in W.KINDS:
        r = c.inputs(kind)
        got = c.emulate(kind)
        worst = {}
        for n, a, ref, A in zip(W.NAMES, got, r["ref"], r["A"]):
            ok = W.within_hard(a, ref, A, r["F"].get(n, 0.0), hard[n])
            assert bool(ok.all()), f"{name} {kind}: {n} outside the hard bound"
            worst[n] = W.ratio(a, ref, A, r["F"].get(n, 0.0))
            assert worst[n] * MARGIN <= W.DISC[n], (name, kind, n, worst[n])
        lines.append(f"  {kind:8s} " + " ".join(f"{n} {v:.3f}" for n, v in worst.items()))
    print(f"\n{name}: design worst err / (u A) (DISC {W.DISC}, HARD {hard}):\n" + "\n".join(lines))


@pytest.mark.parametrize("mutant", list(W.MUTANTS))
def test_every_mutant_fails_the_discriminating_bar(mutant):
    flags, seen_by = W.MUTANTS[mutant]
    best = 0.0
    lines = []
    for name, kind in MUTANT_INPUTS:
        c = case(name)
        r = c.inputs(kind)
        got = c.emulate(kind, **flags)
        seen = {n: W.ratio(got[i], r["ref"][i], r["A"][i], r["F"].get(n, 0.0)) for n, i in ((n, W.NAMES.index(n)) for n in seen_by)}
        best = max([best] + [v / W.DISC[n] for n, v in seen.items()])
        lines.append(f"{name} {kind}: " + " ".join(f"{n} {v:.3g} u A ({v / W.DISC[n]:.3g}x its bar)" for n, v in seen.items()))
    print(f"\n{mutant}: " + "; ".join(lines))
    assert best >= MARGIN, (mutant, lines)


def test_per_chunk_shift_passes_the_norm_gate_and_fails_disc():
    """One power-of-two shift per chunk (from the warpgroup's largest row) instead of one per row: on units that span eight decades
    the small rows lose their bits, yet norm-wise the gradients stay far inside the 2e-5 gate."""
    c = case("graded")
    r = c.inputs("mapping")
    got = c.emulate("mapping", g_shift="chunk")
    seen = {}
    for n in ("gW1", "gW2"):
        i = W.NAMES.index(n)
        nw = float(np.linalg.norm(got[i].astype(np.float64) - r["ref"][i]) / np.linalg.norm(r["ref"][i]))
        seen[n] = W.ratio(got[i], r["ref"][i], r["A"][i], r["F"][n]) / W.DISC[n]
        print(f"\nper-chunk shift, graded decoder, mapping-scale d sdf: {n} norm-wise {nw:.2e} (gate {GATE}), "
              f"element-wise {seen[n]:.3g}x DISC {W.DISC[n]}")
        assert nw < GATE
    # the lost bits sit in gW1's small elements; gW2 sums them into elements that large rows dominate
    assert seen["gW1"] >= MARGIN, seen


def test_hard_grows_with_the_launch():
    """HARD(M, S) counts the fp32 sums the launch makes: more tiles per CTA and more chunks per split mean a larger bound."""
    small, big = W.hard(1), W.hard(776_000)
    assert all(big[n] > small[n] for n in W.NAMES)
    lay = W.layout(776_000)
    assert (lay["grid"], lay["T"], lay["nsplit"], lay["C"]) == (132, 46, 33, 368)
