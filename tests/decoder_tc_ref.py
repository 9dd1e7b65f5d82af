"""Emulator of the tensor-core decoder's arithmetic (nerf-loam_b200/csrc/mlp_tc.cu, k_mlp_wg), the decoders and features its
tests run on, and the error bars they apply.  NumPy only: the CPU test (test_decoder_tc_ref_cpu.py) runs it, the GPU test
(test_gpu_decoder_tc.py) takes its inputs and bars from here.

The model of one wgmma k-step (8 products of tf32 operands into an fp32 accumulator): the products are exact, their sum is exact,
and the accumulator is rounded toward zero to fp32 once per k-step.  Each term of the hi/lo split (ah*bh, ah*bl, al*bh: 3xTF32) is
its own wgmma, so a k-step of a 3-term GEMM is three such roundings.  The kernel's layers, in that model:
  layer 1       z1 = fl(x W0^T + b0)          K = 16, 3 terms; h1 = relu(z1)
  layer 2       z2 = fl(h1 W1^T + b1)         K = 256, 3 terms; h2 = relu(z2)
  output        sdf                           every quad thread t sums columns 8j + 2t + e (ascending) with fmaf, then
                                              (p0 + p1) + (p2 + p3) (two quad shuffles), then + b2
  backward 2    D3 = m2 B,  B = fl(w2[j] W1[j, k])   A is the exact 0/1 mask relu'(h2): 2 terms (a bh, a bl)
                dh1 = m1 ? fl(dsdf D3) : 0
  backward 1    dx = dh1 W0                   K = 256, 3 terms
`terms` (per layer, in the order above: layer 1, layer 2, backward 2, backward 1) counts the terms kept, in the order ah*bh,
ah*bl, al*bh; anything other than the design (3, 3, 2, 3) exists only to build mutants the bars must see.

Bars (u = 2^-24; a1, a2, a_sdf, a_dh1, a_dx are the network and its backward pass run on |x|, |g|, |W|, |b|, tests/decoder_ref.py):
  * Hard per-row bound, from the model.  A 3-term product misses al*bl, ah*rb and ra*b (r: what the split leaves, at most 2^-22
    of the operand): at most 3 2^-22 = 12 u |a||b|.  A k-step's truncation loses less than one fp32 ulp, 2u, of an accumulator
    that is at most the absolute sum.  The bias add is one rounding.  With e_in the error coming in, carried through |W|:
      layer 1     12 + 2 * 3 * 16/8 + 1                 = 25          (x exact)
      layer 2     25 + 12 + 2 * 3 * 256/8 + 1           = 230
      sdf         230 + 64 + 3  (64 fmaf, 2 shuffle adds, + b2)  = 297
      dh1         1 (B = fl(w2 W1)) + 4 (split of B) + 2 * 2 * 256/8 + 1 (x dsdf)  = 134
      dx          134 + 12 + 2 * 3 * 256/8              = 338
    times u times the absolute evaluation (HARD).  It catches layout, bias and ring faults: those are errors of the size of the
    values themselves.
  * Discriminating bar (DISC): the max over rows (elements for dh1, dx) of err / (u a).  Set from the emulator: at least 4x above
    the design's worst case and at least 4x below the lowest mutant worst case on the same inputs (test_decoder_tc_ref_cpu.py
    checks both).  The emulated design reaches about 0.2 (sdf), 10 (dh1) and 3.3 (dx); the mildest mutants about 11 (sdf), 1700
    (dh1) and 150 (dx).  So the bars are 1, 64 and 24.  dh1's design ratio is the largest because an element of dh1 is one dot
    product of 256 terms whose absolute sum can be far above its value.
  * Near-zero margin: a row whose pre-activation is within twice the hard bound of zero (|z1| <= 50 u a1 or |z2| <= 460 u a2,
    about 3e-6 and 2.7e-5 relative) may have its relu' decided either way by a valid evaluation; the tests give it d loss / d sdf
    = 0 and leave it out of the relu'(h2) comparison.  Twice, because an evaluation whose inner sums are not exact (alignment
    truncation inside a k-step) could reach about 1.6e3 u in layer 2 at worst; if the H100 did that, DISC would see it first."""
import numpy as np

U = 2.0 ** -24
DESIGN = (3, 3, 2, 3)
# hard bound, in u times the absolute evaluation (derivation above)
HARD_Z1, HARD_Z2 = 25, 230
HARD = {"sdf": 297, "dh1": 134, "dx": 338}
DISC = {"sdf": 1.0, "dh1": 64.0, "dx": 24.0}
NEAR_Z1, NEAR_Z2 = 2 * HARD_Z1 * U, 2 * HARD_Z2 * U
SCALES = (1e-3, 0.05, 1.0, 10.0)
SEEDS = (2000, 2001, 2002)          # the seeded decoders


# ------------------------------------------------------------------------------------------------ tf32 and fp32 rounding
def rna(a):
    """tf32 round half away from zero, the kernel's tf32_rna_finite: (u + 0x1000) & 0xffffe000 on the fp32 bits.  For finite
    inputs only: at |a| >= (2 - 2^-11) 2^127 the carry reaches the exponent and the result is +-inf (cvt.rna.tf32.f32 rounds to
    inf there as well); the kernels' operands are far from that."""
    u = np.asarray(a, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)


def rna_ref(a):
    """The same rounding without bit tricks: |a| to a multiple of q = 2^(e - 10) (e = floor(log2 |a|), q at least 2^-136, the
    quantum of tf32 subnormals), ties away from zero, in fp64."""
    a = np.asarray(a, np.float32).astype(np.float64)
    m = np.abs(a)
    _, e = np.frexp(np.where(m > 0, m, 1.0))           # m = f 2^e, f in [0.5, 1)
    q = np.maximum(np.ldexp(1.0, e - 11), 2.0 ** -136)
    r = np.floor(m / q + 0.5) * q
    return np.copysign(r, a).astype(np.float32)


def split(a):
    a = np.asarray(a, np.float32)
    hi = rna(a)
    return hi, rna(a - hi)


def trunc32(v):
    """fp64 -> fp32 rounded toward zero.  Where the result is a normal fp32, clearing the 29 low significand bits of the fp64
    truncates it exactly; zeros, subnormals, overflow and NaN take the rounding route (round, then step back toward zero)."""
    f = (np.ascontiguousarray(v, np.float64).view(np.uint64) & np.uint64(0xFFFFFFFFE0000000)).view(np.float64).astype(np.float32)
    a = np.abs(v)
    odd = ~((a >= 2.0 ** -126) & (a < 2.0 ** 128)) & (v != 0)
    if odd.any():
        r = v[odd].astype(np.float32)
        over = np.abs(r.astype(np.float64)) > np.abs(v[odd])
        r[over] = np.nextafter(r[over], np.float32(0))
        f[odd] = r
    return f


def mm(a, b, terms):
    """fp32 [M, K] x [K, N] as the tensor core does it under the k-step model: per k-step of 8 and per term, the exact sum of
    8 products added to the accumulator, which is then truncated to fp32."""
    ah, al = (x.astype(np.float64) for x in split(a))
    bh, bl = (x.astype(np.float64) for x in split(b))
    parts = [(ah, bh), (ah, bl), (al, bh)][:terms]
    c = np.zeros((a.shape[0], b.shape[1]))
    for k0 in range(0, a.shape[1], 8):
        for p, q in parts:
            c = trunc32(c + p[:, k0:k0 + 8] @ q[k0:k0 + 8]).astype(np.float64)
    return c.astype(np.float32)


def _fma32(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ the kernel's layers
def forward(x, P, terms=DESIGN):
    """Emulated k_mlp_wg forward.  x fp32 [M, 16], P fp32 (W0, b0, W1, b1, w2, b2).  Returns (z1, z2, sdf), fp32."""
    W0, b0, W1, b1, w2, b2 = P
    z1 = mm(x, W0.T, terms[0]) + b0
    h1 = np.maximum(z1, np.float32(0))
    z2 = mm(h1, W1.T, terms[1]) + b1
    h2 = np.maximum(z2, np.float32(0))
    ps = []
    for t in range(4):
        p = np.zeros(x.shape[0], np.float32)
        for c in sorted(c for c in range(256) if (c >> 1) & 3 == t):
            p = _fma32(h2[:, c], w2[0, c], p)
        ps.append(p)
    return z1, z2, ((ps[0] + ps[1]) + (ps[2] + ps[3])) + b2[0]


def backward(z1, z2, g, P, terms=DESIGN):
    """Emulated backward layers from the forward's pre-activations and d loss / d sdf g (fp32 [M]).  Returns (dh1, dx), fp32."""
    W0, _, W1, _, w2, _ = P
    B = (w2[0][:, None] * W1).astype(np.float32)                    # B[j, k] = fl(w2[j] W1[j, k]), k_tc_prepare
    D3 = mm((z2 > 0).astype(np.float32), B, terms[2])
    dh1 = np.where(z1 > 0, g[:, None] * D3, np.float32(0)).astype(np.float32)
    return dh1, mm(dh1, W0, terms[3])


# ------------------------------------------------------------------------------------------------ fp64 yardstick
def reference(x, P, g=None):
    """fp64 values and absolute evaluations: dict with z1, z2, sdf, a1, a2, a_sdf, near [M] (and with g: dh1, dx, a_dh1, a_dx)."""
    W0, b0, W1, b1, w2, b2 = (p.astype(np.float64) for p in P)
    xd = x.astype(np.float64)
    z1 = xd @ W0.T + b0
    h1 = np.maximum(z1, 0)
    z2 = h1 @ W1.T + b1
    h2 = np.maximum(z2, 0)
    a1 = np.abs(xd) @ np.abs(W0).T + np.abs(b0)
    a2 = a1 @ np.abs(W1).T + np.abs(b1)
    out = dict(z1=z1, z2=z2, sdf=(h2 @ w2.T + b2)[:, 0], a1=a1, a2=a2, a_sdf=(a2 @ np.abs(w2).T + np.abs(b2))[:, 0])
    out["near"] = (np.abs(z1) <= NEAR_Z1 * a1).any(1) | (np.abs(z2) <= NEAR_Z2 * a2).any(1)
    if g is not None:
        gd = g.astype(np.float64)
        m1, m2 = z1 > 0, z2 > 0
        out["dh1"] = ((gd[:, None] * w2[0] * m2) @ W1) * m1
        out["dx"] = out["dh1"] @ W0
        out["a_dh1"] = ((np.abs(gd)[:, None] * np.abs(w2[0]) * m2) @ np.abs(W1)) * m1
        out["a_dx"] = out["a_dh1"] @ np.abs(W0)
    return out


def ratio(got, ref, a):
    """max of |got - ref| / (u a) over the entries with a > 0 (0 if there are none)."""
    live = a > 0
    if not live.any():
        return 0.0
    return float((np.abs(got.astype(np.float64) - ref)[live] / (U * a[live])).max())


# ------------------------------------------------------------------------------------------------ decoders and features
def seeded_params(seed):
    """fp32 parameters of `torch.manual_seed(seed); lidar.Decoder(width=256)` (nn.Linear's default initialisation), in the
    order of DecoderBuffers.params, as NumPy arrays."""
    import torch
    import torch.nn as nn
    torch.manual_seed(seed)
    l0, l1, l2 = nn.Linear(16, 256), nn.Linear(256, 256), nn.Linear(256, 1)
    return [t.detach().numpy().copy() for t in (l0.weight, l0.bias, l1.weight, l1.bias, l2.weight, l2.bias)]


def trained_scale(P, seed=7):
    """A decoder at trained scale: P's weights x 8, and every layer-1 and layer-2 bias set so that the unit is active on half of
    a fixed batch of N(0, 0.05^2) features (the median of its pre-activation without bias is its -bias)."""
    W0, _, W1, _, w2, b2 = (p.astype(np.float64) for p in P)
    W0, W1, w2 = 8 * W0, 8 * W1, 8 * w2
    x = np.random.default_rng(seed).standard_normal((4096, 16)) * 0.05
    b0 = -np.median(x @ W0.T, axis=0)
    b1 = -np.median(np.maximum(x @ W0.T + b0, 0) @ W1.T, axis=0)
    return [p.astype(np.float32) for p in (W0, b0, W1, b1, w2, b2)]


def dead_layer1(P):
    """P with every layer-1 bias made negative (-|b0| - 0.01): small features switch every layer-1 unit off."""
    out = [p.copy() for p in P]
    out[1] = (-np.abs(P[1]) - np.float32(0.01)).astype(np.float32)
    return out


def dead_row(P):
    """A feature row on which every layer-1 unit is inactive (z1 < 0), if the decoder has one within |x| <= 10, else None.
    Found by a linear program: minimise s subject to W0 x + b0 <= s."""
    from scipy.optimize import linprog
    W0, b0 = P[0].astype(np.float64), P[1].astype(np.float64)
    n = W0.shape[0]
    res = linprog(np.r_[np.zeros(16), 1.0], A_ub=np.c_[W0, -np.ones(n)], b_ub=-b0, bounds=[(-10, 10)] * 16 + [(None, None)],
                  method="highs")
    if not res.success or res.x[16] >= 0:
        return None
    x = res.x[:16].astype(np.float32)
    return x if bool(((x.astype(np.float64) @ W0.T + b0) < 0).all()) else None


def features(M, seed, P=None):
    """fp32 [M, 16]: row r is N(0, 1) times SCALES[r % 4]; rows 1, 2 and 3 (where M reaches them) are all zero, tf32-exact
    (lo = 0) and, when P has one, a row with every layer-1 unit dead."""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((M, 16)) * np.asarray(SCALES)[np.arange(M) % 4, None]).astype(np.float32)
    if M > 1:
        x[1] = 0
    if M > 2:
        x[2] = rna(x[2])
    if M > 3 and P is not None:
        d = dead_row(P)
        if d is not None:
            x[3] = d
    return x


def dsdf(M, seed, x, P):
    """fp32 d loss / d sdf [M], N(0, 0.1^2), 0 on near-zero rows (see the margin above)."""
    g = (np.random.default_rng(seed + 1).standard_normal(M) * 0.1).astype(np.float32)
    g[reference(x, P)["near"]] = 0
    return g
