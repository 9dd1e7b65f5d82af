"""Emulator of the tensor-core decoder's weight-gradient arithmetic (nerf-loam_b200/csrc/mlp_tc.cu: gw0_quarter in k_mlp_wg, and
k_wgrad_tc), the fp64 yardstick with an absolute evaluation per gradient element, and the per-element bars.  NumPy only: the CPU
test (test_decoder_wgrad_ref_cpu.py) runs the emulator, the GPU test (test_gpu_decoder_wgrad_elementwise.py) takes its inputs and
bars from here.  The k-step model, the tf32 split and dh1 are decoder_tc_ref's (u = 2^-24).

What the kernels do, in that model (M samples, S SMs):
  gW0, gb0  k_mlp_wg, grid = min(tiles, S) persistent CTAs over 128-sample tiles (tile t on CTA t mod grid).  Per warpgroup (64
            samples) and per 32-sample block: gW0^T = x^T dh1 on mma.sync m16n8k8, three tf32 terms (xh dh, xh dl, xl dh), each
            its own accumulator restarted every block (4 k-steps of 8); the block adds (t0 + t1) + t2 into the warpgroup's fp32
            running sum in shared memory.  gb0: every thread sums its 16 samples of a column as 8 pairs (dh1[8ks + t] +
            dh1[8ks + t + 4]), two quad shuffles add the 4 threads, and the total goes into the running sum once per tile.  At
            the end a CTA adds its two warpgroups' sums and makes one fp32 atomic per entry.
  G         k_wgrad_tc, grid = 4 tiles (128 x 128 of G^T) x nsplit = max(S / 4, 1) splits; 64-sample chunk ch goes to split
            ch mod nsplit.  Per chunk: z1^T = W0 x^T by 3xTF32 wgmma (K = 16, the training kernel's term order, so the same
            bits as decoder_tc_ref.mm(x, W0^T, 3)), v = fl(dsdf fl(relu(z1 + b0))); per row k of h1^T the power of two 2^s that
            puts the row's largest |v| over the chunk in [2^14, 2^15); fp16 hi = rn(v 2^s), lo = rn(v 2^s - hi); part = hi m2
            + lo m2 on fp16 wgmma (k-steps of 16, truncated after each of the 8 wgmmas, the 0/1 mask exact); tot = fmaf(part,
            2^-s, tot) in fp32 over the split's chunks.
  c, gb2    c[j] = sum_s m2[s, j] dsdf_s: each thread sums 32 samples in fp32, in sample order, into an fp64 total; the two
            halves are added in fp64 and rounded to fp32.  gb2: fp64 sums of dsdf per warp of tile 0, rounded, two atomics per
            split.
  epilogue  gW1[j, k] += fl(w2[j] tot[k, j]) (an atomic per split);  gW2[j] += r with r = fmaf(W1[j, kr], tot[kr, j],
            fl(W1[j, kr + 8] tot[kr + 8, j])) per thread, a 3-level shuffle tree over the 8 row groups of a warp, the 8
            warps' sums added in order, and on the k0 = 0 tiles + b1[j] c (an atomic per CTA: 2 per split);  gb1[j] +=
            fl(w2[j] c) (one per split).
The emulator runs the atomics in one fixed order (CTA index); the bound below holds for every order.

Absolute evaluations (fp64, from decoder_tc_ref.reference's a1 and a_dh1, which carry no rounding; m1, m2 the fp64 relu'):
  A_gW0[n, e] = sum_s a_dh1[s, n] |x[s, e]|        A_gb0[n] = sum_s a_dh1[s, n]
  A_G[j, k]   = sum_s m2[s, j] |dsdf_s| m1[s, k] a1[s, k]   (a unit that is off adds an exact 0, so m1 keeps the sum tight)
  A_c[j]      = sum_s m2[s, j] |dsdf_s|
  A_gW1 = |w2[j]| A_G      A_gW2[j] = sum_k |W1[j, k]| A_G[j, k] + |b1[j]| A_c[j]      A_gb1 = |w2| A_c      A_gb2 = sum |dsdf|
A_gW2 follows the kernel's route through G; the cancellation in sum_k W1 G is the kernel's and the yardstick's alike.

HARD: the per-element bound |got - fp64| <= u (HARD A + F), first order in u (at these depths the higher-order terms stay far
below 1), with every fp32 rounding counted as u of a partial sum that is at most the absolute sum, a k-step truncation as 2u:
  T = tiles per CTA = ceil(tiles / grid), L = live splits = min(nsplit, chunks), C = chunks per split = ceil(chunks / nsplit)
  gW0   134 (dh1, decoder_tc_ref.HARD) + 12 (3 terms: al bl, ah rb, ra b, 2^-22 each) + 2 * 3 * 4 (truncations per block)
        + 2 (t0 + t1 + t2) + 2T (running sum: two blocks per tile) + 1 (the two warpgroups) + grid (atomics)
  gb0   134 + 1 (pair) + 8 (thread's chain) + 2 (quad shuffles) + T + 1 + grid
  G     25 (z1, decoder_tc_ref.HARD_Z1; relu is 1-Lipschitz) + 1 (x dsdf) + 4 (hi + lo leaves 2^-22 of v 2^s while lo is normal)
        + 2 * 2 * 4 (8 truncations) + C (fmaf per chunk; the 2^s scaling is exact)
        and, where lo is subnormal, at most 2^-25 absolute of v 2^s, i.e. 2^-39 of the row's chunk maximum: the floor
        F_G[j, k] = 2^-14 sum_chunks n[c, j] max_(s in c) |dsdf_s| m1 a1[s, k] (n = the chunk's samples with m2[s, j] and dsdf
        != 0; 2^-14 is twice 2^-15 = 2^-39 / u, the factor covering the kernel's v against its absolute evaluation)
  gW1   G + 1 (w2 G) + L                            F_gW1 = |w2| F_G
  gW2   G + 2 (fma pair) + 3 (shuffles) + 8 (warps) + 1 (+ b1 c) + 2L; the b1 c route is shorter (c: 32 + 1, product,
        add, 2L)                                    F_gW2 = sum_k |W1| F_G
  gb1   32 (thread's fp32 chain) + 1 (to fp32) + 1 (w2 c) + L
  gb2   1 (fp64 partial to fp32) + 2L
  (+ 1 each for the higher-order terms.)  T, grid, L and C grow with M and the SM count, hence HARD(M, S).
  Accumulating into gradients that already hold a sum of A1: the atomics then round partial sums up to A1 + A2, so two calls are
  within (HARD(M1) + HARD(M2)) u (A1 + A2) (+ F1 + F2) of the fp64 sum of both.

DISC: the discriminating bar on max err / (u (A + F)) (F = 0 but for gW1 and gW2: where a chunk's d loss / d sdf spans more
decades than fp16 does, the floor is the design's own error, and the bar measures against it), set from the emulator at the CPU test's sample count: at least 4x above the
design's worst case and at least 4x below every mutant's worst case on the same inputs (test_decoder_wgrad_ref_cpu.py checks
both).  At 2 x 128 x 132 + 77 samples the emulated design reaches 3.2 (gW0), 1.4 (gb0), 5.5 (gW1), 1.5 (gb1), 0.31 (gW2) and
0.43 (gb2); on each of the mutant inputs the mildest mutant reaches 70 (gW0 without xl dh), 410 (gW1, G hi only) and 31 (gW2,
G hi only).  So the bars are 16, 32 and 4.  The bias gradients have no mutant of their own (a fault in c or dh1 shows in gW2 or
gW0 first); their bars, 8, 8 and 4, are above 4x the design and above what the H100's other atomic orders reach.
"""
import numpy as np

import decoder_tc_ref as T
from decoder_tc_ref import U, mm, split, trunc32

TM = 128                # samples per training tile (k_mlp_wg)
KC = 64                 # samples per k_wgrad_tc chunk
WN = 256
SMS = 132               # the SM count of an H100 SXM: the CPU test's layout
NAMES = ("gW0", "gb0", "gW1", "gb1", "gW2", "gb2")
DISC = {"gW0": 16.0, "gb0": 8.0, "gW1": 32.0, "gW2": 4.0, "gb1": 8.0, "gb2": 4.0}
KINDS = ("span", "single", "mapping")
# mutant -> (emulator flags, the gradients whose bar must see it)
MUTANTS = {
    "gW0 single-pass tf32": (dict(gw0_terms=1), ("gW0",)),
    "gW0 without xl dh": (dict(gw0_terms=2), ("gW0",)),
    "h1 single-pass tf32": (dict(h1_terms=1), ("gW1", "gW2")),
    "G hi only": (dict(g_lo=False), ("gW1", "gW2")),
    "G unscaled": (dict(g_shift="none"), ("gW1", "gW2")),
    "G one shift per chunk": (dict(g_shift="chunk"), ("gW1", "gW2")),
    "gW2 without b1 c": (dict(b1c=False), ("gW2",)),
}


# ------------------------------------------------------------------------------------------------ launch layout and HARD
def layout(M, sms=SMS):
    tiles = -(-M // TM)
    grid = max(min(tiles, sms), 1)
    chunks = -(-M // KC)
    nsplit = max(sms // 4, 1)
    return dict(tiles=tiles, grid=grid, T=-(-tiles // grid), chunks=chunks, nsplit=nsplit, L=min(nsplit, chunks),
                C=-(-chunks // nsplit))


def hard(M, sms=SMS):
    """{gradient: HARD} in u times the absolute evaluation (derivation in the module docstring)."""
    lay = layout(M, sms)
    Tn, grid, L, Cn = lay["T"], lay["grid"], lay["L"], lay["C"]
    G = 25 + 1 + 4 + 16 + Cn
    return {"gW0": T.HARD["dh1"] + 12 + 24 + 2 + 2 * Tn + 1 + grid + 1,
            "gb0": T.HARD["dh1"] + 1 + 8 + 2 + Tn + 1 + grid + 1,
            "gW1": G + 1 + L + 1,
            "gW2": G + 14 + 2 * L + 1,
            "gb1": 32 + 1 + 1 + L + 1,
            "gb2": 1 + 2 * L + 1}


# ------------------------------------------------------------------------------------------------ fp64 yardstick
def _relu_mask(z):
    return z > 0


def grads64(x, P, g):
    """fp64 weight gradients [gW0, gb0, gW1, gb1, gW2, gb2] (the shapes of the parameters) from fp64 x [M, 16], P and d loss /
    d sdf g [M].  Written with operators NumPy arrays and torch tensors share, so the GPU test runs it on the device."""
    W0, b0, W1, b1, w2, b2 = P
    z1 = x @ W0.T + b0
    m1 = _relu_mask(z1)
    h1 = z1 * m1
    z2 = h1 @ W1.T + b1
    m2 = _relu_mask(z2)
    dz2 = g[:, None] * w2[0] * m2
    dz1 = (dz2 @ W1) * m1
    return [dz1.T @ x, dz1.sum(0), dz2.T @ h1, dz2.sum(0), (g[:, None] * (z2 * m2)).sum(0)[None, :], g.sum(0).reshape(1)]


def absolute64(x, P, g):
    """The absolute evaluations [A_gW0, ..., A_gb2] and the fp16 floors (F_gW1, F_gW2) of the module docstring, fp64, with the
    operators NumPy and torch share (chunk maxima through amax / max)."""
    W0, b0, W1, b1, w2, b2 = P
    ax, ag = abs(x), abs(g)
    z1 = x @ W0.T + b0
    m1 = _relu_mask(z1)
    a1 = (ax @ abs(W0).T + abs(b0)) * m1                  # a1 of the active units
    m2 = _relu_mask(z1 * m1 @ W1.T + b1)
    a_dh1 = ((ag[:, None] * abs(w2[0]) * m2) @ abs(W1)) * m1
    mg = ag[:, None] * m2                                 # m2[s, j] |dsdf_s|
    A_G = mg.T @ a1                                       # [j, k]
    A_c = mg.sum(0)
    # floor: chunk c contributes n[c, j] max_s |dsdf_s| a1[s, k]
    M = x.shape[0]
    nf = M // KC
    v = ag[:, None] * a1
    cnt = 0.0 * mg + (mg > 0)                             # n: 1.0 where m2 and dsdf != 0
    F = 0.0
    if nf:
        mx = v[:nf * KC].reshape(nf, KC, -1)
        mx = mx.amax(1) if hasattr(mx, "amax") else mx.max(1)
        F = cnt[:nf * KC].reshape(nf, KC, -1).sum(1).T @ mx
    if M > nf * KC:
        tail = v[nf * KC:]
        tail = tail.amax(0) if hasattr(tail, "amax") else tail.max(0)
        F = F + cnt[nf * KC:].sum(0)[:, None] * tail[None, :]
    F_G = 2.0 ** -14 * F
    A = [a_dh1.T @ ax, a_dh1.sum(0), abs(w2[0])[:, None] * A_G, abs(w2[0]) * A_c,
         ((abs(W1) * A_G).sum(1) + abs(b1) * A_c)[None, :], ag.sum(0).reshape(1)]
    F = {"gW1": abs(w2[0])[:, None] * F_G, "gW2": (abs(W1) * F_G).sum(1)[None, :]}
    return A, F


def ratio(got, ref, a, f=0.0):
    """max |got - ref| / (u (a + f)) over the entries with a + f > 0 (0 if none; inf if got is not finite there).  f: the
    gradient's fp16 floor, where it has one."""
    got = np.asarray(got, np.float64)
    a = a + f
    live = a > 0
    if not live.any():
        return 0.0
    err = np.abs(got - ref)[live] / (U * a[live])
    return float("inf") if not np.isfinite(err).all() else float(err.max())


def within_hard(got, ref, a, f, h):
    """bool array: |got - ref| <= u (h a + f) (f = 0 where the gradient has no floor)."""
    return np.abs(np.asarray(got, np.float64) - ref) <= U * (h * a + f)


# ------------------------------------------------------------------------------------------------ inputs
def graded(P, seed=5):
    """P with every W0 row and b0 entry of unit k scaled by 10^U(-8, 0): layer-1 units that span eight decades."""
    s = (10.0 ** np.random.default_rng(seed).uniform(-8, 0, WN)).astype(np.float32)
    out = [p.copy() for p in P]
    out[0] = (P[0] * s[:, None]).astype(np.float32)
    out[1] = (P[1] * s).astype(np.float32)
    return out


def raw_dsdf(kind, M, seed):
    """d loss / d sdf [M] fp32 before the near-zero rows are zeroed: span (10^U(-12, 6) with random signs, every chunk holding
    the whole range), single (one N(0, 1) x 1e-3 value per 64-sample chunk), mapping (N(0, 1) x 1e-6: a loss averaged over
    ~1e6 samples)."""
    rng = np.random.default_rng(seed)
    if kind == "span":
        d = np.sign(rng.standard_normal(M)) * 10.0 ** rng.uniform(-12, 6, M)
    elif kind == "single":
        d = np.zeros(M)
        n = -(-M // KC)
        pos = np.minimum(np.arange(n) * KC + rng.integers(0, KC, n), M - 1)
        d[pos] = rng.standard_normal(n) * 1e-3
    elif kind == "mapping":
        d = rng.standard_normal(M) * 1e-6
    else:
        raise ValueError(kind)
    return d.astype(np.float32)


# ------------------------------------------------------------------------------------------------ the emulator
def _f32(a):
    return np.asarray(a, np.float64).astype(np.float32)


def emulate_gw0(x, dh1, sms=SMS, terms=3):
    """gW0 [256, 16] and gb0 [256] as k_mlp_wg forms them from x [M, 16] and its dh1 [M, 256] (both fp32)."""
    M = x.shape[0]
    lay = layout(M, sms)
    grid, Tn = lay["grid"], lay["T"]
    rows = Tn * grid * TM
    xp = np.zeros((rows, 16), np.float32)
    xp[:M] = x
    dp = np.zeros((rows, WN), np.float32)
    dp[:M] = dh1
    xb = xp.reshape(Tn, grid, 2, 2, 32, 16)               # [it, cta, warpgroup, block, sample, e]; tile = it * grid + cta
    db = dp.reshape(Tn, grid, 2, 2, 32, WN)
    S = np.zeros((grid, 2, 16, WN), np.float32)
    Sb = np.zeros((grid, 2, WN), np.float32)
    for it in range(Tn):
        xh, xl = (a.astype(np.float64) for a in split(xb[it]))
        dh, dl = (a.astype(np.float64) for a in split(db[it]))
        acc = []
        for p, q in [(xh, dh), (xh, dl), (xl, dh)][:terms]:
            c = np.zeros((grid, 2, 2, 16, WN))
            for k in range(4):
                c = trunc32(c + np.swapaxes(p[..., 8 * k:8 * k + 8, :], -1, -2) @ q[..., 8 * k:8 * k + 8, :]).astype(np.float64)
            acc.append(c.astype(np.float32))
        blk = acc[0]
        for a in acc[1:]:
            blk = blk + a
        S = S + blk[:, :, 0]
        S = S + blk[:, :, 1]
        d = db[it].reshape(grid, 2, 8, 2, 4, WN)          # row 8 ks + 4 half + t of the warpgroup's 64
        cs = np.zeros((grid, 2, 4, WN), np.float32)
        for ks in range(8):
            cs = cs + (d[:, :, ks, 0] + d[:, :, ks, 1])
        Sb = Sb + ((cs[:, :, 0] + cs[:, :, 1]) + (cs[:, :, 2] + cs[:, :, 3]))
    gW0 = np.zeros((16, WN), np.float32)
    gb0 = np.zeros(WN, np.float32)
    for c in range(grid):
        gW0 = gW0 + (S[c, 0] + S[c, 1])
        gb0 = gb0 + (Sb[c, 0] + Sb[c, 1])
    return gW0.T.copy(), gb0


def _shift(mx):
    """mlp_tc.cu f16_shift: s with mx 2^s in [2^14, 2^15), 0 for mx = 0, at most 126."""
    e = np.frexp(mx.astype(np.float64))[1]
    return np.where(mx == 0, 0, np.minimum(15 - e, 126)).astype(np.int32)


def emulate_g(x, g, m2, P, sms=SMS, h1_terms=3, g_shift="row", g_lo=True, b1c=True, tot=None):
    """gW1, gb1, gW2, gb2 as k_wgrad_tc forms them from x [M, 16], d loss / d sdf g [M] and relu'(h2) m2 [M, 256] (bool), and
    the splits' G^T sums [nsplit, k, j] (pass them back as tot to rerun the epilogue alone)."""
    W0, b0, W1, b1, w2, b2 = P
    M = x.shape[0]
    lay = layout(M, sms)
    ns, nch, Cn, L = lay["nsplit"], lay["chunks"], lay["C"], lay["L"]
    rows = Cn * ns * KC
    vp = np.zeros((rows, WN), np.float32)
    if tot is None:
        h = mm(x, W0.T, h1_terms) + b0
        vp[:M] = (g[:, None] * np.maximum(h, np.float32(0))).astype(np.float32)
    mp = np.zeros((rows, WN), np.float32)
    mp[:M] = m2
    dp = np.zeros(rows, np.float32)
    dp[:M] = g
    vb = vp.reshape(Cn, ns, KC, WN)                       # chunk = it * ns + split
    mb = mp.reshape(Cn, ns, KC, WN).astype(np.float64)
    run = tot is None
    tot = np.zeros((ns, WN, WN), np.float32) if run else tot    # [split, k, j]
    with np.errstate(over="ignore", invalid="ignore"):
        for it in range(Cn if run else 0):
            vc = np.swapaxes(vb[it], 1, 2)                # [split, k, s]
            mx = np.abs(vc).max(2)
            if g_shift == "chunk":                        # one shift for a warpgroup's 64 rows
                mx = np.repeat(mx.reshape(ns, 4, 64).max(2), 64, axis=1)
            s = _shift(mx) if g_shift != "none" else np.zeros(mx.shape, np.int32)
            vs = (vc * np.ldexp(np.float32(1), s)[..., None]).astype(np.float32)
            hi = vs.astype(np.float16)
            lo = (vs - hi.astype(np.float32)).astype(np.float16) if g_lo else np.zeros_like(hi)
            part = np.zeros((ns, WN, WN))
            for kk in range(KC // 16):
                mk = mb[it][:, 16 * kk:16 * kk + 16]
                for piece in (hi, lo):
                    part = trunc32(part + piece[..., 16 * kk:16 * kk + 16].astype(np.float64) @ mk).astype(np.float64)
            tot = (part * np.ldexp(1.0, -s)[..., None] + tot).astype(np.float32)
    # c: per split and sample half, fp32 chains of 32 samples into fp64
    md = mp * dp[:, None]                                  # m2[s, j] dsdf_s, exact
    cb = md.reshape(Cn, ns, 2, 32, WN)
    sc = np.zeros((Cn, ns, 2, WN), np.float32)
    for r in range(32):
        sc = sc + cb[:, :, :, r]
    c = _f32(sc.astype(np.float64).sum(0).sum(1))          # [split, j]
    W1T = W1.T                                             # [k, j]
    gW1 = np.zeros((WN, WN), np.float32)
    gb1 = np.zeros(WN, np.float32)
    gW2 = np.zeros(WN, np.float32)
    gb2 = np.float32(0)
    half = dp.reshape(Cn, ns, 2, 32).astype(np.float64).sum(axis=(0, 3))   # [split, warp]
    for sp in range(L):
        gW1 = gW1 + (w2[0][:, None] * tot[sp].T)
        gb1 = gb1 + w2[0] * c[sp]
        for j0 in (0, 128):
            for k0 in (0, 128):                            # blockIdx order: tile = (j0 / 128) * 2 + k0 / 128
                t = tot[sp, k0:k0 + 128, j0:j0 + 128].reshape(8, 2, 8, 128)     # [warp, half, g, j]
                w = W1T[k0:k0 + 128, j0:j0 + 128].reshape(8, 2, 8, 128)
                r = _f32(w[:, 0].astype(np.float64) * t[:, 0] + (w[:, 1] * t[:, 1]).astype(np.float64))
                r = r[:, 0::2] + r[:, 1::2]
                r = r[:, 0::2] + r[:, 1::2]
                r = r[:, 0] + r[:, 1]                       # [warp, j]
                acc = np.zeros(128, np.float32)
                for wi in range(8):
                    acc = acc + r[wi]
                if k0 == 0 and b1c:
                    acc = _f32(b1[j0:j0 + 128].astype(np.float64) * c[sp, j0:j0 + 128] + acc)
                gW2[j0:j0 + 128] = gW2[j0:j0 + 128] + acc
        for hw in range(2):
            gb2 = np.float32(gb2 + np.float32(half[sp, hw]))
    return [gW1, gb1, gW2[None, :], np.array([gb2], np.float32)], tot


def emulate(x, g, P, sms=SMS, dh1=None, **mut):
    """All six gradients [gW0, gb0, gW1, gb1, gW2, gb2] as the kernels form them.  m1, m2 and dh1's relu' come from fp64 (equal
    to the kernel's on every row with g != 0, by the near-zero margin); dh1 is decoder_tc_ref.backward's (pass it to reuse)."""
    r = T.reference(x, P)
    m2 = r["z2"] > 0
    if dh1 is None:
        dh1 = T.backward(r["z1"], r["z2"], g, P)[0]
    gW0, gb0 = emulate_gw0(x, dh1, sms, mut.get("gw0_terms", 3))
    (gW1, gb1, gW2, gb2), _ = emulate_g(x, g, m2, P, sms, mut.get("h1_terms", 3), mut.get("g_shift", "row"), mut.get("g_lo", True),
                                        mut.get("b1c", True))
    return [gW0, gb0, gW1, gb1, gW2, gb2]
