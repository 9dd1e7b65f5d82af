"""Plain numpy references of the tail of an optimisation iteration (csrc/pose.cu, csrc/loss.cuh and the control kernels of
csrc/render.cu): the SE(3) map, ray generation and pose Jacobian in float64 with the per-entry error bounds of the fp32 kernels,
an fp32 emulation of the Jacobian kernel (with the mutants its bar has to reject), the loss constants and read-out in float64 and
as an fp32 emulation that rounds where the kernels round, and the iteration-control fold written from the header's contract
(include/nerfloam_b200.h sections 3b and 8).  The Adam step is embedding_ref.adam_step.  CPU only.

Error bounds (first order in u = 2^-24; every bound is finally multiplied by SLACK to cover the second-order terms):
* theta^ = sqrtf(w0*w0 + w1*w1 + w2*w2) is one of the six values theta_candidates() lists (contracted into FMAs or not), and
  A, B and their derivatives move exactly by P(theta^) - P(theta) for the worst of them.
* Each polynomial term (-1)^i powf(theta^, 2i) / (float)den_i: POWF_ULP ulp <= 2 POWF_ULP u relative for powf (CUDA C++
  Programming Guide, appendix "Mathematical Functions", single-precision table: powf(x, y) 4 ulp, full range; the build does not
  use -use_fast_math), u for the denominator's cast and u for the division; term 0 is exactly 1.  The fp32 sum of the eleven terms
  in order adds u |S_k| per partial sum S_k.
* The derivatives are summed in double and cast once: u |A'(theta^)|.
* Products and sums of the matrix expressions: u per rounding of each product and partial sum (and 2^-150 absolute per product,
  for the products of w ~ 1e-20 that land in the subnormal range), wherever nvcc contracts a
  multiply-add into an FMA (the build does not pass -fmad=false, so it may); W's entries and E_i W, W E_i are exact."""
from fractions import Fraction
from math import factorial

import numpy as np

import embedding_ref as E

F32 = np.float32
U = 2.0 ** -24
POWF_ULP = 4
SLACK = 1.01
NT = 11                                           # terms of the reference's Taylor polynomials (se3pose.py, i = 0..10)
ETA = 2.0 ** -150                                 # absolute error of a product rounded into the subnormal range
DEN_A = np.array([float(factorial(2 * i + 1)) for i in range(NT)])
DEN_B = np.array([float(factorial(2 * i + 2)) for i in range(NT)])
SGN = np.array([(-1.0) ** i for i in range(NT)])
I2 = 2.0 * np.arange(NT)


# ------------------------------------------------------------------------------------------------ polynomials
def taylor_AB(theta):
    """A, B (se3pose.py's 11-term polynomials), their theta-derivatives and the sums of |term| of each, float64, elementwise over
    theta (any shape).  Returns a dict with A, B, dA, dB, aA, aB, adA, adB."""
    th = np.asarray(theta, np.float64)[..., None]
    p = th ** I2                                                        # theta^(2i); 0^0 = 1
    dp = np.where(I2 > 0, I2 * th ** np.maximum(I2 - 1, 0), 0.0)        # d theta^(2i) / d theta
    tA, tB, dA, dB = SGN * p / DEN_A, SGN * p / DEN_B, SGN * dp / DEN_A, SGN * dp / DEN_B
    return dict(A=tA.sum(-1), B=tB.sum(-1), dA=dA.sum(-1), dB=dB.sum(-1), aA=np.abs(tA).sum(-1), aB=np.abs(tB).sum(-1),
                adA=np.abs(dA).sum(-1), adB=np.abs(dB).sum(-1))


def f32_round(x):
    """A Fraction (or int) rounded once to the nearest fp32, ties to even (float(x) first would round twice)."""
    x = Fraction(x)
    c = F32(float(x))
    best = None
    for y in (np.nextafter(c, F32(-np.inf)), c, np.nextafter(c, F32(np.inf))):
        if not np.isfinite(y):
            continue
        d = abs(Fraction(float(y)) - x)
        if best is None or d < best[0] or (d == best[0] and int(np.asarray(y).view(np.uint32)) % 2 == 0):
            best = (d, y)
    return F32(best[1])


def fma32(a, b, c):
    """fmaf: a*b + c rounded once to fp32."""
    return f32_round(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def theta_candidates(w):
    """[..., 6] float64: every value sqrtf(w0*w0 + w1*w1 + w2*w2) can take in the kernels for fp32 w, one per way nvcc may
    evaluate the sum (w0*w0 rounded; the first addition fused with either product or not; the second fused or not).  sqrtf is
    correctly rounded (the build keeps -prec-sqrt at its default)."""
    w = np.asarray(w, F32)
    out = np.empty(w.shape[:-1] + (6,))
    for idx in np.ndindex(w.shape[:-1]):
        a, b, c = (F32(x) for x in w[idx])
        with np.errstate(under="ignore"):
            aa, bb, cc = F32(a * a), F32(b * b), F32(c * c)
            firsts = (F32(aa + bb), fma32(b, b, aa), fma32(a, a, bb))
            sums = [F32(s + cc) for s in firsts] + [fma32(c, c, s) for s in firsts]
        out[idx] = [float(np.sqrt(F32(s), dtype=F32)) for s in sums]
    return out


def _theta(w):
    """(theta, theta^ candidates, |theta^ - theta| max) for fp32 w [..., 3]."""
    th = np.linalg.norm(np.asarray(w, np.float64), axis=-1)
    c = theta_candidates(w)
    return th, c, np.abs(c - th[..., None]).max(-1)


def _poly(theta, den):
    th = np.asarray(theta, np.float64)[..., None]
    return (SGN * th ** I2 / den).sum(-1), (np.where(I2 > 0, SGN * I2 * th ** np.maximum(I2 - 1, 0) / den, 0.0)).sum(-1)


def _poly_err(w, den):
    """Bounds on |kernel value - exact value at theta| of P = sum_i (-1)^i theta^(2i) / den_i (fp32 term by term, see the module
    doc) and of its derivative (double, cast once), for fp32 w [..., 3].  The move from theta to the kernel's theta^ is taken
    exactly: max over the candidates of |P(theta^) - P(theta)| (float64, 2^-50 of the sum of |terms| for its roundings)."""
    th, cand, eth = _theta(w)
    thm = np.maximum(th, cand.max(-1))[..., None]
    t = SGN * thm ** I2 / den
    dt = np.where(I2 > 0, SGN * I2 * thm ** np.maximum(I2 - 1, 0) / den, 0.0)
    p0, d0 = _poly(th, den)
    pc, dc = _poly(cand, den)
    move = np.abs(pc - p0[..., None]).max(-1) + 2.0 ** -50 * np.abs(t).sum(-1)
    dmove = np.abs(dc - d0[..., None]).max(-1) + 2.0 ** -50 * np.abs(dt).sum(-1)
    term = np.where(I2 > 0, (2 * POWF_ULP + 2) * U * np.abs(t), 0.0).sum(-1)
    partial = U * np.abs(np.cumsum(t, -1)[..., 1:]).sum(-1)
    return term + partial + move, U * np.abs(dc).max(-1) + dmove


# ------------------------------------------------------------------------------------------------ rotation
def skew(w):
    w = np.asarray(w, np.float64)
    z = np.zeros(w.shape[:-1])
    return np.stack([np.stack([z, -w[..., 2], w[..., 1]], -1), np.stack([w[..., 2], z, -w[..., 0]], -1),
                     np.stack([-w[..., 1], w[..., 0], z], -1)], -2)


def _abs_mm(a, b):
    return np.abs(a) @ np.abs(b)


def rotation(w):
    """R = I + A [w]x + B [w]x^2 in float64 for w [..., 3], and the per-entry sum of |terms| 1[diag] + aA |W| + aB (|W| |W|)."""
    w = np.asarray(w, np.float64)
    W = skew(w)
    p = taylor_AB(np.linalg.norm(w, axis=-1))
    A, B = p["A"][..., None, None], p["B"][..., None, None]
    eye = np.eye(3)
    R = eye + A * W + B * (W @ W)
    a = eye + p["aA"][..., None, None] * np.abs(W) + p["aB"][..., None, None] * _abs_mm(W, W)
    return R, a


def rotation_bar(w):
    """Per-entry bound [..., 3, 3] on |R (nl_pose_matrices) - rotation(w)| for fp32 w."""
    w = np.asarray(w, np.float64)
    W = skew(w)
    p = taylor_AB(np.linalg.norm(w, axis=-1))
    eA, _ = _poly_err(w, DEN_A)
    eB, _ = _poly_err(w, DEN_B)
    ex = lambda x: np.asarray(x)[..., None, None]
    AW, BW2, W2a = np.abs(ex(p["A"]) * W), np.abs(ex(p["B"])) * _abs_mm(W, W), _abs_mm(W, W)
    R, _ = rotation(w)
    prop = ex(eA) * np.abs(W) + ex(eB) * W2a + np.abs(ex(p["B"])) * 3 * U * W2a     # A, B and the fp32 W^2 (3 roundings)
    rnd = U * (AW + BW2 + np.abs(np.eye(3) + ex(p["A"]) * W) + np.abs(R)) + 8 * ETA   # two products, two sums (+ W^2's three products)
    return SLACK * (prop + rnd)


# ------------------------------------------------------------------------------------------------ Jacobian
GEN = np.zeros((3, 3, 3))
GEN[0, 1, 2], GEN[0, 2, 1] = -1, 1                  # E_0 = [e_x]x  (pose.cu: E[5] = -1, E[7] = 1)
GEN[1, 0, 2], GEN[1, 2, 0] = 1, -1
GEN[2, 0, 1], GEN[2, 1, 0] = -1, 1


def _dR_parts(w):
    """The four terms of dR/dw_i (i = 0..2) in float64: T1 = A' theta'_i W, T2 = A E_i, T3 = B' theta'_i W^2, T4 = B (E_i W + W E_i),
    each [..., 3(i), 3, 3], with theta'_i = w_i / theta (0 at theta = 0, torch's norm backward)."""
    w = np.asarray(w, np.float64)
    W = skew(w)[..., None, :, :]
    th = np.linalg.norm(w, axis=-1)
    p = taylor_AB(th)
    with np.errstate(invalid="ignore", divide="ignore"):
        dth = np.where(th[..., None] > 0, w / th[..., None], 0.0)[..., None, None]
    ex = lambda x: np.asarray(x)[..., None, None, None]
    EW = GEN @ W + W @ GEN
    return (ex(p["dA"]) * dth * W, ex(p["A"]) * GEN, ex(p["dB"]) * dth * (W @ W), ex(p["B"]) * EW), dth, W, EW, p, th


def pose_grad(w, acc):
    """grad6 = [dL/dt, dL/dw] of acc = (dL/dt[3], dL/dR[3][3] row-major) for w [..., 3], acc [..., 12], float64: dL/dw_i =
    sum G o dR/dw_i; dL/dt = acc[:3] passed through.  Returns (grad6 [..., 6], sum of |terms| [..., 6]), the polynomials expanded
    into their terms."""
    T, dth, W, EW, p, _ = _dR_parts(w)
    G = np.asarray(acc, np.float64)[..., None, 3:].reshape(np.shape(acc)[:-1] + (1, 3, 3))
    dR = sum(T)
    ex = lambda x: np.asarray(x)[..., None, None, None]
    aR = (ex(p["adA"]) * np.abs(dth) * np.abs(W) + ex(p["aA"]) * np.abs(GEN) + ex(p["adB"]) * np.abs(dth) * _abs_mm(W, W)
          + ex(p["aB"]) * (_abs_mm(GEN, W) + _abs_mm(W, GEN)))
    g = (G * dR).sum((-1, -2))
    a = (np.abs(G) * aR).sum((-1, -2))
    acc = np.asarray(acc, np.float64)
    return np.concatenate([acc[..., :3], g], -1), np.concatenate([np.abs(acc[..., :3]), a], -1)


def pose_grad_bar(w, acc):
    """Per-output bound [..., 3] on |dL/dw (nl_pose_grad) - pose_grad(w, acc)| for fp32 w and acc (dL/dt is exact)."""
    (T1, T2, T3, T4), dth, W, EW, p, th = _dR_parts(w)
    eA, edA = _poly_err(w, DEN_A)
    eB, edB = _poly_err(w, DEN_B)
    ex = lambda x: np.asarray(x)[..., None, None, None]
    _, cand, _ = _theta(w)
    w = np.asarray(w, np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        adth = np.abs(np.where(th[..., None] > 0, w / th[..., None], 0.0))
        # theta' = w_i / theta^ (0 where theta^ = 0): exact move over the candidates, and u for the division
        dc = np.where(cand[..., None, :] > 0, w[..., :, None] / cand[..., None, :], 0.0)
        edth = np.abs(dc - adth[..., None] * np.sign(w)[..., None]).max(-1) + U * np.abs(dc).max(-1)
    edth = edth[..., None, None]
    adth = adth[..., None, None]
    W2a = np.abs(W) @ np.abs(W)
    # propagated errors of A', theta', A, B', B and the fp32 W^2 / E W + W E
    prop = ((ex(edA) * adth + np.abs(ex(p["dA"])) * edth) * np.abs(W) + ex(eA) * np.abs(GEN)
            + (ex(edB) * adth + np.abs(ex(p["dB"])) * edth) * W2a + np.abs(ex(p["dB"])) * adth * 3 * U * W2a
            + ex(eB) * np.abs(EW) + np.abs(ex(p["B"])) * U * np.abs(EW))
    a = [np.abs(t) for t in (T1, T2, T3, T4)]
    # roundings: A' theta' (1), * W (1), B' theta' (1), * W^2 (1), A E (exact), B * EW (1), three partial sums
    rnd = U * (2 * a[0] + 2 * a[2] + a[3] + np.abs(T1 + T2) + np.abs(T1 + T2 + T3) + np.abs(T1 + T2 + T3 + T4))
    e_dR = prop + rnd + 16 * ETA                                      # products rounded into the subnormal range (w ~ 1e-20)
    G = np.asarray(acc, np.float64)[..., None, 3:].reshape(np.shape(acc)[:-1] + (1, 3, 3))
    dR = T1 + T2 + T3 + T4
    prod = (G * dR).reshape(dR.shape[:-2] + (9,))
    run = np.abs(np.cumsum(prod, -1)) * (prod != 0)                   # g += G * dR: a partial sum is rounded where a term enters
    e_g = (np.abs(G) * e_dR).sum((-1, -2)) + U * (np.abs(prod).sum(-1) + run.sum(-1)) + 9 * ETA
    return SLACK * e_g


# ------------------------------------------------------------------------------------------------ fp32 emulation of pose_grad_warp
def _powf(x, n):
    return np.power(F32(x), F32(n), dtype=F32)


def emulate_taylor(theta, f32_derivatives=False):
    """taylor_AB of pose.cu for one fp32 theta: values term by term in fp32, derivatives in double then cast (or, the mutant,
    term by term and summed in fp32)."""
    theta = F32(theta)
    a = b = F32(0)
    da = db = 0.0
    fa = fb = F32(0)
    for i in range(NT):
        xp = _powf(theta, 2 * i)
        sg = F32(SGN[i])
        a = F32(a + F32(F32(sg * xp) / F32(DEN_A[i])))
        b = F32(b + F32(F32(sg * xp) / F32(DEN_B[i])))
        if i > 0:
            dxp = (2 * i) * float(theta) ** (2 * i - 1)
            da += SGN[i] * dxp / DEN_A[i]
            db += SGN[i] * dxp / DEN_B[i]
            d32 = F32(F32(2 * i) * _powf(theta, 2 * i - 1))
            fa = F32(fa + F32(F32(sg * d32) / F32(DEN_A[i])))
            fb = F32(fb + F32(F32(sg * d32) / F32(DEN_B[i])))
    return (a, b, fa, fb) if f32_derivatives else (a, b, F32(da), F32(db))


def emulate_rotation(w):
    """rotation_from_w of pose.cu in numpy fp32, unfused, for one fp32 w [3]: [3, 3]."""
    w = np.asarray(w, F32)
    with np.errstate(under="ignore"):
        theta = np.sqrt(F32(F32(w[0] * w[0]) + F32(w[1] * w[1])) + F32(w[2] * w[2]), dtype=F32)
        A, B, _, _ = emulate_taylor(theta)
        W = skew(w).astype(F32)
        W2 = np.array([[F32(F32(F32(W[r, 0] * W[0, c]) + F32(W[r, 1] * W[1, c])) + F32(W[r, 2] * W[2, c])) for c in range(3)] for r in range(3)], F32)
        return F32(F32(np.eye(3, dtype=F32) + F32(A * W)) + F32(B * W2))


MUTANTS = ("no theta'", "E W only", "E_1 sign flipped", "fp32 derivatives")


def emulate_pose_grad(w, G, mutant=None):
    """dL/dw [3] of pose_grad_warp in numpy fp32, unfused, for one fp32 w [3] and G [3,3]; `mutant` one of MUTANTS or None."""
    w = np.asarray(w, F32)
    G = np.asarray(G, F32).reshape(3, 3)
    with np.errstate(under="ignore"):
        theta = np.sqrt(F32(F32(w[0] * w[0]) + F32(w[1] * w[1])) + F32(w[2] * w[2]), dtype=F32)
    A, B, dA, dB = emulate_taylor(theta, mutant == "fp32 derivatives")
    W = skew(w).astype(F32)
    W2 = np.zeros((3, 3), F32)
    for r in range(3):
        for c in range(3):
            W2[r, c] = F32(F32(F32(W[r, 0] * W[0, c]) + F32(W[r, 1] * W[1, c])) + F32(W[r, 2] * W[2, c]))
    out = np.zeros(3, F32)
    for i in range(3):
        Ei = GEN[i].astype(F32)
        if mutant == "E_1 sign flipped" and i == 1:
            Ei = -Ei
        dth = F32(w[i] / theta) if theta > 0 else F32(0)
        if mutant == "no theta'":
            dth = F32(1)
        g = F32(0)
        for r in range(3):
            for c in range(3):
                EW = F32(F32(F32(Ei[r, 0] * W[0, c]) + F32(Ei[r, 1] * W[1, c])) + F32(Ei[r, 2] * W[2, c]))
                WE = F32(F32(F32(W[r, 0] * Ei[0, c]) + F32(W[r, 1] * Ei[1, c])) + F32(W[r, 2] * Ei[2, c]))
                sym = EW if mutant == "E W only" else F32(EW + WE)
                dR = F32(F32(F32(F32(F32(dA * dth) * W[r, c]) + F32(A * Ei[r, c])) + F32(F32(dB * dth) * W2[r, c])) + F32(B * sym))
                g = F32(g + F32(G[r, c] * dR))
        out[i] = g
    return out


# ------------------------------------------------------------------------------------------------ rays
def rays(dirs, ray_frame, Rt12):
    """(ray_o, ray_d) [R, 3] in float64: d = dirs @ R_f^T, o = t_f, f = ray_frame[r] (0 without), and the bound u (3|x R_a0| +
    2|y R_a1| + |z R_a2|) * SLACK on |ray_d (kernel) - d| (x R_a0 rounded, then two explicit fmaf)."""
    Rt = np.asarray(Rt12, np.float64).reshape(-1, 12)
    f = np.zeros(len(dirs), np.int64) if ray_frame is None else np.asarray(ray_frame, np.int64)
    R = Rt[f, :9].reshape(-1, 3, 3)
    d = np.asarray(dirs, np.float64)
    terms = R * d[:, None, :]
    bar = SLACK * U * (3 * np.abs(terms[..., 0]) + 2 * np.abs(terms[..., 1]) + np.abs(terms[..., 2]))
    return Rt[f, 9:], terms.sum(-1), bar


# ------------------------------------------------------------------------------------------------ loss constants
COUNTERS = ("n_hit_rays", "max_samples", "cnt_fs_valid", "cnt_sdf_valid", "pad_fs_rays", "pad_fs_nsamp", "pad_sdf_rays", "pad_sdf_nsamp",
            "pad_sdf_d2", "pad_sdf_d2_nsamp")


def _fma64(a, b, c):
    """fma in double: a*b + c rounded once."""
    return float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _counts(c):
    S = int(c["max_samples"])
    n_fs = int(c["cnt_fs_valid"]) + int(c["pad_fs_rays"]) * S - int(c["pad_fs_nsamp"])
    n_sdf = int(c["cnt_sdf_valid"]) + int(c["pad_sdf_rays"]) * S - int(c["pad_sdf_nsamp"])
    return S, n_fs, n_sdf


def loss_prepare(c, fs_weight, sdf_weight):
    """loss_prepare_dev (render.cu) in float64 from the counters (a dict with COUNTERS): n_fs, n_sdf, w_fs, w_sdf, g_fs, g_sdf,
    pad_fs_sum, pad_sdf_sum (criterion.py's count_nonzero, class weights and mean() denominators)."""
    S, n_fs, n_sdf = _counts(c)
    num = n_fs + n_sdf
    N = int(c["n_hit_rays"]) * S
    w_fs = 1.0 - n_fs / num if num else float("nan")
    w_sdf = 1.0 - n_sdf / num if num else float("nan")
    ok = N > 0 and num > 0
    return dict(n_fs=float(n_fs), n_sdf=float(n_sdf), w_fs=w_fs, w_sdf=w_sdf, g_fs=fs_weight * w_fs / N if ok else 0.0,
                g_sdf=sdf_weight * w_sdf / N if ok else 0.0, pad_fs_sum=float(int(c["pad_fs_rays"]) * S - int(c["pad_fs_nsamp"])),
                pad_sdf_sum=float(c["pad_sdf_d2"]) * S - float(c["pad_sdf_d2_nsamp"]))


def loss_prepare_f32(c, fs_weight, sdf_weight):
    """loss_prepare_dev rounded where it rounds: (float) of the 64-bit counts (round to nearest, also past 2^24), __fadd_rn /
    __fdiv_rn / __fsub_rn, N = (float)(R_hit * S), g = weight * w / N in two fp32 operations, pad_fs_sum = (float) of a 64-bit
    count, pad_sdf_sum = (float)(d2 * S - d2_nsamp) in double.  Returns fp32 values; pad_sdf_sum is a tuple of the values nvcc may
    produce (the double multiply-subtract contracted into one DFMA, or not)."""
    S, n_fs, n_sdf = _counts(c)
    nfs, nsdf = F32(n_fs), F32(n_sdf)
    num = F32(nsdf + nfs)
    with np.errstate(invalid="ignore", divide="ignore"):
        w_fs, w_sdf = F32(F32(1) - F32(nfs / num)), F32(F32(1) - F32(nsdf / num))
        N = F32(int(c["n_hit_rays"]) * S)
        ok = N > 0 and num > 0
        g_fs = F32(F32(F32(fs_weight) * w_fs) / N) if ok else F32(0)
        g_sdf = F32(F32(F32(sdf_weight) * w_sdf) / N) if ok else F32(0)
    d2, d2n = float(c["pad_sdf_d2"]), float(c["pad_sdf_d2_nsamp"])
    pad_sdf = (F32(_fma64(d2, float(S), -d2n)), F32(d2 * float(S) - d2n))
    return dict(n_fs=nfs, n_sdf=nsdf, w_fs=w_fs, w_sdf=w_sdf, g_fs=g_fs, g_sdf=g_sdf, pad_fs_sum=F32(int(c["pad_fs_rays"]) * S - int(c["pad_fs_nsamp"])),
                pad_sdf_sum=pad_sdf)


def loss_finalize(n_hit_rays, max_samples, fs_sum, sdf_sum, pad_fs_sum, pad_sdf_sum, w_fs, w_sdf, fs_weight, sdf_weight):
    """criterion.py's loss from the masked sums in float64: fs_loss = (fs_sum + pad) / N * w_fs, the same for sdf, loss =
    fs_weight fs_loss + sdf_weight sdf_loss.  Returns (fs_loss, sdf_loss, loss)."""
    N = float(int(n_hit_rays) * int(max_samples))
    fs = (float(fs_sum) + float(pad_fs_sum)) / N * float(w_fs)
    sdf = (float(sdf_sum) + float(pad_sdf_sum)) / N * float(w_sdf)
    return fs, sdf, float(fs_weight) * fs + float(sdf_weight) * sdf


def loss_finalize_f32(n_hit_rays, max_samples, fs_sum, sdf_sum, pad_fs_sum, pad_sdf_sum, w_fs, w_sdf, fs_weight, sdf_weight):
    """nl_loss_finalize_dev rounded where it rounds: the quotient in double, cast, times w in fp32.  Returns (fs_loss, sdf_loss,
    losses) where `losses` are the values `fs_weight * fs_loss + sdf_weight * sdf_loss` may take: unfused, or either product
    contracted into an FMA with the other (nvcc may contract; the build leaves -fmad at its default)."""
    N = np.float64(int(n_hit_rays) * int(max_samples))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        fs = F32(F32((np.float64(fs_sum) + np.float64(F32(pad_fs_sum))) / N) * F32(w_fs))
        sdf = F32(F32((np.float64(sdf_sum) + np.float64(F32(pad_sdf_sum))) / N) * F32(w_sdf))
        a, b = F32(fs_weight), F32(sdf_weight)
        if not (np.isfinite(fs) and np.isfinite(sdf)):
            return fs, sdf, (F32(F32(a * fs) + F32(b * sdf)),)
        return fs, sdf, (F32(F32(a * fs) + F32(b * sdf)), fma32(a, fs, F32(b * sdf)), fma32(b, sdf, F32(a * fs)))


# ------------------------------------------------------------------------------------------------ control fold
CTL_ERROR, CTL_SKIPPED, CTL_SKIP_NOW, CTL_ADAM_STEP, CTL_MIN_HIT, CTL_ITERS, CTL_MAX_SAMPLES, CTL_STOPPED, CTL_WORDS = 0, 1, 2, 3, 4, 5, 6, 7, 8
INT32_MAX = 2 ** 31 - 1


def ctl_init():
    """A control block before the first iteration: zero, MIN_HIT = INT32_MAX (header section 8)."""
    c = [0] * CTL_WORDS
    c[CTL_MIN_HIT] = INT32_MAX
    return c


def iter_status(prev, stats):
    """Section 8: fold one iteration's statistics (dict with n_hit_rays, n_samples, error) into a copy of `prev`.  The iteration
    is skipped (render_rays returns None: render_helpers.py:405-409) when R_hit = 0 or error bit 0 is set; a skipped iteration
    does not advance Adam's step."""
    c = list(prev)
    skip = int(stats["n_hit_rays"] <= 0 or bool(stats["error"] & 1))
    c[CTL_ERROR] |= int(stats["error"])
    c[CTL_SKIPPED] += skip
    c[CTL_SKIP_NOW] = skip
    c[CTL_ADAM_STEP] += 1 - skip
    c[CTL_MIN_HIT] = min(c[CTL_MIN_HIT], int(stats["n_hit_rays"]))
    c[CTL_ITERS] += 1
    c[CTL_MAX_SAMPLES] = max(c[CTL_MAX_SAMPLES], int(stats["n_samples"]))
    return c


def iter_status_batch(ctl, totals, stats):
    """Sections 3b and 8 for K problems: problem k is skipped when it was stopped before, or hits nothing (R_hit = 0, error bit 0,
    or no sample); a skip stops it for the rest of the call (render_helpers.py:488-491's `break`) and freezes its Adam step.
    ERROR takes the problem's bit 0 and the call-wide bits 1 and 2 of `totals` (never its bit 0); MAX_SAMPLES the call-wide
    sample count.  Returns the new blocks."""
    out = []
    for c0, s in zip(ctl, stats):
        c = list(c0)
        err = (int(s["error"]) & 1) | (int(totals["error"]) & 6)
        skip = int(bool(c[CTL_STOPPED]) or s["n_hit_rays"] <= 0 or bool(err & 1) or s["n_samples"] <= 0)
        c[CTL_ERROR] |= err
        c[CTL_SKIPPED] += skip
        c[CTL_SKIP_NOW] = skip
        c[CTL_STOPPED] = skip
        c[CTL_ADAM_STEP] += 1 - skip
        c[CTL_MIN_HIT] = min(c[CTL_MIN_HIT], int(s["n_hit_rays"]))
        c[CTL_ITERS] += 1
        c[CTL_MAX_SAMPLES] = max(c[CTL_MAX_SAMPLES], int(totals["n_samples"]))
        out.append(c)
    return out


def scripted_stats(rng, n_iters, K):
    """Per iteration: per-problem statistics (R_hit, S_total, error bit 0 sometimes zero / set) and call-wide totals."""
    out = []
    for _ in range(n_iters):
        ps = []
        for _ in range(K):
            r = rng.random()
            ps.append(dict(n_hit_rays=0 if r < 0.1 else int(rng.integers(1, 2000)), n_samples=0 if 0.1 <= r < 0.15 else int(rng.integers(1, 10 ** 5)),
                           error=int(rng.random() < 0.08) | (int(rng.integers(0, 4)) << 1 if rng.random() < 0.1 else 0)))
        tot = dict(n_hit_rays=sum(s["n_hit_rays"] for s in ps), n_samples=int(rng.integers(0, 10 ** 6)),
                   error=int(rng.integers(0, 8)) if rng.random() < 0.3 else 0)
        out.append((tot, ps))
    return out


# ------------------------------------------------------------------------------------------------ Adam
adam_step = E.adam_step
bf16_bits, bf16_to_f32 = E.bf16_bits, E.bf16_to_f32


# ------------------------------------------------------------------------------------------------ the pose set of the tests
THETAS = (0.0, 1e-20, 1e-23, 1e-7, 1e-3, 0.1, 1.0, 2.0, 3.0, np.pi - 1e-4, np.pi, 3.5, 2 * np.pi)
DIRECTIONS = ((1, 0, 0), (0, -1, 0), (0, 0, 1), (1, 0, 1), (-1, 2, -3), (0.3, -0.8, 0.52))


def pose_set():
    """fp32 poses [n, 6] = [t, w]: every theta of THETAS (1e-20: the squares are subnormal; 1e-23: they underflow to 0, so the
    kernel sees theta = 0 with w != 0) along every direction of DIRECTIONS (axis-aligned, negative components, generic), with
    translations up to 1e3 in size."""
    rng = np.random.default_rng(11)
    out = []
    for th in THETAS:
        for d in DIRECTIONS:
            d = np.asarray(d, np.float64)
            w = d / np.linalg.norm(d) * th
            t = rng.standard_normal(3) * 10.0 ** rng.integers(-2, 4)
            out.append(np.concatenate([t, w]))
    return np.asarray(out, F32)
