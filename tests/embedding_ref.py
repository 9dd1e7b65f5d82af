"""Plain numpy references of the embedding-table path (csrc/gather.cu, csrc/optim.cu): the trilinear gather restated bit for bit in
float32, the gradient scatter, d xyz and the per-frame pose accumulators in float64 together with the sums of absolute terms their
error bounds need, the Adam step (fp32 and bf16 table) in float32 with the kernels' rounding points, and a generator of "dyadic"
inputs on which every fp32 sum of the backward is exact whatever order the atomics and shuffles take.  CPU only."""
import numpy as np

F32 = np.float32


# ------------------------------------------------------------------------------------------------ bf16
def bf16_bits(x):
    """fp32 -> bf16 bits, round to nearest even, NaN kept quiet (nl_f32_to_bf16 in nl_cuda.cuh), in uint32 arithmetic."""
    u = np.ascontiguousarray(x, F32).view(np.uint32)
    nan = (u & np.uint32(0x7fffffff)) > np.uint32(0x7f800000)
    r = (u + np.uint32(0x7fff) + ((u >> np.uint32(16)) & np.uint32(1))) >> np.uint32(16)    # no wrap: finite |x| <= 0x7f7fffff
    q = (u >> np.uint32(16)) | np.uint32(0x40)
    return np.where(nan, q, r).astype(np.uint16)


def bf16_to_f32(bits):
    return (np.asarray(bits, np.uint16).astype(np.uint32) << np.uint32(16)).view(F32)


def bf16_rne(x):
    """fp32 -> nearest bf16, returned as fp32 (nl_round_bf16)."""
    return bf16_to_f32(bf16_bits(x))


# ------------------------------------------------------------------------------------------------ forward
def corner_factors(xyz, vox, centres, voxel_size):
    """The kernel's fp32 trilinear factors: a[M,8,3] (a = p or 1-p per axis, corner k = 4kx + 2ky + kz) and w[M,8] = (ax*ay)*az,
    with p = (x - c) / vs + 0.5 taken in separately rounded fp32 operations (tri_coords / corner_weight)."""
    c = centres[vox].astype(F32)
    p = (xyz.astype(F32) - c) / F32(voxel_size) + F32(0.5)
    a = np.empty((p.shape[0], 8, 3), F32)
    for k in range(8):
        for ax, bit in enumerate((4, 2, 1)):
            a[:, k, ax] = p[:, ax] if k & bit else F32(1.0) - p[:, ax]
    w = (a[:, :, 0] * a[:, :, 1]) * a[:, :, 2]
    return a, w


def _rows(vox, vox2row):
    return vox2row[vox].astype(np.int64)          # [M,8], -1 = vertex without a row


def gather_fwd_f32(xyz, vox, centres, vox2row, emb, voxel_size):
    """k_gather_fwd restated: acc += w_k * f_k in corner order, fp32 mul then fp32 add (nothing contracted); a row id of -1 reads
    as zeros.  emb: the bf16 table as fp32 values [V,16]."""
    _, w = corner_factors(xyz, vox, centres, voxel_size)
    rows = _rows(vox, vox2row)
    acc = np.zeros((xyz.shape[0], emb.shape[1]), F32)
    for k in range(8):
        f = np.where(rows[:, k, None] >= 0, emb[np.maximum(rows[:, k], 0)], F32(0))
        acc = acc + w[:, k, None] * f
    return acc


# ------------------------------------------------------------------------------------------------ backward (float64)
def contributions(vox, vox2row, w, dfeats, round_bf16=True):
    """Per (sample, corner) contributions c = bf16_rne(fp32(g * w_k)) ([M,8,16] fp32) and their row ids [M,8]."""
    c = dfeats.astype(F32)[:, None, :] * w[:, :, None]
    if round_bf16:
        c = bf16_rne(c)
    return c, _rows(vox, vox2row)


def scatter_ref(vox, vox2row, w, dfeats, n_rows, round_bf16=True):
    """d emb: sum over the contributions of every row in float64.  Returns (sum[V,16], n[V,16] = number of contributions,
    abs[V,16] = sum of |c|).  A sample whose corner has no row contributes nothing."""
    c, rows = contributions(vox, vox2row, w, dfeats, round_bf16)
    keep = rows.reshape(-1) >= 0
    r = rows.reshape(-1)[keep]
    c = c.reshape(-1, c.shape[-1])[keep].astype(np.float64)
    s = np.stack([np.bincount(r, weights=c[:, e], minlength=n_rows) for e in range(c.shape[1])], 1)
    a = np.stack([np.bincount(r, weights=np.abs(c[:, e]), minlength=n_rows) for e in range(c.shape[1])], 1)
    n = np.repeat(np.bincount(r, minlength=n_rows)[:, None], c.shape[1], 1)
    return s, n, a


def corner_dots(xyz, vox, centres, vox2row, emb, dfeats, chunk=1 << 15):
    """dot[M,8] = sum_e g_e f_ke (d loss / d w_k) and sum_e |g_e f_ke|, float64, zero where the corner has no row."""
    rows = _rows(vox, vox2row)
    M = len(vox)
    dot, adot = np.zeros((M, 8)), np.zeros((M, 8))
    e64, g64 = emb.astype(np.float64), dfeats.astype(np.float64)
    for s in range(0, M, chunk):
        r = rows[s:s + chunk]
        gf = g64[s:s + chunk, None, :] * np.where(r[:, :, None] >= 0, e64[np.maximum(r, 0)], 0.0)
        dot[s:s + chunk], adot[s:s + chunk] = gf.sum(2), np.abs(gf).sum(2)
    return dot, adot


def dxyz_factors(xyz, vox, centres, voxel_size):
    """[M,3,8] float64: d w_k / d xyz[a] = sign * (product of the other two fp32 factors) / vs."""
    a, _ = corner_factors(xyz, vox, centres, voxel_size)
    a = a.astype(np.float64)
    inv = 1.0 / np.float64(F32(voxel_size))
    out = np.empty((len(vox), 3, 8))
    for ax, (bit, o1, o2) in enumerate(((4, 1, 2), (2, 0, 2), (1, 0, 1))):
        sign = np.array([1.0 if k & bit else -1.0 for k in range(8)])
        out[:, ax] = sign[None, :] * a[:, :, o1] * a[:, :, o2] * inv
    return out


def dxyz_ref(xyz, vox, centres, vox2row, emb, voxel_size, dfeats):
    """(dxyz[M,3], sum of |term|[M,3]) in float64, terms g_e f_ke d w_k / d xyz over the corners k with a row and e = 0..15."""
    dot, adot = corner_dots(xyz, vox, centres, vox2row, emb, dfeats)
    fac = dxyz_factors(xyz, vox, centres, voxel_size)
    return (fac * dot[:, None, :]).sum(2), (np.abs(fac) * adot[:, None, :]).sum(2)


def pose_terms(dxyz, s_ray, s_depth, dir_local):
    """Per-sample pose terms [M,12] = (g, g[a] * depth * d_local[b]) in float64 from the float64 d xyz g."""
    l = dir_local.astype(np.float64)[s_ray] * s_depth.astype(np.float64)[:, None]
    return np.concatenate([dxyz, (dxyz[:, :, None] * l[:, None, :]).reshape(-1, 9)], 1), l


def pose_acc_ref(dxyz, dxyz_abs, s_ray, s_depth, dir_local, ray_frame, n_frames):
    """acc[f] = (dL/dt[3], dL/dR[3x3] row-major), dL/dR[a][b] = sum g[a] * depth * d_local[b] over the samples of frame
    f = ray_frame[s_ray[i]] (frame 0 for every sample when ray_frame is None).  Returns (acc[F,12], sum of |term|[F,12]), where a
    sample's |term| for dL/dt[a] is the sum of |d xyz terms| and for dL/dR[a][b] that times |depth * d_local[b]|."""
    v, l = pose_terms(dxyz, s_ray, s_depth, dir_local)
    va = np.concatenate([dxyz_abs, (dxyz_abs[:, :, None] * np.abs(l)[:, None, :]).reshape(-1, 9)], 1)
    fr = np.zeros(len(s_ray), np.int64) if ray_frame is None else ray_frame[s_ray].astype(np.int64)
    acc = np.stack([np.bincount(fr, weights=v[:, c], minlength=n_frames) for c in range(12)], 1)
    aab = np.stack([np.bincount(fr, weights=va[:, c], minlength=n_frames) for c in range(12)], 1)
    return acc, aab


def gamma(k):
    """Higham's gamma_k = k u / (1 - k u), u = 2^-24: the bound on |prod (1 + d_i)^(+-1) - 1| over k fp32 roundings."""
    k = np.asarray(k, np.float64)
    u = 2.0 ** -24
    return k * u / (1 - k * u)


# ------------------------------------------------------------------------------------------------ Adam
def adam_consts(lr, beta1, beta2, eps, t):
    """The kernel constants as nl_adam_f32 / nl_adam_bf16 form them on the host: double arithmetic, then one cast to float."""
    bc1, bc2 = 1.0 - beta1 ** t, 1.0 - beta2 ** t
    return F32(1.0 - beta1), F32(beta2), F32(1.0 - beta2), F32(eps), F32(lr / bc1), F32(np.sqrt(bc2))


def adam_step(p, g, m, v, lr, beta1, beta2, eps, t, bf16):
    """One Adam step in numpy float32, the arithmetic of optim.cu: m = m + w1 (g - m); v = v b2; v = v + (w2 g) g;
    d = sqrt(v) / bc2_sqrt + eps; p = p + (-step_size) (m / d).  bf16: p, m, v are bf16 values (given as fp32), the fp32 gradient
    is rounded to bf16 first and every line above rounds its result to bf16, as k_adam_bf16 does.  Returns (p, m, v) fp32."""
    w1, b2, w2, e, step_size, bc2_sqrt = adam_consts(lr, beta1, beta2, eps, t)
    r = bf16_rne if bf16 else (lambda x: x)
    p, g, m, v = (np.asarray(x, F32) for x in (p, g, m, v))
    g = r(g)
    m = r(m + w1 * (g - m))
    v = r(v * b2)
    v = r(v + (w2 * g) * g)
    d = r(np.sqrt(v))
    d = r(d / bc2_sqrt)
    d = r(d + e)
    p = r(p + (-step_size) * (m / d))
    return p, m, v


# ------------------------------------------------------------------------------------------------ dyadic inputs
def grid_bits(x):
    """Smallest q >= 0 such that every element of x (float64) is a multiple of 2^-q."""
    x = np.abs(np.asarray(x, np.float64)).ravel()
    x = x[x != 0]
    q = 0
    while x.size and not np.all(np.ldexp(x, q) == np.floor(np.ldexp(x, q))):
        q += 1
        assert q < 1100
    return q


def exact_margin(terms, axis):
    """max over outputs of (sum of |terms| along `axis`) * 2^q / 2^24, q = grid_bits(terms).  Below 1, every term and every partial
    sum of any subset is a multiple of 2^-q below 2^(24-q): each is an fp32 number, so fp32 addition in any order or tree is exact."""
    terms = np.asarray(terms, np.float64)
    if not np.any(terms):
        return 0.0
    return float(np.abs(terms).sum(axis).max() * 2.0 ** (grid_bits(terms) - 24))


def dyadic_problem(rng, vox, n_vox, n_rows, voxel_size=0.5, g_levels=3, f_levels=3, g_density=1.0, empty_vox=(), holes=0.05):
    """Inputs of the backward on which every fp32 operation of k_gather_bwd is exact:
    - voxel_size a power of two and centres on its grid, so p = (x - c) / vs + 0.5 is exact and lies on a 1/8 grid (faces and
      corners included): a, w_k are multiples of 2^-3 and 2^-9;
    - embedding values k/8 and dfeats k/16 with |k| <= f_levels / g_levels (dfeats zero with probability 1 - g_density);
    - dir_local in {0, +-1/2} and depths in {1/2, 1}, so that depth * d_local and its products with d xyz are exact and the pose
      sums of a frame stay exact over ~10^4 samples.
    vox: voxel id per sample.  Voxels in `empty_vox` have no row at any corner; elsewhere a corner has no row with probability
    `holes`.  Row ids are shared between voxels.  Returns a dict of numpy arrays (s_ray = sample index, one sample per ray)."""
    vox = np.asarray(vox, np.int32)
    M = len(vox)
    vs = F32(voxel_size)
    assert np.log2(vs) == np.round(np.log2(vs))
    centres = (rng.integers(-16, 17, size=(n_vox, 3)) * vs).astype(F32)
    vox2row = rng.integers(0, n_rows, size=(n_vox, 8)).astype(np.int32)
    vox2row[rng.random((n_vox, 8)) < holes] = -1
    vox2row[list(empty_vox)] = -1
    j = rng.integers(0, 9, size=(M, 3))
    xyz = (centres[vox] + (j - 4) * (vs / 8)).astype(F32)
    emb = (rng.integers(-f_levels, f_levels + 1, size=(n_rows, 16)) / 8.0).astype(F32)
    g = (rng.integers(-g_levels, g_levels + 1, size=(M, 16)) / 16.0).astype(F32)
    g[rng.random(M) >= g_density] = 0
    dirs = (rng.integers(-1, 2, size=(M, 3)) / 2.0).astype(F32)
    depth = (2.0 ** rng.integers(-1, 1, size=M)).astype(F32)
    return dict(xyz=xyz, vox=vox, centres=centres, vox2row=vox2row, emb=emb, voxel_size=float(vs), dfeats=g,
                s_ray=np.arange(M, dtype=np.int32), s_depth=depth, dir_local=dirs, n_rows=n_rows)


def dyadic_margins(P, layouts=((None, 1),)):
    """Margins (exact below 1, see exact_margin) of every fp32 sum the backward forms on problem P: the 16-term dot products, d xyz
    per axis, the rows' sums of contributions and the frames' pose sums for each (ray_frame or None, n_frames) of `layouts`.  The grids are bounded from above by the grids of the
    factors (a product of multiples of 2^-q1 and 2^-q2 is a multiple of 2^-(q1+q2); bf16 rounding of such a product keeps it one)
    or taken from the terms themselves (d xyz per corner, pose per sample), which are exact in float64.
    All below 1: the kernel's results do not depend on the order of its additions and equal the float64 reference."""
    a, w = corner_factors(P["xyz"], P["vox"], P["centres"], P["voxel_size"])
    qg, qf, qa = grid_bits(P["dfeats"]), grid_bits(P["emb"]), grid_bits(a)
    qi = grid_bits(1.0 / np.float64(P["voxel_size"]))
    dot, adot = corner_dots(P["xyz"], P["vox"], P["centres"], P["vox2row"], P["emb"], P["dfeats"])
    d, da = dxyz_ref(P["xyz"], P["vox"], P["centres"], P["vox2row"], P["emb"], P["voxel_size"], P["dfeats"])
    fac = dxyz_factors(P["xyz"], P["vox"], P["centres"], P["voxel_size"])
    qt = max(grid_bits(fac[s:s + 4096] * dot[s:s + 4096, None, :]) for s in range(0, len(dot), 4096))
    out = {"dot": float(adot.max() * 2.0 ** (qg + qf - 24)), "dxyz": float(da.max() * 2.0 ** (qt - 24))}
    _, _, s = scatter_ref(P["vox"], P["vox2row"], w, P["dfeats"], P["n_rows"])
    out["grad_emb"] = float(s.max() * 2.0 ** (qg + 3 * qa - 24))
    if layouts:
        v, l = pose_terms(d, P["s_ray"], P["s_depth"], P["dir_local"])
        out["depth_dir"] = float(np.abs(l).max() * 2.0 ** (grid_bits(l) - 24))
        qv = grid_bits(v)
        out["pose"] = 0.0
        for ray_frame, n_frames in layouts:
            fr = np.zeros(len(v), np.int64) if ray_frame is None else ray_frame[P["s_ray"]].astype(np.int64)
            s = np.stack([np.bincount(fr, weights=np.abs(v[:, k]), minlength=n_frames) for k in range(12)], 1)
            out["pose"] = max(out["pose"], float(s.max() * 2.0 ** (qv - 24)))
    return out
