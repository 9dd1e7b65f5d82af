"""fp64 restatement of the decoder (16 -> W -> W -> 1, ReLU; nerf-loam_b200/csrc/mlp.cu, lidar.py) and of the loss its training
kernels evaluate in place (mlp.cu k_mlp, criterion.py:92-100).

Everything runs in torch float64 on whatever device the inputs are on, chunked over samples, so that it evaluates the full
776 k-sample case on the GPU.  Parameters are the list (W0 [W,16], b0 [W], W1 [W,W], b1 [W], w2 [1,W], b2 [1]), the order of
DecoderBuffers.params and .grads.

Error scales ("absolute evaluation"): the same network run on |x|, |W| and |b|.  a1 = |x||W0|^T + |b0|, a2 = a1|W1|^T + |b1| and
a_sdf = a2|w2|^T + |b2| bound the magnitude of every term a pre-activation or the output sums, so a dot product of n fp32 terms is
within about n 2^-24 of them.  a_dx is the backward pass run the same way on |g| and |W| (with the fp64 relu' masks)."""
import torch

CHUNK = 1 << 17
U = 2.0 ** -24              # fp32 unit roundoff
NEAR = 1e-4                 # near_zero's relative margin


def params64(dec):
    """The decoder's parameters in fp64, in the order of DecoderBuffers.params."""
    lin = list(dec.pts_linears)
    return [p.detach().double() for p in (lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias, dec.sdf_out.weight, dec.sdf_out.bias)]


def _chunks(n):
    return [(s, min(n, s + CHUNK)) for s in range(0, n, CHUNK)]


def _fwd(x, p):
    W0, b0, W1, b1, w2, b2 = p
    z1 = x @ W0.T + b0
    h1 = z1.clamp_min(0)
    z2 = h1 @ W1.T + b1
    h2 = z2.clamp_min(0)
    return z1, h1, z2, h2, (h2 @ w2.T + b2).reshape(-1)


def forward(x, p, keep=("sdf",)):
    """Chunked fp64 forward.  Returns {name: tensor} for the names in keep, from z1, h1, z2, h2 ([M,W]) and sdf ([M])."""
    M = x.shape[0]
    out = {}
    for s, e in _chunks(M):
        vals = dict(zip(("z1", "h1", "z2", "h2", "sdf"), _fwd(x[s:e].double(), p)))
        for k in keep:
            if k not in out:
                shape = (M,) + tuple(vals[k].shape[1:])
                out[k] = torch.empty(shape, dtype=torch.float64, device=x.device)
            out[k][s:e] = vals[k]
    return out


def absolute(x, p):
    """(a1 [M,W], a2 [M,W], a_sdf [M]) of one chunk: the network run on |x|, |W|, |b| (every term is nonnegative, so the ReLUs
    are identities)."""
    return _fwd(x.double().abs(), [t.abs() for t in p])[0::2]


def near_zero(x, p):
    """bool[M]: rows with a pre-activation within NEAR of zero relative to the absolute sum of its terms: |z1| <= 1e-4 a1 or
    |z2| <= 1e-4 (h1 |W1|^T + |b1|) anywhere (layer 2's terms are those of the computed h1).  Two valid fp32 evaluations may
    disagree on relu' for such a row."""
    W0, b0, W1, b1 = p[:4]
    out = torch.empty(x.shape[0], dtype=torch.bool, device=x.device)
    for s, e in _chunks(x.shape[0]):
        xs = x[s:e].double()
        z1, h1, z2, _, _ = _fwd(xs, p)
        a1 = xs.abs() @ W0.abs().T + b0.abs()
        a2 = h1 @ W1.abs().T + b1.abs()
        out[s:e] = ((z1.abs() <= NEAR * a1).any(dim=1)) | ((z2.abs() <= NEAR * a2).any(dim=1))
    return out


def _bwd(x, g, p, masks=None):
    """One chunk of the backward pass from d loss / d sdf = g: (dx, [gW0, gb0, gW1, gb1, gw2, gb2]).  masks: the relu' masks
    (z1 > 0, z2 > 0) to use; by default the ones of x under p."""
    W0, b0, W1, b1, w2, b2 = p
    z1, h1, z2, h2, _ = _fwd(x, p)
    m1, m2 = (z1 > 0, z2 > 0) if masks is None else masks
    dz2 = g[:, None] * w2[0] * m2
    dz1 = (dz2 @ W1) * m1
    dx = dz1 @ W0
    return dx, [dz1.T @ x, dz1.sum(0), dz2.T @ h1, dz2.sum(0), (g[:, None] * h2).sum(0, keepdim=True), g.sum().reshape(1)], (m1, m2)


def backward(x, g, p, with_abs=False):
    """Chunked fp64 backward from an external g = d loss / d sdf [M].  Returns (dx [M,16], grads) with grads in the order of
    DecoderBuffers.grads; with_abs=True also a_dx [M,16], the same backward on |g|, |W| with the same relu' masks."""
    M = x.shape[0]
    dx = torch.empty((M, 16), dtype=torch.float64, device=x.device)
    a_dx = torch.empty_like(dx) if with_abs else None
    grads = [torch.zeros_like(t) for t in p]
    for s, e in _chunks(M):
        xs, gs = x[s:e].double(), g[s:e].double()
        d, gr, masks = _bwd(xs, gs, p)
        dx[s:e] = d
        for acc, t in zip(grads, gr):
            acc += t
        if with_abs:
            a_dx[s:e] = _bwd(xs.abs(), gs.abs(), [t.abs() for t in p], masks)[0]
    return (dx, grads, a_dx) if with_abs else (dx, grads)


def _errors(sdf, flag, depth, ray, gt_depth, cos, truncation):
    """Per-sample (e_fs, e_sdf) in the dtype of sdf, rounded step by step as the kernel rounds them when sdf is fp32:
    e_fs = sdf - 1; e_sdf = (depth*cos + sdf*trunc) - gt (cos = 1 when absent)."""
    dt = sdf.dtype
    r = ray.long()
    z = depth.to(dt) * (cos[r].to(dt) if cos is not None else 1.0)
    e_fs = sdf - 1.0
    e_sdf = (z + sdf * torch.tensor(truncation, dtype=torch.float32).to(dt).item()) - gt_depth[r].to(dt)
    return e_fs, e_sdf


def loss(sdf, flag, depth, ray, gt_depth, cos, truncation, g_fs, g_sdf):
    """The in-kernel loss (mlp.cu k_mlp, criterion.py:92-100) on sdf [M]:
      flag & 1 (front):    e = sdf - 1,                       adds e^2 to fs_sum,  d loss / d sdf += 2 g_fs e
      flag & 2 (SDF band): e = (depth cos + sdf trunc) - gt,  adds e^2 to sdf_sum, d loss / d sdf += 2 g_sdf trunc e
    g_fs / g_sdf: scalars, or tensors [M] of per-sample constants.  With fp64 sdf everything is fp64.  With the kernel's own fp32
    sdf, e is formed in fp32 with the kernel's roundings and squared and summed in fp64, as the kernel does; only the order of the
    sums differs.  Returns (fs_sum, sdf_sum, dsdf [M] fp64)."""
    fs, sd, dsdf, _ = _loss_terms(sdf, flag, depth, ray, gt_depth, cos, truncation, g_fs, g_sdf)
    return fs, sd, dsdf


def _f32(v):
    return torch.as_tensor(v, dtype=torch.float32).double()


def _loss_terms(sdf, flag, depth, ray, gt_depth, cos, truncation, g_fs, g_sdf):
    """loss() plus the per-sample squared errors (sq_fs, sq_sdf)."""
    e_fs, e_sdf = (e.double() for e in _errors(sdf, flag, depth, ray, gt_depth, cos, truncation))
    trunc = float(_f32(truncation))
    f = flag.long()
    front, band = (f & 1) != 0, (f & 2) != 0
    zero = torch.zeros_like(e_fs)
    sq_fs, sq_sdf = torch.where(front, e_fs * e_fs, zero), torch.where(band, e_sdf * e_sdf, zero)
    gf = g_fs.double() if torch.is_tensor(g_fs) else float(_f32(g_fs))      # the kernel reads them as fp32
    gs = g_sdf.double() if torch.is_tensor(g_sdf) else float(_f32(g_sdf))
    dsdf = torch.where(front, 2.0 * gf * e_fs, zero) + torch.where(band, 2.0 * gs * trunc * e_sdf, zero)
    return float(sq_fs.sum()), float(sq_sdf.sum()), dsdf, (sq_fs, sq_sdf)


def problem_loss(sdf, flag, depth, ray, gt_depth, cos, truncation, rays_per_problem, g_fs, g_sdf):
    """The batched loss (nl_mlp_train_batch): sample m belongs to problem k = ray[m] // rays_per_problem and uses that problem's
    g_fs[k] / g_sdf[k] (sequences of length K).  Returns (fs_sum [K], sdf_sum [K], dsdf [M]) in fp64."""
    K = len(g_fs)
    k = ray.long() // int(rays_per_problem)
    gf = _f32(list(g_fs)).to(sdf.device)
    gs = _f32(list(g_sdf)).to(sdf.device)
    _, _, dsdf, (sq_fs, sq_sdf) = _loss_terms(sdf, flag, depth, ray, gt_depth, cos, truncation, gf[k], gs[k])
    fs = torch.zeros(K, dtype=torch.float64, device=sdf.device).index_add_(0, k, sq_fs)
    sd = torch.zeros(K, dtype=torch.float64, device=sdf.device).index_add_(0, k, sq_sdf)
    return fs, sd, dsdf
