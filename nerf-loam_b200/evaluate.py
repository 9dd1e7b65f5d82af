"""Reconstruction evaluation on the GPU: accuracy, completeness, Chamfer distance and F-score of a mesh against a reference
point cloud (csrc/eval.cu, include/nerfloam_b200.h section 11).

Replaces the evaluation protocol of the reference's Readme.md ("Evaluation"), an external script that samples the mesh on the
host and runs a CPU KD-tree in both directions.  Here the mesh samples, the down-sampled clouds and the distances stay on the
device; only a few totals come back to the host.

    m = evaluate.eval_mesh(verts, faces, gt, n_samples=10**6, res=0.05, threshold=0.1, truncation=0.5, seed=0)
    pts = evaluate.sample_surface(verts, faces, n, seed)                  # f32[n,3] CUDA
    vox = evaluate.voxel_down_sample(points, res, origin)                 # f32[m,3] CUDA, centroids in key order
    d = evaluate.nearest_distances(query, target, truncation)             # f32[len(query)] CUDA

Inputs may be numpy arrays or CPU / CUDA tensors; they are uploaded once.  There is no CPU fallback.
"""
import math

import numpy as np
import torch

from . import _capi

KEY_DIM = 1 << _capi.EVAL_KEY_BITS
MAX_RING = 8          # the search cell is at least truncation / MAX_RING: a query visits at most (2 * MAX_RING + 1)^3 cells


# ---- argument checks (host only; they run before anything touches a device) ------------------------------------------------
def _as_tensor(x, name):
    if isinstance(x, np.ndarray):
        return torch.from_numpy(x)
    if isinstance(x, torch.Tensor):
        return x.detach()
    raise ValueError(f"{name} must be a numpy array or a torch tensor, not {type(x).__name__}")


def _check_points(x, name):
    t = _as_tensor(x, name)
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{name} must have shape [N, 3], got {tuple(t.shape)}")
    if t.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"{name} must be float32 or float64, got {t.dtype}")
    if t.shape[0] >= 2**31 - 1:
        raise ValueError(f"{name} has more than 2^31 - 2 rows")
    return t


def _check_faces(x):
    t = _as_tensor(x, "faces")
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"faces must have shape [T, 3], got {tuple(t.shape)}")
    if t.dtype not in (torch.int32, torch.int64):
        raise ValueError(f"faces must be int32 or int64, got {t.dtype}")
    if t.shape[0] == 0:
        raise ValueError("the mesh has no faces")
    if t.shape[0] >= 2**31:
        raise ValueError("faces has more than 2^31 - 1 rows")
    return t


def _positive(v, name):
    try:
        v = float(v)
    except (TypeError, ValueError):
        raise ValueError(f"{name} must be a number") from None
    if not (math.isfinite(v) and v > 0):
        raise ValueError(f"{name} must be finite and > 0, got {v}")
    return v


def _count(n, name, lo=0):
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or not lo <= int(n) < 2**31:
        raise ValueError(f"{name} must be an integer in [{lo}, 2^31), got {n!r}")
    return int(n)


def _seed(seed):
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= int(seed) < 2**64:
        raise ValueError(f"seed must be an integer in [0, 2^64), got {seed!r}")
    return int(seed)


def _device(*ts):
    for t in ts:
        if t.is_cuda:
            return t.device
    if not torch.cuda.is_available():
        raise RuntimeError("reconstruction evaluation runs on the GPU only (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


# ---- device steps ---------------------------------------------------------------------------------------------------------
def _ws(nbytes, what, dev):
    if nbytes < 0:
        _capi.check(int(nbytes), what)
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)


def _bounds(pts):
    """(f32[6] min / max of the finite rows, i64[1] non-finite rows), on the device, no host read."""
    b = torch.empty(6, dtype=torch.float32, device=pts.device)
    nf = torch.empty(1, dtype=torch.int64, device=pts.device)
    _capi.check(_capi.lib().nl_eval_bounds(pts.shape[0], _capi.ptr(pts), _capi.ptr(b), _capi.ptr(nf), _capi.stream_ptr()), "nl_eval_bounds")
    return b, nf


def _surface(V, F):
    """Areas and their prefix sum in a workspace; returns (workspace, info f64[2] on the device)."""
    lib, dev = _capi.lib(), V.device
    ws = _ws(lib.nl_eval_surface_workspace_bytes(F.shape[0]), "nl_eval_surface_workspace_bytes", dev)
    info = torch.empty(2, dtype=torch.float64, device=dev)
    _capi.check(lib.nl_eval_surface_prepare(V.shape[0], _capi.ptr(V), F.shape[0], _capi.ptr(F), _capi.ptr(ws), ws.numel(), _capi.ptr(info),
                                            _capi.stream_ptr()), "nl_eval_surface_prepare")
    return ws, info


def _check_surface(nf_verts, info):
    nf, (area, bad) = int(nf_verts.item()), info.tolist()
    if nf:
        raise ValueError(f"verts has {nf} rows with non-finite coordinates")
    if bad > 0:
        raise ValueError("faces index a vertex outside [0, len(verts))")
    if not (math.isfinite(area) and area > 0):
        raise ValueError(f"the mesh's total area is {area}")


def _draw(V, F, ws, n, seed, faces_out=False):
    out = torch.empty((n, 3), dtype=torch.float32, device=V.device)
    fid = torch.empty(n, dtype=torch.int32, device=V.device) if faces_out else None
    _capi.check(_capi.lib().nl_eval_sample_surface(V.shape[0], _capi.ptr(V), F.shape[0], _capi.ptr(F), n, seed, _capi.ptr(ws), ws.numel(),
                                                   _capi.ptr(out) if n else None, _capi.ptr(fid) if n and faces_out else None,
                                                   _capi.stream_ptr()), "nl_eval_sample_surface")
    _capi.LAUNCHES += 1
    return out, fid


def _key_span(lo, hi, origin, res):
    """The largest voxel key coordinate a row in [lo, hi] gets; ValueError below the origin or past NL_EVAL_KEY_BITS."""
    for a in range(3):
        k_lo = math.floor((float(lo[a]) - origin[a]) / res)
        k_hi = math.floor((float(hi[a]) - origin[a]) / res)
        if k_lo < 0:
            raise ValueError(f"points lie below the origin on axis {a} ({float(lo[a])} < {origin[a]})")
        if k_hi >= KEY_DIM:
            raise ValueError(f"the extent on axis {a} is {k_hi + 1} voxels of {res}, more than the 2^{_capi.EVAL_KEY_BITS} the voxel key holds")


def _down_sample(P, res, origin, crop=None):
    """Centroids f32[n,3] (capacity n) and counts i64[3] = (cropped, outside the key range, voxels), on the device."""
    lib, dev, n = _capi.lib(), P.device, P.shape[0]
    ws = _ws(lib.nl_eval_voxel_workspace_bytes(n), "nl_eval_voxel_workspace_bytes", dev)
    out = torch.empty((n, 3), dtype=torch.float32, device=dev)
    counts = torch.empty(3, dtype=torch.int64, device=dev)
    _capi.check(lib.nl_eval_voxel_down_sample(n, _capi.ptr(P), origin[0], origin[1], origin[2], res, _capi.ptr(crop), _capi.ptr(ws), ws.numel(),
                                              _capi.ptr(out), None, _capi.ptr(counts), _capi.stream_ptr()), "nl_eval_voxel_down_sample")
    _capi.LAUNCHES += 1
    return out, counts


def search_cell(lo, hi, n, truncation):
    """Cell side of the nearest-distance grid over n target rows inside [lo, hi]: about one surface sample spacing (2 sqrt(A / n)
    with A the bounding box's three face areas, or (V / n)^(1/3) for a volume), at least truncation / MAX_RING so that a query
    visits a bounded number of cells, and large enough that the box fits the 21-bit cell key.  Returns (cell, max_ring)."""
    ex = [max(float(hi[a]) - float(lo[a]), 0.0) for a in range(3)]
    area = ex[0] * ex[1] + ex[1] * ex[2] + ex[0] * ex[2]
    vol = ex[0] * ex[1] * ex[2]
    h = max(2.0 * math.sqrt(area / n), (vol / n) ** (1.0 / 3.0), truncation / MAX_RING, max(ex) / (KEY_DIM - 2))
    ring = math.ceil(truncation / h)
    while ring * h < truncation:
        ring += 1
    return h, ring


def _nearest(Q, T, truncation, lo, hi):
    """d f32[len(Q)] with T's rows inside the box [lo, hi] (host floats)."""
    lib, dev = _capi.lib(), T.device
    n = T.shape[0]
    truncation = float(np.float32(truncation))          # the value the kernel compares against
    cell, ring = search_cell(lo, hi, n, truncation)
    origin = [float(lo[a]) for a in range(3)]
    ws = _ws(lib.nl_eval_nn_workspace_bytes(n), "nl_eval_nn_workspace_bytes", dev)
    d = torch.empty(Q.shape[0], dtype=torch.float32, device=dev)
    bad = torch.empty(1, dtype=torch.int64, device=dev)
    _capi.check(lib.nl_eval_nearest(Q.shape[0], _capi.ptr(Q) if Q.shape[0] else None, n, _capi.ptr(T), origin[0], origin[1], origin[2], cell, ring,
                                    truncation, _capi.ptr(ws), ws.numel(), _capi.ptr(d) if Q.shape[0] else None, _capi.ptr(bad),
                                    _capi.stream_ptr()), "nl_eval_nearest")
    _capi.LAUNCHES += 1
    return d, bad


def _sums(d, threshold):
    lib = _capi.lib()
    ws = _ws(lib.nl_eval_sums_workspace_bytes(d.shape[0]), "nl_eval_sums_workspace_bytes", d.device)
    out = torch.empty(3, dtype=torch.float64, device=d.device)
    _capi.check(lib.nl_eval_distance_sums(d.shape[0], _capi.ptr(d), threshold, _capi.ptr(ws), ws.numel(), _capi.ptr(out), _capi.stream_ptr()),
                "nl_eval_distance_sums")
    return out


# ---- public API -----------------------------------------------------------------------------------------------------------
@torch.no_grad()
def sample_surface(verts, faces, n, seed=0, return_faces=False):
    """n points uniformly by area on the mesh (verts f32[V,3], faces int[T,3]) -> f32[n,3] on the device (and the triangle of each
    sample, i32[n], with return_faces=True).  Sample i depends only on (seed, i) and the mesh: Philox4x32-10 keyed on the seed picks
    the triangle by inverse CDF over an fp64 prefix sum of the areas (zero-area triangles are never picked) and the point by the
    square-root barycentric formula."""
    V, F = _check_points(verts, "verts"), _check_faces(faces)
    if V.shape[0] == 0:
        raise ValueError("the mesh has no vertices")
    n, seed = _count(n, "n"), _seed(seed)
    dev = _device(V, F)
    V = V.to(device=dev, dtype=torch.float32).contiguous()
    F = F.to(device=dev, dtype=torch.int32).contiguous()
    _, nf = _bounds(V)
    ws, info = _surface(V, F)
    _check_surface(nf, info)
    pts, fid = _draw(V, F, ws, n, seed, return_faces)
    return (pts, fid) if return_faces else pts


@torch.no_grad()
def voxel_down_sample(points, res, origin):
    """Voxel centroids of points f32[N,3] on the grid with the given origin (3 numbers) and side res -> f32[M,3] on the device, in
    key order (x major, z minor).  key = floor((p - origin) / res) per axis in fp64; each centroid is an fp64 sum in the order of a
    stable sort by key, rounded to fp32.  Points below the origin, or an extent past 2^21 voxels, raise ValueError."""
    P = _check_points(points, "points")
    if P.shape[0] == 0:
        raise ValueError("points is empty")
    res = _positive(res, "res")
    o = [float(v) for v in np.asarray(origin, dtype=np.float64).reshape(-1)]
    if len(o) != 3 or not all(math.isfinite(v) for v in o):
        raise ValueError(f"origin must be 3 finite numbers, got {origin!r}")
    dev = _device(P)
    P = P.to(device=dev, dtype=torch.float32).contiguous()
    b, nf = _bounds(P)
    nf, b = int(nf.item()), b.tolist()
    if nf:
        raise ValueError(f"points has {nf} rows with non-finite coordinates")
    _key_span(b[:3], b[3:], o, res)
    out, counts = _down_sample(P, res, o)
    m = int(counts[2].item())
    return out[:m]


@torch.no_grad()
def nearest_distances(query, target, truncation):
    """d[i] = min(truncation, min_j |query_i - target_j|) -> f32[len(query)] on the device, computed in fp32 from the fp32 inputs and
    exact below the truncation (a grid of cells over the target, searched ring by ring; see search_cell for the cell size)."""
    Q, T = _check_points(query, "query"), _check_points(target, "target")
    if T.shape[0] == 0:
        raise ValueError("target is empty")
    truncation = _positive(truncation, "truncation")
    dev = _device(Q, T)
    Q = Q.to(device=dev, dtype=torch.float32).contiguous()
    T = T.to(device=dev, dtype=torch.float32).contiguous()
    bt, nft = _bounds(T)
    _, nfq = _bounds(Q)
    nft, nfq, bt = int(nft.item()), int(nfq.item()), bt.tolist()
    if nft or nfq:
        raise ValueError(f"non-finite coordinates: {nfq} query rows, {nft} target rows")
    d, _ = _nearest(Q, T, truncation, bt[:3], bt[3:])
    return d


@torch.no_grad()
def eval_mesh(verts, faces, gt, n_samples=1_000_000, res=0.05, threshold=0.1, truncation=0.5, seed=0):
    """Accuracy, completeness, Chamfer distance and F-score of a mesh (verts f32[V,3], faces int[T,3], as mesh.extract_mesh returns
    them) against a reference point cloud gt f32[N,3] in the same frame.  The product's meshes are in world coordinates with the
    +2000 m pose offset of frame.POSE_OFFSET, so gt has to carry it too.

    1. n_samples points uniformly by area (sample_surface with `seed`);
    2. samples outside gt's bounding box padded by res are dropped (`n_cropped`);
    3. samples and gt are down-sampled (voxel_down_sample) on one grid with origin min(gt) - res: P and G;
    4. d_acc[i] = min(truncation, dist(P_i, G)), d_comp[j] = min(truncation, dist(G_j, P)) (nearest_distances);
    5. accuracy = mean(d_acc), completeness = mean(d_comp), chamfer_l1 = their mean, chamfer_l2 = sqrt((mean(d_acc^2) +
       mean(d_comp^2)) / 2), precision / recall = 100 * fraction of d_acc / d_comp below threshold, fscore = 2PR / (P + R) (0 when
       both are 0).  Every sum is fp64 in a fixed order: two calls return identical dicts.
    Returns those metrics and the counts n_samples, n_cropped, n_pred (|P|) and n_gt (|G|)."""
    V, F, G = _check_points(verts, "verts"), _check_faces(faces), _check_points(gt, "gt")
    if V.shape[0] == 0:
        raise ValueError("the mesh has no vertices")
    if G.shape[0] == 0:
        raise ValueError("gt is empty")
    n = _count(n_samples, "n_samples", lo=1)
    res, threshold, truncation = _positive(res, "res"), _positive(threshold, "threshold"), _positive(truncation, "truncation")
    seed = _seed(seed)
    dev = _device(V, F, G)
    V = V.to(device=dev, dtype=torch.float32).contiguous()
    F = F.to(device=dev, dtype=torch.int32).contiguous()
    G = G.to(device=dev, dtype=torch.float32).contiguous()
    _, nfv = _bounds(V)
    bg, nfg = _bounds(G)
    ws, info = _surface(V, F)
    nfg, bg = int(nfg.item()), bg.tolist()
    if nfg:
        raise ValueError(f"gt has {nfg} rows with non-finite coordinates")
    _check_surface(nfv, info)
    lo, hi = bg[:3], bg[3:]
    origin = [lo[a] - res for a in range(3)]
    _key_span(origin, [hi[a] + res for a in range(3)], origin, res)
    S, _ = _draw(V, F, ws, n, seed)
    P, cp = _down_sample(S, res, origin, crop=torch.tensor(bg, dtype=torch.float32, device=dev))
    Gd, cg = _down_sample(G, res, origin)
    n_cropped, out_p, n_p, _, out_g, n_g = torch.cat([cp, cg]).tolist()
    if out_p or out_g:
        raise RuntimeError(f"nl_eval_voxel_down_sample: {out_p + out_g} rows outside the key range that the host check admitted")
    if n_p == 0:
        raise ValueError("no mesh sample lies inside the bounding box of gt padded by res")
    P, Gd = P[:n_p], Gd[:n_g]
    d_acc, bad_g = _nearest(P, Gd, truncation, lo, hi)
    d_comp, bad_p = _nearest(Gd, P, truncation, [lo[a] - res for a in range(3)], [hi[a] + res for a in range(3)])
    (sa, sa2, ca), (sc, sc2, cc) = torch.stack([_sums(d_acc, threshold), _sums(d_comp, threshold)]).tolist()
    if int((bad_g + bad_p).item()):
        raise RuntimeError("nl_eval_nearest: down-sampled rows fell outside the search grid's box")
    acc, comp = sa / n_p, sc / n_g
    prec, rec = 100.0 * ca / n_p, 100.0 * cc / n_g
    return {"accuracy": acc, "completeness": comp, "chamfer_l1": 0.5 * (acc + comp), "chamfer_l2": math.sqrt(0.5 * (sa2 / n_p + sc2 / n_g)),
            "precision": prec, "recall": rec, "fscore": 2.0 * prec * rec / (prec + rec) if prec + rec > 0 else 0.0,
            "n_samples": n, "n_cropped": int(n_cropped), "n_pred": int(n_p), "n_gt": int(n_g)}
