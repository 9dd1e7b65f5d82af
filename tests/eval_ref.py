"""NumPy / SciPy restatement of nerf-loam_b200/evaluate.py (test infrastructure only, like embedding_ref.py): the crop, the voxel
down-sampling and the metrics with the same formulas, and the nearest distances from scipy's cKDTree in float64.  Surface sampling
is not restated: the tests feed the product's samples to eval_samples."""
import math

import numpy as np
from scipy.spatial import cKDTree

KEY_BITS = 21


def voxel_keys(points, res, origin):
    """floor((p - origin) / res) per axis in float64 -> int64[N,3] (the product's key arithmetic)."""
    p = np.asarray(points, np.float32).astype(np.float64)
    return np.floor((p - np.asarray(origin, np.float64)) / float(res)).astype(np.int64)


def voxel_down_sample(points, res, origin):
    """Centroids f32[M,3] in key order and their packed keys u64[M]: a stable sort by key, float64 sums per voxel in that order."""
    p = np.asarray(points, np.float32)
    k = voxel_keys(p, res, origin)
    if (k < 0).any() or (k >= 1 << KEY_BITS).any():
        raise ValueError("key out of range")
    key = (k[:, 0].astype(np.uint64) << np.uint64(2 * KEY_BITS)) | (k[:, 1].astype(np.uint64) << np.uint64(KEY_BITS)) | k[:, 2].astype(np.uint64)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    heads = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    ends = np.r_[heads[1:], len(ks)]
    ps = p[order].astype(np.float64)
    out = np.empty((len(heads), 3), np.float32)
    for r, (b, e) in enumerate(zip(heads, ends)):
        s = np.zeros(3)
        for j in range(b, e):                       # sequential, like the kernel
            s += ps[j]
        out[r] = (s / (e - b)).astype(np.float32)
    return out, ks[heads]


def voxel_down_sample_fast(points, res, origin):
    """voxel_down_sample with np.add.reduceat (for large inputs; its summation order may differ in the last fp64 bits)."""
    p = np.asarray(points, np.float32)
    k = voxel_keys(p, res, origin)
    if (k < 0).any() or (k >= 1 << KEY_BITS).any():
        raise ValueError("key out of range")
    key = (k[:, 0].astype(np.uint64) << np.uint64(2 * KEY_BITS)) | (k[:, 1].astype(np.uint64) << np.uint64(KEY_BITS)) | k[:, 2].astype(np.uint64)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    heads = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    cnt = np.diff(np.r_[heads, len(ks)])
    s = np.add.reduceat(p[order].astype(np.float64), heads, axis=0)
    return (s / cnt[:, None]).astype(np.float32), ks[heads]


def nearest_distances(query, target, truncation):
    """min(truncation, distance to the nearest target row) in float64 (cKDTree on the fp32 inputs widened to float64)."""
    q = np.asarray(query, np.float32).astype(np.float64)
    t = np.asarray(target, np.float32).astype(np.float64)
    if len(q) == 0:
        return np.zeros(0)
    d, _ = cKDTree(t).query(q, k=1, workers=-1)
    return np.minimum(d, truncation)


def nearest_brute(query, target, truncation):
    q = np.asarray(query, np.float64)
    t = np.asarray(target, np.float64)
    d = np.sqrt(((q[:, None, :] - t[None, :, :]) ** 2).sum(-1)).min(1)
    return np.minimum(d, truncation)


def crop(samples, gt, res):
    """The samples inside gt's bounding box padded by res (float64 comparison), and how many were dropped."""
    s = np.asarray(samples, np.float32)
    g = np.asarray(gt, np.float32)
    lo, hi = g.min(0).astype(np.float64) - res, g.max(0).astype(np.float64) + res
    s64 = s.astype(np.float64)
    keep = ((s64 >= lo) & (s64 <= hi)).all(1)
    return s[keep], int((~keep).sum())


def metrics(d_acc, d_comp, threshold):
    acc, comp = float(np.mean(d_acc)), float(np.mean(d_comp))
    prec = 100.0 * float(np.mean(d_acc < threshold))
    rec = 100.0 * float(np.mean(d_comp < threshold))
    return {"accuracy": acc, "completeness": comp, "chamfer_l1": 0.5 * (acc + comp),
            "chamfer_l2": math.sqrt(0.5 * (float(np.mean(d_acc ** 2)) + float(np.mean(d_comp ** 2)))),
            "precision": prec, "recall": rec, "fscore": 2 * prec * rec / (prec + rec) if prec + rec > 0 else 0.0}


def eval_samples(samples, gt, res, threshold, truncation, fast=True):
    """eval_mesh from step 2 on, given the surface samples."""
    g = np.asarray(gt, np.float32)
    kept, n_cropped = crop(samples, g, res)
    origin = g.min(0).astype(np.float64) - res
    ds = voxel_down_sample_fast if fast else voxel_down_sample
    P, _ = ds(kept, res, origin)
    G, _ = ds(g, res, origin)
    d_acc = nearest_distances(P, G, truncation)
    d_comp = nearest_distances(G, P, truncation)
    out = metrics(d_acc, d_comp, threshold)
    out.update(n_samples=len(samples), n_cropped=n_cropped, n_pred=len(P), n_gt=len(G))
    return out, d_acc, d_comp
