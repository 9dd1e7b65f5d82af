"""relocalise_global on a map of about 10^6 leaf voxels: a street (walls 8 m either side, ground between) along a 3.7 km curved
path, anchors every metre along it at the sensor's height, 5 m radius, 1 m lattice, 72 yaws (about 2.7 M placements).  The scan is
taken from the timed scene: points drawn inside the map's voxels within 40 m of a pose halfway along the path (no occlusion), so
stage 1 counts real hits and stages 2 and 3 have a map to score and refine against.  The decoder is untrained, so stage 3's result
means nothing; its time is that of the default relocalise (512 rays, 25 iterations) from 4 seeds.  Per repeat, alternating:
  - the coarse stage's parts with CUDA events: occupied set, cell table, scan points + scorer, selection;
  - score_poses on 65 535 of the same placements (the most one call takes), scaled per placement to the whole lattice (labelled);
  - a whole relocalise_global call, per stage (its own host-clock diagnostics);
  - the NumPy restatement (tests/globalloc_ref.py) on a host subset of placements, which must give the same counts.
Prints one JSON line: card name and power limit (read in the same run), medians and min-max.

    python scripts/time_relocalise_global.py [--repeats 3] [--length 3700] [--subset 2000]
"""
import argparse
import json
import math
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import nerfloam_b200 as nl  # noqa: E402
import globalloc_ref as ref  # noqa: E402
from nerfloam_b200.criterion import Criterion  # noqa: E402
from time_track_batch import _Args, card  # noqa: E402

VS = 0.3


def path(s):
    """xy and heading of the path at arc parameter s (metres, approximately)."""
    x, y = s, 60.0 * np.sin(s / 300.0)
    return x, y, np.arctan2(0.2 * np.cos(s / 300.0), 1.0)


def street_voxels(length):
    s = np.arange(0.0, length, VS)
    x, y, h = path(s)
    nx, ny = -np.sin(h), np.cos(h)
    parts = []
    for u in np.arange(-8.0, 8.0 + 1e-9, VS):                      # ground
        parts.append(np.stack([x + u * nx, y + u * ny, np.full_like(x, -1.73)], 1))
    for side in (-8.0, 8.0):                                        # walls
        for z in np.arange(-1.7, 4.3, VS):
            parts.append(np.stack([x + side * nx, y + side * ny, np.full_like(x, z)], 1))
    w = np.concatenate(parts) + nl.synthetic.POSE_OFFSET
    return np.unique(np.floor(w / VS).astype(np.int32), axis=0)


def street_scan(vox, length, seed=7, per_voxel=3, max_range=40.0):
    """(points f32[n,3] in the sensor frame, pointsCos f32[n], pose f64[4,4]) of a sensor at the path's midpoint: per_voxel points
    drawn uniformly inside every map voxel within max_range; ground voxels get |n.d| as their cosine, the rest 1."""
    rng = np.random.default_rng(seed)
    x, y, h = path(length / 2)
    pose = np.eye(4)
    pose[:2, :2] = [[np.cos(h), -np.sin(h)], [np.sin(h), np.cos(h)]]
    pose[:3, 3] = [x + nl.synthetic.POSE_OFFSET, y + nl.synthetic.POSE_OFFSET, nl.synthetic.POSE_OFFSET]
    c = (vox.astype(np.float64) + 0.5) * VS
    near = np.linalg.norm(c[:, :2] - pose[:2, 3], axis=1) < max_range
    v = np.repeat(vox[near], per_voxel, axis=0).astype(np.float64)
    w = (v + rng.uniform(0.0, 1.0, v.shape)) * VS
    p = (w - pose[:3, 3]) @ pose[:3, :3]
    r = np.linalg.norm(p, axis=1)
    keep = (r > 1.5) & (r < max_range)
    p, v = p[keep], v[keep]
    ground = v[:, 2] == np.floor((nl.synthetic.POSE_OFFSET - 1.73) / VS)
    cos = np.where(ground, np.abs(p[:, 2]) / np.linalg.norm(p, axis=1), 1.0)
    return p.astype(np.float32), cos.astype(np.float32), pose


def stats(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def probes_of(Rt, points):
    """Per subset placement: the points whose voxel lies inside the grid, i.e. the ones that reach a hash probe."""
    _, ok = ref.voxel_keys(Rt, points, VS, 1 << 18)
    return ok.sum(1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--length", type=float, default=3700.0)
    ap.add_argument("--subset", type=int, default=2000, help="placements restated in NumPy")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_relocalise_global.py measures on the GPU; none found")
    dev = torch.device("cuda")
    gpu = card()
    vox = street_voxels(a.length)
    mu = nl.mapping.MapUpdater(VS, device=dev, reserve_nodes=3 * vox.shape[0], reserve_rows=3 * vox.shape[0])
    ms = mu.insert_voxels(torch.from_numpy(vox))
    s = np.arange(0.0, a.length, 1.0)
    x, y, h = path(s)
    anchors = np.tile(np.eye(4), (s.size, 1, 1))
    anchors[:, 0, 0], anchors[:, 0, 1], anchors[:, 1, 0], anchors[:, 1, 1] = np.cos(h), -np.sin(h), np.sin(h), np.cos(h)
    anchors[:, 0, 3], anchors[:, 1, 3] = x + nl.synthetic.POSE_OFFSET, y + nl.synthetic.POSE_OFFSET
    anchors[:, 2, 3] = nl.synthetic.POSE_OFFSET                      # the sensor's height, as street_voxels places the street
    torch.manual_seed(0)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    crit = Criterion(_Args())
    pts, cos, _ = street_scan(vox, a.length)
    frame = nl.frame.LidarFrame(0, torch.from_numpy(pts), torch.from_numpy(cos), nl.se3pose.OptimizablePose(torch.zeros(6)), new_keyframe=True)
    g = nl.globalloc

    def ev():
        return torch.cuda.Event(enable_timing=True)

    def coarse():
        e = [ev() for _ in range(5)]
        e[0].record()
        m = nl.engine.MapState.view(ms.centres, ms.structure, ms.vox2row, ms.emb)          # no cached set
        occ = g.occupied_set(m, VS)
        e[1].record()
        pl = g.placements(anchors, 5.0, 1.0, 72)
        e[2].record()
        p, _ = g.scan_points(frame, 512)
        counts = g.coarse_scores(pl, occ, p)
        e[3].record()
        ids, _ = g.top_placements(counts, 512, 4096)
        e[4].record()
        torch.cuda.synchronize()
        return [e[i].elapsed_time(e[i + 1]) for i in range(4)], pl, occ, p, counts

    def fine(pl, n=65535):
        T = g.placement_matrices(pl, np.linspace(0, pl.n_placements - 1, n).astype(np.int64))
        p6 = nl.score.poses_from_matrices(T).contiguous()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        nl.score_poses(p6, frame, ms, dec, crit, VS, 512, step_size=0.15, max_distance=40.0)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    def whole():
        torch.manual_seed(1)
        r = nl.relocalise_global(frame, ms, dec, crit, VS, anchors=anchors, step_size=0.15, max_distance=40.0, truncation=0.3, max_voxel_hit=20)
        d = r.diagnostics
        return {k: v * 1e3 for k, v in d.times.items()}, int(d.counts[0]), len(d.seeds), r.hit_mask is not None

    coarse(), fine(g.placements(anchors, 5.0, 1.0, 72), 4096), whole()                      # warm-up
    rec = {k: [] for k in ("occupied_ms", "cells_ms", "score_ms", "select_ms", "score_poses_65535_ms", "call_coarse_ms", "call_fine_ms",
                           "call_refine_ms", "numpy_subset_ms")}
    agree = True
    for _ in range(a.repeats):
        parts, pl, occ, p, counts = coarse()
        for k, v in zip(("occupied_ms", "cells_ms", "score_ms", "select_ms"), parts):
            rec[k].append(v)
        rec["score_poses_65535_ms"].append(fine(pl))
        w, top_count, n_seeds, hit = whole()
        for k in ("coarse", "fine", "refine"):
            rec[f"call_{k}_ms"].append(w[k])
        sub = np.linspace(0, pl.n_placements - 1, a.subset).astype(np.int64)
        T = g.placement_matrices(pl, sub).cpu().numpy()
        Rt = np.concatenate([T[:, :3, :3].reshape(-1, 9), T[:, :3, 3]], 1)
        keys = occ.slots.cpu().numpy()
        keys = np.sort(keys[keys != -1])
        t0 = time.perf_counter()
        want = ref.counts(Rt, p.cpu().numpy(), keys, VS, 1 << 18)
        rec["numpy_subset_ms"].append((time.perf_counter() - t0) * 1e3)
        agree &= bool(np.array_equal(counts.cpu().numpy()[sub], want))
        nonzero_share = float((counts > 0).float().mean())
        probes = int(probes_of(Rt, p.cpu().numpy()).sum())
    P, M = pl.n_placements, 512
    score_ms = statistics.median(rec["score_ms"])
    out = {"bench": "relocalise_global", "gpu": gpu, "leaf_voxels": occ.n_leaves, "set_slots": occ.slots.numel(), "anchors": int(s.size),
           "cells": pl.n_cells, "placements": P, "points": M, "repeats": a.repeats,
           **{k: stats(v) for k, v in rec.items()},
           "scorer_placements_per_s": P / (score_ms * 1e-3), "scorer_lookups_per_s": P * M / (score_ms * 1e-3),
           "score_poses_scaled_to_all_placements_s": statistics.median(rec["score_poses_65535_ms"]) * 1e-3 * P / 65535,
           "numpy_subset_placements": a.subset,
           "numpy_scaled_to_all_placements_s": statistics.median(rec["numpy_subset_ms"]) * 1e-3 * P / a.subset,
           "numpy_agrees": agree, "numpy_subset_nonzero_counts": int((want > 0).sum()),
           "numpy_subset_probe_share": probes / (a.subset * M), "placements_with_hits_share": nonzero_share,
           "best_coarse_count": top_count, "stage3_seeds": n_seeds, "stage3_hit": hit, "scan_points": int(pts.shape[0])}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
