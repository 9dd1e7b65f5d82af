"""track_frames with K = 1, 2, 4, 8, 16 problems of 2048 rays x 25 iterations against K solo track_frame calls, on the KITTI-shape
synthetic scan, captured graph and eager.  Every variant is timed as whole calls (host clock around work that ends in a device
synchronise), warmed up first, alternated over repeats; prints the card, its power limit and one JSON line per (K, mode) with the
median and the spread (min, max) of the repeats.

    python scripts/time_track_batch.py [--repeats 7] [--ks 1,2,4,8,16] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nerfloam_b200 as nl  # noqa: E402
from nerfloam_b200.criterion import Criterion  # noqa: E402


class _Args:
    def __init__(self):
        self.criteria = {"eiko_weight": 0.1, "sdf_weight": 10000.0, "fs_weight": 1.0, "sdf_truncation": 0.3}
        self.data_specs = {"max_depth": 40.0}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--ks", default="1,2,4,8,16")
    ap.add_argument("--iters", type=int, default=25)
    ap.add_argument("--rays", type=int, default=2048)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_track_batch.py measures on the GPU; none found")
    syn = nl.synthetic
    pts, cos, pose = syn.make_scan()                     # KITTI shape: 64 beams x 1300 azimuths
    mu = nl.mapping.MapUpdater(0.3, init_std=0.02, seed=1)
    ms = mu.insert_voxels(torch.from_numpy(syn.voxelize(pts, pose, 0.3)))
    torch.manual_seed(0)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    crit = Criterion(_Args())
    start = nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose)).data.detach().clone()
    fr = nl.frame.LidarFrame(5, torch.from_numpy(pts), torch.from_numpy(cos), nl.se3pose.OptimizablePose(start.clone()), new_keyframe=True)
    kw = dict(N_rays=a.rays, step_size=0.15, num_iterations=a.iters, truncation=0.3, learning_rate=0.01, max_voxel_hit=20, max_distance=40.0)
    starts = [nl.se3pose.OptimizablePose(start + 0.02 * torch.randn(6) * torch.tensor([1.0, 1.0, 1.0, 0.1, 0.1, 0.1])) for _ in range(32)]

    def solo(K, graph):
        for k in range(K):
            nl.render_helpers.track_frame(starts[k], fr, ms, dec, crit, 0.3, cuda_graph=graph, **kw)

    def batch(K, graph):
        nl.track_frames(starts[:K], [fr] * K, ms, dec, crit, 0.3, cuda_graph=graph, **kw)

    dev_card = card()
    print("card:", dev_card, flush=True)
    rows = []
    for K in [int(x) for x in a.ks.split(",")]:
        for graph in (True, False):
            variants = {"batch": lambda: batch(K, graph), "solo": lambda: solo(K, graph)}
            for f in variants.values():          # warm-up: captures, engines, frame uploads
                f(); f()
            torch.cuda.synchronize()
            times = {n: [] for n in variants}
            for _ in range(a.repeats):
                for n, f in variants.items():    # alternated
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    f()
                    torch.cuda.synchronize()
                    times[n].append((time.perf_counter() - t0) * 1e3)
            row = dict(K=K, mode="graph" if graph else "eager", rays=a.rays, iters=a.iters, card=dev_card)
            for n, t in times.items():
                row[n + "_ms"] = round(statistics.median(t), 2)
                row[n + "_min_max_ms"] = [round(min(t), 2), round(max(t), 2)]
            row["speedup"] = round(row["solo_ms"] / row["batch_ms"], 2)
            print(json.dumps(row), flush=True)
            rows.append(row)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_track_batch.json"), "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
