"""Localising against a saved map: a street drive (synthetic.make_street_scan, 0.5 m apart) mapped by slam.NeRFLOAM with the true
poses and KITTI's tracker and mapper values, saved with save_map to a temporary directory, then a second pass over the same route
(new scan noise, shifted 0.5 m and turned 10 degrees) localised in the file with localise.Localiser, on the host and the device octree
alternately.  Per run: the map file's load time, the first scan's placement (relocalise_global: whole call and per stage, then the tracking from it) and the host
milliseconds per scan for load, track (slam.Tracking: ends in a read-back) and score (score_poses at the final pose).  Prints one JSON
line with the card's name and power limit (read in the same run), medians and min-max over the runs, and the worst pose error.

    python scripts/time_localise.py [--map-scans 40] [--scans 32] [--repeats 2]
"""
import argparse
import json
import math
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import nerfloam_b200 as nl  # noqa: E402
from time_track_batch import card  # noqa: E402

SPACING = 0.5


def scan(i, seed, shift=(0.0, 0.0), turn=0.0):
    xyz = (SPACING * i + shift[0], 0.05 * np.sin(0.7 * i) + shift[1], 0.0)
    pts, cos, pose = nl.synthetic.make_street_scan(xyz, 0.01 * np.sin(0.5 * i) + turn, seed=seed)
    pose = pose.astype(np.float64)
    pose[:3, 3] -= nl.synthetic.POSE_OFFSET
    return pts, cos, pose


class Stream:
    def __init__(self, scans, use_gt):
        self.scans, self.use_gt = scans, use_gt

    def __len__(self):
        return len(self.scans)

    def __getitem__(self, i):
        pts, cos, pose = self.scans[i]
        return i, torch.from_numpy(pts), torch.from_numpy(cos), (pose.copy() if self.use_gt else None)

    def get_init_pose(self, i):
        return self.scans[i][2].copy() if self.use_gt else np.eye(4)


def config():
    """KITTI's tracker and mapper values (the reference's configs/kitti/kitti.yaml) with the true poses for the mapping run."""
    return {"dataset": "kitti", "seeding": 777, "data_specs": {"data_path": "", "use_gt": True, "max_depth": 40, "min_depth": 1.5},
            "criteria": {"sdf_weight": 10000.0, "fs_weight": 1, "eiko_weight": 0.1, "sdf_truncation": 0.3},
            "decoder_specs": {"depth": 2, "width": 256, "in_dim": 16, "skips": [], "embedder": "none", "multires": 0},
            "tracker_specs": {"N_rays": 2048, "learning_rate": 0.01, "step_size": 0.2, "max_voxel_hit": 20, "num_iterations": 25},
            "mapper_specs": {"N_rays_each": 2048, "use_local_coord": False, "voxel_size": 0.3, "step_size": 0.5, "window_size": 4,
                             "num_iterations": 25, "max_voxel_hit": 20, "final_iter": False, "mesh_res": 2, "learning_rate_emb": 0.01,
                             "learning_rate_decorder": 0.005, "learning_rate_pose": 0.001, "freeze_frame": 5, "keyframe_gap": 1.0,
                             "remove_back": False, "key_distance": 12},
            "debug_args": {"verbose": False, "mesh_freq": 0}}


def stats(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--map-scans", type=int, default=40)
    ap.add_argument("--scans", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=2, help="runs per octree, alternated")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    with tempfile.TemporaryDirectory() as tmp:
        s = nl.slam.NeRFLOAM(config(), os.path.join(tmp, "run"), data_stream=Stream([scan(i, 2000 + i) for i in range(a.map_scans)], True))
        s.run()
        path = os.path.join(tmp, "run.map")
        s.save_map(path)
        size = os.path.getsize(path)
        n_nodes, n_rows = s.mapper.map.n_nodes, s.mapper.map.n_rows
        del s
        second = [scan(i, 5000 + i, (0.3, 0.4), math.radians(10.0)) for i in range(a.scans)]
        truth = torch.from_numpy(np.stack([p[2] for p in second]))
        runs = {"host": [], "device": []}
        for r in range(a.repeats + 1):                                 # the first round warms every shape up and is not kept
            for octree in ("host", "device"):
                torch.cuda.synchronize()
                loc = nl.localise.Localiser(path, Stream(second, False), generator=torch.Generator().manual_seed(r), octree=octree)
                res = loc.run()
                torch.cuda.synchronize()
                sm = loc.summary(res)
                dt = float((res.poses[:, :3, 3] - truth[:, :3, 3]).norm(dim=-1).max())
                dr = float(torch.linalg.matrix_norm(res.poses[:, :3, :3] - truth[:, :3, :3]).max())
                if r:
                    runs[octree].append(dict(sm, max_translation_error_m=dt, max_rotation_error_fro=dr))
                del loc, res
    out = {"card": card(), "map": {"scans": a.map_scans, "nodes": int(n_nodes), "embedding_rows": int(n_rows), "file_bytes": size},
           "localised_scans": a.scans, "points_per_scan": int(np.mean([p[0].shape[0] for p in second]))}
    for octree, rs in runs.items():
        out[octree] = {"map_load_ms": stats([x["map_load_ms"] for x in rs]),
                       "placement_ms": stats([x["placement"]["ms"] for x in rs]),
                       "placement_track_ms": stats([x["placement"]["track_ms"] for x in rs]),
                       "placement_stages_ms": {k: stats([x["placement"]["stages_ms"][k] for x in rs]) for k in rs[0]["placement"]["stages_ms"]},
                       "placements": rs[0]["placement"]["placements"],
                       "ms_per_scan": {k: stats([x["ms_per_scan"][k] for x in rs]) for k in rs[0]["ms_per_scan"]},
                       "median_loss": stats([x["median_loss"] for x in rs]),
                       "max_translation_error_m": max(x["max_translation_error_m"] for x in rs),
                       "max_rotation_error_fro": max(x["max_rotation_error_fro"] for x in rs)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
