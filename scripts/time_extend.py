"""Growing a saved map with a later drive (slam.NeRFLOAM(..., base_map=...)) against mapping the same drive from scratch: the street of
tests/test_gpu_extend.py (synthetic.street_boxes(length=180)), drive A (12 scans 0.5 m apart) mapped with the true poses and KITTI's
values and saved to a temporary directory, then drive B (shifted 0.5 m, turned 10 degrees, 1 m apart, on past A's coverage):

  * extend: B grown into A's map (the first scan placed with no guess, the saved rows and the decoder held fixed);
  * scratch: B mapped from an empty map by a plain NeRFLOAM run with B's first true pose as its initial pose;

alternately, each with a fresh copy of the map read from the file.  Per run: the median host ms per scan of track, map, update and
publish, the first scan's placement (search and tracking from it) and, for extend, the grown file's size and its load_map time.

Prints one JSON line with the card's name, power limit and SM clock (read in the same run) and medians and min-max over the repeats
(after one warm-up round that is not kept).

    python scripts/time_extend.py [--repeats 3] [--scans 60]
"""
import argparse
import json
import math
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import nerfloam_b200 as nl  # noqa: E402
from time_localise import Stream, config, stats  # noqa: E402
from time_track_batch import card  # noqa: E402

SHIFT, TURN = (0.3, 0.4), math.radians(10.0)
STAGES = ("track", "map", "update", "publish")


class FirstPose(Stream):
    """B's scans with no pose but the first one's true pose as get_init_pose (the scratch run's starting point)."""

    def get_init_pose(self, i):
        return self.scans[i][2].copy()


def scan(boxes, x, i, seed, shift=(0.0, 0.0), turn=0.0):
    xyz = (x + shift[0], 0.05 * np.sin(0.7 * i) + shift[1], 0.0)
    pts, cos, pose = nl.synthetic.make_street_scan(xyz, 0.01 * np.sin(0.5 * i) + turn, boxes=boxes, seed=seed)
    pose = pose.astype(np.float64)
    pose[:3, 3] -= nl.synthetic.POSE_OFFSET
    return pts, cos, pose


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--scans", type=int, default=60, help="scans of drive B, 1 m apart")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    boxes = nl.synthetic.street_boxes(length=180.0)
    A = [scan(boxes, 0.5 * i, i, 2000 + i) for i in range(12)]
    B = [scan(boxes, 1.0 * i, i, 5000 + i, SHIFT, TURN) for i in range(a.scans)]
    runs = {"extend": [], "scratch": []}
    with tempfile.TemporaryDirectory() as tmp:
        s = nl.slam.NeRFLOAM(config(), os.path.join(tmp, "A"), data_stream=Stream(A, True))
        s.run()
        path = os.path.join(tmp, "A.map")
        s.save_map(path)
        del s
        cfg = config()
        cfg["data_specs"]["use_gt"] = False
        for r in range(a.repeats + 1):                                  # the first round warms every shape up and is not kept
            for name in ("extend", "scratch"):
                torch.cuda.synchronize()
                out = os.path.join(tmp, f"{name}{r}")
                if name == "extend":
                    s = nl.slam.NeRFLOAM(cfg, out, data_stream=Stream(B, False), base_map=path)
                else:
                    s = nl.slam.NeRFLOAM(cfg, out, data_stream=FirstPose(B, False))
                sm = s.run()
                truth = np.stack([p[2] for p in B])
                poses = np.loadtxt(os.path.join(out, "misc", "frame_poses.txt"), ndmin=2).reshape(-1, 3, 4)
                sm["max_translation_error_m"] = float(np.linalg.norm(poses[:, :, 3] - truth[:, :3, 3], axis=1).max())
                if name == "extend":
                    grown = os.path.join(tmp, f"grown{r}.map")
                    s.save_map(grown)
                    del s
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    g = nl.slam.load_map(grown)
                    torch.cuda.synchronize()
                    sm["load_ms"] = (time.perf_counter() - t0) * 1e3
                    sm["file_bytes"] = os.path.getsize(grown)
                    sm["rows"], sm["nodes"] = int(g.map.n_rows), int(g.map.n_nodes)
                    del g
                else:
                    del s
                if r:
                    runs[name].append(sm)
    res = {"bench": "extend", "card": card(), "scans_a": len(A), "scans_b": len(B), "repeats": a.repeats}
    for name, rs in runs.items():
        res[name] = {f"{k}_ms_per_scan": stats([x["ms_per_scan"][k] for x in rs]) for k in STAGES}
        res[name]["wall_ms_per_scan"] = stats([x["ms_per_scan_wall"] for x in rs])
        res[name]["max_translation_error_m"] = max(x["max_translation_error_m"] for x in rs)
    ex = runs["extend"]
    res["extend"]["place_search_ms"] = stats([x["base"]["place_ms"]["search"] for x in ex])
    res["extend"]["place_track_ms"] = stats([x["base"]["place_ms"]["track"] for x in ex])
    res["extend"]["grown_file_bytes"] = ex[-1]["file_bytes"]
    res["extend"]["grown_load_ms"] = stats([x["load_ms"] for x in ex])
    res["extend"]["rows"] = {"saved": ex[-1]["base"]["frozen_rows"], "grown": ex[-1]["rows"]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
