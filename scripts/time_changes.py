"""Change detection per scan (changes.ChangeDetector, DESIGN.md §11.7): the street drive of tests/test_gpu_localise.py (12 scans 0.5 m
apart, synthetic.make_street_scan, about 62 k points per scan as in §11.4) mapped by slam.NeRFLOAM with the true poses and KITTI's
values and saved to a temporary directory, then a second pass of 14 scans (shifted 0.5 m and turned 10 degrees):

  * add_scan: host ms per scan (every point rendered, the votes and the added table; it ends in its own read-back), after a warm-up
    scan, against the NumPy restatement (tests/change_ref.py) of the same votes and added counts from the same sample arrays;
  * tracking per scan (Localiser's track stage) with change_specs off and on, alternated, with the generator seeded alike.

Prints one JSON line with the card's name, power limit and SM clock read in the same run, medians and min-max.

    python scripts/time_changes.py [--repeats 3]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import nerfloam_b200 as nl  # noqa: E402
import change_ref as ref  # noqa: E402
from time_localise import Stream, config, scan, stats  # noqa: E402
from time_track_batch import card  # noqa: E402

MAP_SCANS, PASS_SCANS = 12, 14
SHIFT, TURN = (0.3, 0.4), math.radians(10.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    second = [scan(i, 6000 + i, SHIFT, TURN) for i in range(PASS_SCANS)]
    out = {"bench": "changes", "card": card(), "map_scans": MAP_SCANS, "scans": PASS_SCANS, "repeats": a.repeats,
           "specs": nl.changes.CHANGE_SPECS, "points_per_scan": stats([int(s[0].shape[0]) for s in second])}
    with tempfile.TemporaryDirectory() as tmp:
        s = nl.slam.NeRFLOAM(config(), os.path.join(tmp, "run"), data_stream=Stream([scan(i, 2000 + i) for i in range(MAP_SCANS)], True))
        s.run()
        path = os.path.join(tmp, "run.map")
        s.save_map(path)
        del s
        saved = nl.slam.load_map(path)
        track = {"off": [], "on": []}
        add_ms, frames = [], None
        for r in range(a.repeats + 1):                              # the first round warms every shape up and is not kept
            for mode in ("off", "on"):
                loc = nl.localise.Localiser(saved, Stream(second, False), generator=torch.Generator().manual_seed(r),
                                            config={"change_specs": {}} if mode == "on" else None)
                res = loc.run()
                torch.cuda.synchronize()
                if r:
                    track[mode].append(loc.summary(res)["ms_per_scan"]["track"])
                    if mode == "on":
                        add_ms += loc.change_ms[1:]
                        out.setdefault("changes", loc.summary(res)["changes"])
                if mode == "on" and frames is None:
                    frames = [(torch.from_numpy(p[0]), torch.from_numpy(p[1]), res.poses[i].clone()) for i, p in enumerate(second)]
        # the restatement on the arrays of one detector pass
        m, dec = saved.map.map_states["_mapstate"], saved.decoder
        cfg = saved.config
        vs = float(cfg["voxel_size"])
        det = nl.changes.ChangeDetector(m, dec, vs, cfg["criteria"], {"step_size": cfg["tracker_specs"]["step_size"] * vs,
                                                                     "max_distance": cfg["data_specs"]["max_depth"]})
        calls, ref_ms = [], []
        orig = det._votes

        def spy(mm, bufs, dirs, gt, r0, R, status):
            orig(mm, bufs, dirs, gt, r0, R, status)
            e, M = det.eng, det.eng.read_stats().n_samples
            calls.append(tuple(t[:M].cpu().numpy() for t in (e.s_ray, e.s_vox, e.s_depth, e.sdf)) + (gt[r0:r0 + R].cpu().numpy(),))
        det._votes = spy
        occ = ref.leaf_keys(m.centres.cpu().numpy(), m.structure.cpu().numpy(), vs)
        samples = []
        for i, (pts, cos, P) in enumerate(frames):
            T = P.clone()
            T[:3, 3] += nl.frame.POSE_OFFSET
            f = nl.frame.LidarFrame(i, pts, cos, nl.se3pose.OptimizablePose.from_matrix(T.float()), new_keyframe=True)
            calls.clear()
            det.add_scan(f, f.pose)
            Rt = det.Rt12.cpu().numpy()
            t0 = time.perf_counter()
            for s_ray, s_vox, s_depth, sdf, gt in calls:
                ref.votes(s_ray, s_vox, s_depth, sdf, gt, m.n_nodes, det.truncation, det.through)
            ref.added([(pts.numpy(), Rt)], occ, vs)
            ref_ms.append((time.perf_counter() - t0) * 1e3)
            samples.append(sum(c[0].shape[0] for c in calls))
    out["add_scan_ms"] = stats(add_ms)
    out["restatement_ms"] = stats(ref_ms)
    out["samples_per_scan"] = stats(samples)
    out["track_ms_per_scan"] = {k: stats(v) for k, v in track.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
