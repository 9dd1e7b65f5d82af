"""render_helpers.refine_map against the mapper's loop it replaces (P calls of bundle_adjust_frames over random windows with poses and
decoder frozen), on 26 synthetic keyframes in a MapUpdater map whose table holds 400 k or 4 M rows, with KITTI's mapping values
(window 4, 2 x 2048 rays per keyframe, 25 iterations, voxel 0.3 m, embedding rate 0.01, 27 passes) and NCD's (window 5, 15 iterations,
voxel 0.2 m, rate 0.002).  Whole calls are timed (host clock around work that ends in a device synchronise), warmed up first, the two
alternated over the repeats from the same table and seeds; prints one JSON line per (config, capacity) with medians and min-max, the
time per iteration, the bytes per iteration of both Adam steps computed from the row counts, how well the two tables agree (and, for
scale, how well two runs of the same method agree: the fp32 scatter atomics add in a different order every run), and the card, its
power limit and SM clock read in the same run.

    python scripts/time_refine.py [--repeats 3] [--keyframes 26] [--capacities 400000,4000000] [--configs kitti,ncd] [--out DIR]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nerfloam_b200 as nl  # noqa: E402

CONFIGS = {"kitti": dict(window=4, iters=25, voxel=0.3, lr=0.01), "ncd": dict(window=5, iters=15, voxel=0.2, lr=0.002)}
RAYS = 2 * 2048                 # per keyframe: the reference's 2 x n_rays for the random window (mapping.py:187)
DENSE_BYTES_PER_ROW = 320       # grad zero-fill 64 + grad read 64 + p, m, v (bf16 rows) read 96 + write 96
ROWS_BYTES_PER_ROW = 324        # grad read 64 + clear 64 + p, m, v read 96 + write 96 + the row index 4
MARK_BYTES_PER_SAMPLE = 36      # voxel id 4 + eight row ids 32 (plus the flag words, at most 4 per row)


class _Args:
    def __init__(self):
        self.criteria = {"eiko_weight": 0.1, "sdf_weight": 10000.0, "fs_weight": 1.0, "sdf_truncation": 0.3}
        self.data_specs = {"max_depth": 40.0}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def setup(n_kf, capacity, cfg):
    vs = cfg["voxel"]
    mu = nl.mapping.MapUpdater(vs, init_std=0.01, seed=3, reserve_nodes=400_000, reserve_rows=capacity)
    torch.manual_seed(5)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    kg = nl.keyframes.KeyframeGraph(window_size=cfg["window"], keyframe_gap=0.5, key_distance=40.0, n_rays=RAYS // 2, voxel_size=vs)
    ms = None
    for i in range(n_kf):
        xyz, yaw = nl.synthetic.path_pose(i, n_kf, 1.0, "line")
        pts, cos, pose = nl.synthetic.make_scan(seed=1000 + i, sensor_xyz=xyz, yaw=yaw)
        f = nl.frame.LidarFrame(i, torch.from_numpy(pts), torch.from_numpy(cos), nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose)),
                                new_keyframe=True)
        ms = mu.create_voxels(f.points, f.get_pose().detach())
        kg.insert_keyframe(f)
    return mu, dec, kg, ms


def agreement(e0, e_loop, e_ref, lr):
    """test_gpu_refine's criteria: rows left bitwise unchanged by one and not the other, the update's relative norm difference, and the
    share of entries that differ by more than a fifth of one Adam step."""
    same_l = (e_loop.view(torch.int16) == e0.view(torch.int16)).all(1)
    same_r = (e_ref.view(torch.int16) == e0.view(torch.int16)).all(1)
    e0, e_loop, e_ref = e0.float(), e_loop.float(), e_ref.float()
    u_l, u_r = e_loop - e0, e_ref - e0
    return {"unchanged_rows_mismatch": int((same_l != same_r).sum()), "update_rel": float((u_r - u_l).norm() / u_l.norm()),
            "frac_gt_fifth_step": float(((e_ref - e_loop).abs() > lr / 5).float().mean())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--keyframes", type=int, default=26)
    ap.add_argument("--capacities", default="400000,4000000")
    ap.add_argument("--configs", default="kitti,ncd")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rh = nl.render_helpers
    crit = nl.criterion.Criterion(_Args())
    lines = []
    for name in a.configs.split(","):
        cfg = CONFIGS[name]
        caps = [int(c) for c in a.capacities.split(",")] if name == "kitti" else [int(a.capacities.split(",")[0])]
        for capacity in caps:
            mu, dec, kg, ms = setup(a.keyframes, capacity, cfg)
            table = mu._emb_buf
            e0 = table.clone()
            P = len(kg.keyframe_graph) + 1
            kw = dict(voxel_size=cfg["voxel"], step_size=0.5 * cfg["voxel"], N_rays=RAYS, num_iterations=cfg["iters"], truncation=0.3,
                      max_voxel_hit=20, max_distance=40.0)

            def loop():
                for _ in range(P):
                    rh.bundle_adjust_frames(kg.select_optimize_targets(None, "random"), mu.embeddings, ms, dec, crit,
                                            learning_rate=[cfg["lr"], 0.005, 0.001], update_pose=False, update_decoder=False, **kw)

            def refine():
                rh.refine_map(kg, mu.embeddings, ms, dec, crit, learning_rate=cfg["lr"], passes=P, **kw)

            def timed(fn):
                table.copy_(e0)
                random.seed(11)
                torch.manual_seed(12)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                return (time.perf_counter() - t0) * 1e3, table.clone()

            timed(loop)                                         # warm-up: captures, first launches
            timed(refine)
            t = {"loop": [], "refine_map": []}
            tables = {"loop": [], "refine_map": []}
            for _ in range(a.repeats):
                ms_l, e_loop = timed(loop)
                ms_r, e_ref = timed(refine)
                t["loop"].append(ms_l)
                t["refine_map"].append(ms_r)
                for k, e in (("loop", e_loop), ("refine_map", e_ref)):
                    if len(tables[k]) < 2:
                        tables[k].append(e)
            g = rh._RefineGraph._cache["g"]
            state = g.state.tolist()
            n_samples = g.eng.read_stats().n_samples
            rows_last = state[nl._capi.REFINE_PREV]             # rows the last pass listed: what its last iteration's Adam steps
            iters = P * cfg["iters"]
            out = {"config": name, "keyframes": a.keyframes, "passes": P, "iterations": iters, "rays_per_iteration": RAYS * g.F,
                   "table_rows": int(g.V), "repeats": a.repeats,
                   **{f"{k}_ms": {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in t.items()},
                   **{f"{k}_ms_per_iteration": statistics.median(v) / iters for k, v in t.items()},
                   "speedup_median": statistics.median(t["loop"]) / statistics.median(t["refine_map"]),
                   "adam_bytes_per_iteration": {"dense": DENSE_BYTES_PER_ROW * int(g.V),
                                                "row_list_last_pass_max": ROWS_BYTES_PER_ROW * rows_last + MARK_BYTES_PER_SAMPLE * n_samples,
                                                "rows_listed_last_pass": rows_last, "samples_last_iteration": n_samples},
                   "agreement": agreement(e0, e_loop, e_ref, cfg["lr"]),
                   # the same comparison between two runs of one method: the spread the fp32 scatter atomics' order leaves
                   **({f"agreement_{k}_vs_itself": agreement(e0, v[0], v[1], cfg["lr"]) for k, v in tables.items()} if a.repeats > 1 else {}),
                   "card": card()}
            print(json.dumps(out), flush=True)
            lines.append(out)
            del mu, dec, kg, ms, table, e0
            rh._RefineGraph._cache = {}
            rh._MapGraph._cache = {}
            torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_refine.json"), "w") as fh:
            json.dump(lines, fh, indent=1)


if __name__ == "__main__":
    main()
