"""Per-scan time of the whole pipeline (slam.NeRFLOAM): the tracker and the mapper concurrent on two streams against the same lag-one
order driven on one thread, alternated in one process.

    python scripts/time_slam.py [--scans 64] [--runs 3] [--json out.json]

Synthetic 83 k-point canyon scans 0.5 m apart (nl.synthetic), KITTI's tracker and mapper values, the reference's 'current' mapping
window, no periodic mesh.  Reports per mode the median and min-max milliseconds per tracked scan (wall-clock from the first tracked
scan's hand-off to the end of the last mapping step, divided by the tracked scans), each stage's median host milliseconds per scan
and its share of the one-thread scan time, and the card's name and power limit.
"""
import argparse, json, os, subprocess, sys, tempfile, time
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerfloam_b200 as nl


class Stream:
    def __init__(self, scans):
        self.scans = scans

    def __len__(self):
        return len(self.scans)

    def __getitem__(self, i):
        return i, torch.from_numpy(self.scans[i][0]), torch.from_numpy(self.scans[i][1]), None

    def get_init_pose(self, i):
        return np.eye(4)


def config():
    return {"dataset": "kitti", "seeding": 777, "data_specs": {"data_path": "", "use_gt": False, "max_depth": 40, "min_depth": 5},
            "criteria": {"sdf_weight": 10000.0, "fs_weight": 1, "eiko_weight": 0.1, "sdf_truncation": 0.3},
            "decoder_specs": {"depth": 2, "width": 256, "in_dim": 16, "skips": [], "embedder": "none", "multires": 0},
            "tracker_specs": {"N_rays": 2048, "learning_rate": 0.01, "step_size": 0.2, "max_voxel_hit": 20, "num_iterations": 25},
            "mapper_specs": {"N_rays_each": 2048, "use_local_coord": False, "voxel_size": 0.3, "step_size": 0.5, "window_size": 4,
                             "num_iterations": 25, "max_voxel_hit": 20, "final_iter": False, "mesh_res": 2, "learning_rate_emb": 0.01,
                             "learning_rate_decorder": 0.005, "learning_rate_pose": 0.001, "freeze_frame": 5, "keyframe_gap": 8,
                             "remove_back": False, "key_distance": 12},
            "debug_args": {"mesh_freq": 0}}


class Clock:
    """Wraps the mapper's init so that the clock starts when the first scan has been mapped (the capture and init calls excluded)."""
    def __init__(self, s):
        self.t0, init = None, s.mapper.init
        def timed_init(frame):
            v = init(frame)
            torch.cuda.synchronize()
            self.t0 = time.perf_counter()
            return v
        s.mapper.init = timed_init


def run_serial(s):
    tr, mp = s.tracker, s.mapper
    versions = [mp.init(tr.first_frame())]
    ids = tr.frame_ids()
    frame = tr.track(ids[0], versions[0])
    for p in range(1, len(ids) + 1):
        state = mp.optimise(frame)
        if p < len(ids):
            frame = tr.track(ids[p], versions[p - 1])
        versions.append(mp.update(state))


def one(mode, scans, out):
    s = nl.slam.NeRFLOAM(config(), out, data_stream=Stream(scans))
    s.mapper.finish = lambda: None                    # meshes are not part of the per-scan time
    clock = Clock(s)
    if mode == "concurrent":
        nl.slam.run_pipeline(s.tracker, s.mapper, s.streams)
    else:
        run_serial(s)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - clock.t0) * 1e3 / (len(scans) - 1)
    stages = {k: float(np.median(v)) for k, v in {**s.tracker.times, **s.mapper.times}.items() if k != "init"}
    return ms, stages


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=64); ap.add_argument("--runs", type=int, default=3); ap.add_argument("--json", default=None)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    syn = nl.synthetic
    scans = []
    for i in range(a.scans):
        xyz, yaw = syn.path_pose(i, a.scans, 0.5)
        p, c, _ = syn.make_scan(seed=1000 + i, sensor_xyz=xyz, yaw=yaw)
        scans.append((p, c))
    res = {"concurrent": [], "one_thread": []}
    with tempfile.TemporaryDirectory() as tmp:
        one("one_thread", scans[:8], os.path.join(tmp, "warm"))           # module loads, first captures
        for r in range(a.runs):
            for mode in ("one_thread", "concurrent"):
                res[mode].append(one(mode, scans, os.path.join(tmp, f"{mode}{r}")))
    out = {"card": card, "scans": a.scans, "points_per_scan": int(np.mean([s[0].shape[0] for s in scans])), "runs": a.runs}
    base = float(np.median([m for m, _ in res["one_thread"]]))
    for mode, rs in res.items():
        ms = [m for m, _ in rs]
        stages = {k: float(np.median([st[k] for _, st in rs])) for k in rs[0][1]}
        out[mode] = {"ms_per_scan": float(np.median(ms)), "min_max_ms": [float(min(ms)), float(max(ms))], "stage_ms": stages,
                     "stage_share_of_one_thread_scan": {k: round(v / base, 3) for k, v in stages.items()}}
    out["speedup"] = base / out["concurrent"]["ms_per_scan"]
    print(json.dumps(out))
    if a.json:
        json.dump(out, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
