"""Wall-clock time of MapUpdater.create_voxels per scan, host octree against device octree, on two synthetic sequences:
  * demo: 0.3 m voxels, scans 0.5 m apart (the scripts/demo_slam.py setting);
  * fine: 0.2 m voxels (MaiCity / NCD), scans 2 m apart.
Each scan is 83 k points, handed over as device tensors (as the SLAM loop holds them).  The two trees alternate scan by scan, each
timed from a synchronised start to a synchronise after the update.  A warm-up sequence runs first; the sequences are then repeated
--repeats times and the medians of the first scan and of the later scans are reported, with the card and its power limit, as one
JSON line.  Nothing is written to disk.

    python scripts/time_map_update.py [--scans 12] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


SEQUENCES = {"demo": (0.3, 0.5, 1000), "fine": (0.2, 2.0, 2000)}   # voxel size, spacing, seed base


def card(index):
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(index)],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, power = (f.strip() for f in out.split(","))
    return name, power


def scans(name, k, dev):
    import nerfloam_b200 as nl
    vs, spacing, seed = SEQUENCES[name]
    out = []
    for i in range(k):
        pts, _, pose = nl.synthetic.make_scan(seed=seed + i, sensor_xyz=(spacing * i, 0.05 * np.sin(0.7 * i), 0.0), yaw=0.01 * np.sin(0.5 * i))
        out.append((torch.from_numpy(pts).to(dev), torch.from_numpy(pose).to(dev)))
    return vs, out


def run(name, k, dev):
    import nerfloam_b200 as nl
    vs, seq = scans(name, k, dev)
    mus = {o: nl.mapping.MapUpdater(vs, device=dev, octree=o, reserve_nodes=1_000_000, reserve_rows=1_000_000) for o in ("host", "device")}
    ms = {o: [] for o in mus}
    for pts, pose in seq:
        for o, mu in mus.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mu.create_voxels(pts, pose)
            torch.cuda.synchronize()
            ms[o].append((time.perf_counter() - t0) * 1e3)
    assert mus["host"].n_nodes == mus["device"].n_nodes and mus["host"].n_rows == mus["device"].n_rows
    return ms, mus["device"].n_nodes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=12)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_map_update.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    run("demo", 3, dev)                                                  # warm-up
    out = {}
    for name in SEQUENCES:
        first, later, nodes = {"host": [], "device": []}, {"host": [], "device": []}, 0
        for _ in range(a.repeats):
            ms, nodes = run(name, a.scans, dev)
            for o, t in ms.items():
                first[o].append(t[0])
                later[o] += t[1:]
        out[name] = {"voxel_size": SEQUENCES[name][0], "spacing_m": SEQUENCES[name][1], "nodes_after": nodes,
                     **{o: {"first_ms": round(float(np.median(first[o])), 3), "later_ms_median": round(float(np.median(later[o])), 3),
                            "later_ms_max": round(float(np.max(later[o])), 3)} for o in first},
                     "device_faster_on_every_scan": bool(all(d < h for d, h in zip(first["device"] + later["device"], first["host"] + later["host"])))}
    name, power = card(0)
    print(json.dumps({"gpu": name, "power_limit": power, "scans": a.scans, "repeats": a.repeats, "sequences": out}))


if __name__ == "__main__":
    main()
