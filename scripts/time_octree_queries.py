"""Wall-clock time of the octree queries, host tree against device tree, on the two sequences of scripts/time_map_update.py:
  * demo: 0.3 m voxels, scans 0.5 m apart (the scripts/demo_slam.py setting);
  * fine: 0.2 m voxels (MaiCity / NCD), scans 2 m apart; more than 60 k nodes after the first scan.
After each of --scans scans (83 k points) is inserted into both trees, every query runs --repeats times on both, host and device
alternating: get_centres_and_children, get_voxels, get_leaf_voxels, try_insert of the next scan's voxels (a CUDA tensor for the
device tree, a CPU one for the host tree, as each is fed in the SLAM loop) and a pickle round trip (pickle.loads(pickle.dumps)).
Each call is timed from a synchronised start to a synchronise after it; the results are on the host by then.  The two trees'
results are checked equal.  Prints the medians over scans and repeats, the node counts and pickle sizes, the card and its power
limit, as one JSON line.  Nothing is written to disk.

    python scripts/time_octree_queries.py [--scans 4] [--repeats 5]
"""
import argparse
import json
import os
import pickle
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from time_map_update import SEQUENCES, card  # noqa: E402

QUERIES = ("get_centres_and_children", "get_voxels", "get_leaf_voxels", "try_insert", "pickle_round_trip")


def voxel_scans(name, k):
    import nerfloam_b200 as nl
    vs, spacing, seed = SEQUENCES[name]
    out = []
    for i in range(k):
        pts, _, pose = nl.synthetic.make_scan(seed=seed + i, sensor_xyz=(spacing * i, 0.05 * np.sin(0.7 * i), 0.0), yaw=0.01 * np.sin(0.5 * i))
        out.append(nl.synthetic.voxelize(pts, pose, vs))
    return vs, out


def timed(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def same(a, b):
    if isinstance(a, tuple):
        return all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, torch.Tensor):
        return a.dtype == b.dtype and torch.equal(a, b)
    return a == b


def run(name, k, repeats):
    import nerfloam_b200 as nl
    vs, scans = voxel_scans(name, k + 1)
    trees = {"host": nl.svo.Octree(), "device": nl.svo.DeviceOctree()}
    for t in trees.values():
        t.init(256 * 256 * 4, 16, vs)
    ms = {q: {o: [] for o in trees} for q in QUERIES}
    nodes, pickle_bytes = [], {}
    for i in range(k):
        for o, t in trees.items():
            t.insert(torch.from_numpy(scans[i]).cuda() if o == "device" else torch.from_numpy(scans[i]))
        nodes.append(trees["host"].count_nodes())
        nxt = {"host": torch.from_numpy(scans[i + 1]), "device": torch.from_numpy(scans[i + 1]).cuda()}
        calls = {"get_centres_and_children": lambda t, o: t.get_centres_and_children(), "get_voxels": lambda t, o: t.get_voxels(),
                 "get_leaf_voxels": lambda t, o: t.get_leaf_voxels(), "try_insert": lambda t, o: t.try_insert(nxt[o]),
                 "pickle_round_trip": lambda t, o: pickle.loads(pickle.dumps(t)).count_nodes()}
        for _ in range(repeats):
            for q, f in calls.items():
                res = {}
                for o, t in trees.items():
                    dt, res[o] = timed(lambda: f(t, o))
                    ms[q][o].append(dt)
                assert same(res["host"], res["device"]), (name, q)
    for o, t in trees.items():
        pickle_bytes[o] = len(pickle.dumps(t))
    return {"voxel_size": vs, "spacing_m": SEQUENCES[name][1], "nodes_after_each_scan": nodes, "pickle_bytes": pickle_bytes,
            "ms_median": {q: {o: round(float(np.median(v)), 3) for o, v in d.items()} for q, d in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_octree_queries.py needs a CUDA device")
    torch.cuda.set_device(0)
    run("demo", 1, 1)                                                    # warm-up
    out = {name: run(name, a.scans, a.repeats) for name in SEQUENCES}
    name, power = card(0)
    print(json.dumps({"gpu": name, "power_limit": power, "scans": a.scans, "repeats": a.repeats, "sequences": out}))


if __name__ == "__main__":
    main()
