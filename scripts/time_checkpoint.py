"""Wall-clock time of a map checkpoint, host tree against device tree, and of the route the reference takes to get a map back.
Maps:
  * demo: 0.3 m voxels, 12 scans 0.5 m apart (the scripts/demo_slam.py setting);
  * fine: 0.2 m voxels (MaiCity / NCD), 4 scans 2 m apart;
  * large: about 10^6 nodes.  The synthetic street canyon is fixed in the world, so scan k's voxels are shifted by k * 200
    voxels along x (the canyon is 200 voxels long at 0.3 m), each scan adding a fresh stretch of map, until 10^6 nodes.
For each map and tree, --repeats times, host and device alternating:
  * save: MapUpdater.state_dict() + torch.save into memory;
  * load: torch.load(weights_only=True) + MapUpdater.from_state_dict onto the same kind of tree;
  * reference route (host tree): pickle.loads(pickle.dumps(mu.svo)), which replays every inserted scan, then the full export and
    the renumbering of the embedding rows that a restored map needs (export_map + nl_assign_embedding_rows).  One pass numbers
    the rows in a different order than the scan-by-scan updates did, so this route does not even give back the same rows.
Each call is timed from a synchronised start to a synchronise after it.  The restored maps are checked equal to the saved ones.
Prints the medians, node counts, checkpoint bytes per node, the card and its power limit as one JSON line.  Nothing is written
to disk.

    python scripts/time_checkpoint.py [--repeats 3]
"""
import argparse
import ctypes as C
import io
import json
import os
import pickle
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from time_map_update import card  # noqa: E402

TARGET_NODES = 1_000_000


def voxel_scans(vs, spacing, seed, k, shift=0):
    import nerfloam_b200 as nl
    out = []
    for i in range(k):
        pts, _, pose = nl.synthetic.make_scan(seed=seed + i, sensor_xyz=(spacing * i, 0.05 * np.sin(0.7 * i), 0.0), yaw=0.01 * np.sin(0.5 * i))
        out.append(nl.synthetic.voxelize(pts, pose, vs) + np.array([[shift * i, 0, 0]], np.int32))
    return out


def build(vs, scans, until=None):
    import nerfloam_b200 as nl
    mus = {o: nl.mapping.MapUpdater(vs, init_std=0.01, seed=0, octree=o) for o in ("host", "device")}
    for v in scans:
        for mu in mus.values():
            mu.insert_voxels(torch.from_numpy(v))
        if until and mus["device"].n_nodes >= until:
            break
    return mus


def timed(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def same_state(a, b):
    return set(a) == set(b) and all(torch.equal(a[k], b[k]) if isinstance(a[k], torch.Tensor) else a[k] == b[k] for k in a)


def save(mu):
    buf = io.BytesIO()
    torch.save(mu.state_dict(), buf)
    return buf.getvalue()


def load(blob, octree):
    import nerfloam_b200 as nl
    return nl.mapping.MapUpdater.from_state_dict(torch.load(io.BytesIO(blob), weights_only=True), octree=octree)


def reference_route(mu):
    import nerfloam_b200 as nl
    svo = pickle.loads(pickle.dumps(mu.svo))
    _, _, vertex = svo.export_map()
    v = vertex.numpy()
    v2r = np.full(v.shape[0], -1, np.int32)
    rows = nl._capi.lib().nl_assign_embedding_rows(v.ctypes.data_as(C.c_void_p), v.shape[0], v2r.ctypes.data_as(C.c_void_p), 0)
    return rows, v2r


def run(mus, repeats):
    n = mus["host"].n_nodes
    ms = {q: {o: [] for o in mus} for q in ("save", "load")}
    ms["reference_route"] = {"host": []}
    blobs = {}
    for _ in range(repeats):
        for o, mu in mus.items():
            dt, blobs[o] = timed(lambda: save(mu))
            ms["save"][o].append(dt)
            dt, res = timed(lambda: load(blobs[o], o))
            ms["load"][o].append(dt)
            assert same_state(res.state_dict(), mu.state_dict()), o
        dt, (rows, v2r) = timed(lambda: reference_route(mus["host"]))
        ms["reference_route"]["host"].append(dt)
        assert rows == mus["host"].n_rows               # the same vertices, numbered in one pass instead of scan by scan
    assert blobs["host"] == blobs["device"] or same_state(torch.load(io.BytesIO(blobs["host"]), weights_only=True),
                                                          torch.load(io.BytesIO(blobs["device"]), weights_only=True))
    return {"nodes": n, "embedding_rows": mus["host"].n_rows, "checkpoint_bytes": len(blobs["host"]),
            "bytes_per_node": round(len(blobs["host"]) / n, 2),
            "ms_median": {q: {o: round(float(np.median(v)), 3) for o, v in d.items()} for q, d in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_checkpoint.py needs a CUDA device")
    torch.cuda.set_device(0)
    run(build(0.3, voxel_scans(0.3, 0.5, 1000, 2)), 1)                  # warm-up
    maps = {"demo": lambda: build(0.3, voxel_scans(0.3, 0.5, 1000, 12)),
            "fine": lambda: build(0.2, voxel_scans(0.2, 2.0, 2000, 4)),
            "large": lambda: build(0.3, voxel_scans(0.3, 0.0, 1000, 60, shift=200), until=TARGET_NODES)}
    out = {}
    for name, make in maps.items():
        out[name] = run(make(), a.repeats)
        torch.cuda.empty_cache()
    name, power = card(0)
    print(json.dumps({"gpu": name, "power_limit": power, "repeats": a.repeats, "maps": out}))


if __name__ == "__main__":
    main()
