"""evaluate.eval_mesh on the GPU against the NumPy / SciPy restatement on the host (tests/eval_ref.py: cKDTree with workers=-1),
alternating, at 10^6 and 10^7 surface samples on two meshes: an analytic height field (a 1000 x 1000 grid, 2 M triangles, against
4 M points on the same surface) and the mesh of a map trained on four synthetic scans (against their noise-free returns).  The
host side starts from the GPU's surface samples (it does not sample); the GPU side is the whole eval_mesh call from device inputs,
timed with a host clock around a device synchronise after a warm-up.  Both compute the same numbers; the script checks that the
counts agree.  Prints one JSON line: medians and min-max per case, with the card and its power limit.

    python scripts/time_evaluate.py [--repeats 3] [--samples 1000000,10000000] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import nerfloam_b200 as nl  # noqa: E402
import eval_ref as ER  # noqa: E402
from time_track_batch import card  # noqa: E402

KW = dict(res=0.05, threshold=0.1, truncation=0.5, seed=0)


def height_field(n=1000, size=40.0):
    """z = 0.5 sin(x / 3) cos(y / 4) + 2000 over [2000, 2000 + size]^2: the mesh (n x n quads) and 4 n^2 points on the surface."""
    f = lambda x, y: 0.5 * np.sin(x / 3.0) * np.cos(y / 4.0)
    g = np.linspace(0, size, n + 1)
    xx, yy = np.meshgrid(g, g, indexing="ij")
    V = np.c_[xx.reshape(-1) + 2000, yy.reshape(-1) + 2000, f(xx, yy).reshape(-1) + 2000].astype(np.float32)
    i = np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]
    a, b, c, d = i, i + 1, i + n + 1, i + n + 2
    F = np.concatenate([np.stack([a, c, b], -1).reshape(-1, 3), np.stack([b, c, d], -1).reshape(-1, 3)]).astype(np.int32)
    rng = np.random.default_rng(0)
    x, y = rng.uniform(0, size, 4 * n * n), rng.uniform(0, size, 4 * n * n)
    gt = np.c_[x + 2000, y + 2000, f(x, y) + 2000].astype(np.float32)
    return V, F, gt


def demo_map():
    """Four synthetic scans mapped at their true poses (as tests/test_gpu_score_poses.py does), the mesh and the clean returns."""
    dev = torch.device("cuda")
    syn, rh = nl.synthetic, nl.render_helpers
    vs, md, trunc = 0.3, 40.0, 0.3
    crit = nl.criterion.Criterion(SimpleNamespace(criteria={"eiko_weight": 0.1, "sdf_weight": 10000.0, "fs_weight": 1.0, "sdf_truncation": trunc},
                                                  data_specs={"max_depth": md}))
    torch.manual_seed(777)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).to(dev)
    mu = nl.mapping.MapUpdater(vs, device=dev, reserve_nodes=400_000, reserve_rows=400_000)
    mk = lambda i, noise: syn.make_scan(seed=1000 + i, sensor_xyz=(0.5 * i, 0.05 * np.sin(0.7 * i), 0.0), yaw=0.01 * np.sin(0.5 * i), noise_std=noise)
    scans = [mk(i, 0.02) for i in range(4)]
    frames = [nl.frame.LidarFrame(i, torch.from_numpy(s[0]), torch.from_numpy(s[1]), nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(s[2])),
                                  new_keyframe=True) for i, s in enumerate(scans)]
    ms = None
    for i in range(4):
        ms = mu.create_voxels(scans[i][0], torch.from_numpy(scans[i][2]).double())
        for _ in range(6 if i else 12):
            rh.bundle_adjust_frames(frames[:i + 1], mu.embeddings, ms, dec, crit, vs, 0.5 * vs, N_rays=2048, num_iterations=25, truncation=trunc,
                                    max_voxel_hit=20, max_distance=md, learning_rate=[0.01, 0.005, 0.001], update_pose=False, update_decoder=True)
    V, F = nl.mesh.extract_mesh(dec, ms, vs, res=8)
    clean = []
    for i in range(4):
        p, _, pose = mk(i, 0.0)
        clean.append(p.astype(np.float64) @ pose[:3, :3].T.astype(np.float64) + pose[:3, 3])
    return V.cpu().numpy(), F.cpu().numpy(), np.concatenate(clean).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--samples", default="1000000,10000000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_evaluate.py measures on the GPU; none found")
    dev_card = card()
    meshes = {"height_field": height_field(), "demo_map": demo_map()}
    rows = []
    for name, (V, F, gt) in meshes.items():
        Vd, Fd, Gd = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (V, F, gt))
        for n in (int(s) for s in a.samples.split(",")):
            gpu = lambda: nl.evaluate.eval_mesh(Vd, Fd, Gd, n_samples=n, **KW)
            S = nl.evaluate.sample_surface(Vd, Fd, n, KW["seed"]).cpu().numpy()
            host = lambda: ER.eval_samples(S, gt, KW["res"], KW["threshold"], KW["truncation"])[0]
            m_gpu, m_host = gpu(), host()                      # warm-up, and the two agree on the counts
            assert all(m_gpu[k] == m_host[k] for k in ("n_cropped", "n_pred", "n_gt")), (m_gpu, m_host)
            t = {"gpu": [], "host": []}
            for _ in range(a.repeats):
                for k, f in (("gpu", gpu), ("host", host)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    f()
                    torch.cuda.synchronize()
                    t[k].append((time.perf_counter() - t0) * 1e3)
            row = dict(mesh=name, triangles=int(F.shape[0]), gt_points=int(gt.shape[0]), n_samples=n, n_pred=m_gpu["n_pred"], n_gt=m_gpu["n_gt"],
                       accuracy=round(m_gpu["accuracy"], 6), completeness=round(m_gpu["completeness"], 6), fscore=round(m_gpu["fscore"], 4))
            for k, v in t.items():
                row[k + "_ms"] = round(statistics.median(v), 2)
                row[k + "_min_max_ms"] = [round(min(v), 2), round(max(v), 2)]
            row["speedup"] = round(row["host_ms"] / row["gpu_ms"], 1)
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    out = {"card": dev_card, "params": KW, "host_threads": os.cpu_count(), "cases": rows}
    print(json.dumps(out), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_evaluate.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
