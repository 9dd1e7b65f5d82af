"""A miniature of the reference's SLAM loop (src/tracking.py:110-148, src/mapping.py:96-170) on synthetic scans, run entirely through the
drop-in API: per scan  track_frame (captured graph) -> bundle_adjust_frames over the keyframe window (captured graph) -> incremental
map update (MapUpdater) -> publication to the tracker (share.SharedMap); at the end GPU marching cubes.
BASELINE.json config 2 ("KITTI seq 00 tracking+mapping incremental loop") / config 3 ("... + marching cubes") in spirit; prints a
JSON summary (per-stage ms per scan, trajectory error against the synthetic ground truth, and under `reconstruction` the final mesh
scored by evaluate.eval_mesh against the scans' noise-free returns at the true poses).

The mapping window goes through keyframes.KeyframeGraph (a keyframe every second scan, window_size 4): `--selection previous` (the
default) optimises the last four keyframes, `--selection overlap` the four whose voxels overlap the tracked scan's most.  `--path loop`
drives out along +x and back over the same ground (fresh noise seeds), so the last scans revisit the first ones' place.

    python scripts/demo_slam.py [--scans 12] [--spacing 0.5] [--octree host|device] [--selection previous|overlap] [--path line|loop]
                                [--json out.json]

`--data DIR --dataset kitti|maicity` runs the same loop on a recorded sequence through dataset.<name>.DataLoader (points and pointsCos
from the GPU ground segmentation, ground.py): the first scan takes the loader's get_init_pose, every later one is tracked; the
trajectory error is reported against the pose file when it exists, and the `reconstruction` block (synthetic scans only) is left out.
`--scans` then caps the number of scans (default: all).  `--vertical-cell W` (with --data) turns on the ground segmentation's
vertical-structure filter with W-metre columns (GroundParams.vertical_cell; 0, the default, leaves it off).

`--final-iter` runs the mapper's key-scan refinement (mapper_specs.final_iter, src/mapping.py:154-164) before the final mesh:
render_helpers.refine_map over the keyframe graph with KITTI's values (window 4, 2 x 2048 rays per keyframe, 25 iterations, embedding
rate 0.01, len(keyframes) + 1 passes).  The JSON then carries `refine_ms` and, for synthetic scans, `reconstruction_before_refine`
next to `reconstruction` (the refined map's mesh).
"""
import argparse, json, os, sys, time
from types import SimpleNamespace
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerfloam_b200 as nl


def load_sequence(a):
    """(scans [(points, pointsCos)] as numpy, true poses or None, the first scan's pose) of --data through its DataLoader; poses carry
    the offset LidarFrame adds to a supplied pose."""
    import importlib
    loader = importlib.import_module("nerf-loam_b200.dataset." + a.dataset).DataLoader
    has_poses = os.path.exists(os.path.join(a.data, loader.pose_file))
    gp = nl.ground.GroundParams(vertical_cell=a.vertical_cell) if a.vertical_cell > 0 else None
    data = loader(a.data, use_gt=has_poses, ground_params=gp)
    a.scans = len(data) if a.scans is None else min(a.scans, len(data))
    if a.scans < 2:
        raise SystemExit(f"{a.data}: need at least 2 scans, found {len(data)}")
    scans = []
    for i in range(a.scans):
        _, points, pointcos, _ = data[i]
        scans.append((points.numpy(), pointcos.numpy()))
    def shifted(pose):
        pose = np.array(pose, dtype=np.float32)
        pose[:3, 3] += nl.frame.POSE_OFFSET
        return torch.from_numpy(pose)
    gt = [shifted(data.get_init_pose(i)) for i in range(a.scans)] if has_poses else None
    return scans, gt, shifted(data.get_init_pose(0))


def trajectory_errors(est, gt):
    err = [float((e[:3, 3] - g[:3, 3]).norm()) for e, g in zip(est, gt)]
    rot = [float(torch.linalg.matrix_norm(e[:3, :3] - g[:3, :3])) for e, g in zip(est, gt)]
    return {"translation_error_m": {"mean": float(np.mean(err[1:])), "max": float(np.max(err[1:])), "last": err[-1]},
            "rotation_error_fro": {"mean": float(np.mean(rot[1:])), "max": float(np.max(rot[1:]))},
            "per_scan_translation_error_m": [round(e, 4) for e in err]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=None, help="number of scans (default 12, or the whole sequence with --data)"); ap.add_argument("--spacing", type=float, default=0.5)
    ap.add_argument("--init-calls", type=int, default=12); ap.add_argument("--json", default=None)
    ap.add_argument("--ray-selection", default="device", choices=["device", "host"])
    ap.add_argument("--octree", default="host", choices=["host", "device"], help="where MapUpdater keeps the octree (the `update` stage)")
    ap.add_argument("--selection", default="previous", choices=["previous", "overlap"], help="KeyframeGraph.select_optimize_targets method")
    ap.add_argument("--path", default="line", choices=["line", "loop"], help="line: out along +x; loop: out and back over the same ground")
    ap.add_argument("--data", default=None, help="a KITTI- or MaiCity-layout sequence directory instead of synthetic scans")
    ap.add_argument("--dataset", default="kitti", choices=["kitti", "maicity"], help="layout of --data")
    ap.add_argument("--vertical-cell", type=float, default=0.0,
                    help="with --data: column width (m) of the ground segmentation's vertical-structure filter; 0 = off")
    ap.add_argument("--final-iter", action="store_true", help="refine the map over every keyframe (refine_map) before the final mesh")
    a = ap.parse_args()
    if a.vertical_cell != 0.0 and a.data is None:
        ap.error("--vertical-cell applies to --data")
    dev = torch.device("cuda"); syn, rh = nl.synthetic, nl.render_helpers
    vs, md, trunc = 0.3, 40.0, 0.3
    crit = nl.criterion.Criterion(SimpleNamespace(criteria={"eiko_weight": 0.1, "sdf_weight": 10000.0, "fs_weight": 1.0, "sdf_truncation": trunc},
                                                  data_specs={"max_depth": md}))
    torch.manual_seed(777)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).to(dev)
    mu = nl.mapping.MapUpdater(vs, device=dev, reserve_nodes=400_000, reserve_rows=400_000, octree=a.octree)   # embeddings start at zero like the reference
    shared = nl.share.SharedMap(lambda: nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).to(dev))
    mu.readers = shared
    if a.data is None:
        a.scans = 12 if a.scans is None else a.scans
        drive = [syn.path_pose(i, a.scans, a.spacing, a.path) for i in range(a.scans)]
        scans = [syn.make_scan(seed=1000 + i, sensor_xyz=xyz, yaw=yaw) for i, (xyz, yaw) in enumerate(drive)]
        gt = [torch.from_numpy(s[2]) for s in scans]
        init = gt[0]
    else:
        scans, gt, init = load_sequence(a)
    T = {k: [] for k in ("track", "map", "update", "publish")}
    def tick():
        torch.cuda.synchronize(); return time.perf_counter()
    mk = lambda i, pose: nl.frame.LidarFrame(i, torch.from_numpy(scans[i][0]), torch.from_numpy(scans[i][1]), pose, new_keyframe=True)
    lr = [0.01, 0.005, 0.001]
    ba = lambda fr, upd_dec, it=25: rh.bundle_adjust_frames(fr, mu.embeddings, ms, dec, crit, vs, 0.5 * vs, N_rays=2048, num_iterations=it, truncation=trunc,
                                                            max_voxel_hit=20, max_distance=md, learning_rate=lr, update_pose=True, update_decoder=upd_dec,
                                                            ray_selection=a.ray_selection)
    # ---- first scan: map it, then train on it while "waiting for the tracker" (mapping.py:100-108) ----
    f0 = mk(0, nl.se3pose.OptimizablePose.from_matrix(init.clone()))
    t0 = tick()
    ms = mu.create_voxels(scans[0][0], init)
    t_update0 = (tick() - t0) * 1e3
    # key_distance = max_depth: every return of these scans lies inside it, so a keyframe holds the whole scan
    kg = nl.keyframes.KeyframeGraph(window_size=4, keyframe_gap=2 * a.spacing, key_distance=md, n_rays=2048, voxel_size=vs)
    kg.insert_keyframe(f0)
    est, window = [init.clone()], []
    t0 = tick()
    for _ in range(a.init_calls):
        ba([f0], True)
    t_init = (tick() - t0) * 1e3
    shared.publish(ms, dec)
    rel = None
    for i in range(1, a.scans):
        last = est[-1]
        guess = last @ rel if rel is not None else last.clone()                            # constant-velocity model (tracking.py:112-117)
        fr = mk(i, nl.se3pose.OptimizablePose.from_matrix(guess.clone()))
        # KITTI's tracking rate (0.06, /3 from the third scan on).  The first tracked scan has no motion prior: 125 iterations, and a rate of
        # 0.01 because frame index < 2 doubles it -- 0.12 m Adam steps on 0.3 m voxels are bistable (scripts/sweep_tracking_lr.py)
        t0 = tick()
        m_t, dec_t, slot = shared.acquire()
        pose, hit = rh.track_frame(fr.pose, fr, m_t, dec_t, crit, vs, N_rays=2048, step_size=0.2 * vs, num_iterations=25 if rel is not None else 125,
                                   truncation=trunc, learning_rate=0.06 if rel is not None else 0.01, max_voxel_hit=20, max_distance=md, ray_selection=a.ray_selection)
        shared.release(slot)
        T["track"].append((tick() - t0) * 1e3)
        if hit is None:
            pose = nl.se3pose.OptimizablePose.from_matrix(guess.clone())
        fr.pose = nl.se3pose.OptimizablePose(pose.data.detach().cpu().clone())
        t0 = tick()
        window = kg.select_optimize_targets(fr, a.selection)                               # window_size 4 + the tracked frame
        ba(window, upd_dec=(i < 5))                                                          # freeze_frame 5
        T["map"].append((tick() - t0) * 1e3)
        t0 = tick()
        ms = mu.create_voxels(scans[i][0], fr.get_pose().detach())
        T["update"].append((tick() - t0) * 1e3)
        t0 = tick()
        shared.publish(ms, dec)
        T["publish"].append((tick() - t0) * 1e3)
        cur = fr.get_pose().detach().cpu()
        rel = torch.linalg.inv(last) @ cur
        est.append(cur)
        if i % 2 == 0:
            kg.insert_keyframe(fr)
    # the map against the scans' noise-free returns at the true poses, in world coordinates (with the 2000 m offset, like the mesh)
    def score(verts, faces):
        clean = []
        for i, (xyz, yaw) in enumerate(drive):
            p, _, pose = syn.make_scan(seed=1000 + i, sensor_xyz=xyz, yaw=yaw, noise_std=0.0)
            clean.append(p.astype(np.float64) @ pose[:3, :3].T.astype(np.float64) + pose[:3, 3])
        t0 = tick()
        recon = nl.evaluate.eval_mesh(verts, faces, np.concatenate(clean).astype(np.float32), n_samples=1_000_000, res=0.05, threshold=0.1,
                                      truncation=0.5, seed=0)
        recon["ms"] = (tick() - t0) * 1e3
        return recon
    refine = {}
    if a.final_iter:
        if a.data is None:
            refine["reconstruction_before_refine"] = score(*nl.mesh.extract_mesh(dec, ms, vs, res=8))
        t0 = tick()
        rh.refine_map(kg, mu.embeddings, ms, dec, crit, vs, 0.5 * vs, N_rays=2 * 2048, num_iterations=25, truncation=trunc, max_voxel_hit=20,
                      max_distance=md, learning_rate=lr[0])
        refine = {"refine_ms": (tick() - t0) * 1e3, "refine_passes": len(kg.keyframe_graph) + 1, **refine}
    t0 = tick()
    verts, faces = nl.mesh.extract_mesh(dec, ms, vs, res=8)
    t_mesh = (tick() - t0) * 1e3
    if a.data is not None:
        out = {"data": a.data, "dataset": a.dataset, "scans": a.scans, "octree": a.octree, "selection": a.selection,
               **({"vertical_cell": a.vertical_cell} if a.vertical_cell > 0 else {}),
               "last_window_scans": [f.index for f in window], "ground_points": [int((s[1] < 1).sum()) for s in scans],
               "ms_per_scan": {k: float(np.median(v)) for k, v in T.items()}, "ms_first_tracked_scan": T["track"][0], "ms_first_update": t_update0,
               "init_mapping_ms": t_init, "mesh": {"ms": t_mesh, "vertices": int(verts.shape[0]), "triangles": int(faces.shape[0])},
               "map": {"nodes": ms.n_nodes, "embedding_rows": int(mu.n_rows), "last_update": mu.last_update}, **refine}
        if gt is not None:
            out.update(trajectory_errors(est, gt))
        print(json.dumps(out))
        if a.json:
            json.dump(out, open(a.json, "w"), indent=1)
        return
    recon = score(verts, faces)
    errors = trajectory_errors(est, gt)
    out = {"scans": a.scans, "spacing_m": a.spacing, "octree": a.octree, "selection": a.selection, "path": a.path,
           "last_window_scans": [f.index for f in window], "translation_error_m": errors["translation_error_m"],
           "rotation_error_fro": errors["rotation_error_fro"],
           "ms_per_scan": {k: float(np.median(v)) for k, v in T.items()}, "ms_first_tracked_scan": T["track"][0], "ms_first_update": t_update0, "init_mapping_ms": t_init,
           "mesh": {"ms": t_mesh, "vertices": int(verts.shape[0]), "triangles": int(faces.shape[0])},
           "map": {"nodes": ms.n_nodes, "embedding_rows": int(mu.n_rows), "last_update": mu.last_update},
           "reconstruction": recon, **refine,
           "per_scan_translation_error_m": errors["per_scan_translation_error_m"]}
    print(json.dumps(out))
    if a.json:
        json.dump(out, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
