"""Time keyframes.keyframe_overlap (csrc/overlap.cu) against an eager-torch restatement on the same GPU (torch.unique per keyframe plus
torch.isin) and the NumPy restatement of tests/keyframe_ref.py, on synthetic scans: K = 8, 64 and 512 keyframes, each a full scan
(64 beams x 1563 azimuths, ~10^5 returns) or one cropped to |x|, |y|, |z| < key_distance like KeyframeGraph.insert_keyframe.  The three
run alternately in one process; every call ends in a device synchronise.  Prints the card, its power limit and one line per case
(median and min-max in ms), and checks that the three agree.

    python scripts/time_keyframe_overlap.py [--reps 7] [--numpy-reps 3] [--key-distance 20] [--json out.json]
"""
import argparse, json, os, subprocess, sys, time
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import nerfloam_b200 as nl
import keyframe_ref as KR

VS, GD = 0.3, 256 * 256 * 4


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
        return q or torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def frames(K, key_distance, n_base=64):
    """K keyframes along the street (x in [-10, 10]), cycling n_base distinct scans, plus the current scan at x = 0."""
    syn = nl.synthetic
    base = []
    for j in range(n_base + 1):
        x = -10.0 + 20.0 * j / n_base
        pts, cos, pose = syn.make_scan(seed=500 + j, sensor_xyz=(x, 0.3 * np.sin(j), 0.0), yaw=0.02 * np.sin(0.3 * j))
        if key_distance is not None:
            keep = np.all(np.abs(pts) < key_distance + 0.01, axis=1)
            pts, cos = pts[keep], cos[keep]
        base.append((torch.from_numpy(pts), torch.from_numpy(cos), torch.from_numpy(pose)))
    mk = lambda i, b: nl.frame.LidarFrame(i, b[0], b[1], nl.se3pose.OptimizablePose.from_matrix(b[2].clone()), new_keyframe=True)
    cur = mk(0, base[n_base // 2])
    return cur, [mk(1 + k, base[k % n_base]) for k in range(K)]


def matrices(fr):
    pose6 = torch.stack([f.pose.data.detach().float() for f in fr]).cuda().contiguous()
    Rt = torch.empty((len(fr), 12), dtype=torch.float32, device="cuda")
    nl._capi.check(nl._capi.lib().nl_pose_matrices(len(fr), nl._capi.ptr(pose6), nl._capi.ptr(Rt), nl._capi.stream_ptr()))
    return Rt


def torch_keys(pts, Rt):
    """keys (int64) of the points inside the grid, and the number outside: the definitions in eager torch, fp64."""
    p = pts.double()
    R, t = Rt[:9].double().view(3, 3), Rt[9:].double()
    w = torch.stack([((R[i, 0] * p[:, 0] + R[i, 1] * p[:, 1]) + R[i, 2] * p[:, 2]) + t[i] for i in range(3)], 1)
    v = torch.floor(w / VS)
    inside = ((v >= 0) & (v < GD)).all(1)
    vi = v[inside].long()
    return (vi[:, 0] << 36) | (vi[:, 1] << 18) | vi[:, 2], (~inside).sum()


def eager(cur, kfs):
    Rt = matrices([cur] + kfs)
    fk, _ = torch_keys(nl.render_helpers._frame_points(cur, "cuda"), Rt[0])
    fset = torch.unique(fk)
    shared, kv, out = [], [], []
    for k, f in enumerate(kfs):
        keys, o = torch_keys(nl.render_helpers._frame_points(f, "cuda"), Rt[k + 1])
        u = torch.unique(keys)
        shared.append(torch.isin(u, fset).sum()); kv.append(torch.tensor(u.numel(), device="cuda")); out.append(o)
    return torch.cat([torch.stack(shared), torch.stack(kv), torch.stack(out), torch.tensor([fset.numel()], device="cuda")]).cpu()


def kernel(cur, kfs):
    return nl.keyframes._overlap_counts(cur, kfs, VS, GD).cpu()


def restated(cur, kfs, Rt):
    r = KR.overlap(cur.points.numpy(), [f.points.numpy() for f in kfs], Rt, VS, GD)
    return torch.from_numpy(np.r_[r["shared"], r["kf_voxels"], r["outside"], [r["frame_voxels"]]])


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7); ap.add_argument("--numpy-reps", type=int, default=3)
    ap.add_argument("--key-distance", type=float, default=20.0); ap.add_argument("--sizes", default="8,64,512")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    info = card()
    print(f"card: {info}")
    rows = []
    for K in [int(x) for x in a.sizes.split(",")]:
        for crop in (None, a.key_distance):
            cur, kfs = frames(K, crop)
            n_pts = sum(f.num_point for f in kfs)
            Rt = matrices([cur] + kfs).cpu().numpy()
            ref = kernel(cur, kfs)                                      # warm-up: uploads every scan once (cached per frame object)
            assert torch.equal(eager(cur, kfs), ref), "eager torch and the kernel disagree"
            t = {"kernel": [], "torch": [], "numpy": []}
            for r in range(a.reps):
                ms, out = timed(lambda: kernel(cur, kfs)); t["kernel"].append(ms); assert torch.equal(out, ref)
                ms, out = timed(lambda: eager(cur, kfs)); t["torch"].append(ms); assert torch.equal(out, ref)
                if r < a.numpy_reps:
                    ms, out = timed(lambda: restated(cur, kfs, Rt)); t["numpy"].append(ms); assert torch.equal(out, ref)
            row = {"K": K, "scan": "full" if crop is None else f"cropped {crop:g} m", "points": n_pts}
            for k, v in t.items():
                row[k] = {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v)), "runs": len(v)}
            rows.append(row)
            print(f"K={K:4d} {row['scan']:>14s} points={n_pts:>9d}  " + "  ".join(
                f"{k} {row[k]['median_ms']:9.2f} ms ({row[k]['min_ms']:.2f}-{row[k]['max_ms']:.2f})" for k in t), flush=True)
            del cur, kfs
            torch.cuda.empty_cache()
    if a.json:
        json.dump({"card": info, "voxel_size": VS, "rows": rows}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
