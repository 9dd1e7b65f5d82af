"""Time ground.points_and_cos (csrc/ground.cu) with the vertical-structure filter off and on, and dataset.kitti.DataLoader.__getitem__,
against the NumPy restatement of tests/ground_ref.py on the host, on synthetic 64 x 1563 scans (synthetic.make_scan, ~10^5 returns) and,
with --data, on the scans of a KITTI-layout sequence.  The cases run alternately in one process; every GPU call ends in a device
synchronise.  Prints the card, its power limit and SM clock and one line per case (median and min-max in ms), and checks that the
labels agree with the restatements (tests/ground_vertical_ref.py for the filter).

    python scripts/time_ground.py [--reps 9] [--numpy-reps 3] [--scans 4] [--vertical-cell 0.2] [--profile] [--data DIR] [--json out.json]

--profile adds, in a pass of its own on the first synthetic scan, each kernel's device time per segment_ground call (torch.profiler).
"""
import argparse, json, os, subprocess, sys, tempfile, time
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import nerfloam_b200 as nl
import ground_ref as GR
import ground_vertical_ref as GV


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
        return q or torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def stats(v):
    return {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v)), "runs": len(v)}


def kernel_times(dev, params, calls=20):
    """Device time per segment_ground call, from torch.profiler's CUDA activities: {kernel or memset name: us per call}."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        nl.ground.segment_ground(dev, params)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            nl.ground.segment_ground(dev, params)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", None)
        t = e.self_cuda_time_total if t is None else t
        if t > 0:
            out[e.key] = t / calls
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def short(name):
    for k in ("k_fit<true>", "k_fit<false>", "k_fitILb1", "k_fitILb0", "k_columns", "k_vertical", "k_bin", "k_gather", "k_cos", "Memset",
              "Onesweep", "Histogram", "ExclusiveSum", "ScanKernel", "ScanInit"):
        if k in name:
            return k.replace("ILb1", "<true>").replace("ILb0", "<false>")
    return name[:40]


def write_kitti(root, scans):
    os.makedirs(os.path.join(root, "velodyne"), exist_ok=True)
    for i, p in enumerate(scans):
        np.concatenate([p, np.zeros((len(p), 1), np.float32)], 1).tofile(os.path.join(root, "velodyne", f"{i:06d}.bin"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9); ap.add_argument("--numpy-reps", type=int, default=3)
    ap.add_argument("--scans", type=int, default=4); ap.add_argument("--data", default=None); ap.add_argument("--json", default=None)
    ap.add_argument("--vertical-cell", type=float, default=0.2, help="column width (m) of the filtered case")
    ap.add_argument("--profile", action="store_true", help="also sum each kernel's device time per call (torch.profiler), filter off and on")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_ground.py needs a CUDA device")
    info = card()
    print(f"card: {info}")
    params = nl.ground.GroundParams()
    params_v = nl.ground.GroundParams(vertical_cell=a.vertical_cell)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        synthetic = [nl.synthetic.make_scan(seed=2000 + i, sensor_xyz=(0.5 * i, 0.0, 0.0))[0] for i in range(a.scans)]
        write_kitti(tmp, synthetic)
        sources = [("synthetic 64x1563", tmp)] + ([("data " + a.data, a.data)] if a.data else [])
        for name, path in sources:
            loader = nl.dataset.kitti.DataLoader(path)
            for i in range(min(a.scans, len(loader))):
                raw = loader.read_points(i)
                dev = torch.from_numpy(raw).cuda()
                ref = GR.segment(raw, params)
                kern = lambda: nl.ground.points_and_cos(dev, params)
                kern_v = lambda: nl.ground.points_and_cos(dev, params_v)
                timed(kern); timed(kern_v); timed(lambda: loader[i])    # warm-up
                t = {"points_and_cos (device input)": [], "points_and_cos, vertical filter on": [], "__getitem__ (file to CPU tensors)": [],
                     "restatement (host)": []}
                for r in range(a.reps):
                    ms, out = timed(kern); t["points_and_cos (device input)"].append(ms)
                    ms, out = timed(kern_v); t["points_and_cos, vertical filter on"].append(ms)
                    ms, item = timed(lambda: loader[i]); t["__getitem__ (file to CPU tensors)"].append(ms)
                    if r < a.numpy_reps:
                        ms, _ = timed(lambda: GR.segment(raw, params)); t["restatement (host)"].append(ms)
                g = int((ref["label"] == 1).sum())
                agree = float((nl.ground.segment_ground(dev, params).label.cpu().numpy() == ref["label"]).mean())
                ref_v = GV.segment(raw, params_v)
                gv = nl.ground.segment_ground(dev, params_v)
                agree_v = float((gv.label.cpu().numpy() == ref_v["label"]).mean())
                n_vert = int(gv.vertical.sum())
                row = {"source": name, "scan": i, "points": int(len(raw)), "ground": g, "label_agreement": agree, "vertical": n_vert,
                       "ground_filtered": int(ref_v["label"].sum()), "label_agreement_filtered": agree_v}
                row.update({k: stats(v) for k, v in t.items()})
                rows.append(row)
                print(f"{name} scan {i}: {len(raw)} points, {g} ground, labels agree {agree:.6f}; filtered {n_vert} vertical, "
                      f"{row['ground_filtered']} ground, labels agree {agree_v:.6f}  " + "  ".join(
                    f"{k} {row[k]['median_ms']:.3f} ms ({row[k]['min_ms']:.3f}-{row[k]['max_ms']:.3f})" for k in t), flush=True)
        kt = None
        if a.profile:                                                    # in a pass of its own: tracing slows the host
            dev = torch.from_numpy(synthetic[0]).cuda()
            kt = {"off": kernel_times(dev, params), "on": kernel_times(dev, params_v)}
            for mode, t in kt.items():
                merged = {}
                for k, v in t.items():
                    merged[short(k)] = merged.get(short(k), 0.0) + v
                print(f"device time per segment_ground call, filter {mode}: {sum(t.values()):.1f} us  " +
                      "  ".join(f"{k} {v:.1f}" for k, v in merged.items()), flush=True)
    if a.json:
        json.dump({"card": info, "rows": rows, "device_us_per_call": kt}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
