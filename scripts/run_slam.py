"""Run a whole sequence the way the reference's `python demo/run.py config.yaml` does: the tracker and the mapper concurrent on two
CUDA streams (slam.NeRFLOAM), writing mesh/*.ply and misc/frame_poses*.txt under the output directory.

    python scripts/run_slam.py CONFIG [--data DIR] [--out DIR] [--selection current|previous|overlap] [--init-calls 12]
                               [--save-map PATH] [--base-map FILE]

CONFIG is the reference's YAML layout (base_config merged).  --data replaces data_specs.data_path; --out defaults to
log_dir/exp_name/<time> like src/loggers.py:17-18.  Prints a JSON summary: scans, keyframes, milliseconds per scan per stage (host
wall-clock of each role's steps), the wall time and the refinement times.  --save-map also writes the finished run's map, decoder,
trajectory and settings to PATH (NeRFLOAM.save_map), which scripts/localise.py localises later drives in.  --base-map FILE grows
the map in FILE with this sequence instead of starting an empty one (NeRFLOAM's base_map: the first scan placed with no pose guess,
the saved rows and the decoder held fixed); with --save-map the grown map, its trajectory the saved one followed by this sequence's.
"""
import argparse, json, os, sys
from datetime import datetime
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerfloam_b200 as nl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config")
    ap.add_argument("--data", default=None, help="sequence directory (overrides data_specs.data_path)")
    ap.add_argument("--out", default=None, help="output directory (default: log_dir/exp_name/<time>)")
    ap.add_argument("--selection", default="current", choices=nl.slam.SELECTIONS, help="the mapping window (reference: current)")
    ap.add_argument("--init-calls", type=int, default=12, help="mapping calls on the first scan")
    ap.add_argument("--save-map", default=None, metavar="PATH", help="write the finished run's map to PATH (slam.NeRFLOAM.save_map)")
    ap.add_argument("--base-map", default=None, metavar="FILE", help="grow the map in FILE (a --save-map file) with this sequence")
    a = ap.parse_args()
    cfg = nl.slam.load_config(a.config)
    if a.data is not None:
        cfg.data_specs["data_path"] = a.data
    out = a.out or os.path.join(getattr(cfg, "log_dir", "./logs"), getattr(cfg, "exp_name", "run"),
                                datetime.strftime(datetime.now(), "%Y-%m-%d-%H-%M-%S"))
    slam = nl.slam.NeRFLOAM(cfg, out, selection=a.selection, init_calls=a.init_calls, base_map=a.base_map)
    summary = slam.run()
    if a.save_map is not None:
        slam.save_map(a.save_map)
        summary["map_file"] = a.save_map
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
