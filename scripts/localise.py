"""Localise a drive in a saved map (localise.Localiser): the first scan placed with no pose guess, the rest tracked against the frozen
map, writing frame_poses.txt.

    python scripts/localise.py MAP --data DIR [--out DIR] [--octree host|device] [--start 0] [--end -1] [--read-offset 1]
                               [--recover | --recovery-specs JSON] [--changes | --change-specs JSON]

MAP is a file written by `scripts/run_slam.py --save-map` (slam.NeRFLOAM.save_map).  DIR is read with the dataset loader the map's run
used (its data_specs' depth gates, no poses).  Prints a JSON summary: scans, the map file's load time, median host ms per scan for
load, track and score, the first scan's placement (ms, per-stage ms, placements searched) and the median loss.  --recover turns on the
recovery of lost scans with its default settings (localise.RECOVERY_SPECS), --recovery-specs '{"global_interval": 3}' with those
overridden; the summary then has the scans per status and the ms of a local and a global step, and --out gets frame_status.txt.
--changes reports what changed since the map was saved (localise's change detection with changes.CHANGE_SPECS), --change-specs
'{"min_votes": 5}' with those overridden; the summary then has the voxel totals and --out gets changes_removed.ply, changes_added.ply
and changes.txt.
"""
import argparse, importlib, json, os, sys, time
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerfloam_b200 as nl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("map", help="map file (scripts/run_slam.py --save-map)")
    ap.add_argument("--data", required=True, help="sequence directory in the layout of the map's dataset")
    ap.add_argument("--out", default=None, help="where frame_poses.txt goes (default: not written)")
    ap.add_argument("--octree", default="host", choices=["host", "device"], help="where the map's octree is restored")
    ap.add_argument("--start", type=int, default=0)
    ap.add_argument("--end", type=int, default=-1)
    ap.add_argument("--read-offset", type=int, default=1)
    ap.add_argument("--recover", action="store_true", help="recover lost scans with the default recovery_specs")
    ap.add_argument("--recovery-specs", type=json.loads, default=None, metavar="JSON",
                    help="recover lost scans with these recovery_specs over the defaults (implies --recover)")
    ap.add_argument("--changes", action="store_true", help="report changes against the map with the default change_specs")
    ap.add_argument("--change-specs", type=json.loads, default=None, metavar="JSON",
                    help="report changes with these change_specs over the defaults (implies --changes)")
    a = ap.parse_args()
    specs = a.recovery_specs if a.recovery_specs is not None else ({} if a.recover else None)
    change = a.change_specs if a.change_specs is not None else ({} if a.changes else None)
    config = {}
    if specs is not None:
        config["recovery_specs"] = specs
    if change is not None:
        config["change_specs"] = change
    t0 = time.perf_counter()
    saved = nl.slam.load_map(a.map, octree=a.octree)
    ds = saved.config["data_specs"]
    loader = importlib.import_module(f"nerf-loam_b200.dataset.{saved.config['dataset']}").DataLoader
    data = loader(a.data, use_gt=False, max_depth=ds.get("max_depth", -1), min_depth=ds.get("min_depth", -1))
    loc = nl.localise.Localiser(saved, data, out_dir=a.out, config=config or None)
    torch.cuda.synchronize()
    loc.load_ms = (time.perf_counter() - t0) * 1e3           # the map file read and restored, and the loader set up
    summary = loc.summary(loc.run(a.start, a.end, a.read_offset))
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
