"""Recovering lost scans while localising in a saved map (localise.Localiser with recovery_specs): the street drive of
tests/test_gpu_localise.py (12 scans 0.5 m apart, synthetic.make_street_scan) mapped by slam.NeRFLOAM with the true poses and KITTI's
values and saved to a temporary directory, then three second passes (shifted 0.5 m and turned 10 degrees):

  * healthy: 14 scans, localised with recovery off and on alternately: host ms per scan for track and score (the lost rule reuses
    the score, so tracking should not change), and whether any scan was flagged;
  * gap: the same pass with scans 5-7 dropped, recovery on: ms per local recovery (relocalise + the score of its pose);
  * jump: 6 scans, then a restart 4.7 m ahead, 1.9 m aside and turned 40 degrees, recovery on: ms per global recovery (the first
    scan's search and tracking + the score of its pose).

Prints one JSON line with the card's name, power limit and SM clock (read in the same run), medians and min-max over the repeats
(after one warm-up round that is not kept), the status counts and the worst pose error of each drive.

    python scripts/time_localise_recovery.py [--repeats 3]
"""
import argparse
import json
import math
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import nerfloam_b200 as nl  # noqa: E402
from time_localise import Stream, config, scan, stats  # noqa: E402
from time_track_batch import card  # noqa: E402

MAP_SCANS = 12
SHIFT, TURN = (0.3, 0.4), math.radians(10.0)


def drives():
    second = [scan(i, 6000 + i, SHIFT, TURN) for i in range(14)]
    jump = second[:6] + [scan(k, 7000 + k, (8.0, -1.5), TURN + math.radians(40.0)) for k in range(6)]
    return {"healthy": second, "gap": [s for i, s in enumerate(second) if i not in (5, 6, 7)], "jump": jump}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    runs = {"healthy_off": [], "healthy_on": [], "gap": [], "jump": []}
    with tempfile.TemporaryDirectory() as tmp:
        s = nl.slam.NeRFLOAM(config(), os.path.join(tmp, "run"), data_stream=Stream([scan(i, 2000 + i) for i in range(MAP_SCANS)], True))
        s.run()
        path = os.path.join(tmp, "run.map")
        s.save_map(path)
        del s
        saved = nl.slam.load_map(path)
        d = drives()
        for r in range(a.repeats + 1):                                  # the first round warms every shape up and is not kept
            for name, scans, on in (("healthy_off", d["healthy"], False), ("healthy_on", d["healthy"], True), ("gap", d["gap"], True),
                                    ("jump", d["jump"], True)):
                torch.cuda.synchronize()
                loc = nl.localise.Localiser(saved, Stream(scans, False), generator=torch.Generator().manual_seed(r),
                                            config={"recovery_specs": {}} if on else None)
                res = loc.run()
                torch.cuda.synchronize()
                truth = torch.from_numpy(np.stack([p[2] for p in scans]))
                sm = loc.summary(res)
                sm["max_translation_error_m"] = float((res.poses[:, :3, 3] - truth[:, :3, 3]).norm(dim=-1).max())
                sm["max_rotation_error_fro"] = float(torch.linalg.matrix_norm(res.poses[:, :3, :3] - truth[:, :3, :3]).max())
                sm["recover_ms"] = {k: list(loc.times.get(f"recover_{k}", [])) for k in ("local", "global")}
                if r:
                    runs[name].append(sm)
                del loc, res
    out = {"bench": "localise_recovery", "card": card(), "map_scans": MAP_SCANS, "repeats": a.repeats,
           "scans": {k: len(v) for k, v in drives().items()}, "specs": nl.localise.RECOVERY_SPECS}
    for name in ("healthy_off", "healthy_on"):
        rs = runs[name]
        out[name] = {"track_ms_per_scan": stats([x["ms_per_scan"]["track"] for x in rs]),
                     "score_ms_per_scan": stats([x["ms_per_scan"]["score"] for x in rs]),
                     "counts": [x.get("recovery", {}).get("counts") for x in rs],
                     "max_translation_error_m": max(x["max_translation_error_m"] for x in rs),
                     "max_rotation_error_fro": max(x["max_rotation_error_fro"] for x in rs)}
    for name, step in (("gap", "local"), ("jump", "global")):
        rs = runs[name]
        every = [ms for x in rs for ms in x["recover_ms"][step]]
        out[name] = {f"{step}_recovery_ms": stats(every) if every else None, "counts": [x["recovery"]["counts"] for x in rs],
                     "recover_ms": [x["recover_ms"] for x in rs],
                     "max_translation_error_m": max(x["max_translation_error_m"] for x in rs),
                     "max_rotation_error_fro": max(x["max_rotation_error_fro"] for x in rs)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
