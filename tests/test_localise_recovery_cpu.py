"""The Localiser's recovery of lost scans without a GPU: the lost rule and its history window, recovery_specs validation, and the
fallback order of run() with tracking, scoring, relocalise and relocalise_global replaced by stubs of a scripted drive."""
import importlib
import json
import math

import numpy as np
import pytest
import torch

from test_localise_cpu import _saved, _Stream

localise = importlib.import_module("nerf-loam_b200.localise")
slam = importlib.import_module("nerf-loam_b200.slam")
se3 = importlib.import_module("nerf-loam_b200.se3pose")
globalloc = importlib.import_module("nerf-loam_b200.globalloc")
OFFSET = importlib.import_module("nerf-loam_b200.frame").POSE_OFFSET

SPECS = dict(localise.RECOVERY_SPECS)


# -- the rule -----------------------------------------------------------------------------------------------------------------
def test_lost_rule():
    s = dict(SPECS, lost_hit_fraction=0.5, lost_loss_ratio=4.0)
    assert not localise.is_lost(1.0, 0.9, [1.0], s)
    assert localise.is_lost(1.0, 0.49, [1.0], s)                      # too few hits
    assert not localise.is_lost(1.0, 0.5, [1.0], s)                   # the bound itself passes
    assert localise.is_lost(float("nan"), 0.9, [1.0], s) and localise.is_lost(float("inf"), 0.9, [1.0], s)
    assert not localise.is_lost(4.0, 0.9, [1.0], s) and localise.is_lost(4.0001, 0.9, [1.0], s)  # strictly above ratio x median
    assert not localise.is_lost(1e9, 0.9, [], s)                      # no history: only the hit and finiteness tests
    assert localise.is_lost(float("nan"), 0.9, [], s)
    # the median of an even window is the mean of its middle two
    assert not localise.is_lost(10.0, 0.9, [1.0, 2.0, 3.0, 4.0], s) and localise.is_lost(10.01, 0.9, [1.0, 2.0, 3.0, 4.0], s)


def test_lost_rule_history_window():
    """Only the last HISTORY accepted losses count."""
    s = dict(SPECS, lost_loss_ratio=4.0)
    assert localise.HISTORY == 10
    old_high = [100.0] * 5 + [1.0] * 10                               # window: ten 1s
    assert localise.is_lost(5.0, 0.9, old_high, s)
    old_low = [1.0] * 5 + [100.0] * 10                                # window: ten 100s
    assert not localise.is_lost(5.0, 0.9, old_low, s)
    nine = [100.0] * 6 + [1.0] * 9                                    # window: one 100 and nine 1s
    assert localise.is_lost(5.0, 0.9, nine, s)
    mixed = [1.0] * 5 + [100.0] * 5 + [1.0] * 5                       # window: five 100s, five 1s -> median 50.5
    assert not localise.is_lost(200.0, 0.9, mixed, s) and localise.is_lost(203.0, 0.9, mixed, s)


# -- settings -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("specs,match", [
    ({"lost_hit": 0.5}, "lost_hit"),
    ({"lost_hit_fraction": float("nan")}, "lost_hit_fraction"),
    ({"lost_hit_fraction": 1.5}, "lost_hit_fraction"),
    ({"lost_hit_fraction": -0.1}, "lost_hit_fraction"),
    ({"lost_hit_fraction": "0.5"}, "lost_hit_fraction"),
    ({"lost_loss_ratio": float("inf")}, "lost_loss_ratio"),
    ({"lost_loss_ratio": 0.5}, "lost_loss_ratio"),
    ({"global_interval": 0}, "global_interval"),
    ({"global_interval": 2.5}, "global_interval"),
    ({"global_interval": True}, "global_interval"),
    ({"global_interval": None}, "global_interval"),
])
def test_recovery_specs_rejected(specs, match):
    with pytest.raises(ValueError, match=match):
        localise.recovery_specs(specs)
    with pytest.raises(ValueError, match=match):
        localise.Localiser(_saved(), _Stream(2), config={"recovery_specs": specs})


def test_recovery_specs_accepted():
    assert localise.Localiser(_saved(), _Stream(2)).recovery is None                            # off without the key
    assert localise.Localiser(_saved(), _Stream(2), config={"recovery_specs": {}}).recovery == SPECS
    got = localise.Localiser(_saved(), _Stream(2), config={"recovery_specs": {"global_interval": np.int64(3), "lost_loss_ratio": 2}}).recovery
    assert got == dict(SPECS, global_interval=3, lost_loss_ratio=2.0) and type(got["global_interval"]) is int
    assert localise.recovery_specs({"lost_hit_fraction": 0.0, "lost_loss_ratio": 1.0, "global_interval": 1.0})["global_interval"] == 1
    with pytest.raises(ValueError, match="dict"):
        localise.Localiser(_saved(), _Stream(2), config={"recovery_specs": None})


# -- the fallback order on a scripted drive -----------------------------------------------------------------------------------
# Scan i lies at x = TRUTH[i] (metres, no rotation).  The stub tracker converges to the truth from within BASIN of it and ends 100 m
# past its start otherwise; the stub score gives loss 1 within 0.1 m of the truth and 50 elsewhere.  Scan 8 is one the map cannot
# explain: tracking hits nothing, its score is NaN with no hits, and neither search places it.
TRUTH = [0.0, 1.0, 4.0, 5.0, 20.0, 21.0, 22.0, 23.0, None, 24.0]
BASIN = 1.5
GLOBAL = {4: None, 6: "truth", 8: None}                     # what relocalise_global finds per scan
LOCAL_NO_HIT = {6, 8}                                       # where relocalise hits nothing; elsewhere out of reach it settles wrongly
WANT = ["tracked", "tracked", "local", "tracked", "lost", "lost", "global", "tracked", "lost", "tracked"]


def _x(pose):
    return float(pose.data.detach().reshape(-1)[0]) - OFFSET


def _pose(x):
    return se3.OptimizablePose(torch.tensor([OFFSET + x, OFFSET, OFFSET, 0.0, 0.0, 0.0]))


class _Drive:
    def __init__(self, monkeypatch):
        self.log = []
        monkeypatch.setattr(slam.rh, "track_frame", self.track_frame)
        monkeypatch.setattr(localise.Localiser, "score", lambda loc, frame: self.score(frame))
        monkeypatch.setattr(localise, "relocalise", self.relocalise)
        monkeypatch.setattr(localise, "relocalise_global", self.relocalise_global)
        # Tracking's stage clock also records the CUDA stream it ran on
        monkeypatch.setattr(slam.Tracking, "_tick", lambda tr, stage, t0: tr.times.setdefault(stage, []).append(0.0))

    def track_frame(self, pose, frame, map_state, decoder, crit, voxel_size, N_rays, step_size, num_iterations, *a, **kw):
        x, truth = _x(pose), TRUTH[frame.index]
        self.log.append(("track", frame.index, num_iterations, round(x, 3)))
        if truth is None:
            return _pose(x), None
        return (_pose(truth) if abs(x - truth) < BASIN else _pose(x + 100.0)), torch.ones(4, dtype=torch.bool)

    def score(self, frame):
        truth = TRUTH[frame.index]
        if truth is None:
            return float("nan"), 0.0
        return (1.0 + 0.01 * frame.index if abs(_x(frame.pose) - truth) < 0.1 else 50.0), 0.9

    def relocalise(self, frame, guess, *a, xy_range=2.0, **kw):
        x, truth = _x(guess), TRUTH[frame.index]
        self.log.append(("local", frame.index, round(x, 3)))
        if frame.index in LOCAL_NO_HIT:
            return _pose(x), None, None
        return (_pose(truth) if abs(x - truth) <= xy_range else _pose(x + 0.5)), torch.ones(4, dtype=torch.bool), None

    def relocalise_global(self, frame, *a, anchors, **kw):
        self.log.append(("global", frame.index))
        found = GLOBAL.get(frame.index)
        diag = globalloc.Diagnostics(10, None, None, None, [], {"coarse": 0.0, "fine": 0.0, "refine": 0.0})
        if found is None:
            return globalloc.GlobalResult(_pose(0.0), None, float("nan"), diag)
        return globalloc.GlobalResult(_pose(TRUTH[frame.index]), torch.ones(4, dtype=torch.bool), 1.0, diag)


def _run(monkeypatch, tmp_path, specs):
    drive = _Drive(monkeypatch)
    s = _saved()
    config = {"tracker_specs": {"num_iterations": 7}}
    if specs is not None:
        config["recovery_specs"] = specs
    loc = localise.Localiser(s, _Stream(len(TRUTH)), config=config, out_dir=str(tmp_path))
    res = loc.run(init_pose=np.eye(4))
    return drive, loc, res


def test_fallback_order(monkeypatch, tmp_path):
    drive, loc, res = _run(monkeypatch, tmp_path, {"global_interval": 2})
    assert res.status == WANT
    N, N5 = 7, 35
    assert drive.log == [
        ("track", 1, N5, 0.0),                  # no motion prior yet
        ("track", 2, N, 2.0),                   # constant velocity: 2 m short of the truth after a gap, outside the basin
        ("local", 2, 2.0),                      # local first, around the constant-velocity guess; accepted
        ("track", 3, N5, 4.0),                  # the motion model restarts from the re-placed scan
        ("track", 4, N, 6.0),                   # a restart 14 m away
        ("local", 4, 6.0),                      # settles wrongly: rejected by its score, falls through
        ("global", 4),                          # places nothing: lost
        ("track", 5, N5, 5.0),                  # tracked from scan 3, the last accepted scan, not from the lost scan 4
        ("local", 5, 5.0),                      # rejected; the global search ran one scan ago (global_interval 2): lost
        ("track", 6, N5, 5.0),
        ("local", 6, 5.0),                      # no hit
        ("global", 6),                          # two scans later the global search runs again and places it
        ("track", 6, N5, 22.0),                 # ... tracked from the placement like the first scan
        ("track", 7, N5, 22.0),
        ("track", 8, N, 24.0),                  # a scan the map cannot explain
        ("local", 8, 24.0),
        ("global", 8),                          # a new run of lost scans: the global search is allowed at once
        ("track", 9, N5, 23.0),                 # from scan 7, not from the lost scan 8
    ]
    x = res.poses[:, 0, 3].numpy()
    want_x = [0, 1, 4, 5, 106, 105, 22, 23, 24, 24]           # lost scans keep their tracked pose (scan 8: the guess)
    assert np.allclose(x, want_x, atol=1e-3), x
    loss = res.loss.numpy()
    assert loss[4] == 50.0 and loss[5] == 50.0 and math.isnan(loss[8]) and res.hit_fraction[8] == 0.0   # and their tracked scores
    assert loss[2] == pytest.approx(1.02) and loss[6] == pytest.approx(1.06)                           # re-placed: their own score
    assert loc.tracker.rel_pose is not None and loc.tracker.last_frame.index == 9
    lines = (tmp_path / "frame_status.txt").read_text().splitlines()
    assert lines == [f"{i} {s}" for i, s in enumerate(WANT)]
    sm = loc.summary(res)
    json.dumps(sm)
    assert sm["recovery"]["counts"] == {"tracked": 5, "local": 1, "global": 1, "lost": 3}
    assert set(sm["recovery"]["ms"]) == {"local", "global"} and all(v >= 0 for v in sm["recovery"]["ms"].values())
    assert len(loc.times["recover_local"]) == 5 and len(loc.times["recover_global"]) == 3
    assert not set(sm["ms_per_scan"]) & {"recover_local", "recover_global", "place", "polish"}


def test_global_interval_one_searches_every_lost_scan(monkeypatch, tmp_path):
    drive, _, res = _run(monkeypatch, tmp_path, {"global_interval": 1})
    assert [e[1] for e in drive.log if e[0] == "global"] == [4, 5, 6, 8]
    assert res.status == WANT


def test_wide_interval_leaves_later_lost_scans_to_the_local_step(monkeypatch, tmp_path):
    """Once scan 4's search fails, nothing is accepted again, so no later scan of the run is searched globally: every later scan is
    tracked from scan 3 (5 m), far outside the basin, and is lost."""
    drive, _, res = _run(monkeypatch, tmp_path, {"global_interval": 10})
    assert [e[1] for e in drive.log if e[0] == "global"] == [4]
    assert res.status == WANT[:4] + ["lost"] * 6
    assert [e[3] for e in drive.log if e[0] == "track" and e[1] > 4] == [5.0] * 5


def test_recovery_off_is_the_plain_tracker(monkeypatch, tmp_path):
    drive, loc, res = _run(monkeypatch, tmp_path, None)
    assert res.status is None and all(e[0] == "track" for e in drive.log)
    assert not (tmp_path / "frame_status.txt").exists() and "recovery" not in loc.summary(res)
    assert (tmp_path / "frame_poses.txt").exists()
    assert not any(k.startswith("recover_") for k in loc.times)
