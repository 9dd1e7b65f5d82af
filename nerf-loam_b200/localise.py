"""Localise a sequence in a saved map: the first scan placed with no pose guess, every later one tracked against the frozen map.

    saved = slam.load_map("run.map")                       # written by slam.NeRFLOAM.save_map after run()
    loc = Localiser(saved, dataset.kitti.DataLoader(seq_dir, max_depth=40, min_depth=5), out_dir=out)
    result = loc.run()                                     # poses, losses, hit fractions; out/frame_poses.txt

  * First scan: globalloc.relocalise_global, anchored on the saved trajectory (POSE_OFFSET added back, since the map carries it),
    then tracked from that placement like a scan without a motion prior (num_iterations x 5) at the later scans' rate.  An explicit
    init_pose skips the search and that tracking.  If no placement hits the map, run() raises: there is no constant pose to fall back
    to.
  * Later scans: slam.Tracking, the reference's tracker rules unchanged (tracking.py:98-144): the constant-velocity guess,
    num_iterations x 5 while there is no relative pose, the guess when no ray hits.  Tracking reads the map through FrozenMap, which
    serves SharedMap's acquire / release over the one loaded map.
  * The map never changes: no create_voxels, no bundle adjustment, no publication.  The captured tracking iteration
    (render_helpers._TrackGraph) is keyed on the map's and the decoder's addresses, so it is captured once per tracking rate (the
    reference doubles the rate for scan indices below 2) and replayed for every scan.
  * Per scan, the loss and the fraction of rays that hit the map come from one score_poses(..., deterministic=True) call at the final
    pose, on rays spread evenly over the scan: track_frame only reports a loss through loss_log, which turns its captured graph off.
  * Recovery (opt-in, config key "recovery_specs"; DESIGN.md §11.5): a tracked scan whose hit fraction or loss fails the lost rule
    (is_lost) is re-placed by score.relocalise around the constant-velocity guess, then, at most once every global_interval scans
    while scans stay lost, by the first scan's search over the whole saved trajectory.  A re-placement counts only if its own score
    passes the rule; otherwise the scan keeps its tracked pose and is reported lost.  After either, the motion model restarts from
    the last accepted scan.  The map is frozen, so a wrong decision changes one reported pose and nothing else.
  * Changes (opt-in, config key "change_specs"; DESIGN.md §11.7): after the drive, every scan that is not lost goes to a
    changes.ChangeDetector at its final pose, which reports the saved voxels the drive sees through (removed) and the voxels where its
    returns land outside the map (added).  It reports and does not edit the map.

Not covered here: updating the map (slam.NeRFLOAM's base_map grows a saved map with a later drive, placing its first scan with
place_scan; DESIGN.md §11.6), loop closure.
"""
import contextlib
import copy
import math
import os
import time
from collections import namedtuple
from types import SimpleNamespace

import numpy as np
import torch

from . import _capi
from . import render_helpers as rh
from .changes import ChangeDetector, change_specs, write_changes
from .frame import POSE_OFFSET, LidarFrame
from .globalloc import relocalise_global
from .score import relocalise, score_poses
from .se3pose import OptimizablePose
from .slam import SavedMap, Tracking, _merge, constant_velocity_guess, load_map, write_poses

# relocalise_global's settings for the first scan (config key "global_specs" overrides them): the search of DESIGN.md §3.4 around
# every saved pose, and its refinement with 1024 rays, 150 iterations at rate 0.01 (the rate Adam steps at, whatever the scan's index)
GLOBAL_SPECS = dict(radius=5.0, xy_step=1.0, yaw_steps=72, n_points=512, n_candidates=4096, n_seeds=4, N_rays=1024, refine_iterations=150,
                    learning_rate=0.01)

# the lost rule's settings (config key "recovery_specs" turns recovery on and overrides them; DESIGN.md §11.5 says what they rest on):
# a scan is lost when its hit fraction is below lost_hit_fraction or its loss exceeds lost_loss_ratio x the median loss of the last
# HISTORY accepted scans; while scans stay lost, the global search runs at most once every global_interval scans
RECOVERY_SPECS = dict(lost_hit_fraction=0.5, lost_loss_ratio=3.0, global_interval=5)
HISTORY = 10
STATUSES = ("tracked", "local", "global", "lost")
_NOT_PER_SCAN = ("place", "polish", "recover_local", "recover_global")          # Localiser.times entries summary() reports apart


def recovery_specs(specs):
    """RECOVERY_SPECS with `specs` merged over them, checked: ValueError naming an unknown key or a value out of range."""
    if not isinstance(specs, dict):
        raise ValueError(f"recovery_specs must be a dict, got {specs!r}")
    out = dict(RECOVERY_SPECS)
    for k, v in specs.items():
        if k not in RECOVERY_SPECS:
            raise ValueError(f"recovery_specs: unknown key {k!r} (known: {', '.join(RECOVERY_SPECS)})")
        if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or not math.isfinite(float(v)):
            raise ValueError(f"recovery_specs: {k} must be a finite number, got {v!r}")
        out[k] = v
    if not 0.0 <= float(out["lost_hit_fraction"]) <= 1.0:
        raise ValueError(f"recovery_specs: lost_hit_fraction must lie in [0, 1], got {out['lost_hit_fraction']}")
    if not float(out["lost_loss_ratio"]) >= 1.0:
        raise ValueError(f"recovery_specs: lost_loss_ratio must be >= 1 (below 1 it flags healthy scans), got {out['lost_loss_ratio']}")
    if int(out["global_interval"]) != out["global_interval"] or int(out["global_interval"]) < 1:
        raise ValueError(f"recovery_specs: global_interval must be an integer >= 1, got {out['global_interval']}")
    return {"lost_hit_fraction": float(out["lost_hit_fraction"]), "lost_loss_ratio": float(out["lost_loss_ratio"]),
            "global_interval": int(out["global_interval"])}


def is_lost(loss, hit_fraction, accepted_losses, specs):
    """The lost rule: True when the loss is not finite, the hit fraction is below specs["lost_hit_fraction"], or the loss exceeds
    specs["lost_loss_ratio"] x the median of the last HISTORY entries of accepted_losses (the losses of the accepted scans so far, in
    order; with none, only the first two tests apply)."""
    if not math.isfinite(loss) or hit_fraction < specs["lost_hit_fraction"]:
        return True
    window = list(accepted_losses)[-HISTORY:]
    return bool(window) and loss > specs["lost_loss_ratio"] * float(np.median(window))


def _rate_argument(rate, index):
    """The learning_rate argument that makes track_frame / track_frames step at `rate` on a scan of this index: they double the rate
    below index 2 and divide it by 3 from there (the reference's rule, render_helpers.py:448-450), which is meant for a run's first
    scans, not for a search's refinement.  Halving and doubling are exact, so rate / 3 at index 0 or 1 gives later scans' rate bits."""
    return rate / 2 if index < 2 else rate * 3


def _cpu_pose(pose):
    p = OptimizablePose(pose.data.detach().cpu().float().clone())
    p.requires_grad_(False)
    return p


def forked_rng(generator):
    """With a generator, a context under which torch's global generators are seeded from one draw of it and restored afterwards
    (torch.random.fork_rng); with None, nothing: the caller draws from torch's global generators."""
    if generator is None:
        return contextlib.nullcontext()
    seed = int(torch.randint(0, 2 ** 62, (1,), generator=generator))
    stack = contextlib.ExitStack()
    stack.enter_context(torch.random.fork_rng(devices=[torch.cuda.current_device()]))
    torch.manual_seed(seed)
    return stack


def _tracking_kw(tr):
    return dict(step_size=tr.step_size, truncation=tr.sdf_truncation, max_voxel_hit=tr.max_voxel_hit, max_distance=tr.max_distance)


def place_scan(frame, map_state, decoder, tracker, anchors, global_specs, generator=None):
    """The search with no pose guess: relocalise_global anchored on every pose of `anchors` (f64[S,4,4] in the map frame, POSE_OFFSET
    included) with global_specs (GLOBAL_SPECS' keys), under forked_rng(generator), then track_frame from its placement with
    `tracker`'s settings (a slam.Tracking).  Localiser's first scan and its global recovery use it, and so does slam.NeRFLOAM's first
    scan when it extends a saved map.  Returns (GlobalResult, the pose as a CPU OptimizablePose or None when no placement hits the
    map, search ms, tracking ms or None); frame.pose is not touched."""
    tr = tracker
    g = dict(global_specs)
    search = {k: g.pop(k) for k in ("radius", "xy_step", "yaw_steps", "n_points", "n_candidates", "n_seeds") if k in g}
    g["learning_rate"] = _rate_argument(g["learning_rate"], frame.index)
    t0 = time.perf_counter()
    with forked_rng(generator):
        res = relocalise_global(frame, map_state, decoder, tr.loss_criteria, tr.voxel_size, anchors=anchors, **search, **_tracking_kw(tr), **g)
    search_ms = (time.perf_counter() - t0) * 1e3
    if res.hit_mask is None:
        return res, None, search_ms, None
    # the search's refinement ends at its own rate; the scan is then tracked from the placement like a scan without a motion prior
    # (num_iterations x 5) at the rate of every later scan, so its pose is as settled as theirs
    t0 = time.perf_counter()
    pose, hit = rh.track_frame(OptimizablePose(res.pose.data.detach().cpu().float().clone()), frame, map_state, decoder,
                               tr.loss_criteria, tr.voxel_size, tr.N_rays, tr.step_size, tr.num_iterations * 5, tr.sdf_truncation,
                               _rate_argument(tr.learning_rate / 3, frame.index), tr.max_voxel_hit, tr.max_distance, generator=generator)
    polish_ms = (time.perf_counter() - t0) * 1e3
    return res, _cpu_pose(pose if hit is not None else res.pose), search_ms, polish_ms


def trajectory_anchors(trajectory):
    """A saved trajectory (f64[S,4,4] without POSE_OFFSET) as place_scan's anchors: a copy with POSE_OFFSET added, since the map
    carries it."""
    anchors = torch.as_tensor(np.asarray(trajectory, dtype=np.float64)).clone()
    anchors[:, :3, 3] += POSE_OFFSET
    return anchors


def place_first(frame, map_state, decoder, tracker, anchors, global_specs, generator, times, who):
    """A sequence's first scan placed in a saved map with no pose guess: place_scan, then frame.pose = its pose.  times["place"] gets
    the search's ms and, when it succeeded, times["polish"] the tracking's.  Raises NerfLoamError naming `who` when no placement
    hits the map.  Returns the GlobalResult.  Localiser.place and slam.NeRFLOAM's base_map both use it."""
    res, pose, search_ms, polish_ms = place_scan(frame, map_state, decoder, tracker, anchors, global_specs, generator)
    times["place"] = [search_ms]
    if pose is None:
        raise _capi.NerfLoamError(f"{who}: scan {frame.index} could not be placed: no placement within "
                                  f"{global_specs['radius']} m of the saved trajectory hits the map")
    times["polish"] = [polish_ms]
    frame.pose = pose
    return res


Localisation = namedtuple("Localisation", ["scan_ids", "poses", "loss", "hit_fraction", "placement", "status", "changes"])
Localisation.__doc__ = """Localiser.run's result, per scan in order: scan_ids i64[S], poses f64[S,4,4] in the map frame without POSE_OFFSET
(what frame_poses.txt holds), loss f64[S] and hit_fraction f64[S] (score_poses at the final pose), placement: the first scan's
globalloc.GlobalResult (None when an init_pose was given), and status: with recovery on, a list of S codes from STATUSES ("tracked":
the tracker's pose passed the lost rule, "local" / "global": re-placed by that step, "lost": nothing passed, the tracked pose is
kept; the first scan is "tracked"), None with recovery off, and changes: with change detection on, the changes.Changes of every scan
that is not lost, None with it off."""


class FrozenMap:
    """share.SharedMap's reader interface over a map that never changes: acquire(version) returns the same (map_state, decoder) for
    every version, with nothing to wait for, and release(slot) does nothing.  slam.Tracking reads its map through this."""

    def __init__(self, map_state, decoder):
        self.map_state, self.decoder = map_state, decoder

    def acquire(self, version=None):
        return self.map_state, self.decoder, None

    def release(self, slot):
        pass


class Localiser:
    """Localises the scans of `data_stream` in a saved map.

    saved: a map file (slam.write_map) or a slam.SavedMap (load_map's result, or NeRFLOAM.saved_map() of a finished run).
    data_stream: a loader with __len__ and __getitem__ -> (index, points, pointsCos, pose or None) like dataset.<name>.DataLoader;
    a scan that comes with a pose is passed through untracked, as the run's tracker does (build the loader with use_gt=False).
    config: overrides merged over the file's config, e.g. {"tracker_specs": {"num_iterations": 50}} or {"global_specs": {...}}
    (relocalise_global's settings, GLOBAL_SPECS); voxel_size is the map's and cannot change.  {"recovery_specs": {...}} turns
    recovery of lost scans on (RECOVERY_SPECS; {} for the defaults); without the key run() does what it did before recovery existed.
    {"change_specs": {...}} turns change detection on (changes.CHANGE_SPECS; {} for the defaults); without it no detector is built.
    generator: a CPU torch.Generator every draw comes from (tracking's, and a seed for each search -- the first scan's and every
    recovery's -- which runs under a forked torch RNG); None draws from torch's global generators.  octree: where a map file is restored
    ("host" or "device").  out_dir: where run() writes frame_poses.txt, frame_status.txt with recovery on and changes.write_changes
    files with change detection on (None: nowhere)."""

    def __init__(self, saved, data_stream, config=None, generator=None, octree="host", out_dir=None):
        if not isinstance(saved, SavedMap):
            t0 = time.perf_counter()
            saved = load_map(saved, octree=octree)
            torch.cuda.synchronize()
            self.load_ms = (time.perf_counter() - t0) * 1e3
        else:
            self.load_ms = None
        cfg = _merge(copy.deepcopy(dict(saved.config)), copy.deepcopy(dict(config or {})))
        if float(cfg["voxel_size"]) != saved.map.voxel_size:
            raise ValueError(f"Localiser: voxel_size is the map's ({saved.map.voxel_size}), not {cfg['voxel_size']}")
        self.saved, self.data_stream, self.generator, self.out_dir = saved, data_stream, generator, out_dir
        self.args = SimpleNamespace(criteria=cfg["criteria"], data_specs=cfg["data_specs"], dataset=cfg["dataset"],
                                    tracker_specs={"start_frame": 0, "end_frame": -1, "read_offset": 1, **cfg["tracker_specs"]},
                                    mapper_specs={"voxel_size": float(cfg["voxel_size"])})
        self.global_specs = {**GLOBAL_SPECS, **cfg.get("global_specs", {})}
        self.recovery = recovery_specs(cfg["recovery_specs"]) if "recovery_specs" in cfg else None
        self.change_specs = change_specs(cfg["change_specs"]) if "change_specs" in cfg else None
        self.change_ms = []
        self.map_state = saved.map.map_states["_mapstate"]
        self.frozen = FrozenMap(self.map_state, saved.decoder)
        self.tracker = Tracking(self.args, data_stream, self.frozen, generator)
        self.anchors = trajectory_anchors(saved.trajectory)
        self.times = {}

    # -- the first scan -------------------------------------------------------------------------------------------------
    def _rng(self):
        return forked_rng(self.generator)

    def place(self, frame, init_pose=None):
        """Sets frame.pose for the first scan: init_pose (4x4 in the map frame, without POSE_OFFSET) or relocalise_global over the
        saved trajectory, tracked from there.  Returns the GlobalResult (None with an init_pose); raises NerfLoamError when no
        placement hits the map."""
        if init_pose is not None:
            T = torch.as_tensor(np.array(init_pose, dtype=np.float64)).clone()
            if T.shape != (4, 4) or not bool(torch.isfinite(T).all()):
                raise ValueError("Localiser: init_pose must be a finite 4x4 matrix")
            T[:3, 3] += POSE_OFFSET
            frame.pose = OptimizablePose.from_matrix(T.float())
            frame.pose.requires_grad_(False)
            return None
        return place_first(frame, self.map_state, self.saved.decoder, self.tracker, self.anchors, self.global_specs, self.generator,
                           self.times, "Localiser")

    def _tracking_kw(self):
        return _tracking_kw(self.tracker)

    def _search(self, frame):
        """place_scan over this map, its saved trajectory and global_specs, drawing from the Localiser's generator."""
        return place_scan(frame, self.map_state, self.saved.decoder, self.tracker, self.anchors, self.global_specs, self.generator)

    # -- recovery -------------------------------------------------------------------------------------------------------
    def _local(self, frame, guess):
        """score.relocalise around the 4x4 guess with its default lattice (N_rays, refine_iterations and the rate from global_specs):
        the re-placed pose as a CPU OptimizablePose, or None when no hypothesis hits the map."""
        g = self.global_specs
        with self._rng():
            pose, hit, _ = relocalise(frame, OptimizablePose.from_matrix(guess), self.map_state, self.saved.decoder,
                                      self.tracker.loss_criteria, self.tracker.voxel_size, N_rays=g["N_rays"],
                                      refine_iterations=g["refine_iterations"],
                                      learning_rate=_rate_argument(g["learning_rate"], frame.index), **self._tracking_kw())
        return None if hit is None else _cpu_pose(pose)

    def _recover(self, frame, guess, accepted_losses, global_allowed):
        """The fallback order for a lost scan: the local search around the guess, then, if global_allowed, the search with no guess.
        Each re-placement is scored and kept only if it passes the lost rule.  Returns (status, (loss, hit fraction) of the kept pose),
        or ("lost", None) with frame.pose left as it was."""
        steps = [("local", lambda: self._local(frame, guess))]
        if global_allowed:
            steps.append(("global", lambda: self._search(frame)[1]))
        tracked = frame.pose
        for name, step in steps:
            t0 = time.perf_counter()
            pose, ok = step(), False
            if pose is not None:
                frame.pose = pose
                sc = self.score(frame)
                ok = not is_lost(*sc, accepted_losses, self.recovery)
            self.times.setdefault(f"recover_{name}", []).append((time.perf_counter() - t0) * 1e3)
            if ok:
                return name, sc
        frame.pose = tracked
        return "lost", None

    # -- scoring --------------------------------------------------------------------------------------------------------
    def score(self, frame):
        """(loss, hit fraction) of the frame at its pose: one score_poses call, deterministic, on N_rays rays spread evenly over the
        scan (every point when it has fewer)."""
        t0 = time.perf_counter()
        n = int(frame.points.shape[0])
        N = min(int(self.tracker.N_rays), n)
        ids = (torch.arange(N, dtype=torch.int64) * n) // N
        sc = score_poses(frame.pose.data.detach().reshape(1, 6).float(), frame, self.map_state, self.saved.decoder, self.tracker.loss_criteria,
                         self.tracker.voxel_size, step_size=self.tracker.step_size, max_distance=self.tracker.max_distance,
                         deterministic=True, ray_ids=ids)
        loss, hit = float(sc.loss[0]), int(sc.hit_rays[0])
        self.times.setdefault("score", []).append((time.perf_counter() - t0) * 1e3)
        return loss, hit / N

    # -- the sequence ---------------------------------------------------------------------------------------------------
    def run(self, start_frame=0, end_frame=-1, read_offset=1, init_pose=None):
        """Localises scans start_frame .. end_frame (clamped to the last; -1: the last) whose index is divisible by read_offset, the
        first scan always.  Returns a Localisation and, with out_dir, writes out_dir/frame_poses.txt (slam.write_poses) and, with
        recovery on, out_dir/frame_status.txt ("<scan id> <status>" per line).  With recovery on, each tracked scan is judged by
        is_lost against the losses of the accepted scans (the first scan counts as accepted); a lost one goes through _recover, and a
        global step runs only if none ran in the current run of lost scans within the last global_interval scans."""
        tr, n = self.tracker, len(self.data_stream)
        if not 0 <= int(start_frame) < n:
            raise ValueError(f"Localiser.run: start_frame {start_frame} outside the stream's {n} scans")
        if int(read_offset) < 1:
            raise ValueError(f"Localiser.run: read_offset must be >= 1, got {read_offset}")
        tr.end_frame = min(end_frame if end_frame > 0 else n - 1, n - 1)
        tr.read_offset = int(read_offset)
        tr.last_frame, tr.rel_pose, tr.times = None, None, {}
        self.times = {}
        t0 = time.perf_counter()
        index, points, pointcos, _ = self.data_stream[int(start_frame)]
        tr._tick("load", t0)
        first = LidarFrame(index, points, pointcos, OptimizablePose(torch.zeros(6)), new_keyframe=True)
        placement = self.place(first, init_pose)
        tr.last_frame, tr.start_frame = first, int(start_frame) + 1
        frames, scores = [first], [self.score(first)]
        status = None if self.recovery is None else ["tracked"]
        accepted, last_global = [scores[0][0]], None            # losses of the accepted scans; where the current lost run last searched
        for fid in tr.frame_ids():
            ref, rel = tr.last_frame, tr.rel_pose
            f = tr.track(fid, 0)
            frames.append(f)
            scores.append(self.score(f))
            if status is None:
                continue
            # a scan that came with a pose was passed through untracked (it has no relative pose): there is no track to judge
            if f.rel_pose is None or not is_lost(*scores[-1], accepted, self.recovery):
                status.append("tracked")
                accepted.append(scores[-1][0])
                last_global = None
                continue
            pos = len(frames) - 1
            global_allowed = last_global is None or pos - last_global >= self.recovery["global_interval"]
            code, sc = self._recover(f, constant_velocity_guess(ref.get_pose(), rel), accepted, global_allowed)
            status.append(code)
            if global_allowed and code != "local":
                last_global = pos
            if code == "lost":                                  # the scan keeps its tracked pose and score; tracking restarts from ref
                tr.last_frame = ref
            else:
                scores[-1] = sc
                accepted.append(sc[0])
                last_global = None
                tr.last_frame = f
            tr.rel_pose = None                                  # the next scan is tracked like one without a motion prior
        poses = torch.stack([f.get_pose().detach().double() for f in frames])
        poses[:, :3, 3] -= POSE_OFFSET
        scan_ids = [int(f.index) for f in frames]
        if self.out_dir is not None:
            os.makedirs(self.out_dir, exist_ok=True)
            write_poses(os.path.join(self.out_dir, "frame_poses.txt"), poses.numpy())
            if status is not None:
                with open(os.path.join(self.out_dir, "frame_status.txt"), "w") as fh:
                    fh.writelines(f"{i} {s}\n" for i, s in zip(scan_ids, status))
        self.times.update(tr.times)
        changes = None if self.change_specs is None else self.detect_changes(frames, status)
        return Localisation(torch.tensor(scan_ids, dtype=torch.int64), poses,
                            torch.tensor([s[0] for s in scores], dtype=torch.float64), torch.tensor([s[1] for s in scores], dtype=torch.float64),
                            placement, status, changes)

    def detect_changes(self, frames, status):
        """Every frame whose status is not "lost" (every frame with recovery off) into a new ChangeDetector at its final pose; returns
        its Changes and, with out_dir, writes them there.  change_ms gets each add_scan's host ms (ending in its read-back)."""
        det = ChangeDetector(self.map_state, self.saved.decoder, self.tracker.voxel_size, self.args.criteria, self._tracking_kw(), self.change_specs)
        self.change_ms = []
        for i, f in enumerate(frames):
            if status is not None and status[i] == "lost":
                continue
            t0 = time.perf_counter()
            det.add_scan(f, f.pose)
            self.change_ms.append((time.perf_counter() - t0) * 1e3)
        changes = det.result()
        if self.out_dir is not None:
            write_changes(self.out_dir, changes)
        return changes

    def summary(self, result):
        """A JSON-ready summary of run()'s result: scans, the map file's load time, median host ms per scan per stage (load, track,
        score; tracking's stages end in a read-back), the first scan's placement (ms, stage times, placements searched), the median
        loss and the smallest hit fraction.  The placement's ms is the relocalise_global call; its track_ms the tracking from it.  With
        recovery on, "recovery": the scans per status and the median ms of a local and of a global step (each with the score of its
        pose; None where the step never ran).  With change detection on, "changes": the scans added, the confirmed, removed,
        unobserved and added voxel totals and the median ms of an add_scan."""
        p = result.placement
        place = None
        if p is not None:
            place = {"ms": self.times["place"][0], "stages_ms": {k: v * 1e3 for k, v in p.diagnostics.times.items()},
                     "placements": int(p.diagnostics.n_placements), "loss": float(p.loss), "track_ms": self.times["polish"][0]}
        out = {"scans": int(result.scan_ids.numel()), "map_load_ms": self.load_ms,
               "ms_per_scan": {k: float(np.median(v)) for k, v in self.times.items() if k not in _NOT_PER_SCAN},
               "placement": place, "median_loss": float(result.loss.median()), "min_hit_fraction": float(result.hit_fraction.min()),
               "out_dir": self.out_dir}
        if result.status is not None:
            out["recovery"] = {"counts": {s: result.status.count(s) for s in STATUSES},
                               "ms": {s: float(np.median(self.times[f"recover_{s}"])) if f"recover_{s}" in self.times else None
                                      for s in ("local", "global")}}
        if result.changes is not None:
            c = result.changes
            out["changes"] = {"scans": c.n_scans, "confirmed": c.n_confirmed, "removed": c.n_removed, "unobserved": c.n_unobserved,
                              "added": int(len(c.added_centres)), "ms_per_scan": float(np.median(self.change_ms)) if self.change_ms else None}
        return out
