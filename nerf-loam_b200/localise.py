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

Not covered: recovering a scan that is lost partway through, updating the map, loop closure.
"""
import contextlib
import copy
import os
import time
from collections import namedtuple
from types import SimpleNamespace

import numpy as np
import torch

from . import _capi
from . import render_helpers as rh
from .frame import POSE_OFFSET, LidarFrame
from .globalloc import relocalise_global
from .score import score_poses
from .se3pose import OptimizablePose
from .slam import SavedMap, Tracking, _merge, load_map, write_poses

# relocalise_global's settings for the first scan (config key "global_specs" overrides them): the search of DESIGN.md §3.4 around
# every saved pose, and its refinement with 1024 rays, 150 iterations at rate 0.01 (the rate Adam steps at, whatever the scan's index)
GLOBAL_SPECS = dict(radius=5.0, xy_step=1.0, yaw_steps=72, n_points=512, n_candidates=4096, n_seeds=4, N_rays=1024, refine_iterations=150,
                    learning_rate=0.01)


def _rate_argument(rate, index):
    """The learning_rate argument that makes track_frame / track_frames step at `rate` on a scan of this index: they double the rate
    below index 2 and divide it by 3 from there (the reference's rule, render_helpers.py:448-450), which is meant for a run's first
    scans, not for a search's refinement.  Halving and doubling are exact, so rate / 3 at index 0 or 1 gives later scans' rate bits."""
    return rate / 2 if index < 2 else rate * 3


Localisation = namedtuple("Localisation", ["scan_ids", "poses", "loss", "hit_fraction", "placement"])
Localisation.__doc__ = """Localiser.run's result, per scan in order: scan_ids i64[S], poses f64[S,4,4] in the map frame without POSE_OFFSET
(what frame_poses.txt holds), loss f64[S] and hit_fraction f64[S] (score_poses at the final pose), and placement: the first scan's
globalloc.GlobalResult (None when an init_pose was given)."""


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
    (relocalise_global's settings, GLOBAL_SPECS); voxel_size is the map's and cannot change.
    generator: a CPU torch.Generator every draw comes from (tracking's, and a seed for the first scan's search, which runs under a
    forked torch RNG); None draws from torch's global generators.  octree: where a map file is restored ("host" or "device").
    out_dir: where run() writes frame_poses.txt (None: nowhere)."""

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
        self.map_state = saved.map.map_states["_mapstate"]
        self.frozen = FrozenMap(self.map_state, saved.decoder)
        self.tracker = Tracking(self.args, data_stream, self.frozen, generator)
        self.anchors = torch.as_tensor(np.asarray(saved.trajectory, dtype=np.float64)).clone()
        self.anchors[:, :3, 3] += POSE_OFFSET
        self.times = {}

    # -- the first scan -------------------------------------------------------------------------------------------------
    def _rng(self):
        """With a generator, the search draws from torch's global generators seeded from it, restored afterwards."""
        if self.generator is None:
            return contextlib.nullcontext()
        seed = int(torch.randint(0, 2 ** 62, (1,), generator=self.generator))
        stack = contextlib.ExitStack()
        stack.enter_context(torch.random.fork_rng(devices=[torch.cuda.current_device()]))
        torch.manual_seed(seed)
        return stack

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
        tr = self.tracker
        g = dict(self.global_specs)
        search = {k: g.pop(k) for k in ("radius", "xy_step", "yaw_steps", "n_points", "n_candidates", "n_seeds") if k in g}
        g["learning_rate"] = _rate_argument(g["learning_rate"], frame.index)
        t0 = time.perf_counter()
        with self._rng():
            res = relocalise_global(frame, self.map_state, self.saved.decoder, tr.loss_criteria, tr.voxel_size, anchors=self.anchors, **search,
                                    step_size=tr.step_size, truncation=tr.sdf_truncation, max_voxel_hit=tr.max_voxel_hit,
                                    max_distance=tr.max_distance, **g)
        self.times["place"] = [(time.perf_counter() - t0) * 1e3]
        if res.hit_mask is None:
            raise _capi.NerfLoamError(f"Localiser: scan {frame.index} could not be placed: no placement within {search.get('radius', 5.0)} m "
                                      f"of the saved trajectory hits the map")
        # the search's refinement ends at its own rate; the scan is then tracked from the placement like a scan without a motion prior
        # (num_iterations x 5) at the rate of every later scan, so its pose is as settled as theirs
        t0 = time.perf_counter()
        pose, hit = rh.track_frame(OptimizablePose(res.pose.data.detach().cpu().float().clone()), frame, self.map_state, self.saved.decoder,
                                   tr.loss_criteria, tr.voxel_size, tr.N_rays, tr.step_size, tr.num_iterations * 5, tr.sdf_truncation,
                                   _rate_argument(tr.learning_rate / 3, frame.index), tr.max_voxel_hit, tr.max_distance,
                                   generator=self.generator)
        self.times["polish"] = [(time.perf_counter() - t0) * 1e3]
        frame.pose = OptimizablePose((pose if hit is not None else res.pose).data.detach().cpu().float().clone())
        frame.pose.requires_grad_(False)
        return res

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
        first scan always.  Returns a Localisation and, with out_dir, writes out_dir/frame_poses.txt (slam.write_poses)."""
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
        for fid in tr.frame_ids():
            f = tr.track(fid, 0)
            frames.append(f)
            scores.append(self.score(f))
        poses = torch.stack([f.get_pose().detach().double() for f in frames])
        poses[:, :3, 3] -= POSE_OFFSET
        if self.out_dir is not None:
            os.makedirs(self.out_dir, exist_ok=True)
            write_poses(os.path.join(self.out_dir, "frame_poses.txt"), poses.numpy())
        self.times.update(tr.times)
        return Localisation(torch.tensor([int(f.index) for f in frames], dtype=torch.int64), poses,
                            torch.tensor([s[0] for s in scores], dtype=torch.float64), torch.tensor([s[1] for s in scores], dtype=torch.float64),
                            placement)

    def summary(self, result):
        """A JSON-ready summary of run()'s result: scans, the map file's load time, median host ms per scan per stage (load, track,
        score; tracking's stages end in a read-back), the first scan's placement (ms, stage times, placements searched), the median
        loss and the smallest hit fraction.  The placement's ms is the relocalise_global call; its track_ms the tracking from it."""
        p = result.placement
        place = None
        if p is not None:
            place = {"ms": self.times["place"][0], "stages_ms": {k: v * 1e3 for k, v in p.diagnostics.times.items()},
                     "placements": int(p.diagnostics.n_placements), "loss": float(p.loss), "track_ms": self.times["polish"][0]}
        return {"scans": int(result.scan_ids.numel()), "map_load_ms": self.load_ms,
                "ms_per_scan": {k: float(np.median(v)) for k, v in self.times.items() if k not in ("place", "polish")}, "placement": place,
                "median_loss": float(result.loss.median()), "min_hit_fraction": float(result.hit_fraction.min()), "out_dir": self.out_dir}
