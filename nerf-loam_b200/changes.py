"""Change detection against a saved map (DESIGN.md §11.7, include/nerfloam_b200.h section 16): which saved voxels a later drive sees
through, which it confirms, and where its returns land on ground the map does not hold.

    det = ChangeDetector(map_state, decoder, voxel_size, criteria, tracking_kw, specs={})
    for frame in localised_scans:
        det.add_scan(frame, frame.pose)                    # every point of the scan, at its final pose in the map frame
    ch = det.result()                                      # Changes
    write_changes(out_dir, ch)                             # changes_removed.ply, changes_added.ply, changes.txt

  * Votes: each scan point's ray is rendered against the saved map as score_poses renders it (the same traversal and NL_MAX_HITS
    voxel cap, the tracker's step size and max_distance, the deterministic sampling constant) and the decoder's SDF is evaluated at
    every sample.  Per ray and voxel, with d = range - sample depth: a "through" vote when every sample has d > truncation + margin
    and the SDF reaches <= 0 there (the ray crosses a surface the map holds, in space the scan says is empty); a "surface" vote when
    some sample has |d| <= truncation.  A saved voxel is removed when through >= min_votes and through >= ratio x (through +
    surface), confirmed when it has surface votes and is not removed, unobserved when it has none.
  * Added: a scan point whose voxel floor(p_world / voxel_size) is not a leaf of the saved map (globalloc.OccupiedSet) is counted
    per voxel with the number of distinct scans that hit it; a voxel is added with at least min_points points from min_scans scans.
  * The map is only read.  Nothing draws from a random generator.
"""
import math
import os
from collections import namedtuple

import numpy as np
import torch

from . import _capi
from . import render_helpers as rh
from .engine import DecoderBuffers, MapState, SDFEngine
from .frame import POSE_OFFSET
from .globalloc import MAX_GRID_DIM, occupied_set
from .se3pose import OptimizablePose

# The defaults (config key "change_specs" overrides them; DESIGN.md §11.7 says what they rest on): margin in voxel sizes beyond the
# truncation that a through vote's samples must lie in front of the return; min_votes and ratio of the removed rule; min_points and
# min_scans of the added rule.
CHANGE_SPECS = dict(margin=1.0, min_votes=3, ratio=0.8, min_points=5, min_scans=2)
_COUNTS = ("min_votes", "min_points", "min_scans")

CHUNK_RAYS = 1 << 15                  # rays per render call
SAMPLES_PER_RAY = rh.SAMPLES_PER_RAY_TRACK
ADDED_SLOTS = 1 << 18                 # initial slots of the added table; it grows when a scan would fill more than half of it

Changes = namedtuple("Changes", ["removed_centres", "removed_ids", "through", "surface", "n_confirmed", "n_removed", "n_unobserved",
                                 "added_centres", "added_points", "added_scans", "n_scans"])
Changes.__doc__ = """ChangeDetector.result(), on the host: removed_centres f64[R,3] (map frame, POSE_OFFSET removed) and removed_ids i64[R]
of the removed voxels in node order, with their through and surface vote counts i64[R]; the totals of confirmed, removed and
unobserved saved voxels; added_centres f64[A,3] of the added voxels in key order with their point and scan counts i64[A]; the scans
added."""


def change_specs(specs):
    """CHANGE_SPECS with `specs` merged over them, checked: ValueError naming an unknown key, a value that is not a finite number,
    ratio outside (0, 1], margin below 0, or a count below 1 (or not an integer)."""
    if not isinstance(specs, dict):
        raise ValueError(f"change_specs must be a dict, got {specs!r}")
    out = dict(CHANGE_SPECS)
    for k, v in specs.items():
        if k not in CHANGE_SPECS:
            raise ValueError(f"change_specs: unknown key {k!r} (known: {', '.join(CHANGE_SPECS)})")
        if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or not math.isfinite(float(v)):
            raise ValueError(f"change_specs: {k} must be a finite number, got {v!r}")
        out[k] = v
    if not 0.0 < float(out["ratio"]) <= 1.0:
        raise ValueError(f"change_specs: ratio must lie in (0, 1], got {out['ratio']}")
    if not float(out["margin"]) >= 0.0:
        raise ValueError(f"change_specs: margin must be >= 0, got {out['margin']}")
    for k in _COUNTS:
        if int(out[k]) != out[k] or not 1 <= int(out[k]) < 2 ** 32:
            raise ValueError(f"change_specs: {k} must be an integer >= 1, got {out[k]}")
    return {"margin": float(out["margin"]), "ratio": float(out["ratio"]), **{k: int(out[k]) for k in _COUNTS}}


def _pose6(pose):
    if isinstance(pose, OptimizablePose):
        p = pose.data.detach()
    else:
        p = torch.as_tensor(pose).detach()
        if p.shape == (4, 4):
            p = OptimizablePose.from_matrix(p.float()).data.detach()
    p = p.reshape(-1).float()
    if p.numel() != 6 or not bool(torch.isfinite(p).all()):
        raise ValueError("ChangeDetector.add_scan: pose must be an OptimizablePose, a 6-vector or a 4x4 matrix, finite")
    return p.reshape(1, 6)


class ChangeDetector:
    """Accumulates the change votes of a later drive against a saved map.

    map_state: the saved map's MapState (or a map_states dict); decoder: its decoder; voxel_size: the map's; criteria: the map's
    criteria (sdf_truncation is the truncation T); tracking_kw: the tracker's ray settings, step_size and max_distance in metres
    (localise's _tracking_kw); specs: CHANGE_SPECS overrides.  chunk_rays: rays per render call; the sampler's strata depend on the
    rays rendered together (render_rays' batch quirks, as in the reference), so the votes depend on it.  samples_per_ray and
    added_slots size the first sample list and the added table; both grow when a scan needs more, and results do not depend on them."""

    def __init__(self, map_state, decoder, voxel_size, criteria, tracking_kw, specs=None, *, chunk_rays=CHUNK_RAYS, samples_per_ray=SAMPLES_PER_RAY,
                 added_slots=ADDED_SLOTS, grid_dim=MAX_GRID_DIM):
        self.specs = change_specs({} if specs is None else specs)
        self.dev = torch.device("cuda", torch.cuda.current_device())
        self.m = map_state if isinstance(map_state, MapState) else MapState.from_map_states(map_state, self.dev)
        self.decoder, self.vs, self.grid_dim = decoder, float(voxel_size), int(grid_dim)
        self.truncation = float(np.float32(criteria["sdf_truncation"]))
        self.through = float(np.float32(float(criteria["sdf_truncation"]) + self.specs["margin"] * self.vs))
        self.cfg = rh._cfg(tracking_kw["step_size"], self.vs, tracking_kw["max_distance"])
        if int(chunk_rays) < 1 or int(samples_per_ray) < 1:
            raise ValueError("ChangeDetector: chunk_rays and samples_per_ray must be >= 1")
        self.chunk_rays, self.cap = int(chunk_rays), int(chunk_rays) * int(samples_per_ray)
        self.occ = occupied_set(self.m, self.vs, self.grid_dim)
        self.votes = torch.zeros((self.m.n_nodes, 2), dtype=torch.int32, device=self.dev)       # u32 counters
        self.state = torch.zeros(4, dtype=torch.int32, device=self.dev)
        self.Rt12 = torch.empty(12, dtype=torch.float32, device=self.dev)
        self.eng = None
        self.slots = 0
        self._table(int(added_slots))
        self.n_scans = 0
        self.redos = {"samples": 0, "added": 0}

    # -- device state -----------------------------------------------------------------------------------------------------
    def _table(self, slots):
        """A new added table of `slots` (a power of two >= 2^10) with the old one's keys moved into it."""
        slots = max(1024, 1 << (int(slots) - 1).bit_length())
        keys = torch.empty(slots, dtype=torch.int64, device=self.dev)
        vals = torch.empty((slots, 3), dtype=torch.int32, device=self.dev)
        old = (self.slots, _capi.ptr(self.keys), _capi.ptr(self.vals)) if self.slots else (0, None, None)
        _capi.check(_capi.lib().nl_change_rehash(*old, slots, _capi.ptr(keys), _capi.ptr(vals), _capi.ptr(self.state), _capi.stream_ptr()),
                    "nl_change_rehash")
        _capi.LAUNCHES += 2
        self.slots, self.keys, self.vals = slots, keys, vals

    def _engine(self, R):
        if self.eng is None or self.eng.max_rays < R or self.eng.max_samples < self.cap:
            self.eng = None
            self.eng = SDFEngine(max(R, self.chunk_rays), self.cap, self.dev)
        return self.eng

    def _votes(self, m, bufs, dirs, gt, r0, R, status):
        """Render rays [r0, r0 + R) of the scan at self.Rt12 and add their votes (nl_change_votes); status i32[2] records an
        overflowed sample list instead."""
        eng = self._engine(R)
        lib, st = _capi.lib(), _capi.stream_ptr()
        _capi.check(lib.nl_rays_from_poses(R, _capi.ptr(dirs[r0:r0 + R]), None, _capi.ptr(self.Rt12), _capi.ptr(eng.ray_o), _capi.ptr(eng.ray_d), st),
                    "nl_rays_from_poses")
        _capi.LAUNCHES += 1
        eng.forward(m, bufs, R, self.cfg, None, None, None, 0, True)
        _capi.check(lib.nl_change_votes(eng.max_samples, eng.stats.data_ptr(), _capi.ptr(eng.s_ray), _capi.ptr(eng.s_vox), _capi.ptr(eng.s_depth),
                                        _capi.ptr(eng.sdf), _capi.ptr(gt[r0:r0 + R]), _capi.ptr(eng.ray_offset), self.m.n_nodes,
                                        self.truncation, self.through, _capi.ptr(self.votes), _capi.ptr(status), st), "nl_change_votes")
        _capi.LAUNCHES += 1

    def _added(self, pts, scan):
        o = self.occ
        _capi.check(_capi.lib().nl_change_added(pts.shape[0], _capi.ptr(pts), _capi.ptr(self.Rt12), self.vs, self.grid_dim, _capi.ptr(o.slots),
                                                o.slots.numel(), self.slots, _capi.ptr(self.keys), _capi.ptr(self.vals), scan, _capi.ptr(self.state),
                                                _capi.stream_ptr()), "nl_change_added")
        _capi.LAUNCHES += 2

    # -- the interface ----------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def add_scan(self, frame, pose):
        """Adds every point of `frame` at `pose` (an OptimizablePose, 6-vector or 4x4 matrix in the map frame, POSE_OFFSET included):
        its rays' votes, rendered in chunks of chunk_rays, and its added-voxel hits.  One read-back of the overflow flags at the end;
        an overflowed chunk is rendered again with a larger sample list, an overflowed added table is grown and the scan inserted again."""
        if self.n_scans >= 2 ** 32 - 1:
            raise ValueError("ChangeDetector: too many scans")
        dev, lib, st = self.dev, _capi.lib(), _capi.stream_ptr()
        pose6 = _pose6(pose).to(dev).contiguous()
        _capi.check(lib.nl_pose_matrices(1, _capi.ptr(pose6), _capi.ptr(self.Rt12), st), "nl_pose_matrices")
        _capi.LAUNCHES += 1
        dirs = rh._frame_arrays(frame, dev)[0]
        pts = rh._frame_points(frame, dev)
        gt = torch.norm(pts, 2, -1).contiguous()                # the measured depth along the unit ray: the point's range
        n = int(pts.shape[0])
        bufs = DecoderBuffers.of(self.decoder, dev)
        chunks = list(range(0, n, self.chunk_rays))
        status = torch.zeros((len(chunks) + 1, 2), dtype=torch.int32, device=dev)
        for c, r0 in enumerate(chunks):
            self._votes(self.m, bufs, dirs, gt, r0, min(self.chunk_rays, n - r0), status[c])
        self._added(pts, self.n_scans)
        status[-1, 0] = self.state[2]
        flags = status.cpu()
        for c, r0 in enumerate(chunks):
            while int(flags[c, 0]):
                if int(flags[c, 0]) & 4:
                    rh._check_ctl([4], "ChangeDetector.add_scan")
                rh._check_sample_total(int(flags[c, 1]), "ChangeDetector.add_scan")
                self.cap = max(2 * self.cap, int(int(flags[c, 1]) * 1.25) + 1024)
                self.redos["samples"] += 1
                status[c].zero_()
                self._votes(self.m, bufs, dirs, gt, r0, min(self.chunk_rays, n - r0), status[c])
                flags[c] = status[c].cpu()
        if int(flags[-1, 0]):
            committed = int(self.state[0])
            self._table(4 * (committed + n))
            self.redos["added"] += 1
            self._added(pts, self.n_scans)
        self.n_scans += 1

    @torch.no_grad()
    def result(self):
        """The Changes of every scan added so far (two read-backs)."""
        sp, lib = self.specs, _capi.lib()
        n = self.m.n_nodes
        ws_bytes = int(lib.nl_change_finish_workspace_bytes(n, self.slots))
        if ws_bytes < 0:
            _capi.check(ws_bytes, "nl_change_finish_workspace_bytes")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.dev)
        removed = torch.empty(n, dtype=torch.int32, device=self.dev)
        added = torch.empty(self.slots, dtype=torch.int64, device=self.dev)
        added_vals = torch.empty((self.slots, 2), dtype=torch.int32, device=self.dev)
        totals = torch.empty(4, dtype=torch.int64, device=self.dev)
        _capi.check(lib.nl_change_finish(n, _capi.ptr(self.m.structure), _capi.ptr(self.votes), sp["min_votes"], sp["ratio"], self.slots,
                                         _capi.ptr(self.keys), _capi.ptr(self.vals), sp["min_points"], sp["min_scans"], _capi.ptr(ws), ws_bytes,
                                         _capi.ptr(removed), _capi.ptr(added), _capi.ptr(added_vals), _capi.ptr(totals), _capi.stream_ptr()),
                    "nl_change_finish")
        _capi.LAUNCHES += 5
        n_conf, n_rem, n_unobs, n_add = totals.tolist()
        ids = removed[:n_rem].long()
        votes = self.votes[ids].cpu().long() & 0xffffffff
        centres = self.m.centres[ids].double().cpu() - POSE_OFFSET
        keys = added[:n_add].cpu()
        vals = added_vals[:n_add].cpu().long() & 0xffffffff
        mask = (1 << 18) - 1
        vox = torch.stack([(keys >> 36) & mask, (keys >> 18) & mask, keys & mask], -1).double()
        return Changes(centres.numpy(), ids.cpu().numpy(), votes[:, 0].numpy(), votes[:, 1].numpy(), int(n_conf), int(n_rem), int(n_unobs),
                       ((vox + 0.5) * self.vs - POSE_OFFSET).numpy(), vals[:, 0].numpy(), vals[:, 1].numpy(), self.n_scans)


def write_changes(out_dir, changes):
    """out_dir/changes_removed.ply and changes_added.ply (vertex-only PLY files of the removed and added voxel centres, map frame) and
    changes.txt (the totals, then one line per voxel: "removed <x> <y> <z> <through> <surface>" / "added <x> <y> <z> <points>
    <scans>")."""
    from .slam import write_ply
    os.makedirs(out_dir, exist_ok=True)
    ch = changes
    write_ply(os.path.join(out_dir, "changes_removed.ply"), np.asarray(ch.removed_centres, dtype=np.float64).reshape(-1, 3), np.zeros((0, 3)))
    write_ply(os.path.join(out_dir, "changes_added.ply"), np.asarray(ch.added_centres, dtype=np.float64).reshape(-1, 3), np.zeros((0, 3)))
    with open(os.path.join(out_dir, "changes.txt"), "w") as fh:
        fh.write(f"scans {ch.n_scans}\nconfirmed {ch.n_confirmed}\nremoved {ch.n_removed}\nunobserved {ch.n_unobserved}\n"
                 f"added {len(ch.added_centres)}\n")
        for c, t, s in zip(np.asarray(ch.removed_centres).reshape(-1, 3), ch.through, ch.surface):
            fh.write(f"removed {c[0]:.4f} {c[1]:.4f} {c[2]:.4f} {int(t)} {int(s)}\n")
        for c, p, s in zip(np.asarray(ch.added_centres).reshape(-1, 3), ch.added_points, ch.added_scans):
            fh.write(f"added {c[0]:.4f} {c[1]:.4f} {c[2]:.4f} {int(p)} {int(s)}\n")
