"""relocalise_global: place a scan anywhere in a trained map with no pose guess (include/nerfloam_b200.h section 15, DESIGN.md §3.4).

`track_frame` converges from a few decimetres and degrees, and `relocalise` widens that to a ±30° × ±2 m lattice around a guess.
Neither finds a scan whose pose is unknown: the first scan of a run localised against a saved map, a tracker that has been wrong for a
while, a run that re-enters a mapped area.  The reference only gets such a pose from ground truth or a constant (`get_init_pose`).

The search has three stages.
  1. Coarse (csrc/globalloc.cu): every placement of the scan over a lattice of positions (xy_step, within `radius` of an anchor pose)
     × yaw_steps headings is scored by how many of n_points scan points land in an occupied map voxel, one hash lookup per point;
     the n_candidates highest counts are kept, exactly and deterministically.
  2. Fine: score_poses (the SDF loss with its free-space term) on those candidates; select_hypotheses drops those whose loss is not
     finite or that hit less than min_hit_fraction of the best hit count.
  3. Refine: relocalise (its local lattice, then track_frames) from the first n_seeds surviving candidates, in coarse order, at least
     seed_separation apart in xy; the refined pose of lowest loss (among those with enough hits) wins.  Stage 2's loss does not
     order the seeds: one iteration's loss ranks placements a lattice step off the truth below wrong ones (DESIGN.md §3.4).

Before stage 2 a call reads the device twice: the cell count (with the map's leaf count when its occupied set is not built yet) and
the selected placement ids.
"""
import math
import time
from collections import namedtuple

import numpy as np
import torch

from . import _capi
from . import render_helpers as rh
from .engine import MapState
from .score import poses_from_matrices, relocalise, score_poses, select_hypotheses
from .se3pose import OptimizablePose

MAX_POINTS = _capi.GLOBALLOC_MAX_POINTS
MAX_GRID_DIM = 1 << 18                      # voxel keys of 3 x 18 bits
CHUNK = 1 << 22                             # placements per scorer launch

OccupiedSet = namedtuple("OccupiedSet", ["slots", "n_leaves", "voxel_size", "grid_dim"])
OccupiedSet.__doc__ = """The map's leaf voxels as a device hash set: slots i64[pow2 >= 2 n_leaves] holding the keys vx << 36 | vy << 18 | vz
(-1 in empty slots)."""

Placements = namedtuple("Placements", ["cells", "n_cells", "n_placements", "anchors", "xy_step", "yaw_steps", "radius"])
Placements.__doc__ = """The search lattice: cells i32[n_cells, 3] = (i, j, anchor) on the device in ascending (i, j); placement id = cell x
yaw_steps + k.  anchors f64[A, 12] on the device (3x4, row-major)."""

Diagnostics = namedtuple("Diagnostics", ["n_placements", "ids", "counts", "score", "seeds", "times"])
Diagnostics.__doc__ = """n_placements searched; ids / counts i32 (device) of the coarse candidates, best first; score: stage 2's ScoreResult
(indexed like ids); seeds: the coarse ranks stage 3 started from; times: seconds per stage ('coarse', 'fine', 'refine'), host
clock between the stages' own read-backs."""

GlobalResult = namedtuple("GlobalResult", ["pose", "hit_mask", "loss", "diagnostics"])
GlobalResult.__doc__ = """relocalise_global's result: pose (OptimizablePose), hit_mask (None when no refined pose hit the map), loss (float,
the refined pose's score_poses loss; NaN when nothing hit) and Diagnostics."""


def _check(rc, what):
    if rc < 0:
        raise ValueError(f"{what}: {_capi.lib().nl_last_error().decode()}")
    return rc


def _anchor_array(anchors):
    """Anchor poses -> f64[A, 12] (3x4 row-major) on the host.  Accepts [A,4,4] / [A,3,4] arrays or tensors, or a list of 4x4 / 3x4
    matrices or OptimizablePose."""
    if isinstance(anchors, (list, tuple)):
        rows = []
        for a in anchors:
            m = a.matrix().detach() if isinstance(a, OptimizablePose) else a
            rows.append(np.asarray(m.cpu() if isinstance(m, torch.Tensor) else m, dtype=np.float64)[:3, :4])
        A = np.stack(rows) if rows else np.zeros((0, 3, 4))
    else:
        A = np.asarray(anchors.detach().cpu() if isinstance(anchors, torch.Tensor) else anchors, dtype=np.float64)
        if A.ndim != 3 or A.shape[1:] not in ((4, 4), (3, 4)):
            raise ValueError(f"relocalise_global: anchors must be [A,4,4] or [A,3,4], got shape {A.shape}")
        A = A[:, :3, :4]
    if A.shape[0] < 1:
        raise ValueError("relocalise_global: need at least one anchor")
    if not np.isfinite(A).all():
        raise ValueError("relocalise_global: anchors must be finite")
    return np.ascontiguousarray(A.reshape(-1, 12))


def _check_lattice(A, radius, xy_step, yaw_steps):
    """The C ABI's own checks (anchors, radius, xy_step, lattice size) and yaw_steps, all on the host."""
    if isinstance(yaw_steps, bool) or int(yaw_steps) != yaw_steps or int(yaw_steps) < 1:
        raise ValueError(f"relocalise_global: yaw_steps must be an int >= 1, got {yaw_steps!r}")
    ws = _capi.lib().nl_globalloc_cells_workspace_bytes(A.shape[0], A.ctypes.data, float(radius), float(xy_step))
    return _check(int(ws), "relocalise_global")


def _map_state(map_states):
    dev = torch.device("cuda", torch.cuda.current_device())
    m = map_states if isinstance(map_states, MapState) else MapState.from_map_states(map_states, dev)
    if m.n_nodes < 1:
        raise ValueError("relocalise_global: the map is empty")
    return m


def _check_grid(voxel_size, grid_dim):
    if not (float(voxel_size) > 0.0) or not math.isfinite(float(voxel_size)):
        raise ValueError(f"relocalise_global: voxel_size must be finite and > 0, got {voxel_size}")
    g = int(grid_dim)
    if g != grid_dim or not 0 < g <= MAX_GRID_DIM or g & (g - 1):
        raise ValueError(f"relocalise_global: grid_dim must be a power of two <= 2^18, got {grid_dim}")


def _set_cache(m):
    return m._cache_ref if m._cache_ref is not None else m.__dict__.setdefault("_globalloc_cache", {})


def _cached_set(m, voxel_size, grid_dim):
    key = ("globalloc_occupied", float(voxel_size), int(grid_dim), m.n_nodes, m.structure.data_ptr())
    return key, _set_cache(m).get(key)


def _build_set(m, voxel_size, grid_dim, n_leaves, key):
    slots = _check(int(_capi.lib().nl_globalloc_occupied_slots(int(n_leaves))), "relocalise_global")
    s = torch.empty(slots, dtype=torch.int64, device=m.centres.device)
    _capi.check(_capi.lib().nl_globalloc_occupied(m.n_nodes, _capi.ptr(m.centres), _capi.ptr(m.structure), float(voxel_size), int(grid_dim), slots,
                                                  _capi.ptr(s), _capi.stream_ptr()), "nl_globalloc_occupied")
    _capi.LAUNCHES += 1
    occ = OccupiedSet(s, int(n_leaves), float(voxel_size), int(grid_dim))
    _set_cache(m)[key] = occ
    return occ


def _count_leaves(m, out):
    _capi.check(_capi.lib().nl_globalloc_count_leaves(m.n_nodes, _capi.ptr(m.structure), _capi.ptr(out), _capi.stream_ptr()),
                "nl_globalloc_count_leaves")
    _capi.LAUNCHES += 1


def occupied_set(map_states, voxel_size, grid_dim=MAX_GRID_DIM):
    """The map's finest-level voxels (the set Octree.get_leaf_voxels() returns) as an OccupiedSet, built on the device from the
    MapState's structural arrays and kept with the map (like its packed children), so later calls reuse it.  Building it reads the
    leaf count back once."""
    _check_grid(voxel_size, grid_dim)
    m = _map_state(map_states)
    key, occ = _cached_set(m, voxel_size, grid_dim)
    if occ is None:
        n = torch.empty(1, dtype=torch.int64, device=m.centres.device)
        _count_leaves(m, n)
        occ = _build_set(m, voxel_size, grid_dim, int(n.item()), key)
    return occ


def _cells_begin(A, radius, xy_step, ws_bytes, count_out, dev):
    d_anchors = torch.from_numpy(A).to(dev)
    ws = torch.empty(int(ws_bytes), dtype=torch.uint8, device=dev)
    _capi.check(_capi.lib().nl_globalloc_cells(A.shape[0], A.ctypes.data, _capi.ptr(d_anchors), float(radius), float(xy_step), _capi.ptr(ws),
                                               int(ws_bytes), _capi.ptr(count_out), _capi.stream_ptr()), "nl_globalloc_cells")
    _capi.LAUNCHES += 1
    return d_anchors, ws


def _cells_finish(A, d_anchors, ws, radius, xy_step, yaw_steps, n_cells):
    if n_cells < 1:
        raise ValueError("relocalise_global: no lattice point lies within radius of an anchor")
    if n_cells * int(yaw_steps) > 2 ** 31 - 1:
        raise ValueError(f"relocalise_global: {n_cells} cells x {yaw_steps} yaws exceed the 2^31 - 1 placement ids")
    cells = torch.empty((n_cells, 3), dtype=torch.int32, device=d_anchors.device)
    _capi.check(_capi.lib().nl_globalloc_cells_finish(A.shape[0], A.ctypes.data, float(radius), float(xy_step), int(n_cells), _capi.ptr(ws),
                                                      ws.numel(), _capi.ptr(cells), _capi.stream_ptr()), "nl_globalloc_cells_finish")
    _capi.LAUNCHES += 1
    return Placements(cells, int(n_cells), int(n_cells) * int(yaw_steps), d_anchors, float(xy_step), int(yaw_steps), float(radius))


def placements(anchors, radius=5.0, xy_step=1.0, yaw_steps=72):
    """The search lattice (Placements): lattice points (i, j) x xy_step within radius of an anchor's xy, each with its nearest anchor,
    in ascending (i, j), and yaw_steps headings each.  Reads the cell count back once."""
    A = _anchor_array(anchors)
    ws_bytes = _check_lattice(A, radius, xy_step, yaw_steps)
    dev = torch.device("cuda", torch.cuda.current_device())
    n = torch.empty(1, dtype=torch.int64, device=dev)
    d_anchors, ws = _cells_begin(A, radius, xy_step, ws_bytes, n, dev)
    return _cells_finish(A, d_anchors, ws, radius, xy_step, yaw_steps, int(n.item()))


def placement_matrices(pl, ids):
    """f32[n, 4, 4] (device) of the placements `ids`: rotation Rz(2 pi k / Y - psi_a) R_a and translation (q_x, q_y, t_a,z), formed
    in fp64 and rounded to fp32 by the device function the coarse scorer uses.  Host ids outside [0, n_placements) raise
    ValueError; device ids outside it get a NaN matrix (checking them on the host would need a read-back)."""
    ids = torch.as_tensor(ids)
    if ids.dtype.is_floating_point or ids.dtype == torch.bool:
        raise ValueError(f"placement_matrices: ids must be integers, got {ids.dtype}")
    if not ids.is_cuda and ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= pl.n_placements):
        raise ValueError(f"placement_matrices: ids must lie in [0, {pl.n_placements})")
    ids = ids.to(pl.cells.device, torch.int64).reshape(-1).contiguous()
    n = ids.numel()
    Rt = torch.empty((n, 12), dtype=torch.float32, device=pl.cells.device)
    _capi.check(_capi.lib().nl_globalloc_matrices(n, _capi.ptr(ids), pl.n_cells, _capi.ptr(pl.cells), _capi.ptr(pl.anchors), pl.yaw_steps, pl.xy_step,
                                                  _capi.ptr(Rt), _capi.stream_ptr()), "nl_globalloc_matrices")
    _capi.LAUNCHES += 1
    T = torch.zeros((n, 4, 4), dtype=torch.float32, device=pl.cells.device)
    T[:, :3, :3] = Rt[:, :9].view(n, 3, 3)
    T[:, :3, 3] = Rt[:, 9:]
    T[:, 3, 3] = 1.0
    return T


def _check_points(n_points, frame):
    if isinstance(n_points, bool) or int(n_points) != n_points or not 1 <= int(n_points) <= MAX_POINTS:
        raise ValueError(f"relocalise_global: 1 <= n_points <= {MAX_POINTS}, got {n_points!r}")
    if int(n_points) > int(frame.points.shape[0]):
        raise ValueError(f"relocalise_global: n_points ({n_points}) exceeds the scan's {frame.points.shape[0]} points")


def scan_points(frame, n_points=512, point_ids=None, generator=None):
    """The M scan points of the coarse score: f32[M, 3] (sensor frame, device) and their row ids i32[M].  One nl_select_rays draw
    from the scan's non-ground rows (pointsCos == 1), or from all rows when fewer than M are non-ground; the seed comes from torch's
    CUDA generator (or `generator`).  point_ids pins the rows.  No host synchronisation."""
    dev = torch.device("cuda", torch.cuda.current_device())
    pts_all = rh._frame_points(frame, dev)
    if point_ids is not None:
        ids = torch.as_tensor(point_ids).reshape(-1).cpu().long()
        if not 1 <= ids.numel() <= MAX_POINTS:
            raise ValueError(f"relocalise_global: 1 <= len(point_ids) <= {MAX_POINTS}, got {ids.numel()}")
        if int(ids.min()) < 0 or int(ids.max()) >= pts_all.shape[0]:
            raise ValueError(f"relocalise_global: point_ids must index the scan's {pts_all.shape[0]} points")
        ids = ids.to(dev)
        return pts_all[ids].contiguous(), ids.to(torch.int32)
    _check_points(n_points, frame)
    M, n_all = int(n_points), int(pts_all.shape[0])
    cos = frame.pointsCos.float().reshape(-1).to(dev)
    ground = (cos != 1.0).to(torch.int8)
    order = torch.argsort(ground, stable=True)              # non-ground rows first, each part in row order
    n_ng = (ground == 0).sum().reshape(1)
    n_dev = torch.where(n_ng >= M, n_ng, torch.full_like(n_ng, n_all))
    sorted_pts = pts_all[order].contiguous()
    sorted_cos = cos[order].contiguous()
    out = torch.empty((M, 3), dtype=torch.float32, device=dev)
    junk = torch.empty((2, M), dtype=torch.float32, device=dev)
    idx = torch.empty(M, dtype=torch.int32, device=dev)
    seed = rh._seed_from_cuda(dev, generator)
    _capi.check(_capi.lib().nl_select_rays(1, n_all, M, _capi.ptr(n_dev), _capi.ptr(seed), 0, _capi.ptr(sorted_pts), _capi.ptr(sorted_cos),
                                           _capi.ptr(sorted_cos), _capi.ptr(out), _capi.ptr(junk[0]), _capi.ptr(junk[1]), _capi.ptr(idx),
                                           _capi.stream_ptr()), "nl_select_rays")
    _capi.LAUNCHES += 1
    return out, order[idx.long()].to(torch.int32)


def _score(pl, occ, pts, chunk):
    counts = torch.empty(pl.n_placements, dtype=torch.int32, device=pl.cells.device)
    for p0 in range(0, pl.n_placements, chunk):
        n = min(chunk, pl.n_placements - p0)
        _capi.check(_capi.lib().nl_globalloc_score(p0, n, pl.n_cells, _capi.ptr(pl.cells), _capi.ptr(pl.anchors), pl.yaw_steps, pl.xy_step,
                                                   pts.shape[0], _capi.ptr(pts), _capi.ptr(occ.slots), occ.slots.numel(), occ.voxel_size,
                                                   occ.grid_dim, _capi.ptr(counts), _capi.stream_ptr()), "nl_globalloc_score")
        _capi.LAUNCHES += 1
    return counts


def coarse_scores(pl, occ, points, chunk=CHUNK):
    """i32[n_placements] (device): for every placement, how many of points f32[M, 3] (sensor frame) land in an occupied voxel of
    occ (voxel.cuh's arithmetic: fp64 world point from the fp32 matrix and point, floor(w / voxel_size)).  The placements run in
    launches of at most `chunk`; the counts do not depend on it."""
    if isinstance(chunk, bool) or int(chunk) != chunk or int(chunk) < 1:
        raise ValueError(f"coarse_scores: chunk must be a positive int, got {chunk!r}")
    pts = torch.as_tensor(points).to(pl.cells.device, torch.float32).reshape(-1, 3).contiguous()
    if not 1 <= pts.shape[0] <= MAX_POINTS:
        raise ValueError(f"coarse_scores: 1 <= number of points <= {MAX_POINTS}, got {pts.shape[0]}")
    return _score(pl, occ, pts, int(chunk))


def top_placements(counts, n_points, n_select):
    """The n_select placements of highest count, ranked by (count desc, id asc): (ids i32[n_select], counts i32[n_select]) on the
    device.  A histogram of the counts, the threshold from its suffix sums, a stable compaction and a sort of the selected.  Counts
    outside [0, n_points] are ignored; if fewer than n_select remain, the rest of both outputs is -1."""
    counts = counts.to(torch.int32).contiguous()
    P = counts.numel()
    ws_bytes = _check(int(_capi.lib().nl_globalloc_select_workspace_bytes(P, int(n_points), int(n_select))), "top_placements")
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=counts.device)
    ids = torch.empty(int(n_select), dtype=torch.int32, device=counts.device)
    sel = torch.empty(int(n_select), dtype=torch.int32, device=counts.device)
    _capi.check(_capi.lib().nl_globalloc_select(P, _capi.ptr(counts), int(n_points), int(n_select), _capi.ptr(ws), ws_bytes, _capi.ptr(ids),
                                                _capi.ptr(sel), _capi.stream_ptr()), "nl_globalloc_select")
    _capi.LAUNCHES += 1
    return ids, sel


def _distinct_seeds(xy, order, n_seeds, separation):
    """Ranks (into order) of the first n_seeds candidates whose xy lies at least `separation` from every earlier pick."""
    picked = []
    for r, c in enumerate(order):
        if all(float(np.hypot(*(xy[c] - xy[order[q]]))) >= separation for q in picked):
            picked.append(r)
            if len(picked) == n_seeds:
                break
    return picked


@torch.no_grad()
def relocalise_global(frame, map_states, sdf_network, loss_criteria, voxel_size, *, anchors, radius=5.0, xy_step=1.0, yaw_steps=72,
                      n_points=512, n_candidates=4096, n_seeds=4, seed_separation=2.0, grid_dim=MAX_GRID_DIM, point_ids=None,
                      chunk=CHUNK, **relocalise_kw):
    """Localise `frame` in the map with no pose guess.  The search covers xy lattice points (xy_step apart) within `radius` of an
    anchor pose (4x4 or 3x4 in the map frame, POSE_OFFSET included) x yaw_steps headings; roll, pitch and height come from the nearest
    anchor.  Stage 1 counts, per placement, the n_points non-ground scan points in occupied voxels and keeps the n_candidates best;
    stage 2 scores those with score_poses and drops the ones select_hypotheses rejects; stage 3 runs relocalise (relocalise_kw: its
    keywords and track_frames') from the first n_seeds survivors in coarse order at least seed_separation metres apart and keeps the
    refined pose of lowest loss.  point_ids pins stage 1's points.  Returns GlobalResult(pose, hit_mask, loss, diagnostics)."""
    for name, v, lo, hi in (("n_candidates", n_candidates, 1, _capi.SCORE_MAX_PROBLEMS), ("n_seeds", n_seeds, 1, _capi.BATCH_MAX_PROBLEMS)):
        if isinstance(v, bool) or int(v) != v or not lo <= int(v) <= hi:
            raise ValueError(f"relocalise_global: {lo} <= {name} <= {hi}, got {v!r}")
    if not (float(seed_separation) >= 0.0) or not math.isfinite(float(seed_separation)):
        raise ValueError(f"relocalise_global: seed_separation must be finite and >= 0, got {seed_separation}")
    if isinstance(chunk, bool) or int(chunk) != chunk or int(chunk) < 1:
        raise ValueError(f"relocalise_global: chunk must be a positive int, got {chunk!r}")
    _check_grid(voxel_size, grid_dim)
    A = _anchor_array(anchors)
    ws_bytes = _check_lattice(A, radius, xy_step, yaw_steps)
    if point_ids is None:
        _check_points(n_points, frame)
    m = _map_state(map_states)
    dev = m.centres.device
    t0 = time.perf_counter()

    # stage 1: one read for the cell count (and the leaf count when the set is new), one for the selected ids
    key, occ = _cached_set(m, voxel_size, grid_dim)
    counts2 = torch.zeros(2, dtype=torch.int64, device=dev)
    if occ is None:
        _count_leaves(m, counts2[:1])
    d_anchors, ws = _cells_begin(A, radius, xy_step, ws_bytes, counts2[1:], dev)
    n_leaves, n_cells = counts2.tolist()
    if occ is None:
        occ = _build_set(m, voxel_size, grid_dim, n_leaves, key)
    pl = _cells_finish(A, d_anchors, ws, radius, xy_step, yaw_steps, n_cells)
    pts, _ = scan_points(frame, n_points, point_ids)
    counts = _score(pl, occ, pts, int(chunk))
    ids, sel = top_placements(counts, pts.shape[0], min(int(n_candidates), pl.n_placements))
    ids_h = ids.cpu()
    t1 = time.perf_counter()

    # stage 2
    T = placement_matrices(pl, ids)
    pose6 = poses_from_matrices(T).contiguous()
    score_kw = {k: relocalise_kw[k] for k in ("step_size", "max_distance", "deterministic") if k in relocalise_kw}
    N_rays = int(relocalise_kw.get("N_rays", 512))
    sc = score_poses(pose6, frame, m, sdf_network, loss_criteria, voxel_size, N_rays, **score_kw)
    # stage 2 filters (finite loss, enough hits) but does not reorder: a one-iteration loss ranks placements 1 m and a few degrees
    # off the truth below wrong ones that sit in poorly constrained space, while the coarse count ranks the true cell first
    # (DESIGN.md §3.4), so the seeds follow the coarse order
    order = sorted(select_hypotheses(sc.loss, sc.hit_rays, ids_h.numel(), relocalise_kw.get("min_hit_fraction", 0.5)).tolist())
    xy = T[:, :2, 3].double().cpu().numpy()
    seeds = _distinct_seeds(xy, order, int(n_seeds), float(seed_separation))
    t2 = time.perf_counter()

    # stage 3
    refined = []
    for r in seeds:
        p, hit, _ = relocalise(frame, pose6[order[r]].cpu(), m, sdf_network, loss_criteria, voxel_size, **relocalise_kw)
        if hit is not None:
            refined.append((p, hit))
    best, loss = None, float("nan")
    if refined:
        final = score_poses(torch.stack([p.data.detach().reshape(6).float() for p, _ in refined]), frame, m, sdf_network, loss_criteria,
                            voxel_size, ray_ids=sc.ray_ids, **dict(score_kw, deterministic=True))
        # the lowest loss among the poses that hit at least min_hit_fraction of the best hit count, as in stage 2: a pose at the
        # map's edge that hits a few rays well would otherwise win
        pick = select_hypotheses(final.loss, final.hit_rays, 1, relocalise_kw.get("min_hit_fraction", 0.5))
        if pick.numel():
            best = int(pick[0])
            loss = float(final.loss[best])
    t3 = time.perf_counter()
    diag = Diagnostics(pl.n_placements, ids, sel, sc, [order[r] for r in seeds], {"coarse": t1 - t0, "fine": t2 - t1, "refine": t3 - t2})
    if best is None:
        first = order[0] if order else 0
        return GlobalResult(OptimizablePose(pose6[first].cpu().clone()).cuda(), None, loss, diag)
    return GlobalResult(refined[best][0], refined[best][1], loss, diag)
