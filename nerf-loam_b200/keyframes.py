"""The mapper's keyframe graph (src/mapping.py:114-116, 205-225, 266-281): when a tracked scan becomes a keyframe, and which keyframes
a mapping call optimises.

Besides the reference's 'current', 'previous' and 'random' windows this offers 'overlap', which the reference declares and leaves
unimplemented (mapping.py:219-221): the window_size keyframes whose voxels overlap the current scan's most (IoU of the voxel sets).
When a sequence returns to a place it has mapped before, those are the old keyframes of that place, so the mapping call reconciles
the revisit with them instead of training the shared embeddings and decoder on the recent keyframes only.

The counts come from csrc/overlap.cu (include/nerfloam_b200.h section 12) against every keyframe at its current pose, in one pass
with no host synchronisation; select_optimize_targets reads them back once.  Their voxel keys are computed in fp64 and may differ
by one voxel, at voxel boundaries, from MapUpdater.create_voxels' fp32 matmul; the selection is a heuristic, so that is harmless.
"""
import random
from collections import namedtuple
from fractions import Fraction

import torch

from . import _capi
from .frame import LidarFrame
from .render_helpers import _frame_points

SLOT_BUDGET = 1 << 25        # keyframe table slots (8 B each: 256 MB), a power of two >= MIN_SLOTS; larger sets go in passes
MIN_SLOTS = 1 << 10
MAX_GRID_DIM = 1 << 18       # voxel keys of 3 x 18 bits
METHODS = ("current", "previous", "random", "overlap")

Overlap = namedtuple("Overlap", ["shared", "kf_voxels", "frame_voxels", "outside"])
Overlap.__doc__ = """Device int64 counts: shared[k] = |V_k n V_c|, kf_voxels[k] = |V_k|, frame_voxels = |V_c| (0-dim),
outside[k] = keyframe k's points whose voxel lies outside [0, grid_dim)^3."""


def _check_grid(voxel_size, grid_dim):
    if isinstance(grid_dim, bool) or int(grid_dim) != grid_dim or not (0 < grid_dim <= MAX_GRID_DIM) or int(grid_dim) & (int(grid_dim) - 1):
        raise ValueError(f"grid_dim must be a power of two <= 2^18, got {grid_dim}")
    if not (float(voxel_size) > 0.0) or float(voxel_size) == float("inf"):
        raise ValueError(f"voxel_size must be finite and > 0, got {voxel_size}")


def _table_slots(counts):
    """Slots of the keyframe table: room for every point at load 1/2, at most SLOT_BUDGET (then the keyframes go in passes)."""
    largest = max(counts, default=0)
    if 2 * largest > SLOT_BUDGET:
        raise ValueError(f"a keyframe of {largest} points does not fit the keyframe table of {SLOT_BUDGET} slots (at most {SLOT_BUDGET // 2})")
    return min(max(MIN_SLOTS, 1 << (2 * sum(counts) - 1).bit_length()), SLOT_BUDGET)


def _overlap_counts(frame, keyframes, voxel_size, grid_dim):
    """The device buffer int64[3K + 1] = (shared, kf_voxels, outside, frame_voxels) of nl_keyframe_overlap."""
    _check_grid(voxel_size, grid_dim)
    dev = torch.device("cuda", torch.cuda.current_device())
    keyframes = list(keyframes)
    K = len(keyframes)
    pts = _frame_points(frame, dev)
    kf_pts = [_frame_points(kf, dev) for kf in keyframes]
    counts = [int(p.shape[0]) for p in kf_pts]
    slots = _table_slots(counts)
    pose6 = torch.stack([f.pose.data.detach().float().reshape(6).cpu() for f in [frame] + keyframes]).to(dev)
    lib = _capi.lib()
    st = _capi.stream_ptr()
    Rt12 = torch.empty((K + 1, 12), dtype=torch.float32, device=dev)
    _capi.check(lib.nl_pose_matrices(K + 1, _capi.ptr(pose6), _capi.ptr(Rt12), st), "nl_pose_matrices")
    host = torch.tensor([[p.data_ptr() for p in kf_pts], counts], dtype=torch.int64).reshape(2, K)
    table = host.pin_memory().to(dev, non_blocking=True) if K else host.to(dev)
    ws_bytes = lib.nl_keyframe_overlap_workspace_bytes(int(pts.shape[0]), slots)
    if ws_bytes < 0:
        _capi.check(int(ws_bytes), "nl_keyframe_overlap_workspace_bytes")
    ws = torch.empty(int(ws_bytes), dtype=torch.uint8, device=dev)
    out = torch.empty(3 * K + 1, dtype=torch.int64, device=dev)
    _capi.check(lib.nl_keyframe_overlap(int(pts.shape[0]), _capi.ptr(pts), K, _capi.ptr(table[0]), _capi.ptr(table[1]), _capi.ptr(host[1]),
                                        _capi.ptr(Rt12), float(voxel_size), int(grid_dim), slots, _capi.ptr(ws), int(ws_bytes),
                                        _capi.ptr(out), st), "nl_keyframe_overlap")
    _capi.LAUNCHES += 2
    return out


def keyframe_overlap(frame, keyframes, voxel_size, grid_dim=256 * 256 * 4):
    """Voxel overlap of `frame`'s scan with each keyframe, every scan at its current pose (frame.pose.data, kf.pose.data), on the GPU.
    Voxels are floor(world / voxel_size) in fp64 (include/nerfloam_b200.h section 12); grid_dim must be a power of two <= 2^18 and
    voxels outside [0, grid_dim)^3 are not counted.  Returns an Overlap of device int64 tensors; nothing is read back."""
    K = len(keyframes)
    out = _overlap_counts(frame, keyframes, voxel_size, grid_dim)
    return Overlap(out[:K], out[K:2 * K], out[3 * K], out[2 * K:3 * K])


def _host_ints(x):
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu()
        return [int(v) for v in x.reshape(-1).tolist()]
    try:
        return [int(v) for v in x]
    except TypeError:
        return [int(x)]


def rank_by_overlap(shared, kf_voxels, frame_voxels, window_size):
    """Indices of the window_size keyframes of highest IoU s / (|V_k| + |V_c| - s) (0 when the denominator is 0), ties to the later
    keyframe, returned in graph order (which keeps bundle_adjust_frames' ray layout deterministic).  Pure host code; the IoUs are
    compared exactly."""
    s, kv = _host_ints(shared), _host_ints(kf_voxels)
    (fv,) = _host_ints(frame_voxels)
    if len(s) != len(kv):
        raise ValueError("shared and kf_voxels must have one entry per keyframe")
    if window_size < 0:
        raise ValueError("window_size must not be negative")
    iou = [Fraction(a, b + fv - a) if b + fv - a > 0 else Fraction(0) for a, b in zip(s, kv)]
    order = sorted(range(len(s)), key=lambda k: (iou[k], k), reverse=True)
    return sorted(order[:window_size])


class KeyframeGraph:
    """The mapper's keyframe bookkeeping under the reference's names (Mapping.keyframe_graph / current_keyframe / insert_keyframe /
    select_optimize_targets and the keyframe-gap test of mapping.py:114-115)."""

    def __init__(self, window_size, keyframe_gap, key_distance, n_rays, voxel_size, grid_dim=256 * 256 * 4):
        _check_grid(voxel_size, grid_dim)
        self.window_size, self.keyframe_gap, self.key_distance, self.n_rays = window_size, keyframe_gap, key_distance, n_rays
        self.voxel_size, self.grid_dim = voxel_size, grid_dim
        self.keyframe_graph = []
        self.current_keyframe = None

    def needs_keyframe(self, frame):
        """mapping.py:114-115: the tracked frame has moved more than keyframe_gap from the current keyframe (always true for the first)."""
        if self.current_keyframe is None:
            return True
        d = frame.pose.translation().detach().cpu() - self.current_keyframe.pose.translation().detach().cpu()
        return bool(torch.norm(d) > self.keyframe_gap)

    def insert_keyframe(self, frame):
        """mapping.py:266-281: the frame's points with |x|, |y|, |z| < key_distance + 0.01 in the sensor frame become a keyframe that
        SHARES the frame's pose object (later bundle adjustments move both).  ValueError below 2 n_rays points."""
        valid = self.key_distance + 0.01
        p = frame.points
        mask = (torch.abs(p[:, 0]) < valid) & (torch.abs(p[:, 1]) < valid) & (torch.abs(p[:, 2]) < valid)
        kf = LidarFrame(frame.index, p[mask], frame.get_pointsCos()[mask], frame.pose, new_keyframe=True)
        if kf.points.shape[0] < 2 * self.n_rays:
            raise ValueError("valid_distance too small")
        self.current_keyframe = kf
        self.keyframe_graph.append(kf)
        return kf

    def select_optimize_targets(self, tracked_frame=None, selection_method="previous", generator=None):
        """mapping.py:205-225 with 'overlap' implemented: the window of keyframes (plus the tracked frame when it is not the current
        keyframe).  'overlap' ranks the keyframes by voxel IoU with tracked_frame, or with the current keyframe when tracked_frame
        is None.  A graph of at most window_size keyframes returns every keyframe.  An unknown method raises ValueError.
        generator: a CPU torch.Generator that 'random' draws its window from (torch.randperm) instead of the `random` module."""
        if selection_method not in METHODS:
            raise ValueError(f"selection method {selection_method!r} unknown (one of {', '.join(METHODS)})")
        if selection_method == "current":
            if tracked_frame is None:
                raise ValueError("select one track frame")
            return [tracked_frame]
        if len(self.keyframe_graph) <= self.window_size:
            targets = self.keyframe_graph[:]
        elif selection_method == "random" and generator is not None:
            targets = [self.keyframe_graph[i] for i in torch.randperm(len(self.keyframe_graph), generator=generator)[:self.window_size].tolist()]
        elif selection_method == "random":
            targets = random.sample(self.keyframe_graph, self.window_size)
        elif selection_method == "previous":
            targets = self.keyframe_graph[-self.window_size:]
        else:
            ref = tracked_frame if tracked_frame is not None else self.current_keyframe
            K = len(self.keyframe_graph)
            c = _overlap_counts(ref, self.keyframe_graph, self.voxel_size, self.grid_dim).cpu()     # the one read-back
            idx = rank_by_overlap(c[:K], c[K:2 * K], c[3 * K], self.window_size)
            targets = [self.keyframe_graph[i] for i in idx]
        if tracked_frame is not None and tracked_frame is not self.current_keyframe:
            targets.append(tracked_frame)
        return targets
