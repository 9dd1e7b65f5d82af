"""Ground segmentation and incidence cosines of one LiDAR scan on the GPU: the (points, pointsCos) the reference's data loaders build
with the external Patchwork++ library and a host KD-tree (src/dataset/kitti.py:40-70).

The segmentation is this project's own definition (DESIGN.md section 12; tests/ground_ref.py restates it in NumPy): a concentric
zone model, seeds from each patch's lowest points, num_iter principal-component plane fits, and an uprightness and elevation verdict.
A ground point's cosine is |n.p| / |p| with n the normal of the ground patch whose mean is nearest; every other point gets 1.  It
follows Patchwork++'s structure and parameter names but claims no parity with it.  The kernels are csrc/ground.cu
(include/nerfloam_b200.h section 13); a call reads back only the four counts.

GroundParams.vertical_cell > 0 turns on the vertical-structure filter (DESIGN.md section 12.1; tests/ground_vertical_ref.py): a return
whose xy column of that width holds returns spread over more than vertical_height in z takes no part in the plane fits and is
non-ground, so walls stop tilting the ground normals next to them.  It is off by default, and off gives exactly the unfiltered results.
"""
import math
from collections import namedtuple
from dataclasses import dataclass

import numpy as np
import torch

from . import _capi


@dataclass(frozen=True)
class GroundParams:
    """Patchwork++'s parameter names; ranges are xy radii in metres.  elevation_thr applies to the first four global rings (ground
    needs mean z + sensor_height below it); flatness_thr is carried for completeness and not used."""
    sensor_height: float = 1.723
    min_range: float = 2.7
    max_range: float = 80.0
    num_rings_each_zone: tuple = (2, 4, 4, 4)
    num_sectors_each_zone: tuple = (16, 32, 54, 32)
    uprightness_thr: float = 0.707
    elevation_thr: tuple = (0.523, 0.746, 0.879, 1.125)
    flatness_thr: tuple = (0.0005, 0.000725, 0.001, 0.001)
    num_iter: int = 3
    num_lpr: int = 20
    num_min_pts: int = 10
    th_seeds: float = 0.125
    th_dist: float = 0.125
    adaptive_seed_margin: float = -1.2
    vertical_cell: float = 0.0          # column width of the vertical filter in metres; 0 = off
    vertical_height: float = 0.3        # a column whose z extent exceeds it (strictly) is vertical

    @property
    def n_patches(self):
        return sum(r * s for r, s in zip(self.num_rings_each_zone, self.num_sectors_each_zone))

    def to_c(self):
        for name in ("num_rings_each_zone", "num_sectors_each_zone", "elevation_thr", "flatness_thr"):
            if len(getattr(self, name)) != 4:
                raise ValueError(f"{name} must have one entry per zone (4)")
        cell, height = float(self.vertical_cell), float(self.vertical_height)
        if not (math.isfinite(cell) and cell >= 0.0):
            raise ValueError(f"vertical_cell must be finite and >= 0 (0 = off), got {cell}")
        if cell > 0.0:
            if not (math.isfinite(height) and height > 0.0):
                raise ValueError(f"vertical_height must be positive and finite when vertical_cell > 0, got {height}")
            if not float(self.max_range) / cell <= 2.0 ** 30:
                raise ValueError(f"vertical_cell {cell} too small: the cell keys need max_range / vertical_cell <= 2^30")
        c = _capi.GroundParams()
        for name in ("sensor_height", "min_range", "max_range", "uprightness_thr", "th_seeds", "th_dist", "adaptive_seed_margin",
                     "vertical_cell", "vertical_height"):
            setattr(c, name, float(getattr(self, name)))
        for name in ("num_iter", "num_lpr", "num_min_pts"):
            setattr(c, name, int(getattr(self, name)))
        for name in ("num_rings_each_zone", "num_sectors_each_zone"):
            getattr(c, name)[:] = [int(v) for v in getattr(self, name)]
        for name in ("elevation_thr", "flatness_thr"):
            getattr(c, name)[:] = [float(v) for v in getattr(self, name)]
        return c


Ground = namedtuple("Ground", ["label", "cos", "patch", "patches", "counts", "vertical"])
Ground.__doc__ = """Device tensors: label u8[N] (1 = ground), cos f32[N], patch i32[N] (-1 outside the ranges), patches (PatchRecords),
counts i64[4] = (ground, non-ground, outside, non-finite); non-ground includes the outside rows.  vertical u8[N] (1 = vertical
structure) when the vertical filter is on, None when it is off."""
PatchRecords = namedtuple("PatchRecords", ["mean", "normal", "d", "lambda_min", "n_points", "n_ground", "ground", "ring", "n_vertical"])
PatchRecords.__doc__ = """One row per patch (zone by zone, ring by ring, sector by sector): mean f64[P,3], normal f64[P,3] (n_z >= 0),
d f64[P], lambda_min f64[P] (NaN without a complete fit), n_points (vertical points included), n_ground, ground (verdict), ring
(global ring), n_vertical (0 with the filter off) i32[P]."""


def _device_points(points):
    if isinstance(points, np.ndarray):
        points = torch.from_numpy(points)
    if not isinstance(points, torch.Tensor):
        raise TypeError("points must be a numpy array or a torch tensor")
    if points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] not in (3, 4):
        raise ValueError(f"points must be float32 [N,3] or [N,4], got {tuple(points.shape)} {points.dtype}")
    dev = torch.device("cuda", torch.cuda.current_device()) if not points.is_cuda else points.device
    return points.to(dev).contiguous()


def _workspace(lib, n, dev):
    ws_bytes = lib.nl_ground_workspace_bytes(n)
    if ws_bytes < 0:
        _capi.check(int(ws_bytes), "nl_ground_workspace_bytes")
    return torch.empty(int(ws_bytes), dtype=torch.uint8, device=dev), int(ws_bytes)


def _segment(pts, params):
    params = params or GroundParams()
    cp = params.to_c()
    lib = _capi.lib()
    n, dev = int(pts.shape[0]), pts.device
    ws, ws_bytes = _workspace(lib, n, dev)
    label = torch.empty(n, dtype=torch.uint8, device=dev)
    cos = torch.empty(n, dtype=torch.float32, device=dev)
    patch = torch.empty(n, dtype=torch.int32, device=dev)
    raw = torch.empty((max(params.n_patches, 0), _capi.GROUND_PATCH_BYTES), dtype=torch.uint8, device=dev)
    counts = torch.empty(4, dtype=torch.int64, device=dev)
    vertical = None
    with torch.cuda.device(dev):
        if params.vertical_cell > 0:
            vws_bytes = lib.nl_ground_vertical_workspace_bytes(n)
            if vws_bytes < 0:
                _capi.check(int(vws_bytes), "nl_ground_vertical_workspace_bytes")
            vws = torch.empty(int(vws_bytes), dtype=torch.uint8, device=dev)
            vertical = torch.empty(n, dtype=torch.uint8, device=dev)
            _capi.check(lib.nl_ground_segment_vertical(n, _capi.ptr(pts), int(pts.shape[1]), cp, _capi.ptr(ws), ws_bytes, _capi.ptr(vws),
                                                       int(vws_bytes), _capi.ptr(label), _capi.ptr(cos), _capi.ptr(patch), _capi.ptr(raw),
                                                       _capi.ptr(vertical), _capi.ptr(counts), _capi.stream_ptr()), "nl_ground_segment_vertical")
        else:
            _capi.check(lib.nl_ground_segment(n, _capi.ptr(pts), int(pts.shape[1]), cp, _capi.ptr(ws), ws_bytes, _capi.ptr(label), _capi.ptr(cos),
                                              _capi.ptr(patch), _capi.ptr(raw), _capi.ptr(counts), _capi.stream_ptr()), "nl_ground_segment")
    _capi.LAUNCHES += 1
    host = counts.cpu()                                                       # the one read-back
    if int(host[3]):
        raise ValueError(f"points has {int(host[3])} rows with a non-finite coordinate")
    f64, i32 = raw.view(torch.float64), raw.view(torch.int32)
    rec = PatchRecords(f64[:, 0:3], f64[:, 3:6], f64[:, 6], f64[:, 7], i32[:, 16], i32[:, 17], i32[:, 18], i32[:, 19], i32[:, 20])
    return Ground(label, cos, patch, rec, counts, vertical), ws, ws_bytes


def segment_ground(points, params=None):
    """Ground labels and incidence cosines of one scan (float32 [N,3] or [N,4] in the sensor frame; a fourth column is ignored),
    numpy or torch, on the current CUDA device.  Returns a Ground of device tensors.  A row with a NaN or inf raises ValueError, and so
    do invalid vertical-filter settings."""
    return _segment(_device_points(points), params)[0]


def points_and_cos(points, params=None):
    """(points f32[N,3], pointcos f32[N], index i32[N]) on the device: the ground points first, then the rest, each half in input
    order; index[k] is the input row of output row k."""
    pts = _device_points(points)
    g, ws, ws_bytes = _segment(pts, params)
    n = int(pts.shape[0])
    out = torch.empty((n, 3), dtype=torch.float32, device=pts.device)
    cos = torch.empty(n, dtype=torch.float32, device=pts.device)
    index = torch.empty(n, dtype=torch.int32, device=pts.device)
    with torch.cuda.device(pts.device):
        _capi.check(_capi.lib().nl_ground_partition(n, _capi.ptr(pts), int(pts.shape[1]), _capi.ptr(g.label), _capi.ptr(g.cos), _capi.ptr(ws),
                                                    ws_bytes, _capi.ptr(out), _capi.ptr(cos), _capi.ptr(index), _capi.stream_ptr()),
                    "nl_ground_partition")
    _capi.LAUNCHES += 1
    return out, cos, index
