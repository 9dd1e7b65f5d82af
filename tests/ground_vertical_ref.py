"""NumPy restatement of the vertical-structure filter of the ground segmentation (DESIGN.md section 12.1, csrc/ground.cu): flag the
vertical rows, run tests/ground_ref.py's segmentation on the other rows, and map its results back.  `params` is any object with
GroundParams' fields, vertical_cell and vertical_height included.

A row is vertical when it is finite, inside [min_range, max_range), and the returns of its xy column -- the cell
(floor(x / vertical_cell), floor(y / vertical_cell)), fp64 from the fp32 row -- spread over more than vertical_height in z.  A vertical
row is never a seed candidate nor in any fit; it is labelled non-ground with cos 1.  With vertical_cell = 0 nothing is vertical and
the result is ground_ref.segment's."""
import numpy as np

import ground_ref as GR


def vertical_flags(points, p):
    """(vertical bool[N], cell-edge margin f64[N] in cells (inf where the filter does not apply), extent f64[N] of each row's cell)."""
    P = np.asarray(points, np.float32)
    n = P.shape[0]
    vert, margin, extent = np.zeros(n, bool), np.full(n, np.inf), np.full(n, np.nan)
    cell = float(p.vertical_cell)
    if cell == 0.0 or n == 0:
        return vert, margin, extent
    pid = GR.bin_points(P, p)[0]
    rows = np.flatnonzero(pid >= 0)
    if rows.size == 0:
        return vert, margin, extent
    X = P[rows, :3].astype(np.float64)
    qx, qy = X[:, 0] / cell, X[:, 1] / cell
    cx, cy = np.floor(qx).astype(np.int64), np.floor(qy).astype(np.int64)
    _, inv = np.unique(np.stack([cx, cy], 1), axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    lo = np.full(inv.max() + 1, np.inf)
    hi = np.full(inv.max() + 1, -np.inf)
    np.minimum.at(lo, inv, X[:, 2])
    np.maximum.at(hi, inv, X[:, 2])
    ext = (hi - lo)[inv]
    vert[rows] = ext > float(p.vertical_height)
    margin[rows] = np.minimum(np.abs(qx - np.round(qx)), np.abs(qy - np.round(qy)))
    extent[rows] = ext
    return vert, margin, extent


def segment(points, p):
    """ground_ref.segment's dict for the whole scan with the filter applied, plus vertical u8[N], cell_margin f64[N] and extent f64[N];
    the patch records gain n_vertical, and their n_points counts every row of the patch."""
    P = np.asarray(points, np.float32)
    n = P.shape[0]
    vert, cell_margin, extent = vertical_flags(P, p)
    keep = np.flatnonzero(~vert)
    r = GR.segment(P[keep], p)
    pid, zone, gring, edge_margin = GR.bin_points(P, p)
    label = np.zeros(n, np.uint8)
    cos = np.ones(n, np.float32)
    tie = np.full(n, np.inf)
    label[keep], cos[keep], tie[keep] = r["label"], r["cos"], r["tie"]
    NP = GR.n_patches(p)
    rec = dict(r["patches"])
    rec["n_points"] = np.bincount(pid[pid >= 0], minlength=NP).astype(np.int64)
    rec["n_vertical"] = np.bincount(pid[vert], minlength=NP).astype(np.int64)
    finite = np.isfinite(P[:, :3]).all(1)
    n_ground = int(label.sum())
    counts = np.array([n_ground, n - n_ground, int((finite & (pid < 0)).sum()), int((~finite).sum())], np.int64)
    return dict(label=label, cos=cos, patch=pid, zone=zone, ring=gring, edge_margin=edge_margin, tie=tie, counts=counts, patches=rec,
                vertical=vert.astype(np.uint8), cell_margin=cell_margin, extent=extent)
