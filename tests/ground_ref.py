"""NumPy restatement of the ground segmentation (nerf-loam_b200/ground.py, csrc/ground.cu, DESIGN.md section 12), written from the
definitions, step by step, for the kernel tests to compare against value by value.  `params` is any object with GroundParams' fields.

Besides the results, it reports what the comparison needs to exempt: each point's distance to its nearest bin edge (in bin widths),
each patch's smallest eigenvalue gap and smallest margin to a seed or th_dist cut, each verdict's margin to its thresholds, and each
ground point's relative gap between its nearest and second-nearest ground-patch mean."""
import numpy as np

TWO_PI = 2.0 * np.pi


def zone_edges(p):
    lo, hi = float(p.min_range), float(p.max_range)
    return (lo, (7.0 * lo + hi) / 8.0, (3.0 * lo + hi) / 4.0, (lo + hi) / 2.0, hi)


def n_patches(p):
    return sum(r * s for r, s in zip(p.num_rings_each_zone, p.num_sectors_each_zone))


def bin_points(points, p):
    """(patch id i64[N] (-1 outside or not finite), zone i64[N], global ring i64[N], edge margin f64[N] in bin widths)."""
    P = np.asarray(points, np.float32)
    n = P.shape[0]
    x, y = P[:, 0].astype(np.float64), P[:, 1].astype(np.float64)
    finite = np.isfinite(P[:, :3]).all(1)
    with np.errstate(invalid="ignore"):
        r = np.sqrt(x * x + y * y)
        th = np.arctan2(y, x)
    th = np.where(th < 0.0, th + TWO_PI, th)
    b = zone_edges(p)
    pid, zone, gring = np.full(n, -1, np.int64), np.full(n, -1, np.int64), np.full(n, -1, np.int64)
    margin = np.full(n, np.inf)
    with np.errstate(invalid="ignore", divide="ignore"):
        for e in (b[0], b[4]):
            margin = np.where(finite, np.minimum(margin, np.abs(r - e) / e), margin)
    off = roff = 0
    for z in range(4):
        rings, secs = int(p.num_rings_each_zone[z]), int(p.num_sectors_each_zone[z])
        with np.errstate(invalid="ignore"):
            m = finite & (r >= b[z]) & (r < b[z + 1])
        w, ws = (b[z + 1] - b[z]) / rings, TWO_PI / secs
        qr, qs = (r[m] - b[z]) / w, th[m] / ws
        ring = np.minimum(np.floor(qr), rings - 1).astype(np.int64)
        sec = np.minimum(np.floor(qs), secs - 1).astype(np.int64)
        pid[m] = off + ring * secs + sec
        zone[m] = z
        gring[m] = roff + ring
        margin[m] = np.minimum(margin[m], np.minimum(np.abs(qr - np.round(qr)), np.abs(qs - np.round(qs))))
        off += rings * secs
        roff += rings
    return pid, zone, gring, margin


def eig3(C):
    """Cyclic Jacobi on a symmetric 3x3, the kernel's order of operations: (eigenvalues f64[3], eigenvectors as columns f64[3,3])."""
    A = [[float(C[i][j]) for j in range(3)] for i in range(3)]
    V = [[1.0 if i == j else 0.0 for j in range(3)] for i in range(3)]
    for _ in range(32):
        off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2]
        dia = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2]
        if not off > 1e-40 * dia:
            break
        for p, q in ((0, 1), (0, 2), (1, 2)):
            r = 3 - p - q
            apq = A[p][q]
            if apq == 0.0:
                continue
            theta = (A[q][q] - A[p][p]) / (2.0 * apq)
            t = 0.5 / theta if abs(theta) > 1e150 else (1.0 if theta >= 0.0 else -1.0) / (abs(theta) + np.sqrt(theta * theta + 1.0))
            cs = 1.0 / np.sqrt(t * t + 1.0)
            sn = t * cs
            A[p][p] -= t * apq
            A[q][q] += t * apq
            A[p][q] = A[q][p] = 0.0
            arp, arq = A[r][p], A[r][q]
            A[r][p] = A[p][r] = cs * arp - sn * arq
            A[r][q] = A[q][r] = sn * arp + cs * arq
            for k in range(3):
                vkp, vkq = V[k][p], V[k][q]
                V[k][p] = cs * vkp - sn * vkq
                V[k][q] = sn * vkp + cs * vkq
    return np.array([A[0][0], A[1][1], A[2][2]]), np.array(V)


def _min_eig(C):
    lam, V = eig3(C)
    m = 0
    if lam[1] < lam[m]:
        m = 1
    if lam[2] < lam[m]:
        m = 2
    return lam[m], V[:, m].copy(), float(np.sort(lam)[1] - lam[m])


def segment(points, p):
    """The segmentation of one scan: a dict of label u8[N], cos f32[N], patch i64[N], counts (ground, non-ground, outside, non-finite),
    the per-patch records (mean, normal, d, lambda_min, n_points, n_ground, ground, ring) and the margins listed above."""
    P = np.asarray(points, np.float32)
    n = P.shape[0]
    X = P[:, :3].astype(np.float64)
    pid, zone, gring, edge_margin = bin_points(P, p)
    NP = n_patches(p)
    nan3 = np.full((NP, 3), np.nan)
    rec = dict(mean=nan3.copy(), normal=nan3.copy(), d=np.full(NP, np.nan), lambda_min=np.full(NP, np.nan), n_points=np.zeros(NP, np.int64),
               n_ground=np.zeros(NP, np.int64), ground=np.zeros(NP, np.int64), ring=np.zeros(NP, np.int64),
               eig_gap=np.full(NP, np.inf), cut_margin=np.full(NP, np.inf), verdict_margin=np.full(NP, np.inf))
    off = np.cumsum([0] + [r * s for r, s in zip(p.num_rings_each_zone, p.num_sectors_each_zone)])
    roff = np.cumsum([0] + list(p.num_rings_each_zone))
    for q in range(NP):
        z = int(np.searchsorted(off, q, side="right") - 1)
        rec["ring"][q] = roff[z] + (q - off[z]) // p.num_sectors_each_zone[z]
    label = np.zeros(n, np.uint8)
    key = np.where(pid < 0, NP, pid)
    order = np.argsort(key, kind="stable")
    starts = np.searchsorted(key[order], np.arange(NP + 1))
    seed_floor = float(p.adaptive_seed_margin) * float(p.sensor_height)
    for q in range(NP):
        idx = order[starts[q]:starts[q + 1]]
        cnt = idx.size
        rec["n_points"][q] = cnt
        if cnt < p.num_min_pts or cnt == 0:
            continue
        Q = X[idx]
        cand = ~((q < off[1]) & (Q[:, 2] < seed_floor))
        zc = np.sort(Q[cand, 2])
        if zc.size == 0:
            continue
        k = min(int(p.num_lpr), zc.size)
        s = 0.0
        for v in zc[:k]:
            s += float(v)
        cut = s / k + float(p.th_seeds)
        sel = cand & (Q[:, 2] < cut)
        margin = float(np.min(np.abs(Q[cand, 2] - cut)))
        ok = True
        for _ in range(int(p.num_iter)):
            S = Q[sel]
            if S.shape[0] < 3:
                ok = False
                break
            mu = S.mean(0)
            D = S - mu
            C = D.T @ D / S.shape[0]
            lam, nrm, gap = _min_eig(C)
            if nrm[2] < 0.0:
                nrm = -nrm
            d = -((nrm[0] * mu[0] + nrm[1] * mu[1]) + nrm[2] * mu[2])
            dist = Q @ nrm + d
            margin = min(margin, float(np.min(np.abs(dist - float(p.th_dist)))))
            sel = dist < float(p.th_dist)
        if not ok:
            continue
        ring = int(rec["ring"][q])
        rec["mean"][q], rec["normal"][q], rec["d"][q], rec["lambda_min"][q], rec["eig_gap"][q] = mu, nrm, d, lam, gap
        rec["cut_margin"][q] = margin
        up = nrm[2] >= float(p.uprightness_thr)
        vm = abs(nrm[2] - float(p.uprightness_thr))
        low = True
        if ring < 4:
            h = mu[2] + float(p.sensor_height)
            low = h < float(p.elevation_thr[ring])
            vm = min(vm, abs(h - float(p.elevation_thr[ring])))
        rec["verdict_margin"][q] = vm
        if up and low:
            rec["ground"][q] = 1
            rec["n_ground"][q] = int(sel.sum())
            label[idx[sel]] = 1
    cos = np.ones(n, np.float32)
    tie = np.full(n, np.inf)
    gp = np.flatnonzero(rec["ground"])
    gi = np.flatnonzero(label)
    if gi.size:
        M, Nn = rec["mean"][gp], rec["normal"][gp]
        for c0 in range(0, gi.size, 8192):
            rows = gi[c0:c0 + 8192]
            Y = X[rows]
            d2 = ((Y[:, None, 0] - M[None, :, 0]) ** 2 + (Y[:, None, 1] - M[None, :, 1]) ** 2) + (Y[:, None, 2] - M[None, :, 2]) ** 2
            a = np.argmin(d2, axis=1)
            best = d2[np.arange(rows.size), a]
            if gp.size > 1:
                second = np.partition(d2, 1, axis=1)[:, 1]
                tie[rows] = (second - best) / np.maximum(best, 1e-300)
            nn = Nn[a]
            dot = (nn[:, 0] * Y[:, 0] + nn[:, 1] * Y[:, 1]) + nn[:, 2] * Y[:, 2]
            cos[rows] = (np.abs(dot) / np.sqrt((Y[:, 0] * Y[:, 0] + Y[:, 1] * Y[:, 1]) + Y[:, 2] * Y[:, 2])).astype(np.float32)
    finite = np.isfinite(P[:, :3]).all(1)
    n_ground = int(label.sum())
    counts = np.array([n_ground, n - n_ground, int((finite & (pid < 0)).sum()), int((~finite).sum())], np.int64)
    return dict(label=label, cos=cos, patch=pid, zone=zone, ring=gring, edge_margin=edge_margin, tie=tie, counts=counts, patches=rec)


def points_and_cos(points, p):
    """(points f32[N,3] ground first, each half in input order; pointcos f32[N]; index i64[N] into the input)."""
    r = segment(points, p)
    index = np.concatenate([np.flatnonzero(r["label"] == 1), np.flatnonzero(r["label"] == 0)])
    return np.asarray(points, np.float32)[index, :3], r["cos"][index], index
