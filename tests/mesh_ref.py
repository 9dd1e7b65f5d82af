"""Yardsticks of mesh extraction (render_helpers.scores_device -> csrc/mc.cu -> mesh.extract_mesh), NumPy only.

emit_ref restates nl_mc_count + nl_mc_emit exactly, vectorised over voxels, with the case table read from nl_mc_case_table (a host
function; tests/test_mc_cpu.py pins it to oracle/mc.py):
  * per-voxel vertex and triangle counts, their exclusive offsets in int64;
  * the vertices of a voxel in lattice-edge-id order (axis-major, then i, j, k), at
        v = ((p * inv) - 0.5) * vs + c,    p = (i, j, k) with t = s0 / (s0 - s1) added along the edge's axis, inv = 1 / (res - 1),
    every operation rounded separately in fp32, as the kernel writes it;
  * the triangles in voxel-major, cell-major, table order, as vertex ids voff + rank.
A lattice value counts as inside when it is < 0: NaN, +0 and -0 are outside.

vertex_fp64 gives the crossing in fp64 from the same fp32 inputs, c + ((i + s0 / (s0 - s1)) / (res - 1) - 0.5) vs, and a
per-coordinate bar on the kernel's error.  u = 2^-24; every fp32 rounding of a value x is x (1 + d), |d| <= u.  With X the exact
p / (res - 1) in [0, 1], r = X - 0.5, w = r vs and o = w + c (all exact, fp64), the eight roundings contribute, to first order,
  s0 - s1        t (1 + d1)^-1                     u |t|                 (t in [0, 1]: s0 and s1 have opposite signs)
  the division   t (1 + d2)                        u |t|
  i + t          p (1 + d3)                        u |p|
  the rounding of inv = 1/(res-1)                  u |X|                 (carried through p * inv)
  * inv                                            u |X|
  - 0.5                                            u |r|
  * vs                                             u |w|
  + c                                              u |o|
The first five are errors in X and reach the output times vs:
    bar = u [ vs ((2 |t| + |p|) / (res - 1) + 2 |X| + |r|) + |w| + |o| ]      (t = 0 on the other two coordinates)
plus a relative 2^-20 and an absolute 2^-149 vs for the second-order terms and a subnormal t.  Lattices with |s| >= 2^126 are
left out of the fp64 check (s0 - s1 can overflow there; the restatement alone pins them), and so is every non-finite vertex.

The lattice yardstick restates scores_device: lattice point = fp32(linspace(-0.5, 0.5, res) * vs) + centre (two fp32 roundings,
render_helpers._lattice_offsets), features by embedding_ref.gather_fwd_f32 (bit-exact), sdf in fp64 by decoder_ref.forward within
decoder_tc_ref's HARD bar (width 256, tensor cores) or (2W + 20) u a_sdf (widths 32-128, CUDA cores)."""
import ctypes as C
import itertools

import numpy as np

F32 = np.float32
U = 2.0 ** -24


# ------------------------------------------------------------------------------------------------ the case table
_TABLE = None


def case_table():
    """(tri u8[256,16], ntri u8[256], edge_corner u8[12,2]) from nl_mc_case_table (host only)."""
    global _TABLE
    if _TABLE is None:
        import nerfloam_b200 as nl
        tri = np.zeros((256, 16), np.uint8); nt = np.zeros(256, np.uint8); ec = np.zeros((12, 2), np.uint8)
        assert nl._capi.lib().nl_mc_case_table(tri.ctypes.data_as(C.c_void_p), nt.ctypes.data_as(C.c_void_p),
                                                 ec.ctypes.data_as(C.c_void_p)) == 0
        _TABLE = tri, nt, ec
    return _TABLE


# ------------------------------------------------------------------------------------------------ lattice edges
def _edges(sdf):
    """Per voxel, every lattice edge in the kernel's id order: (s0 [n,E], s1 [n,E], axis [E], ijk [E,3]) with E = 3 res^2 (res-1).
    Axis a's edges run over the lattice with res - 1 points along a, row-major in (i, j, k)."""
    n, res = sdf.shape[0], sdf.shape[1]
    s0, s1, axis, ijk = [], [], [], []
    for a in range(3):
        lo = [slice(None)] * 4; hi = [slice(None)] * 4
        lo[a + 1] = slice(0, res - 1); hi[a + 1] = slice(1, res)
        ne = res * res * (res - 1)
        s0.append(sdf[tuple(lo)].reshape(n, ne)); s1.append(sdf[tuple(hi)].reshape(n, ne))
        shape = [res, res, res]; shape[a] = res - 1
        g = np.stack(np.meshgrid(*[np.arange(m) for m in shape], indexing="ij"), -1).reshape(-1, 3)
        axis.append(np.full(len(g), a)); ijk.append(g)
    return np.concatenate(s0, 1), np.concatenate(s1, 1), np.concatenate(axis), np.concatenate(ijk)


def _edge_id(axis, i, j, k, res):
    """edge_encode of csrc/mc.cu."""
    m, nea = res - 1, res * res * (res - 1)
    return np.where(axis == 0, (i * res + j) * res + k,
                    np.where(axis == 1, nea + (i * m + j) * res + k, 2 * nea + (i * res + j) * m + k))


def _centres_of(centres, vox_ids, n):
    c = np.asarray(centres, F32).reshape(-1, 3)
    return c[np.arange(n) if vox_ids is None else np.asarray(vox_ids, np.int64)]


def vertices_f32(s0, s1, axis, ijk, c, res, voxel_size, inv=None, swap=None):
    """The kernel's vertex formula in fp32 (every step rounded separately) for crossed edges with values s0, s1, base point ijk
    [V,3] along `axis` [V] and centre c [V,3].  inv / swap exist to build mutants: a different inv, or two axes exchanged."""
    with np.errstate(all="ignore"):
        t = (s0 - s1).astype(F32)
        t = (s0 / t).astype(F32)
        p = ijk.astype(F32)
        p[np.arange(len(p)), axis] = (p[np.arange(len(p)), axis] + t).astype(F32)
        if swap is not None:
            p[:, list(swap)] = p[:, list(swap)[::-1]]
        inv = F32(1.0) / F32(res - 1) if inv is None else F32(inv)
        return ((p * inv - F32(0.5)) * F32(voxel_size) + c).astype(F32)


def emit_ref(sdf, centres, voxel_size, vox_ids=None, chunk=256):
    """nl_mc_count + nl_mc_emit restated.  sdf f32 [n,res,res,res], centres f32 [N,3], vox_ids [n] rows of centres (None: row v).
    Returns dict nvert, ntri (int32 [n]), voff, toff (int64 [n], exclusive), totals (int64 (V, T)), verts f32 [V,3],
    faces int64 [T,3] (ids voff + rank), vert_vox / tri_vox int64 (the voxel of each row)."""
    tri, ntri_tab, ec = case_table()
    sdf = np.asarray(sdf, F32)
    n, res = sdf.shape[0], sdf.shape[1]
    m = res - 1
    cen = _centres_of(centres, vox_ids, n)
    nvert, ntri = np.zeros(n, np.int64), np.zeros(n, np.int64)
    verts, faces_local, vert_vox, tri_vox = [], [], [], []
    # corner c of cell (ci, cj, ck) sits at (ci + (c & 1), cj + (c >> 1 & 1), ck + (c >> 2 & 1))
    cell = np.stack(np.meshgrid(np.arange(m), np.arange(m), np.arange(m), indexing="ij"), -1).reshape(-1, 3)
    for v0 in range(0, n, chunk):
        s = sdf[v0:v0 + chunk]
        nb = s.shape[0]
        s0, s1, axis, ijk = _edges(s)
        cross = (s0 < 0) != (s1 < 0)                                       # [nb, E]
        rank = np.cumsum(cross, 1) - 1
        nvert[v0:v0 + nb] = cross.sum(1)
        vv, ee = np.nonzero(cross)                                          # voxel-major, edge-id order
        verts.append(vertices_f32(s0[vv, ee], s1[vv, ee], axis[ee], ijk[ee], cen[v0 + vv], res, voxel_size))
        vert_vox.append(v0 + vv)
        cfg = np.zeros((nb, len(cell)), np.int64)
        for c in range(8):
            cfg |= (s[:, cell[:, 0] + (c & 1), cell[:, 1] + (c >> 1 & 1), cell[:, 2] + (c >> 2 & 1)] < 0).astype(np.int64) << c
        nt = ntri_tab[cfg].astype(np.int64)                                 # [nb, ncell]
        ntri[v0:v0 + nb] = nt.sum(1)
        tv, tc, tq = np.nonzero(np.arange(5)[None, None, :] < nt[:, :, None])   # voxel-major, cell-major, table order
        f = np.empty((len(tv), 3), np.int64)
        for r in range(3):
            e = tri[cfg[tv, tc], 3 * tq + r].astype(np.int64)
            c0 = ec[e, 0].astype(np.int64)
            b = cell[tc] + np.stack([c0 & 1, c0 >> 1 & 1, c0 >> 2 & 1], 1)
            f[:, r] = rank[tv, _edge_id(e >> 2, b[:, 0], b[:, 1], b[:, 2], res)]
        faces_local.append(f)
        tri_vox.append(v0 + tv)
    voff = np.concatenate([[0], np.cumsum(nvert)[:-1]]).astype(np.int64) if n else np.zeros(0, np.int64)
    toff = np.concatenate([[0], np.cumsum(ntri)[:-1]]).astype(np.int64) if n else np.zeros(0, np.int64)
    cat = lambda xs, shape, dt: np.concatenate(xs) if xs else np.zeros(shape, dt)
    vert_vox, tri_vox = cat(vert_vox, (0,), np.int64), cat(tri_vox, (0,), np.int64)
    faces = cat(faces_local, (0, 3), np.int64) + (voff[tri_vox][:, None] if n else 0)
    return dict(nvert=nvert.astype(np.int32), ntri=ntri.astype(np.int32), voff=voff, toff=toff,
                totals=np.array([nvert.sum(), ntri.sum()], np.int64), verts=cat(verts, (0, 3), F32).reshape(-1, 3),
                faces=faces, vert_vox=vert_vox, tri_vox=tri_vox)


# ------------------------------------------------------------------------------------------------ fp64 crossing and its bar
def vertex_fp64(sdf, centres, voxel_size, vox_ids=None):
    """(v [V,3] fp64, bar [V,3], checked bool [V]) for every crossed edge, in emit_ref's order.  `checked`: the voxel's lattice
    is finite with |s| < 2^126 (the others are pinned by the restatement alone)."""
    sdf = np.asarray(sdf, F32)
    n, res = sdf.shape[0], sdf.shape[1]
    cen = _centres_of(centres, vox_ids, n).astype(np.float64)
    flat = sdf.reshape(n, res ** 3)
    ok_vox = np.isfinite(flat).all(1) & (np.abs(flat) < 2.0 ** 126).all(1)
    s0, s1, axis, ijk = _edges(sdf)
    cross = (s0 < 0) != (s1 < 0)
    vv, ee = np.nonzero(cross)
    a, b = s0[vv, ee].astype(np.float64), s1[vv, ee].astype(np.float64)
    with np.errstate(all="ignore"):
        t = a / (a - b)
    onaxis = np.arange(3)[None, :] == axis[ee][:, None]
    p = ijk[ee].astype(np.float64) + np.where(onaxis, t[:, None], 0.0)
    vs = np.float64(F32(voxel_size))
    X = p / (res - 1)
    r = X - 0.5
    w = r * vs
    o = w + cen[vv]
    at = np.where(onaxis, np.abs(t)[:, None], 0.0)
    bar = U * (vs * ((2 * at + np.abs(p)) / (res - 1) + 2 * np.abs(X) + np.abs(r)) + np.abs(w) + np.abs(o))
    bar = bar * (1 + 2.0 ** -20) + 2.0 ** -149 * vs
    return o, bar, ok_vox[vv] & np.isfinite(o).all(1)


def fp64_ratio(got, sdf, centres, voxel_size, vox_ids=None):
    """max over the checked vertices and coordinates of |got - fp64| / bar (0 when nothing is checked)."""
    v, bar, ok = vertex_fp64(sdf, centres, voxel_size, vox_ids)
    if not ok.any():
        return 0.0
    return float((np.abs(np.asarray(got, np.float64)[ok] - v[ok]) / bar[ok]).max())


def same_f32(a, b):
    """Bit-equal float32 arrays, except that any NaN equals any NaN (the kernel's NaN is 0x7fffffff, NumPy's 0xffc00000)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)))


# ------------------------------------------------------------------------------------------------ oracle/mc.py
def _boundary(tris):
    """Directed boundary edges of oriented triangles (interior diagonals cancel): equal for two fans of the same polygons."""
    cnt = {}
    for t in tris:
        for i in range(3):
            a, b = t[i], t[(i + 1) % 3]
            if cnt.get((b, a), 0) > 0:
                cnt[(b, a)] -= 1
            else:
                cnt[(a, b)] = cnt.get((a, b), 0) + 1
    return sorted(k for k, v in cnt.items() for _ in range(v))


def check_against_oracle(ref, sdf, centres, voxel_size, voxels, vox_ids=None):
    """ref = emit_ref(sdf, centres, ...) (or the kernel's output in the same layout: verts, faces, voff, toff, nvert, ntri)
    against oracle/mc.py for the listed voxels: the vertex dict in order (the oracle's dict runs over the edges in the kernel's
    id order), bit for bit, and the triangles cell by cell as oriented boundaries over those vertex indices."""
    from oracle import mc as OM
    res = sdf.shape[1]
    cen = np.asarray(centres, np.float32)[np.arange(sdf.shape[0]) if vox_ids is None else np.asarray(vox_ids)]
    for v in voxels:
        with np.errstate(all="ignore"):                                    # inf / NaN lattices
            want_v, _ = OM.marching_cubes_voxel(sdf[v], cen[v], voxel_size)
        vo, nv = int(ref["voff"][v]), int(ref["nvert"][v])
        assert nv == len(want_v), v
        got = ref["verts"][vo:vo + nv]
        assert same_f32(got, np.array([np.asarray(p, np.float32) for p in want_v.values()]).reshape(-1, 3)), v
        pos = {k: r for r, k in enumerate(want_v)}
        gpos = range(nv)
        neg = sdf[v] < 0
        to = int(ref["toff"][v])
        for ci, cj, ck in itertools.product(range(res - 1), repeat=3):
            neg8 = {(x, y, z): bool(neg[ci + x, cj + y, ck + z]) for x, y, z in itertools.product((0, 1), repeat=3)}
            want = [tuple(pos[(a, ci + x, cj + y, ck + z)] for (a, x, y, z) in t) for t in OM.cell_polygons(neg8)]
            f = np.asarray(ref["faces"][to:to + len(want)], np.int64) - vo
            assert len(want) == 0 or (f.min() >= 0 and f.max() < nv), (v, ci, cj, ck)
            assert _boundary([tuple(gpos[i] for i in t) for t in f]) == _boundary(want), (v, ci, cj, ck)
            to += len(want)
        assert to == int(ref["toff"][v]) + int(ref["ntri"][v]), v


# ------------------------------------------------------------------------------------------------ the lattice
def lattice_offsets(res, voxel_size):
    """fp32 [res^3, 3]: linspace(-0.5, 0.5, res) on the meshgrid (torch's fp32 linspace, as _lattice_offsets takes it) times
    fp32(voxel_size), one rounding."""
    import torch
    lin = torch.linspace(-0.5, 0.5, res).numpy().astype(F32)
    g = np.stack(np.meshgrid(lin, lin, lin, indexing="ij"), -1).reshape(-1, 3)
    return (g * F32(voxel_size)).astype(F32)


def lattice_points(centres, res, voxel_size):
    """fp32 [n, res^3, 3]: offsets + centre, one more rounding."""
    return (lattice_offsets(res, voxel_size)[None] + np.asarray(centres, F32)[:, None, :]).astype(F32)


# ------------------------------------------------------------------------------------------------ test inputs
CENTRES = ((0.15, 0.11, 0.17), (1.05, 0.95, 1.12), (-80.15, 37.2, -79.9), (2000.41, 2000.38, 2000.47))


def random_centres(rng, n, voxel_size):
    """n fp32 centres cycling over the four magnitudes of CENTRES, each jittered by up to a few voxels."""
    base = np.asarray(CENTRES)[np.arange(n) % len(CENTRES)]
    return (base + rng.uniform(-3, 3, size=(n, 3)) * voxel_size).astype(F32)


def random_lattices(rng, n, res):
    """f32 [n,res,res,res]: about a third of the voxels cross zero (N(0,1) plus an offset in [-0.8, 0.8], or a smooth plane
    through the voxel), a third are all positive and a third all negative."""
    kind = np.arange(n) % 3
    s = rng.standard_normal((n, res, res, res))
    g = np.stack(np.meshgrid(*[np.linspace(-1, 1, res)] * 3, indexing="ij"), -1)
    for v in range(n):
        if kind[v] == 0:
            if v % 2:
                nrm = rng.standard_normal(3)
                s[v] = g @ (nrm / np.linalg.norm(nrm)) + rng.uniform(-0.5, 0.5) + 0.05 * s[v]
            else:
                s[v] += rng.uniform(-0.8, 0.8)
        elif kind[v] == 1:
            s[v] = np.abs(s[v]) + rng.uniform(0.01, 1)
        else:
            s[v] = -np.abs(s[v]) - rng.uniform(0.01, 1)
    return (s * rng.uniform(0.01, 3, size=(n, 1, 1, 1))).astype(F32)


def alternating(res, n=1, rng=None):
    """f32 [n,res,res,res] of sign (-1)^(i+j+k) (every edge crosses: 3 res^2 (res-1) vertices, 4 triangles per cell); magnitudes
    1, or in [0.1, 10] from rng."""
    i = np.indices((res, res, res)).sum(0)
    sign = np.where(i % 2 == 0, 1.0, -1.0)
    mag = np.ones((n, res, res, res)) if rng is None else np.exp(rng.uniform(np.log(0.1), np.log(10), size=(n, res, res, res)))
    return (sign[None] * mag).astype(F32)
