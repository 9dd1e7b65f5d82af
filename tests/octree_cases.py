"""Octree insertion cases for the comparison with the compiled reference octree (tests/octree_ref_child.py).

A case is a grid, a list of int32 [n,3] batches inserted one after the other, the try_insert probe batches and has_voxel points
asked after every batch, and for the restore cases the batch after which the tree is pickled.  Every corner of every batch lies in
[0, grid_dim): the reference does not bound-check (an out-of-grid corner aliases through `x & edge`), and the product refuses
such a batch, which its own tests check.

All cases are deterministic and built from numpy and the product's synthetic scans alone."""
import functools

import numpy as np

INC = np.array([[0, 0, 0], [0, 0, 1], [0, 1, 0], [0, 1, 1], [1, 0, 0], [1, 0, 1], [1, 1, 0], [1, 1, 1]], np.int32)  # corner j


class Case:
    def __init__(self, grid_dim, voxel_size, batches, probes=None, points=None, restore_after=None, drive=False):
        self.grid_dim = int(grid_dim)
        self.voxel_size = float(voxel_size)
        self.batches = [np.ascontiguousarray(b, dtype=np.int32).reshape(-1, 3) for b in batches]
        for b in self.batches:
            assert b.size == 0 or (b.min() >= 0 and b.max() <= self.grid_dim - 2), "a corner outside the grid"
        self.probes = [np.ascontiguousarray(p, dtype=np.int32).reshape(-1, 3) for p in (probes if probes is not None else default_probes(self))]
        self.points = np.ascontiguousarray(points if points is not None else default_points(self), dtype=np.int32).reshape(-1, 3)
        self.restore_after = restore_after
        self.drive = drive

    def arrays(self):
        """The case as the flat dict of arrays tests/octree_ref_child.py reads."""
        d = {"grid_dim": np.int64(self.grid_dim), "voxel_size": np.float64(self.voxel_size), "n_batches": np.int64(len(self.batches)),
             "n_probes": np.int64(len(self.probes)), "points": self.points}
        d.update({f"batch{i}": b for i, b in enumerate(self.batches)})
        d.update({f"probe{i}": p for i, p in enumerate(self.probes)})
        return d


def default_probes(case, seed=0):
    """try_insert probes: every batch but the empty ones (so each is also asked before it is inserted), every batch's first point,
    and in-grid random points."""
    rng = np.random.default_rng(seed)
    g = case.grid_dim
    probes = [b for b in case.batches if b.shape[0]]
    probes += [b[:1] for b in case.batches if b.shape[0]]
    probes.append(rng.integers(0, g - 1, (64, 3)))
    return probes[:24]


def default_points(case, seed=1):
    """has_voxel points: inserted points and their far corners (cells that exist), the grid's last cell on each axis, and random cells."""
    rng = np.random.default_rng(seed)
    g = case.grid_dim
    pts = [np.zeros((1, 3), np.int32), np.full((1, 3), g - 1, np.int32), np.eye(3, dtype=np.int32) * (g - 1)]
    for b in case.batches:
        if b.shape[0]:
            k = b[rng.integers(0, b.shape[0], min(8, b.shape[0]))]
            pts += [k, k + 1]
    pts.append(rng.integers(0, g, (32, 3)))
    return np.concatenate(pts).astype(np.int32)


# -- drives: the sequences of tests/test_gpu_device_octree.py --------------------------------------------------------------------
def _vox(scan, vs):
    from nerfloam_b200 import synthetic
    pts, _, pose = scan
    return synthetic.voxelize(pts, pose, vs)


def demo():             # scripts/demo_slam.py: 12 scans 0.5 m apart at 0.3 m
    from nerfloam_b200 import synthetic as syn
    return 0.3, 256 * 256 * 4, [_vox(syn.make_scan(seed=1000 + i, sensor_xyz=(0.5 * i, 0.05 * np.sin(0.7 * i), 0.0), yaw=0.01 * np.sin(0.5 * i)), 0.3)
                                for i in range(12)]


def kitti():            # 6 scans 1 m apart
    from nerfloam_b200 import synthetic as syn
    return 0.3, 256 * 256 * 4, [_vox(syn.make_scan(n_beams=32, n_az=240, seed=100 + i, sensor_xyz=(1.0 * i, 0.0, 0.0)), 0.3) for i in range(6)]


def fine():             # MaiCity / NCD: 0.2 m voxels, scans 2 m apart; the first is a whole scan into an empty tree
    from nerfloam_b200 import synthetic as syn
    return 0.2, 256 * 256 * 4, [_vox(syn.make_scan(seed=2000 + i, sensor_xyz=(2.0 * i, 0.0, 0.0), min_depth=1.5, max_depth=50.0), 0.2)
                                for i in range(3)]


def batch_shapes():     # a shuffled scan, only repeated points, another scan, the first re-inserted, an empty batch, one point, one point x3
    from nerfloam_b200 import synthetic as syn
    a = _vox(syn.make_scan(n_beams=16, n_az=400, seed=5), 0.3)
    b = _vox(syn.make_scan(n_beams=16, n_az=400, seed=6, sensor_xyz=(3.0, 1.0, 0.0)), 0.3)
    rng = np.random.default_rng(1)
    rep = a[rng.integers(0, a.shape[0], 5000)]
    single = (b[:1] + np.array([[40, -30, 7]], np.int32)).astype(np.int32)
    return 0.3, 256 * 256 * 4, [a[rng.permutation(a.shape[0])], rep, b, a, np.zeros((0, 3), np.int32), single, np.repeat(b[7:8], 3, 0)]


def _drive_probes(batches):
    """The second and the last scan (asked before and after they are inserted, as a mapper asks), half of the first, a single
    point, and a batch of cells in the grid but away from the drive."""
    full = [b for b in batches if b.shape[0]]
    return [full[min(1, len(full) - 1)], full[-1], full[0][: full[0].shape[0] // 2], full[0][:1], full[0][:2000] + 300]


# -- grid edges ----------------------------------------------------------------------------------------------------------------
def _around(q, hi):
    """The up to 8 valid points that have leaf q as a corner."""
    p = np.asarray(q, np.int32) - INC
    return p[((p >= 0) & (p <= hi)).all(1)]


def grid_edges(g):
    """Batches at the grid's edges, each corner inside [0, g):
    - one point per root octant, 0 or g - 2 on every axis (the lowest and highest valid cells);
    - the 8 points around the centre leaf g/2, one per root octant, all sharing that corner leaf;
    - the 8 points around leaf g - 2 next to the upper faces, sharing it;
    - points whose corners fill whole 2x2x2 blocks (even coordinates: the 8 leaves of one level-(L-1) node), the top block included;
    - every combination of 0, g/2 - 1, g/2 and g - 2 per axis (cells on both sides of the mid-planes)."""
    hi = g - 2
    vals = sorted({0, hi, max(g // 2 - 1, 0), min(g // 2, hi)})
    octants = np.array([[hi if (o >> a) & 1 else 0 for a in range(3)] for o in range(8)], np.int32)
    straddle = np.array([[x, y, z] for x in vals for y in vals for z in vals], np.int32)
    evens = sorted({0, hi - hi % 2, (g // 2) - (g // 2) % 2 if g // 2 <= hi else 0})
    blocks = np.array([[x, hi - hi % 2, z] for x in evens for z in evens], np.int32)
    return [octants, _around(np.full(3, g // 2), hi), _around(np.full(3, hi), hi), blocks, straddle]


# -- promotion: FEATURE leaves turned SURFACE by later batches -----------------------------------------------------------------
def promotion(n_batches=50, per=20, g=256, seed=11):
    """Batch b holds `per` points: about half are a far corner (j > 0) of an earlier batch's point, i.e. a leaf that batch created
    as FEATURE, which this batch's j = 0 corner turns SURFACE; the rest are new cells, some on the upper faces."""
    rng = np.random.default_rng(seed)
    lo = max(0, g - 24)
    batches, seen = [], np.zeros((0, 3), np.int32)
    for b in range(n_batches):
        new = rng.integers(lo, g - 1, (per, 3)).astype(np.int32)
        if seen.shape[0]:
            k = per // 2 + int(rng.integers(-(per // 4), per // 4 + 1))
            src = seen[rng.integers(0, seen.shape[0], k)]
            promoted = src + INC[rng.integers(1, 8, k)]
            new[:k] = np.minimum(promoted, g - 2)
        new[-1, rng.integers(0, 3)] = g - 2
        batches.append(new)
        seen = np.concatenate([seen, new])
    return batches


# -- random trees --------------------------------------------------------------------------------------------------------------
def random_tree(i):
    """Tree i of the random family: grid 2^(1 + i mod 18), 1..8 batches of log-uniform 1..20 000 points, clustered next to the grid's
    faces (each axis near 0, near g - 2 or anywhere, within a spread of 2^k)."""
    rng = np.random.default_rng(1000 + i)
    L = 1 + i % 18
    g = 1 << L
    n_batches = 1 + int(rng.integers(0, 8))
    if i == 0:
        n_batches = 8
    batches = []
    for b in range(n_batches):
        n = int(np.exp(rng.uniform(0, np.log(20_000))))
        if (i, b) == (1, 0):
            n = 20_000
        if (i, b) == (2, 0):
            n = 1
        spread = min(g - 1, 1 << int(rng.integers(0, 6)))
        centre = np.empty(3, np.int64)
        for a in range(3):
            side = rng.integers(0, 3)
            centre[a] = 0 if side == 0 else (g - 2 if side == 1 else rng.integers(0, g - 1))
        pts = centre + rng.integers(-spread, spread + 1, (n, 3))
        batches.append(np.clip(pts, 0, g - 2).astype(np.int32))
    return g, batches


# -- try_insert's int32 truncation ---------------------------------------------------------------------------------------------
def morton(p):
    """The 63-bit Morton key of int coordinates [n,3] (x | y << 1 | z << 2, 21 bits per axis), as uint64."""
    p = np.asarray(p, np.int64).reshape(-1, 3)
    key = np.zeros(p.shape[0], np.uint64)
    for b in range(21):
        for a in range(3):
            key |= (((p[:, a] >> b) & 1).astype(np.uint64)) << np.uint64(3 * b + a)
    return key


def corner_keys(p):
    p = np.asarray(p, np.int64).reshape(-1, 3)
    return np.unique(morton((p[:, None, :] + INC[None]).reshape(-1, 3)))


def truncation(g):
    """A cluster A and its copies shifted by one bit above Morton bit 31 (z + 1024 is bit 32; at 2^18 also x + 2048, bit 33, and
    y + 2048, bit 34): their corner keys share their low 32 bits.  Probes: A with its copies (colliding), A alone and a copy alone
    (controls, no collision), A with cells not in the tree."""
    rng = np.random.default_rng(g)
    base = np.array([100, 200, 8], np.int32) if g == 1 << 11 else np.array([131_000, 70_000, 5], np.int32)
    a = base + rng.integers(0, 6, (40, 3)).astype(np.int32)
    shifts = [np.array([0, 0, 1024], np.int32)]
    if g == 1 << 18:
        shifts += [np.array([2048, 0, 0], np.int32), np.array([0, 2048, 0], np.int32)]
    copies = [a + s for s in shifts]
    batches = [a, *copies]
    probes = [np.concatenate([a, *copies]), np.concatenate([a, copies[0]]), a, copies[0], np.concatenate([a, a + np.array([0, 0, 3], np.int32)])]
    return batches, probes


def low_words_collide(probe, inserted):
    """True if the probe's corner keys that are in the tree (the corner keys of `inserted`) repeat a low 32-bit word."""
    k = np.intersect1d(corner_keys(probe), corner_keys(inserted))
    return np.unique(k & np.uint64(0xFFFFFFFF)).shape[0] < k.shape[0]


# -- the suite -----------------------------------------------------------------------------------------------------------------
N_RANDOM = 40
EDGE_GRIDS = (2, 4, 8, 1024, 1 << 18)


def names():
    return (["drive_demo", "drive_kitti", "drive_fine", "batch_shapes", "promotion_feature_to_surface", "promotion_small_grid"]
            + [f"grid_edges_{g}" for g in EDGE_GRIDS]
            + ["truncated_keys_2048", "truncated_keys_262144", "restore_demo_after_5", "restore_kitti_after_2"]
            + [f"random_{i:02d}" for i in range(N_RANDOM)])


@functools.lru_cache(maxsize=None)
def case(name):
    if name.startswith("drive_") or name.startswith("restore_"):
        seq = name.split("_")[1]
        vs, g, batches = {"demo": demo, "kitti": kitti, "fine": fine}[seq]()
        k = int(name.rsplit("_", 1)[1]) if name.startswith("restore_") else None
        return Case(g, vs, batches, probes=_drive_probes(batches), restore_after=k, drive=True)
    if name == "batch_shapes":
        vs, g, batches = batch_shapes()
        return Case(g, vs, batches, probes=_drive_probes(batches) + [np.repeat(batches[-1], 2, 0), np.zeros((0, 3), np.int32)])
    if name == "promotion_feature_to_surface":
        return Case(256, 0.4, promotion())
    if name == "promotion_small_grid":         # the same at grid 8, where almost every corner is shared
        return Case(8, 1.0, promotion(n_batches=48, per=4, g=8, seed=12))
    if name.startswith("grid_edges_"):
        g = int(name.rsplit("_", 1)[1])
        return Case(g, 0.5, grid_edges(g))
    if name.startswith("truncated_keys_"):
        g = int(name.rsplit("_", 1)[1])
        batches, probes = truncation(g)
        return Case(g, 0.3, batches, probes=probes)
    if name.startswith("random_"):
        g, batches = random_tree(int(name.split("_")[1]))
        return Case(g, 0.25, batches)
    raise KeyError(name)
