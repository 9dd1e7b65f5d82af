"""The ray front end (nl_render_samples: traversal -> hit scan -> sampler -> sample scan -> compact sample list) past the inputs of
the golden scenes: several sampler chunks per batch, the single-block scans, all three traversal kernels on octrees built to reach
their branches, and calls whose sample total passes 2^31.

Yardsticks: the sampler is compared with the oracle's restatement of the reference wrapper (oracle.kernels.ray_sample, which keeps
the reference's 800-ray launches), the hit lists with the compiled reference `svo_intersect` where oracle/_ref was built, else
with the oracle's C restatement.  The hit planes are read from SDFEngine.workspace, which depends on carve() in csrc/render.cu:
h_idx, then h_min, then h_max (each [20][R] 4-byte words, 256-byte aligned), then nvalid [R].

Run as a script (`python tests/test_gpu_front_end.py scan-child OUT.npz`) it computes the scan cases in a process of its own, so
that the NL_SCAN / NL_SCAN_STAGE variables, which nl_render_samples reads once per process, take effect."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from util import product_map, ref_grid

pytestmark = pytest.mark.gpu

MAX_HITS = 20
INT32_MAX = 2 ** 31 - 1
HERE = os.path.abspath(__file__)


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


# ------------------------------------------------------------------------------------------------------------------ helpers
def _ws_offsets(R):
    plane = (4 * MAX_HITS * R + 255) // 256 * 256
    return plane, 3 * plane          # bytes per hit plane, start of nvalid


def hit_planes(eng, R):
    """(idx i32[R,20], min f32[R,20], max f32[R,20], nvalid i32[R]) of the last render_samples call (carve() layout)."""
    plane, nv = _ws_offsets(R)
    n = MAX_HITS * R
    w = eng.workspace
    idx = w[:4 * n].view(torch.int32).view(MAX_HITS, R)
    mn = w[plane:plane + 4 * n].view(torch.float32).view(MAX_HITS, R)
    mx = w[2 * plane:2 * plane + 4 * n].view(torch.float32).view(MAX_HITS, R)
    nvalid = w[nv:nv + 4 * R].view(torch.int32)
    return idx.T.cpu().numpy(), mn.T.cpu().numpy(), mx.T.cpu().numpy(), nvalid.cpu().numpy()


def dummy_state(nl, centres, structure):
    """A MapState for the front end alone (no embeddings are read before the gather)."""
    n = centres.shape[0]
    return nl.engine.MapState(torch.as_tensor(centres), torch.as_tensor(structure), torch.full((n, 8), -1, dtype=torch.int32),
                              torch.zeros((1, 16), dtype=torch.bfloat16), "cuda")


def render(nl, ms, ro, rd, cfg, cap, packed=True, **kw):
    """render_samples on a fresh engine; grows the capacity once if the sample list did not fit."""
    R = ro.shape[0]
    ro = torch.as_tensor(ro).cuda().contiguous()
    rd = torch.as_tensor(rd).cuda().contiguous()
    for _ in range(2):
        eng = nl.engine.SDFEngine(R, cap, want_decoder_grads=False)
        eng.use_packed_octree = packed
        eng.render_samples(ms, R, cfg, ro, rd, **kw)
        st = eng.read_stats()
        if not st.error & 2:
            break
        cap = st.n_samples + 1024
    assert st.error == 0, st.error
    return eng, st


def outputs(eng, st, R):
    M = st.n_samples
    o = {k: np.array(getattr(st, k)) for k in ("n_hit_rays", "max_hits", "max_samples", "n_samples", "max_steps_ceil", "error")}
    o.update(hit_rank=eng.hit_rank[:R].cpu().numpy(), ray_nsamp=eng.ray_nsamp[:R].cpu().numpy(),
             ray_offset=eng.ray_offset[:R].cpu().numpy(), s_ray=eng.s_ray[:M].cpu().numpy(), s_vox=eng.s_vox[:M].cpu().numpy(),
             s_depth=eng.s_depth[:M].cpu().numpy(), s_xyz=eng.s_xyz[:M].cpu().numpy(), s_flag=eng.s_flag[:M].cpu().numpy())
    return o


def exclusive_cumsum(x):
    return np.concatenate([[0], np.cumsum(x.astype(np.int64))[:-1]])


# ------------------------------------------------------------------------------------------------------------------ A. chunks
CHUNK_CFG = dict(step_size=0.15, voxel_size=0.3, max_distance=40.0, truncation=0.3, max_depth=40.0, fs_weight=1.0, sdf_weight=1.0)


@pytest.fixture(scope="module")
def chunk_scene(nl):
    """Three synthetic scans from different sensor positions in one map; the rays of all three that hit it."""
    syn = nl.synthetic
    mu = nl.mapping.MapUpdater(0.3)
    ro, rd = [], []
    for i in range(3):
        pts, cos, pose = syn.make_scan(seed=4100 + i, sensor_xyz=(2.0 * i, 0.7 * i, 0.0), yaw=0.05 * i)
        ms = mu.insert_voxels(torch.from_numpy(syn.voxelize(pts, pose, 0.3)))
        d = (pts.astype(np.float32) @ pose[:3, :3].astype(np.float32).T).astype(np.float32)
        rd.append((d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32))
        ro.append(np.broadcast_to(pose[:3, 3].astype(np.float32), d.shape))
    ro, rd = np.concatenate(ro), np.concatenate(rd)
    eng, st = render(nl, ms, ro, rd, CHUNK_CFG, cap=40 * ro.shape[0])
    hit = eng.hit_rank[:ro.shape[0]].cpu().numpy() >= 0
    assert hit.sum() >= 245_000, hit.sum()
    return ms, np.ascontiguousarray(ro[hit]), np.ascontiguousarray(rd[hit])


def interleave_misses(ro_hit, rd_hit):
    """Every third ray misses (it starts 500 m above the map and points up), so that hit rank != ray index."""
    n = ro_hit.shape[0]
    R = n + (n + 1) // 2
    is_hit = (np.arange(R) % 3) != 1
    is_hit[np.flatnonzero(is_hit)[n:]] = False
    ro = np.zeros((R, 3), np.float32); ro[:, 2] = 500.0
    rd = np.zeros((R, 3), np.float32); rd[:, 2] = 1.0
    ro[is_hit], rd[is_hit] = ro_hit, rd_hit
    return ro, rd, np.flatnonzero(is_hit)


def loss_flags(depth, cos, gt, trunc, max_depth):
    """criterion.py:67-82 per sample: bit0 front_mask, bit1 sdf_mask."""
    f32 = np.float32
    z = (depth * cos).astype(f32)
    front = z < (gt - f32(trunc)).astype(f32)
    back = z > (gt + f32(trunc)).astype(f32)
    dm = (gt > 0) & (gt < f32(max_depth))
    return (front.astype(np.uint8) | ((~front & ~back & dm).astype(np.uint8) << 1)).astype(np.uint8)


@pytest.mark.parametrize("n_hit", [160_000, 160_001, 165_123, 245_000])
def test_sampler_chunks_match_the_reference_wrapper(nl, chunk_scene, n_hit):
    """R_hit past 200 x 800 hit rays: the reference launches its sampler in 800-ray chunks per batch, and both tail quirks depend
    on a ray's slot in its chunk and on the chunk's first ray.  Compared with the oracle's restatement of that wrapper, exactly."""
    from oracle import kernels as OK
    ms, ro_all, rd_all = chunk_scene
    ro, rd, hitpos = interleave_misses(ro_all[:n_hit], rd_all[:n_hit])
    R = ro.shape[0]
    rng = np.random.default_rng(n_hit)
    cos = rng.uniform(0.5, 1.0, R).astype(np.float32)
    gt = rng.uniform(0.0, 45.0, R).astype(np.float32)
    kw = dict(gt_depth=torch.from_numpy(gt).cuda(), cos=torch.from_numpy(cos).cuda())
    eng, st = render(nl, ms, ro, rd, CHUNK_CFG, cap=40 * n_hit, **kw)
    assert st.n_hit_rays == n_hit
    P = st.max_hits
    idx, mn, mx, _ = hit_planes(eng, R)
    inter = {"intersected_voxel_idx": idx[hitpos, :P], "min_depth": mn[hitpos, :P], "max_depth": mx[hitpos, :P]}
    Kp = -(-n_hit // 200)
    max_steps = st.max_steps_ceil + P
    noise = np.random.default_rng(7 + n_hit).uniform(0.001, 0.999, (200, Kp, max_steps)).astype(np.float32)
    chunk1 = np.zeros(R, bool)
    chunk1[hitpos[(np.arange(n_hit) % Kp) >= 800]] = True
    nsamp = {}
    for noise_kind in ("random", "half"):
        for compat in (True, False):
            nz = torch.from_numpy(noise.reshape(200 * Kp, max_steps)).cuda() if noise_kind == "random" else None
            eng, st = render(nl, ms, ro, rd, CHUNK_CFG, cap=40 * n_hit, noise=nz, reference_compat=compat, **kw)
            o = outputs(eng, st, R)
            nsamp[noise_kind, compat] = o["ray_nsamp"]
            # what holds for either setting: ranks, offsets, positions and loss flags of the list the kernels produced
            assert o["n_hit_rays"] == n_hit and o["max_hits"] == P
            assert np.array_equal(o["hit_rank"][hitpos], np.arange(n_hit)) and (np.delete(o["hit_rank"], hitpos) == -1).all()
            assert np.array_equal(o["ray_offset"], exclusive_cumsum(o["ray_nsamp"]))
            assert o["n_samples"] == o["ray_nsamp"].sum() and o["max_samples"] == o["ray_nsamp"].max()
            assert np.array_equal(o["s_ray"], np.repeat(np.arange(R), o["ray_nsamp"]))
            r = o["s_ray"]
            xyz = (ro[r] + (rd[r] * o["s_depth"][:, None]).astype(np.float32)).astype(np.float32)
            assert np.array_equal(o["s_xyz"].view(np.int32), xyz.view(np.int32))
            assert np.array_equal(o["s_flag"], loss_flags(o["s_depth"], cos[r], gt[r], CHUNK_CFG["truncation"], CHUNK_CFG["max_depth"]))
            if not compat:
                continue
            ref = OK.ray_sample(inter, step_size=CHUNK_CFG["step_size"], fixed=noise_kind == "half",
                                noise=noise if noise_kind == "random" else None)
            si, sd = ref["sampled_point_voxel_idx"], ref["sampled_point_depth"]
            valid = si != -1
            assert o["max_samples"] == si.shape[1]
            assert np.array_equal(o["ray_nsamp"][hitpos], valid.sum(1))
            assert np.array_equal(o["s_vox"], si[valid])
            assert np.array_equal(o["s_depth"].view(np.int32), sd[valid].view(np.int32))
    diff = {k: int((nsamp[k, True] != nsamp[k, False])[chunk1].sum()) for k in ("random", "half")}
    print(f"\n[chunks] R_hit={n_hit} Kp={Kp} chunk-1 rays={int(chunk1.sum())} chunk-1 rays whose count the quirks change={diff}")
    if Kp > 800 + 1:
        assert diff["random"] > 0 and diff["half"] > 0      # the quirks ran in chunk 1


# ------------------------------------------------------------------------------------------------------------------ B. scans
SCAN_CFG = dict(step_size=0.25, voxel_size=1.0, max_distance=100.0)
SCAN_SIZES = [1, 3, 4095, 4096, 4097, 3 * 4096 + 1, 82_720]
SCAN_KEYS = ("n_hit_rays", "max_hits", "max_samples", "n_samples", "error", "hit_rank", "ray_nsamp", "ray_offset", "s_ray", "s_vox",
             "s_depth")


def block_state(nl):
    vox = np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.int32)
    m = product_map(vox, 1.0, grid_dim=16)
    return dummy_state(nl, m["centres"], m["structure"])


def block_rays(R, pattern, seed):
    """Rays at the 8^3 block [0, 8)^3: hits come from 20-30 m away aimed at a random point inside, misses point away from it."""
    rng = np.random.default_rng(seed)
    u = rng.normal(size=(R, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    target = rng.uniform(0.0, 8.0, (R, 3))
    ro = (target + rng.uniform(20.0, 30.0, (R, 1)) * u).astype(np.float32)
    rd = (-u).astype(np.float32)
    hit = {"miss": np.zeros(R, bool), "hit": np.ones(R, bool), "random": rng.random(R) < 0.5}[pattern]
    rd[~hit] = u[~hit]
    return ro, rd, hit


def scan_cases(nl):
    ms = block_state(nl)
    out = {}
    for R in SCAN_SIZES:
        for pattern in ("miss", "hit", "random"):
            ro, rd, _ = block_rays(R, pattern, R)
            eng, st = render(nl, ms, ro, rd, SCAN_CFG, cap=64 * R, rng_seed=777)
            o = outputs(eng, st, R)
            o["nvalid"] = hit_planes(eng, R)[3]
            for k in SCAN_KEYS + ("nvalid",):
                out[f"{R}/{pattern}/{k}"] = o[k]
    return out


def test_chained_scan_equals_both_single_block_scans(nl):
    """Tile edges, one tile, three rays: the chained scans against the single-block scans, staged and unstaged (NL_SCAN=single,
    NL_SCAN_STAGE=0, each in a process of its own), bit for bit; ranks and offsets are the cumulative sums of the per-ray counts."""
    mine = scan_cases(nl)
    for key, o in _by_case(mine).items():
        R = o["hit_rank"].shape[0]
        flags = o["nvalid"] > 0
        assert np.array_equal(o["hit_rank"], np.where(flags, np.cumsum(flags) - 1, -1)), key
        assert o["n_hit_rays"] == flags.sum() and (o["ray_nsamp"][~flags] == 0).all()
        assert np.array_equal(o["ray_offset"], exclusive_cumsum(o["ray_nsamp"])) and o["n_samples"] == o["ray_nsamp"].sum(), key
        if key[1] == "hit":
            assert flags.all()
        if key[1] == "miss":
            assert not flags.any()
    with tempfile.TemporaryDirectory() as tmp:
        for env in ({"NL_SCAN": "single"}, {"NL_SCAN": "single", "NL_SCAN_STAGE": "0"}):
            path = os.path.join(tmp, "scan.npz")
            subprocess.run([sys.executable, HERE, "scan-child", path], env=dict(os.environ, **env), check=True, timeout=900)
            with np.load(path) as z:
                other = {k: z[k] for k in z.files}
            assert other.keys() == mine.keys()
            for k in mine:
                assert np.array_equal(mine[k], other[k]), (env, k)


def _by_case(flat):
    cases = {}
    for k, v in flat.items():
        R, pattern, name = k.split("/")
        cases.setdefault((int(R), pattern), {})[name] = v
    return cases


@pytest.mark.parametrize("R", [4 * 1024 * 1024, 4 * 1024 * 1024 + 1])
def test_scans_at_the_chained_limit_and_past_it(nl, R):
    """1024 tiles (the last chained size) and one ray more (the single-block scan, chosen without any variable): ~100 k hit rays
    scattered among misses give the same sample list as the hit rays alone -- the hit order, R_hit and P are the same, so the
    sampler's quirks are too, and the noise is indexed by hit rank.  Needs about 2.5 GB of device memory (1 GB of it the hit planes)."""
    ms = block_state(nl)
    n_hit = 100_003
    ro_h, rd_h, _ = block_rays(n_hit, "hit", 5)
    rng = np.random.default_rng(R)
    pos = np.sort(rng.choice(R, n_hit, replace=False))
    ro, rd, _ = block_rays(R, "miss", 6)
    ro[pos], rd[pos] = ro_h, rd_h
    cap = 64 * n_hit
    noise = torch.rand((n_hit, 128), generator=torch.Generator().manual_seed(3)).clamp_(0.001, 0.999).cuda()
    for kw in (dict(noise=noise), dict()):
        eng, st = render(nl, ms, ro_h, rd_h, SCAN_CFG, cap, **kw)
        assert st.max_steps_ceil + st.max_hits <= 128
        a = outputs(eng, st, n_hit)
        eng, st = render(nl, ms, ro, rd, SCAN_CFG, cap, **kw)
        b = outputs(eng, st, R)
        for k in ("n_hit_rays", "max_hits", "max_samples", "n_samples", "s_vox", "s_depth", "s_xyz"):
            assert np.array_equal(a[k], b[k]), k
        assert a["n_hit_rays"] == n_hit
        assert np.array_equal(b["hit_rank"][pos], np.arange(n_hit)) and (np.delete(b["hit_rank"], pos) == -1).all()
        assert np.array_equal(b["ray_nsamp"][pos], a["ray_nsamp"]) and np.array_equal(b["ray_offset"][pos], a["ray_offset"])
        assert np.array_equal(b["s_ray"], pos[a["s_ray"]])
        del eng
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------ C. traversal
def _octree_cases(nl):
    """(name, voxel_size, centres, structure, ray origins, ray directions, max_distance)."""
    rng = np.random.default_rng(11)
    cases = []

    def rays_for(lo, hi, vs, n):
        """Axis rays with +-0 components, origins on faces / edges / corners and inside voxels, corner diagonals, random rays."""
        ext = (hi - lo) * vs
        o, d = [], []
        g = lambda k: rng.integers(int(lo), int(hi) + 1, (k, 3)).astype(np.float32) * np.float32(vs)   # lattice points
        for axis in range(3):
            for sgn in (1.0, -1.0):
                for zero in (0.0, -0.0):
                    k = n // 24
                    dd = np.full((k, 3), zero, np.float32); dd[:, axis] = sgn
                    oo = rng.uniform(lo * vs, hi * vs, (k, 3)).astype(np.float32)
                    oo[:, axis] = (lo * vs - 1.0) if sgn > 0 else (hi * vs + 1.0)
                    oo[: k // 2, (axis + 1) % 3] = g(k // 2)[:, 0]                                   # on a face plane
                    o.append(oo); d.append(dd)
        k = n // 4
        signs = rng.choice([-1.0, 1.0], (k, 3)).astype(np.float32)
        o.append(g(k)); d.append(signs * np.float32(rng.choice([1.0, 0.125], (k, 1))))            # diagonals through corners
        o.append(rng.uniform(lo * vs, hi * vs, (k, 3)).astype(np.float32))                         # inside voxels
        u = rng.normal(size=(k, 3)); d.append((u / np.linalg.norm(u, axis=1, keepdims=True)).astype(np.float32))
        c = (lo + hi) / 2 * vs
        u = rng.normal(size=(k, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
        o.append((c + 1.5 * ext * u).astype(np.float32)); d.append((-u + rng.normal(scale=0.1, size=u.shape)).astype(np.float32))
        return np.concatenate(o), np.concatenate(d)

    vox = np.stack(np.meshgrid(*[np.arange(16)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.int32)
    m = product_map(vox, 1.0, grid_dim=32)      # the octree takes coordinates in [0, grid_dim - 2]
    ro, rd = rays_for(0, 16, 1.0, 6000)
    cases.append(("solid16", 1.0, m["centres"], m["structure"], ro, rd, 100.0))
    cases.append(("solid16_clip", 1.0, m["centres"], m["structure"], ro, rd, 2.5))

    vox = (rng.choice(64, (40, 3)) * 4).astype(np.int32)                                          # single-child chains
    m = product_map(vox, 0.5, grid_dim=256)
    tgt = (vox[rng.integers(0, 40, 3000)] + rng.uniform(0, 1, (3000, 3))) * 0.5
    u = rng.normal(size=(3000, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    ro2 = (tgt + 20 * u).astype(np.float32)
    ro, rd = rays_for(0, 256, 0.5, 2400)
    cases.append(("chains", 0.5, m["centres"], m["structure"], np.concatenate([ro, ro2]), np.concatenate([rd, (-u).astype(np.float32)]),
                  200.0))

    m = product_map(np.zeros((1, 3), np.int32), 1.0, grid_dim=2)      # the root is a leaf parent (grid_dim 2 admits voxel 0 only)
    ro, rd = rays_for(0, 2, 1.0, 2400)
    cases.append(("grid2", 1.0, m["centres"], m["structure"], ro, rd, 100.0))

    # a root of side 1: the octree refuses grid_dim 1 (nl_octree_create needs a power of two >= 2), so the one-node map is built here
    ro, rd = rays_for(0, 1, 1.0, 1200)
    cases.append(("root_side1", 1.0, np.array([[0.5, 0.5, 0.5]], np.float32), np.array([[-1] * 8 + [1]], np.int32), ro, rd, 100.0))

    gd = 1 << 18                                                                                  # 18 levels below the root
    vox = rng.integers(0, gd - 2, (300, 3)).astype(np.int32)
    vox = np.concatenate([vox, vox[:100] + np.array([1, 0, 0], np.int32)])                       # some neighbours
    m = product_map(vox, 0.125, grid_dim=gd)
    k = 3000
    tgt = (vox[rng.integers(0, vox.shape[0], k)] + rng.uniform(0, 1, (k, 3))) * 0.125
    u = rng.normal(size=(k, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    axis = np.zeros((k, 3)); axis[np.arange(k), rng.integers(0, 3, k)] = 1.0
    u[: k // 3] = axis[: k // 3]
    cases.append(("levels18", 0.125, m["centres"], m["structure"], (tgt + 3.0 * u).astype(np.float32), (-u).astype(np.float32), 50.0))
    return cases


def _ref_planes(g, ro, rd, centres, structure, vs, md):
    """Expected [R,20] planes: svo_intersect (compiled reference, batched 4 ways like its wrapper, else the oracle's restatement)
    followed by the reference's sort and clipping (oracle.kernels.ray_intersect)."""
    from oracle import kernels as OK
    R = ro.shape[0]
    if g is not None:
        pad = (-R) % 4
        o = np.concatenate([ro, np.repeat(ro[:1], pad, 0)]); d = np.concatenate([rd, np.repeat(rd[:1], pad, 0)])
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        K = o.shape[0] // 4
        pts = t(centres)[None].expand(4, -1, -1).contiguous(); ch = t(structure)[None].expand(4, -1, -1).contiguous()
        i, a, b = g.svo_intersect(t(o.reshape(4, K, 3)), t(d.reshape(4, K, 3)), pts, ch, float(vs), MAX_HITS)
        raw = [x.cpu().numpy().reshape(4 * K, MAX_HITS)[:R] for x in (i, a, b)]
    else:
        raw = OK.svo_intersect(ro, rd, centres, structure, vs, MAX_HITS)
    out, _ = OK.ray_intersect(None, None, None, None, vs, max_distance=md, raw=raw)
    idx = np.full((R, MAX_HITS), -1, np.int32); mn = np.full((R, MAX_HITS), np.float32(md)); mx = mn.copy()
    h = out["intersected_voxel_idx"].shape[1]
    idx[:, :h], mn[:, :h], mx[:, :h] = out["intersected_voxel_idx"], out["min_depth"], out["max_depth"]
    return idx, mn, mx, g is not None


def _branch_counts(ro, rd, centres, structure, vs, md, idx, mn):
    """What the case reached: rays through a node with > 4 children, rays with > 20 candidate leaves, rays with tied min_depth,
    entries removed by each clipping condition alone."""
    from oracle import kernels as OK
    i64, a64, b64 = OK.svo_intersect(ro, rd, centres, structure, vs, 64)
    nch = (structure[:, :8] > -1).sum(1)
    parent = np.full(structure.shape[0], -1)
    for p in np.flatnonzero(nch):
        parent[structure[p, :8][structure[p, :8] > -1]] = p
    leaves = i64[i64 > -1]
    wide = np.zeros(i64.shape, bool)
    wide[i64 > -1] = nch[np.maximum(parent[leaves], 0)] > 4
    valid = idx > -1
    s = np.sort(np.where(valid, mn, np.inf), 1)
    ties = ((s[:, 1:] == s[:, :-1]) & np.isfinite(s[:, 1:])).any(1)
    i20, a20, b20 = OK.svo_intersect(ro, rd, centres, structure, vs, MAX_HITS)
    e = i20 > -1
    far, late = b20 > np.float32(2 * md), a20 > np.float32(md)
    return dict(wide=int(wide.any(1).sum()), over20=int(((i64 > -1).sum(1) > MAX_HITS).sum()), ties=int(ties.sum()),
                clip_max=int((e & far & ~late).sum()), clip_min=int((e & late & ~far).sum()))


def test_three_traversals_agree_with_the_reference_on_edge_octrees(nl):
    """k_traverse_coop<8> (R <= 32768), k_traverse_coop<4> (the same rays padded past 32768 with misses) and the thread-per-ray
    k_traverse_sort: hit planes bit-identical to each other and equal to the reference's svo_intersect + sort + clipping.  Each
    case asserts the branches it was built for."""
    g = ref_grid()
    for name, vs, centres, structure, ro, rd, md in _octree_cases(nl):
        centres = np.ascontiguousarray(np.asarray(centres), np.float32)
        structure = np.ascontiguousarray(np.asarray(structure), np.int32)
        ms = dummy_state(nl, centres, structure)
        R = ro.shape[0]
        assert R <= 32768
        cfg = dict(step_size=0.5 * vs, voxel_size=vs, max_distance=md)
        pad = 32768 + 64 - R
        far = np.float32(4 * vs * structure[0, 8] + 1000.0)
        ro4 = np.concatenate([ro, np.full((pad, 3), far, np.float32)]); rd4 = np.concatenate([rd, np.tile(np.float32([[1, 0, 0]]), (pad, 1))])
        planes = []
        for rays, packed in (((ro, rd), True), ((ro4, rd4), True), ((ro, rd), False)):
            eng, st = render(nl, ms, rays[0], rays[1], cfg, cap=64 * rays[0].shape[0], packed=packed)
            planes.append([p[:R] for p in hit_planes(eng, rays[0].shape[0])])
        for p in planes[1:]:
            for x, y in zip(planes[0], p):
                assert np.array_equal(x.view(np.int32), y.view(np.int32)), name
        idx, mn, mx, nv = planes[0]
        assert np.array_equal(nv, (idx > -1).sum(1))
        eidx, emn, emx, exact = _ref_planes(g, ro, rd, centres, structure, vs, md)
        if exact:
            assert np.array_equal(idx, eidx), name
            assert np.array_equal(mn.view(np.int32), emn.view(np.int32)) and np.array_equal(mx.view(np.int32), emx.view(np.int32)), name
        else:     # the oracle's 1/x against __fdividef: the same leaves, depths to 2e-6; exact where the reciprocals are
            key = lambda i, a: np.lexsort((i, np.round(a, 4)), -1)
            assert np.array_equal(np.sort(idx, 1), np.sort(eidx, 1)), name
            np.testing.assert_allclose(np.take_along_axis(mn, key(idx, mn), 1), np.take_along_axis(emn, key(eidx, emn), 1), rtol=2e-6, atol=1e-6)
            pow2 = np.all((rd == 0) | (np.frexp(np.abs(rd))[0] == 0.5), 1)
            assert np.array_equal(idx[pow2], eidx[pow2]) and np.array_equal(mn[pow2], emn[pow2]), name
        c = _branch_counts(ro, rd, centres, structure, vs, md, idx, mn)
        print(f"\n[traverse] {name}: rays={R} hit={int((nv > 0).sum())} {c} yardstick={'reference' if exact else 'oracle'}")
        assert (nv > 0).sum() > R // 10, name
        if name == "solid16":
            assert c["wide"] > 0 and c["ties"] > 0 and c["over20"] > 0 and (nv == MAX_HITS).any()
        if name == "grid2":
            assert structure[0, 8] == 2 and (nv == 1).sum() > 0
        if name == "solid16_clip":
            assert c["clip_max"] > 0 and c["clip_min"] > 0
        if name == "levels18":
            assert structure[0, 8] == 1 << 18
        if name == "root_side1":
            assert structure[0, 8] == 1 and (nv == 1).sum() > 0


# ------------------------------------------------------------------------------------------------------------------ D. 2^31
GUARD = 1 << 16
SENTINEL = 0x5A5A5A5A


def _line_state(nl):
    """20 voxels in a row along x; a ray along +x through them sees 20 m of voxels."""
    vox = np.stack([np.arange(20), np.zeros(20, int), np.zeros(20, int)], 1).astype(np.int32)
    m = product_map(vox, 1.0, grid_dim=32)
    return dummy_state(nl, m["centres"], m["structure"])


def _line_rays(R, n_hit):
    ro = np.tile(np.float32([[-1.0, 0.37, 0.61]]), (R, 1))
    rd = np.tile(np.float32([[1.0, 0.0, 0.0]]), (R, 1))
    rd[n_hit:, 0] = -1.0
    return ro, rd


def _render_guarded(nl, ms, ro, rd, step, cap):
    """nl_render_samples with every sample array inside sentinel-filled guard regions of GUARD elements on both sides.  Without the
    reference's tail quirks (which depend on a ray's slot in its sampler chunk), so that identical rays get identical counts."""
    dev = torch.device("cuda")
    R = ro.shape[0]
    lib = nl._capi.lib()
    n = GUARD + cap + GUARD
    bufs = dict(s_ray=torch.full((n,), SENTINEL, dtype=torch.int32, device=dev), s_vox=torch.full((n,), SENTINEL, dtype=torch.int32, device=dev),
                s_depth=torch.full((n,), SENTINEL, dtype=torch.int32, device=dev), s_xyz=torch.full((n, 3), SENTINEL, dtype=torch.int32, device=dev),
                s_flag=torch.full((n,), 0x5A, dtype=torch.uint8, device=dev))
    ws = torch.empty(int(lib.nl_render_workspace_bytes(R)), dtype=torch.uint8, device=dev)
    stats = torch.zeros(nl.engine.STATS_BYTES, dtype=torch.uint8, device=dev)
    per_ray = {k: torch.empty(R, dtype=torch.int32, device=dev) for k in ("hit_rank", "ray_nsamp", "ray_offset")}
    o, d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    a = nl._capi.RenderArgs()
    a.n_rays, a.n_nodes, a.sample_capacity, a.reference_compat = R, ms.n_nodes, cap, 0
    a.voxel_size, a.step_size, a.max_distance = 1.0, step, 100.0
    a.d_centres, a.d_structure, a.d_packed_children = ms.centres.data_ptr(), ms.structure.data_ptr(), ms.packed_children().data_ptr()
    a.d_ray_o, a.d_ray_d = o.data_ptr(), d.data_ptr()
    a.d_workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    a.d_stats = stats.data_ptr()
    a.d_hit_rank, a.d_ray_nsamp, a.d_ray_offset = (per_ray[k].data_ptr() for k in ("hit_rank", "ray_nsamp", "ray_offset"))
    a.d_s_ray, a.d_s_vox, a.d_s_depth = (bufs[k].data_ptr() + 4 * GUARD for k in ("s_ray", "s_vox", "s_depth"))
    a.d_s_xyz, a.d_s_flag = bufs["s_xyz"].data_ptr() + 12 * GUARD, bufs["s_flag"].data_ptr() + GUARD
    nl._capi.check(lib.nl_render_samples(C.byref(a), nl._capi.stream_ptr()), "nl_render_samples")
    torch.cuda.synchronize()
    st = nl._capi.RenderStats.from_buffer_copy(stats.cpu().numpy().tobytes())
    host = {k: v.cpu().numpy() for k, v in bufs.items()}
    for k, v in host.items():
        s = 0x5A if k == "s_flag" else SENTINEL
        assert (v[:GUARD] == s).all() and (v[GUARD + cap:] == s).all(), f"{k} written outside [0, capacity)"
    return st, {k: v.cpu().numpy() for k, v in per_ray.items()}, host


@pytest.mark.parametrize("case", ["across_tiles", "one_tile", "just_below"])
def test_sample_totals_past_2_31_saturate_and_write_nothing_out_of_bounds(nl, case):
    """A call may ask for 2^31 samples or more (8192 rays of ~3e5 samples each).  The totals are summed in 64 bits: above
    INT32_MAX n_samples saturates there with the capacity bit set, offsets saturate, nothing is written outside the arrays,
    and render_rays refuses the call; just below, the total and every offset are exact."""
    ms = _line_state(nl)
    cap = 1 << 16
    if case == "across_tiles":         # 2 tiles of ~1.2e9 samples: the carry passes 2^31
        R, n_hit, step = 8192, 8192, 20.0 / 288_000
    elif case == "one_tile":           # one tile of ~2.4e9 samples: the tile total itself passes 2^31
        R, n_hit, step = 4096, 4096, 20.0 / 576_000
    else:
        step = 20.0 / 263_000
        st1, pr1, _ = _render_guarded(nl, ms, *_line_rays(1, 1), step, cap)
        per = int(pr1["ray_nsamp"][0])
        R, n_hit = 8192, INT32_MAX // per
        assert n_hit < R
    st, pr, host = _render_guarded(nl, ms, *_line_rays(R, n_hit), step, cap)
    nsamp = pr["ray_nsamp"].astype(np.int64)
    assert (nsamp[:n_hit] > 0).all() and (nsamp[n_hit:] == 0).all() and len(set(nsamp[:n_hit])) == 1
    total = int(nsamp.sum())
    print(f"\n[2^31] {case}: rays={R} hit={n_hit} samples per ray={nsamp[0]} total={total} (2^31 = {2 ** 31})")
    assert st.n_hit_rays == n_hit and np.array_equal(pr["hit_rank"], np.where(np.arange(R) < n_hit, np.arange(R), -1))
    assert st.error & 2
    offs = exclusive_cumsum(nsamp)
    if case == "just_below":
        assert total <= INT32_MAX and total > INT32_MAX - nsamp[0]
        assert st.n_samples == total and np.array_equal(pr["ray_offset"], offs)
    else:
        assert total > INT32_MAX
        assert st.n_samples == INT32_MAX and np.array_equal(pr["ray_offset"], np.minimum(offs, INT32_MAX))
    expect_ray = np.repeat(np.arange(R), np.minimum(nsamp, cap))[:cap]
    assert np.array_equal(host["s_ray"][GUARD:GUARD + cap], expect_ray)
    if case != "just_below":
        dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
        ro, rd = _line_rays(R, n_hit)
        with pytest.raises(nl._capi.NerfLoamError, match="2\\^31"):
            nl.render_helpers.render_rays(torch.from_numpy(ro).cuda()[None], torch.from_numpy(rd).cuda()[None], ms, dec, step, 1.0, 0.3,
                                          10, 100.0, deterministic=True)


if __name__ == "__main__" and len(sys.argv) == 3 and sys.argv[1] == "scan-child":
    import nerfloam_b200 as _nl
    np.savez(sys.argv[2], **scan_cases(_nl))
