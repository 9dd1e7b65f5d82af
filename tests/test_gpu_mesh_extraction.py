"""GPU tests of mesh extraction (render_helpers.scores_device -> csrc/mc.cu -> mesh.extract_mesh) against the yardsticks of
tests/mesh_ref.py: the exact restatement emit_ref (counts, int64 offsets, vertices bit for bit, faces), the fp64 crossing within
its derived bar, oracle/mc.py as an independent check, and the lattice (points, features, sdf) against fp32 / fp64 restatements.
Lattice values count as inside when they are < 0: NaN, +0 and -0 are outside, as in the kernel and emit_ref."""
import sys

import numpy as np
import pytest
import torch

import decoder_ref as DR
import decoder_tc_ref as TR
import embedding_ref as ER
import mesh_ref as MR
from util import Args

pytestmark = pytest.mark.gpu

F32 = np.float32
VS = 0.3
INT32_MAX = 2 ** 31 - 1
SENT_V, SENT_F = -12345.5, -12345            # what the capacity tests prefill the outputs with


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


# ------------------------------------------------------------------------------------------------ calling the kernels
def _count(nl, sdf):
    """nl_mc_count on a device lattice f32 [n,res,res,res] -> (nvert, ntri, voff, toff) int32 [n] and totals int64 [2]."""
    n, res = sdf.shape[0], sdf.shape[1]
    counts = torch.full((4, max(n, 1)), -7, dtype=torch.int32, device="cuda")
    totals = torch.full((2,), -7, dtype=torch.int64, device="cuda")
    C = nl._capi
    C.check(C.lib().nl_mc_count(n, res, C.ptr(sdf), C.ptr(counts[0]), C.ptr(counts[1]), C.ptr(counts[2]), C.ptr(counts[3]),
                                C.ptr(totals), C.stream_ptr()), "nl_mc_count")
    c = counts[:, :n].cpu().numpy()
    return c[0], c[1], c[2], c[3], totals.cpu().numpy()


def _emit(nl, sdf, centres, voff, toff, vcap, tcap, vrows, trows, vox_ids=None, res=None):
    """nl_mc_emit into sentinel-filled buffers of vrows / trows rows.  Returns (rc, verts, faces) (numpy)."""
    C = nl._capi
    n = sdf.shape[0]
    verts = torch.full((vrows, 3), SENT_V, dtype=torch.float32, device="cuda")
    faces = torch.full((trows, 3), SENT_F, dtype=torch.int32, device="cuda")
    rc = C.lib().nl_mc_emit(n, sdf.shape[1] if res is None else res, VS, C.ptr(sdf), C.ptr(centres), C.ptr(vox_ids), C.ptr(voff),
                            C.ptr(toff), vcap, tcap, C.ptr(verts) if vrows else None, C.ptr(faces) if trows else None, C.stream_ptr())
    return rc, verts.cpu().numpy(), faces.cpu().numpy()


def _ndiff(a, b):
    """Rows of two f32 [V,3] arrays that differ in any bit (NaN equal to NaN)."""
    same = (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
    return int((~same).any(1).sum())


def check_exact(nl, sdf, centres, vox_ids=None, oracle_voxels=(), tag=""):
    """Counts, offsets and totals of nl_mc_count, and verts / faces of marching_cubes_device, equal emit_ref's; checked vertices
    within the fp64 bar; the listed voxels also against oracle/mc.py.  Returns (emit_ref's dict, the fp64 ratio)."""
    sdf = np.ascontiguousarray(sdf, F32)
    centres = np.ascontiguousarray(centres, F32)
    d_sdf, d_cen = torch.from_numpy(sdf).cuda(), torch.from_numpy(centres).cuda()
    d_ids = None if vox_ids is None else torch.from_numpy(np.asarray(vox_ids, np.int32)).cuda()
    ref = MR.emit_ref(sdf, centres, VS, vox_ids=vox_ids)
    nv, nt, voff, toff, tot = _count(nl, d_sdf)
    assert np.array_equal(nv, ref["nvert"]) and np.array_equal(nt, ref["ntri"]), tag
    assert np.array_equal(voff.astype(np.int64), ref["voff"]) and np.array_equal(toff.astype(np.int64), ref["toff"]), tag
    assert np.array_equal(tot, ref["totals"]), (tag, tot, ref["totals"])
    v, f = nl.mesh.marching_cubes_device(d_sdf, d_cen, VS, vox_ids=d_ids)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    assert v.shape == ref["verts"].shape and f.shape == ref["faces"].shape, tag
    nd = _ndiff(v, ref["verts"])
    assert nd == 0, f"{tag}: {nd} of {len(v)} vertices differ from the separately rounded fp32 formula"
    assert np.array_equal(f.astype(np.int64), ref["faces"]), tag
    ratio = MR.fp64_ratio(v, sdf, centres, VS, vox_ids)
    assert ratio <= 1.0, (tag, ratio)
    if oracle_voxels:
        got = dict(verts=v, faces=f, voff=voff, toff=toff, nvert=nv, ntri=nt)
        MR.check_against_oracle(got, sdf, centres, VS, oracle_voxels, vox_ids)
    return ref, ratio


# ------------------------------------------------------------------------------------------------ 1. every res
@pytest.mark.parametrize("res", range(2, 17))
def test_every_res_against_the_restatement(nl, res):
    """Random lattices (a third crossing, a third all positive, a third all negative) around centres near 0.15, 1.05, -80.15 and
    2000.41 m: exact against emit_ref, within the fp64 bar, two crossing voxels through oracle/mc.py."""
    rng = np.random.default_rng(500 + res)
    n = 36 if res <= 8 else 15
    sdf = MR.random_lattices(rng, n, res)
    centres = MR.random_centres(rng, n, VS)
    ref, ratio = check_exact(nl, sdf, centres, oracle_voxels=(0, 3), tag=f"res {res}")
    assert ref["totals"][1] > 0
    print(f"res {res}: {ref['totals'][0]} vertices, {ref['totals'][1]} triangles, worst fp64 error {ratio:.3f} of the bar")


# ------------------------------------------------------------------------------------------------ 2. res 2: every configuration
def test_res2_every_sign_configuration(nl):
    """res 2 (mapper_specs.mesh_res of the shipped configs): one voxel per sign configuration of its 8 corners, magnitudes
    log-uniform in [1e-3, 10] so that the crossings land at varied t."""
    rng = np.random.default_rng(2)
    cfg = np.arange(256)
    inside = (cfg[:, None] >> np.arange(8)[None]) & 1
    mag = np.exp(rng.uniform(np.log(1e-3), np.log(10), size=(256, 8)))
    sdf = np.empty((256, 2, 2, 2), F32)
    for c in range(8):
        sdf[:, c & 1, c >> 1 & 1, c >> 2 & 1] = np.where(inside[:, c] == 1, -mag[:, c], mag[:, c])
    centres = MR.random_centres(rng, 256, VS)
    ref, _ = check_exact(nl, sdf, centres, oracle_voxels=range(256), tag="res 2 configurations")
    _, ntri, _ = MR.case_table()
    assert np.array_equal(ref["ntri"], ntri[cfg].astype(np.int32))


# ------------------------------------------------------------------------------------------------ 3. worst case per voxel
@pytest.mark.parametrize("res", range(2, 17))
def test_alternating_lattice(nl, res):
    """Every edge crosses: 3 res^2 (res-1) vertices and 4 triangles per cell.  At res 16 that is 11 520 vertices (the top of the
    int16 rank table, 45 vertex tiles) and 13 500 triangles (14 cell tiles)."""
    rng = np.random.default_rng(30 + res)
    sdf = np.concatenate([MR.alternating(res), -MR.alternating(res, rng=rng)])
    centres = MR.random_centres(rng, 2, VS)
    ref, _ = check_exact(nl, sdf, centres, oracle_voxels=(0, 1) if res <= 8 else (1,), tag=f"alternating res {res}")
    assert ref["nvert"].tolist() == [3 * res * res * (res - 1)] * 2
    assert ref["ntri"].tolist() == [4 * (res - 1) ** 3] * 2


# ------------------------------------------------------------------------------------------------ 4. the scan's tile edges
@pytest.mark.parametrize("n", (0, 1, 1023, 1024, 1025, 2047, 4097, 70_001))
def test_voxel_counts_at_the_scan_edges(nl, n):
    """k_mc_scan runs in tiles of 1024 voxels: totals in int64 and every offset, around the tile edges and over 69 tiles."""
    rng = np.random.default_rng(n)
    sdf = (rng.standard_normal((n, 2, 2, 2)) + rng.uniform(-1.5, 1.5, size=(n, 1, 1, 1))).astype(F32)
    centres = MR.random_centres(rng, n, VS)
    ref, _ = check_exact(nl, sdf, centres, tag=f"{n} voxels")
    if n > 1000:
        assert 0 < ref["totals"][1] and (ref["nvert"] == 0).any() and (ref["nvert"] > 0).mean() > 0.3


# ------------------------------------------------------------------------------------------------ 5. vox_ids
def test_vox_ids(nl):
    """The indirection extract_mesh always uses: a permutation, and a strided subset of a larger centre table."""
    rng = np.random.default_rng(5)
    n, res = 200, 4
    sdf = MR.random_lattices(rng, n, res)
    centres = MR.random_centres(rng, n, VS)
    check_exact(nl, sdf, centres, vox_ids=rng.permutation(n).astype(np.int32), tag="permutation")
    table = MR.random_centres(rng, 3 * n + 7, VS)
    ids = np.arange(5, 3 * n + 7, 3)[:n].astype(np.int32)
    ref, _ = check_exact(nl, sdf, table, vox_ids=ids, oracle_voxels=(0, 3), tag="strided")
    alt = MR.emit_ref(sdf, table[ids], VS)
    assert MR.same_f32(alt["verts"], ref["verts"]) and np.array_equal(alt["faces"], ref["faces"])


# ------------------------------------------------------------------------------------------------ 6. value edges
FMAX = float(np.finfo(F32).max)
POOLS = {
    "signed zeros": (0.0, -0.0, -1.0, -0.25, 1.0),
    "subnormals": (1e-45, -1e-45, 1.4e-44, -1.4e-44, 1.0, -1.0),
    "equal magnitudes": (0.7, -0.7),
    "inf and NaN": (np.inf, -np.inf, np.nan, 1.0, -1.0, 0.5),
    "near FLT_MAX": (FMAX, -FMAX, 3e38, -3e38, 1e38, -1e38, 1.0, -1.0),
}


@pytest.mark.parametrize("pool", POOLS)
@pytest.mark.parametrize("res", (2, 3, 5))
def test_value_edges(nl, pool, res):
    """Lattice values drawn from one pool of edge values per test.  Bit parity with emit_ref, NaN positions included (NaN counts
    as outside); the finite lattices with |s| < 2^126 also within the fp64 bar."""
    rng = np.random.default_rng(100 * list(POOLS).index(pool) + res)
    vals = np.asarray(POOLS[pool], F32)
    n = 64
    sdf = vals[rng.integers(0, len(vals), size=(n, res, res, res))]
    sdf[0] = MR.alternating(res)[0] * vals[vals != 0][0]                    # every edge an equal-magnitude pair
    centres = MR.random_centres(rng, n, VS)
    ref, _ = check_exact(nl, sdf, centres, oracle_voxels=(0, 1), tag=f"{pool} res {res}")
    assert ref["totals"][0] > 0
    if pool == "inf and NaN":
        assert np.isnan(ref["verts"]).any()


# ------------------------------------------------------------------------------------------------ 7. capacities
def test_capacities(nl):
    """nl_mc_emit with vertex / triangle capacities 0, 1 and total - 1 writes exactly the prefix emit_ref gives and nothing past
    it; capacities above INT32_MAX, res 1 and res 17 are refused without writing anything."""
    rng = np.random.default_rng(7)
    n, res = 40, 4
    sdf = MR.random_lattices(rng, n, res)
    centres = MR.random_centres(rng, n, VS)
    ref = MR.emit_ref(sdf, centres, VS)
    V, T = (int(x) for x in ref["totals"])
    d_sdf, d_cen = torch.from_numpy(sdf).cuda(), torch.from_numpy(centres).cuda()
    _, _, voff, toff, _ = _count(nl, d_sdf)
    d_voff, d_toff = torch.from_numpy(voff).cuda(), torch.from_numpy(toff).cuda()
    pad = 64
    for vcap, tcap in ((0, 0), (1, 1), (V - 1, T - 1), (0, T - 1), (V - 1, 0), (V, T)):
        rc, v, f = _emit(nl, d_sdf, d_cen, d_voff, d_toff, vcap, tcap, V + pad, T + pad)
        assert rc == 0
        assert MR.same_f32(v[:vcap], ref["verts"][:vcap]) and (v[vcap:] == F32(SENT_V)).all(), (vcap, tcap)
        assert np.array_equal(f[:tcap].astype(np.int64), ref["faces"][:tcap]) and (f[tcap:] == SENT_F).all(), (vcap, tcap)
    for vcap, tcap in ((INT32_MAX + 1, T), (V, INT32_MAX + 1), (2 ** 40, 2 ** 40)):
        rc, v, f = _emit(nl, d_sdf, d_cen, d_voff, d_toff, vcap, tcap, V + pad, T + pad)
        assert rc != 0 and "INT32_MAX" in nl._capi.lib().nl_last_error().decode()
        assert (v == F32(SENT_V)).all() and (f == SENT_F).all()
    C = nl._capi
    cnt = torch.zeros((4, n), dtype=torch.int32, device="cuda")
    tot = torch.zeros(2, dtype=torch.int64, device="cuda")
    for bad in (1, 17):
        assert C.lib().nl_mc_count(n, bad, C.ptr(d_sdf), C.ptr(cnt[0]), C.ptr(cnt[1]), C.ptr(cnt[2]), C.ptr(cnt[3]), C.ptr(tot),
                                   C.stream_ptr()) != 0
        rc, v, f = _emit(nl, d_sdf, d_cen, d_voff, d_toff, V, T, V + pad, T + pad, res=bad)
        assert rc != 0 and (v == F32(SENT_V)).all() and (f == SENT_F).all()
    assert not cnt.any() and not tot.any()


# ------------------------------------------------------------------------------------------------ 8. totals past int32
def test_totals_past_int32(nl):
    """159 073 voxels of the alternating res-16 lattice: 1.83e9 vertices and 2 147 485 500 > INT32_MAX triangles.  nl_mc_count's
    int64 totals are exact; marching_cubes_device raises ValueError before it allocates the outputs (22 GB + 26 GB)."""
    n, res = 159_073, 16
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    centres = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
    one = torch.from_numpy(MR.alternating(res)).cuda()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    sdf = one.expand(n, res, res, res).contiguous()                         # 2.6 GB, built on the device
    try:
        nv, nt, voff, toff, tot = _count(nl, sdf)
        assert tot.tolist() == [11_520 * n, 13_500 * n] and tot[1] > INT32_MAX and tot[0] <= INT32_MAX
        assert (nv == 11_520).all() and (nt == 13_500).all()
        fits = 13_500 * np.arange(n, dtype=np.int64) <= INT32_MAX             # the int32 offsets are exact up to INT32_MAX
        assert np.array_equal(toff[fits].astype(np.int64), 13_500 * np.arange(n)[fits])
        assert np.array_equal(voff.astype(np.int64), 11_520 * np.arange(n))
        with pytest.raises(ValueError, match="INT32_MAX"):
            nl.mesh.marching_cubes_device(sdf, centres, VS)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        # the lattice, plus two sets of counts (4 n int32) and totals, each rounded up to the allocator's 2 MB blocks
        assert peak <= sdf.numel() * 4 + 2 * (16 * n + (2 << 20)), peak
        print(f"peak device memory above the start: {peak / 1e9:.3f} GB")
    finally:
        del sdf
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ 9. the lattice of a trained map
@pytest.fixture(scope="module", params=(256, 64), ids=("w256", "w64"))
def trained_map(request, nl):
    """A map of one synthetic scan and a decoder of the given width trained on it for 30 bundle_adjust_frames iterations."""
    width = request.param
    syn = nl.synthetic
    pts, cos, pose = syn.make_scan(n_beams=16, n_az=200, seed=4)
    mu = nl.mapping.MapUpdater(VS, init_std=0.05, seed=7)
    ms = mu.insert_voxels(torch.from_numpy(syn.voxelize(pts, pose, VS)))
    torch.manual_seed(1)
    dec = nl.lidar.Decoder(depth=2, width=width, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    frames = [nl.frame.LidarFrame(0, torch.from_numpy(pts), torch.from_numpy(cos),
                                  nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose.copy())), new_keyframe=True)]
    torch.manual_seed(9)
    nl.render_helpers.bundle_adjust_frames(frames, ms.emb, ms, dec, nl.criterion.Criterion(Args()), VS, 0.5 * VS, N_rays=1024,
                                           num_iterations=30, truncation=0.3, max_voxel_hit=20, max_distance=40.0,
                                           learning_rate=[0.01, 0.005, 0.001], update_pose=False, update_decoder=True,
                                           deterministic=True, ray_selection="host")
    torch.cuda.synchronize()
    return ms, dec, width


def _sdf_bar(width, feats, P):
    """(fp64 sdf, u a_sdf, the bar in units of u a_sdf) for the decoder of this width: tensor cores (256): HARD of decoder_tc_ref,
    the bound derived from its k-step model; CUDA cores (32-128): (2W + 20) (tests/test_gpu_decoder_simt.py).  decoder_tc_ref's
    DISC (1 u a_sdf) is calibrated on its emulator's inputs; the trained map's lattice reaches about 1.5 u a_sdf on an H100, so
    the ratio is printed, not asserted against DISC."""
    ref = DR.forward(feats, P)["sdf"]
    a_sdf = torch.cat([DR.absolute(feats[s:e], P)[2] for s, e in DR._chunks(feats.shape[0])])
    return ref, TR.U * a_sdf, (TR.HARD["sdf"] if width == 256 else 2 * width + 20)


@pytest.mark.parametrize("res", (2, 8, 16))
def test_lattice_against_fp64(nl, trained_map, res, monkeypatch):
    """scores_device on a trained map: lattice points bit-equal to fp32(linspace * vs) + centre, features bit-equal to
    gather_fwd_f32, sdf within the decoder's bar, bit-identical output when the voxels are split unevenly into launches, and
    get_scores' rows without embeddings one constant, decoder(0) within the bar."""
    rh = nl.render_helpers
    ms, dec, width = trained_map
    every = (ms.vox2row[:, 0] >= 0).nonzero().view(-1)
    nodes = every[::max(1, -(-len(every) * res ** 3 // 300_000))]           # at most ~300 k lattice points
    seen = []
    orig = rh.mlp_forward

    def spy(*args):                                                          # mlp_forward(bufs, M, None, feats, out)
        seen.append((sys._getframe(1).f_locals["xyz"].clone(), args[3].clone()))
        return orig(*args)
    monkeypatch.setattr(rh, "mlp_forward", spy)
    lat, got_nodes = rh.scores_device(dec, ms, VS, res, nodes=nodes)
    monkeypatch.undo()
    assert torch.equal(got_nodes, nodes) and lat.shape == (len(nodes), res ** 3)
    xyz = torch.cat([s[0] for s in seen]).cpu().numpy()
    feats = torch.cat([s[1] for s in seen])
    cen, ids = ms.centres.cpu().numpy(), nodes.cpu().numpy()
    want_xyz = MR.lattice_points(cen[ids], res, VS).reshape(-1, 3)
    assert MR.same_f32(xyz, want_xyz)
    vox = np.repeat(ids.astype(np.int32), res ** 3)
    want_f = ER.gather_fwd_f32(want_xyz, vox, cen, ms.vox2row.cpu().numpy(), ms.emb.float().cpu().numpy(), VS)
    assert MR.same_f32(feats.cpu().numpy(), want_f)
    P = [p.cuda() for p in DR.params64(dec)]
    ref, ua, bar = _sdf_bar(width, feats, P)
    ratio = float(((lat.reshape(-1).double() - ref).abs() / ua).max())
    print(f"w{width} res {res}: {len(nodes)} voxels, sdf in [{float(lat.min()):.3f}, {float(lat.max()):.3f}], "
          f"worst |sdf - fp64| = {ratio:.3f} u a_sdf (bar {bar})")
    assert ratio <= bar, ratio
    assert float(lat.min()) < 0 < float(lat.max())                           # the trained map's zero level runs through it
    lat2, _ = rh.scores_device(dec, ms, VS, res, nodes=nodes, chunk=1000)
    assert torch.equal(lat2.view(torch.int32), lat.view(torch.int32))
    if res == 2:
        full = rh.get_scores(dec, ms, VS, bits=2).view(ms.n_nodes, -1)
        lat_all, _ = rh.scores_device(dec, ms, VS, 2)
        assert torch.equal(full[every.cpu()].view(torch.int32), lat_all.cpu().view(torch.int32))
        rest = torch.ones(ms.n_nodes, dtype=torch.bool)
        rest[every.cpu()] = False
        const = full[rest]
        assert const.shape[0] > 0 and bool((const == const.reshape(-1)[0]).all())
        zero = torch.zeros((1, 16), dtype=torch.float32, device="cuda")
        r0, ua0, bar0 = _sdf_bar(width, zero, P)
        assert abs(float(const.reshape(-1)[0]) - float(r0[0])) <= bar0 * float(ua0[0])


# ------------------------------------------------------------------------------------------------ 10. extract_mesh end to end
@pytest.mark.parametrize("res", (2, 8))
def test_extract_mesh_end_to_end(nl, trained_map, res):
    """extract_mesh equals emit_ref on the kernel's own lattice with vox_ids = the nodes, and every vertex lies inside its own
    voxel's cube within the fp64 bar."""
    ms, dec, width = trained_map
    lat, nodes = nl.render_helpers.scores_device(dec, ms, VS, res)
    v, f = nl.mesh.extract_mesh(dec, ms, VS, res=res)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    sdf = lat.view(-1, res, res, res).cpu().numpy()
    cen, ids = ms.centres.cpu().numpy(), nodes.cpu().numpy().astype(np.int32)
    ref = MR.emit_ref(sdf, cen, VS, vox_ids=ids)
    assert f.shape[0] > 100
    assert MR.same_f32(v, ref["verts"]) and np.array_equal(f.astype(np.int64), ref["faces"])
    o, bar, ok = MR.vertex_fp64(sdf, cen, VS, ids)
    assert ok.all() and float((np.abs(v - o) / bar).max()) <= 1.0
    c = cen[ids[ref["vert_vox"]]].astype(np.float64)
    assert bool((np.abs(v.astype(np.float64) - c) <= np.float64(F32(VS)) / 2 + bar).all())
