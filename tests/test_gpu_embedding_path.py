"""The embedding-table path against the numpy references of tests/embedding_ref.py, exactly where exactness is defined:
- k_gather_fwd bit for bit against gather_fwd_f32;
- k_gather_bwd<0|1|2> on dyadic inputs (every fp32 sum exact in any order) equal to the float64 reference for d emb, d xyz and the
  pose accumulators, over a catalogue of run shapes, output combinations, frame layouts and a device-side count.  The merge level is
  read once per process (NL_GATHER_MERGE), so each level runs in a child process: this file run as a script;
- k_gather_bwd on a real sample list within Higham's gamma bound of the float64 reference;
- nl_adam_{f32,bf16}[_ctl] bit for bit against adam_step."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import embedding_ref as ER  # noqa: E402

pytestmark = pytest.mark.gpu
F32 = np.float32
SENTINEL = F32(-7777.25)


@pytest.fixture(scope="module")
def nl():
    import torch
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


def _grid_stride():
    """Samples per grid-stride iteration of the persistent gather kernels: (SMs * 16) blocks of 128."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 128


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------------------------------------ a. forward
def _fwd_problem(rng, M, vs, n_vox=5000, n_rows=20000):
    centres = (rng.integers(-400, 400, size=(n_vox, 3)) * 0.25).astype(F32)
    vox2row = rng.integers(0, n_rows, size=(n_vox, 8)).astype(np.int32)
    vox2row[rng.random((n_vox, 8)) < 0.1] = -1                          # vertices without a row
    vox2row[:3] = -1                                                    # voxels without any row
    vox = rng.integers(0, n_vox, size=M).astype(np.int32)
    u = rng.uniform(-0.5, 0.5, size=(M, 3)) * vs
    snap = rng.random(M) < 0.25                  # on the 1/8 lattice of the voxel: faces and edges (p = 0 or 1 on some axis)
    u[snap] = (rng.integers(0, 9, size=(int(snap.sum()), 3)) - 4) * (vs / 8)
    corner = rng.random(M) < 0.05                # corners: p in {0, 1} on every axis
    u[corner] = rng.choice([-0.5, 0.5], size=(int(corner.sum()), 3)) * vs
    xyz = (centres[vox] + u.astype(F32)).astype(F32)
    emb = ER.bf16_rne(rng.standard_normal((n_rows, 16)).astype(F32))
    return xyz, vox, centres, vox2row, emb


@pytest.mark.parametrize("M", [1, 31, 32, 33, 127, 128, 129, 300_001])
def test_gather_forward_bit_exact(nl, M):
    """Power-of-two voxel (faces and corners exactly representable) and a 0.3 m voxel (rounded division), every M around the
    warp and block edges and one past the persistent grid (grid-stride loop)."""
    import torch
    cap, lib = nl._capi, nl._capi.lib()
    for vs in (0.25, 0.3):
        rng = np.random.default_rng(M * 7 + int(vs * 100))
        xyz, vox, centres, vox2row, emb = _fwd_problem(rng, M, vs)
        ref = ER.gather_fwd_f32(xyz, vox, centres, vox2row, emb, vs)
        t = [_cuda(a) for a in (xyz, vox, centres, vox2row)]
        e = torch.from_numpy(ER.bf16_bits(emb).view(np.int16)).cuda().view(torch.bfloat16)
        out = torch.empty((M, 16), dtype=torch.float32, device="cuda")
        cap.check(lib.nl_gather_trilinear_fwd(M, None, *[cap.ptr(x) for x in t], cap.ptr(e), vs, cap.ptr(out), cap.stream_ptr()))
        got = out.cpu().numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (vs, int((got != ref).sum()))


def test_gather_forward_device_count(nl):
    """A device-side count below M: rows up to the count are the reference's, rows past it keep their sentinel."""
    import torch
    cap, lib = nl._capi, nl._capi.lib()
    M = _grid_stride() + 4099
    rng = np.random.default_rng(11)
    xyz, vox, centres, vox2row, emb = _fwd_problem(rng, M, 0.3)
    e = torch.from_numpy(ER.bf16_bits(emb).view(np.int16)).cuda().view(torch.bfloat16)
    t = [_cuda(a) for a in (xyz, vox, centres, vox2row)]
    for n in (0, 1, 33, _grid_stride() + 1, M - 1):
        ref = ER.gather_fwd_f32(xyz[:n], vox[:n], centres, vox2row, emb, 0.3)
        out = torch.full((M, 16), float(SENTINEL), dtype=torch.float32, device="cuda")
        cnt = torch.tensor([n], dtype=torch.int32, device="cuda")
        cap.check(lib.nl_gather_trilinear_fwd(M, cap.ptr(cnt), *[cap.ptr(x) for x in t], cap.ptr(e), 0.3,
                                              cap.ptr(out), cap.stream_ptr()))
        got = out.cpu().numpy()
        assert np.array_equal(got[:n].view(np.uint32), ref.view(np.uint32)), n
        assert np.all(got[n:] == SENTINEL), n


# ------------------------------------------------------------------------------------------------ b. backward, dyadic, every merge level
N_VOX, N_ROWS, EMPTY = 4096, 6000, 0          # voxel 0 has no row at any corner


class _Ids:
    """Voxel ids 1..N_VOX-1 in turn: consecutive draws always differ."""

    def __init__(self):
        self.i = 0

    def __call__(self):
        self.i = self.i % (N_VOX - 1) + 1
        return self.i


def catalogue_sequence(rng, n_tail=1517):
    """Voxel id per sample: every run length 1..9 at every start lane 0..31 (one 64-sample segment each, the run preceded either by
    singletons or by another run ending just before it; runs past lane 31 cross into the next warp), runs split by a voxel without
    rows, ray-like random runs, and a partial last warp."""
    ids = _Ids()
    seq = []
    for L in range(1, 10):
        for s in range(32):
            seg = [ids() for _ in range(64)]
            if (L + s) % 2 and s > 0:
                a = ids()
                seg[:s] = [a] * s
            b = ids()
            seg[s:s + L] = [b] * L
            if s + L < 64 and seg[s + L] == b:
                seg[s + L] = ids()
            seq += seg
    for _ in range(8):                                                   # runs separated by a voxel without rows
        b = ids()
        seq += [b] * 3 + [EMPTY] + [b] * 5 + [EMPTY, EMPTY] + [b] * 2 + [EMPTY] + [b] * 9 + [ids()]
    end = len(seq) + 1500
    while len(seq) < end:                                                # ray-like runs
        seq += [ids()] * int(rng.geometric(0.2))
    seq += [ids() for _ in range(n_tail)]
    for blk in (3, 17, 40):                                              # runs across block boundaries
        seq[128 * blk - 3:128 * blk + 6] = [ids()] * 9
    return np.array(seq, np.int32)


def stride_sequence(rng, M, stride):
    """M samples past one grid-stride iteration: ray-like runs (geometric lengths), voxels without rows in between, and runs that
    cross the warp, block and grid-stride boundaries."""
    ids = _Ids()
    seq = []
    while len(seq) < M:
        seq += [EMPTY] if rng.random() < 0.02 else [ids()] * int(rng.geometric(0.15))
    seq = seq[:M]
    for c in (32 * 7, 128 * 5, 128 * 777, stride - 128, stride):
        seq[c - 3:c + 5] = [ids()] * 8
    return np.array(seq, np.int32)


def frame_layout(M, F, kind):
    """ray_frame per ray (= per sample here): 'warp' = one frame per 32 samples, 'mixed' = the frame changes at every sample."""
    i = np.arange(M)
    return ((i // 32) % F if kind == "warp" else (i + i // 32) % F).astype(np.int32)


def _launches(stride):
    """(case name, problem kwargs, sequence builder) and the launches: outputs, frames, device count."""
    cases = {
        "catalogue": dict(seq=lambda r: catalogue_sequence(r), g_density=1.0, levels=1),
        "stride": dict(seq=lambda r: stride_sequence(r, 300_001, stride), g_density=1 / 16, levels=1),
        "hot": dict(seq=lambda r: np.full(100_000, 7, np.int32), g_density=1.0, levels=1),
    }
    L = []
    for c in cases:
        L += [dict(case=c, out="emb"), dict(case=c, out="dxyz")]
    L += [dict(case="catalogue", out="track"), dict(case="stride", out="track")]
    for F in (1, 3, 31, 32, 1024):
        for kind in (("warp",) if F == 1 else ("warp", "mixed")):
            L.append(dict(case="catalogue", out="all", F=F, frames=kind))
    L += [dict(case="stride", out="all", F=3, frames="mixed"), dict(case="stride", out="all", F=1024, frames="warp")]
    L += [dict(case="catalogue", out="all", F=3, frames="mixed", count=-1000),      # device-side count = M - 1000, NaN past it
          dict(case="stride", out="all", F=32, frames="warp", count=stride + 77)]
    return cases, L


def make_problems(stride):
    cases, launches = _launches(stride)
    P = {}
    for i, (name, c) in enumerate(cases.items()):
        rng = np.random.default_rng(1000 + i)
        P[name] = ER.dyadic_problem(rng, c["seq"](rng), N_VOX, N_ROWS, g_levels=c["levels"], f_levels=c["levels"], g_density=c["g_density"],
                                    empty_vox=(EMPTY,))
    for ln in launches:
        M = len(P[ln["case"]]["vox"])
        ln["M"] = M
        ln["count"] = (M + ln["count"] if ln["count"] < 0 else ln["count"]) if "count" in ln else None
    return P, launches


def expected(P, ln):
    """float64 reference of one launch: {name: array}."""
    n = ln["M"] if ln["count"] is None else ln["count"]
    p = {k: (v[:n] if isinstance(v, np.ndarray) and v.shape[:1] == (ln["M"],) else v) for k, v in P.items()}
    _, w = ER.corner_factors(p["xyz"], p["vox"], p["centres"], p["voxel_size"])
    out = {}
    if ln["out"] in ("emb", "all"):
        out["grad_emb"] = ER.scatter_ref(p["vox"], p["vox2row"], w, p["dfeats"], P["n_rows"])[0]
    d, da = ER.dxyz_ref(p["xyz"], p["vox"], p["centres"], p["vox2row"], p["emb"], p["voxel_size"], p["dfeats"])
    if ln["out"] in ("dxyz", "all"):
        out["dxyz"] = np.concatenate([d, np.full((ln["M"] - n, 3), SENTINEL, np.float64)])
    if ln["out"] in ("track", "all"):
        rf = None if ln["out"] == "track" else frame_layout(ln["M"], ln["F"], ln["frames"])
        out["pose_acc"] = ER.pose_acc_ref(d, da, p["s_ray"], p["s_depth"], p["dir_local"], rf, 1 if rf is None else ln["F"])[0]
    return out


def run_child(inp, outp):
    """Child process: every launch of `inp` at the merge level NL_GATHER_MERGE names; outputs and the kernel name to `outp`."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    import nerfloam_b200 as nl
    cap, lib = nl._capi, nl._capi.lib()
    z = np.load(inp)
    launches = json.loads(str(z["launches"]))
    dev = {}
    res, kname = {}, None
    for j, ln in enumerate(launches):
        c = ln["case"]
        if c not in dev:
            dev[c] = {k: _cuda(z[f"{c}__{k}"]) for k in ("xyz", "vox", "centres", "vox2row", "s_ray", "s_depth", "dir_local")}
            dev[c]["emb"] = torch.from_numpy(ER.bf16_bits(z[f"{c}__emb"]).view(np.int16)).cuda().view(torch.bfloat16)
            dev[c]["n_rows"] = int(z[f"{c}__n_rows"])
            dev[c]["vs"] = float(z[f"{c}__voxel_size"])
        d, M = dev[c], ln["M"]
        g = z[f"{c}__dfeats"].copy()
        cnt = None
        if ln["count"] is not None:
            g[ln["count"]:] = np.nan
            cnt = torch.tensor([ln["count"]], dtype=torch.int32, device="cuda")
        g = _cuda(g)
        o = ln["out"]
        ge = torch.zeros((d["n_rows"], 16), dtype=torch.float32, device="cuda") if o in ("emb", "all") else None
        dx = torch.full((M, 3), float(SENTINEL), dtype=torch.float32, device="cuda") if o in ("dxyz", "all") else None
        F = ln.get("F", 1)
        pa = torch.zeros((F, 12), dtype=torch.float32, device="cuda") if o in ("track", "all") else None
        rf = _cuda(frame_layout(M, F, ln["frames"])) if o == "all" else None
        pose = pa is not None

        def launch():
            cap.check(lib.nl_gather_trilinear_bwd(
                M, cap.ptr(cnt), cap.ptr(d["xyz"]), cap.ptr(d["vox"]), cap.ptr(d["centres"]), cap.ptr(d["vox2row"]), cap.ptr(d["emb"]),
                d["vs"], cap.ptr(g), 1, cap.ptr(ge), cap.ptr(dx), cap.ptr(d["s_ray"]) if pose else None,
                cap.ptr(d["s_depth"]) if pose else None, cap.ptr(d["dir_local"]) if pose else None, cap.ptr(rf), F, cap.ptr(pa),
                cap.stream_ptr()), "nl_gather_trilinear_bwd")

        if kname is None:
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                launch()
                torch.cuda.synchronize()
            kname = [e.name for e in prof.events() if "k_gather_bwd" in e.name][0]
        else:
            launch()
        for k, t in (("grad_emb", ge), ("dxyz", dx), ("pose_acc", pa)):
            if t is not None:
                res[f"{j}__{k}"] = t.cpu().numpy()
    np.savez(outp, kernel=np.array(kname), **res)


@pytest.fixture(scope="module")
def merge_runs(nl, tmp_path_factory):
    """Problems, launches and, per merge level, the child's outputs and the name of the kernel it ran."""
    d = tmp_path_factory.mktemp("gather_bwd")
    stride = _grid_stride()
    P, launches = make_problems(stride)
    arrays = {f"{c}__{k}": np.asarray(v) for c, p in P.items() for k, v in p.items()}
    inp = os.path.join(d, "in.npz")
    np.savez(inp, launches=np.array(json.dumps(launches)), **arrays)
    runs = {}
    for level in (0, 1, 2):
        outp = os.path.join(d, f"out{level}.npz")
        env = dict(os.environ, NL_GATHER_MERGE=str(level))
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), inp, outp]
        subprocess.run(cmd, env=env, cwd=ROOT, check=True, timeout=300)
        runs[level] = dict(np.load(outp))
    refs = [expected(P[ln["case"]], ln) for ln in launches]
    return P, launches, runs, refs


def test_dyadic_inputs_are_exactly_summable(merge_runs):
    """The premise of the exact comparisons: every fp32 sum the backward forms on these inputs is exact in any order."""
    P, launches = merge_runs[:2]
    for name, p in P.items():
        layouts = [(None, 1) if ln["out"] == "track" else (frame_layout(ln["M"], ln["F"], ln["frames"]), ln["F"])
                   for ln in launches if ln["case"] == name and ln["out"] in ("track", "all")]
        m = ER.dyadic_margins(p, layouts)
        assert max(m.values()) < 1, (name, m)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_gather_backward_dyadic_exact(merge_runs, level):
    """grad_emb, dxyz and pose_acc equal the float64 reference exactly: no contribution dropped, doubled or credited to the wrong
    row or frame, for every run shape, output combination, frame layout and device-side count."""
    P, launches, runs, refs = merge_runs
    r = runs[level]
    assert f"k_gather_bwd<{level}>" in str(r["kernel"]), str(r["kernel"])
    for j, (ln, ref) in enumerate(zip(launches, refs)):
        assert set(ref) == {k.split("__")[1] for k in r if k.startswith(f"{j}__")}, ln
        for k, want in ref.items():
            got = r[f"{j}__{k}"].astype(np.float64)
            bad = np.argwhere(got != want)
            assert bad.size == 0, (ln, k, len(bad), bad[:5].tolist(), got[tuple(bad[0])], want[tuple(bad[0])])


def test_gather_backward_merge_levels_agree_bit_for_bit(merge_runs):
    runs = merge_runs[2]
    keys = [k for k in runs[0] if k != "kernel"]
    assert keys and all(set(k for k in runs[lv] if k != "kernel") == set(keys) for lv in (1, 2))
    for k in keys:
        a = runs[0][k].view(np.uint32)
        assert np.array_equal(a, runs[1][k].view(np.uint32)) and np.array_equal(a, runs[2][k].view(np.uint32)), k


# ------------------------------------------------------------------------------------------------ c. backward, real samples, bound
# Rounded fp32 operations per term in k_gather_bwd (the compiler may contract a multiply into a following add, which only removes
# roundings).  d xyz[a] = fl(1/vs) * sum_k (dot_k * (+-1) * a_b * a_c), dot_k = fma chain over e = 0..15:
DOT_ROUNDINGS = 16            # each fma of the dot product rounds once; the first term passes through all 16
CORNER_ROUNDINGS = 2          # * a_b, * a_c (the sign is exact)
CORNER_SUM_ROUNDINGS = 8      # gx += over the 8 corners
SCALE_ROUNDINGS = 2           # fl(1 / voxel_size) and the multiplication by it
DXYZ_ROUNDINGS = DOT_ROUNDINGS + CORNER_ROUNDINGS + CORNER_SUM_ROUNDINGS + SCALE_ROUNDINGS
POSE_R_EXTRA = 2              # l = d_local * depth, then g * l


def test_gather_backward_real_samples_within_bound(nl):
    """The sample list of SDFEngine.render_samples over a MapUpdater map of a synthetic scan (the traversal's own run structure),
    three frames laid out like bundle_adjust_frames, random fp32 dfeats, round_bf16 = 1.  Per element |got - ref| <= gamma_k * sum
    |term|, with k = (number of terms - 1) summation roundings plus the per-term roundings counted above."""
    import torch
    cap, lib = nl._capi, nl._capi.lib()
    dev = torch.device("cuda")
    syn = nl.synthetic
    pts, cos, pose = syn.make_scan(n_beams=32, n_az=900, seed=5)
    vs = 0.3
    mu = nl.mapping.MapUpdater(vs, init_std=0.05, seed=3, device=dev)
    ms = mu.insert_voxels(torch.from_numpy(syn.voxelize(pts, pose, vs)))
    P = torch.from_numpy(pts).to(dev)
    dirs_all = P / (P.norm(dim=-1, keepdim=True) + 1e-8)
    N, F = 6000, 3
    g = torch.Generator().manual_seed(9)
    sel = torch.randperm(dirs_all.shape[0], generator=g)[:N * F].to(dev)
    dirs = dirs_all[sel].contiguous()
    fid = torch.arange(F, dtype=torch.int32, device=dev).repeat_interleave(N).contiguous()
    p0 = nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose)).data.detach().float()
    pose6 = torch.stack([p0 + torch.tensor([0.05 * f, -0.03 * f, 0.02 * f, 0.002 * f, 0.0, -0.001 * f]) for f in range(F)]).to(dev).contiguous()
    cfg = dict(step_size=0.15, voxel_size=vs, max_distance=40.0)
    eng = nl.engine.SDFEngine(N * F, N * F * 48, dev)
    eng.rays_from_poses(pose6, dirs, fid)
    eng.render_samples(ms, N * F, cfg)
    st = eng.read_stats()
    M, Mc = st.n_samples, eng.max_samples
    assert st.error == 0 and 100_000 < M < Mc
    torch.manual_seed(4)
    dfe = torch.randn((Mc, 16), device=dev) * 1e-3
    grad_emb = torch.zeros((ms.emb.shape[0], 16), dtype=torch.float32, device=dev)
    dxyz = torch.empty((Mc, 3), dtype=torch.float32, device=dev)
    pose_acc = torch.zeros((F, 12), dtype=torch.float32, device=dev)
    cap.check(lib.nl_gather_trilinear_bwd(Mc, eng.n_samples_dev, cap.ptr(eng.s_xyz), cap.ptr(eng.s_vox), cap.ptr(ms.centres),
                                          cap.ptr(ms.vox2row), cap.ptr(ms.emb), vs, cap.ptr(dfe), 1, cap.ptr(grad_emb), cap.ptr(dxyz),
                                          cap.ptr(eng.s_ray), cap.ptr(eng.s_depth), cap.ptr(dirs), cap.ptr(fid), F, cap.ptr(pose_acc),
                                          cap.stream_ptr()))
    xyz, vox = eng.s_xyz[:M].cpu().numpy(), eng.s_vox[:M].cpu().numpy()
    s_ray, s_depth = eng.s_ray[:M].cpu().numpy(), eng.s_depth[:M].cpu().numpy()
    centres, vox2row = ms.centres.cpu().numpy(), ms.vox2row.cpu().numpy()
    emb = ms.emb.float().cpu().numpy()
    gf = dfe[:M].cpu().numpy()
    _, w = ER.corner_factors(xyz, vox, centres, vs)
    ratios = {}
    # d emb: contributions are exact fp32 values (bf16-rounded products): only the n - 1 additions of each row round
    ref, n, a = ER.scatter_ref(vox, vox2row, w, gf, emb.shape[0])
    err = np.abs(grad_emb.cpu().numpy() - ref)
    bound = ER.gamma(np.maximum(n - 1, 0)) * a
    assert np.all(err <= bound), int((err > bound).sum())
    ratios["grad_emb"] = float((err[bound > 0] / bound[bound > 0]).max())
    assert int((n > 1).sum()) > 0 and np.all(err[n <= 1] == 0)
    # d xyz
    d, da = ER.dxyz_ref(xyz, vox, centres, vox2row, emb, vs, gf)
    err = np.abs(dxyz[:M].cpu().numpy() - d)
    bound = ER.gamma(DXYZ_ROUNDINGS) * da
    assert np.all(err <= bound), int((err > bound).sum())
    ratios["dxyz"] = float((err[bound > 0] / bound[bound > 0]).max())
    # pose: per-sample terms summed over the frame's samples in some order (warp tree, shared and global atomics)
    acc, aab = ER.pose_acc_ref(d, da, s_ray, s_depth, dirs.cpu().numpy(), fid.cpu().numpy(), F)
    cnt = np.bincount(fid.cpu().numpy()[s_ray], minlength=F)[:, None]
    k = (cnt - 1) + DXYZ_ROUNDINGS + np.array([0] * 3 + [POSE_R_EXTRA] * 9)[None, :]
    err = np.abs(pose_acc.cpu().numpy() - acc)
    bound = ER.gamma(k) * aab
    assert np.all(err <= bound), (err / bound).max()
    ratios["pose_acc"] = float((err / bound).max())
    print("max |got - ref| / bound:", json.dumps(ratios), f"M={M}")


# ------------------------------------------------------------------------------------------------ d. Adam
def _adam_inputs(rng, n, bf16):
    """Parameters, moments and gradients with the special cases spread over the vector: g = 0, g so small that w2 g g underflows
    (denominator = eps), large g, bf16 ties, negative values, zero moments, and second moments so small that eps is not negligible
    in the denominator."""
    p = rng.standard_normal(n).astype(F32) * F32(0.05)
    m = rng.standard_normal(n).astype(F32) * F32(1e-2)
    v = np.abs(rng.standard_normal(n)).astype(F32) * F32(1e-4)
    g = rng.standard_normal(n).astype(F32)
    k = n // 8
    g[:k] = 0
    g[k:2 * k] = rng.choice([-1, 1], k) * F32(1e-25)
    m[k:2 * k] = 0
    v[k:2 * k] = 0
    g[2 * k:3 * k] *= F32(1e5)
    m[3 * k:4 * k] = 0
    v[3 * k:4 * k] = 0
    tie = (rng.integers(0x3c00, 0x4100, 2 * k).astype(np.uint32) << 16) | 0x8000     # exactly half way between two bf16
    g[4 * k:5 * k] = tie[:k].view(F32) * rng.choice([-1, 1], k)
    p[5 * k:6 * k] = tie[k:].view(F32) * F32(0.0625)
    v[6 * k:7 * k] = 10.0 ** rng.uniform(-19, -13, k)                  # sqrt(v) / bc2_sqrt near eps: each rounding of d shows
    g[6 * k:7 * k] = 0
    if bf16:
        p, m, v = ER.bf16_rne(p), ER.bf16_rne(m), ER.bf16_rne(v)
    return p, g, m, v


def _adam_dev(nl, p, m, v, bf16):
    import torch
    if bf16:
        return [torch.from_numpy(ER.bf16_bits(x).view(np.int16)).cuda().view(torch.bfloat16) for x in (p, m, v)]
    return [_cuda(x) for x in (p, m, v)]


def _host(t):
    import torch
    return t.float().cpu().numpy() if t.dtype == torch.bfloat16 else t.cpu().numpy()


def _eq(a, b):
    return np.array_equal(np.asarray(a, F32).view(np.uint32), np.asarray(b, F32).view(np.uint32))


HP = dict(lr=0.01, beta1=0.9, beta2=0.999, eps=1e-8)


@pytest.mark.parametrize("bf16", [False, True])
def test_adam_trajectory_bit_exact(nl, bf16):
    """nl_adam_f32 / nl_adam_bf16 over 12 steps equal adam_step bit for bit, moments included."""
    cap, lib = nl._capi, nl._capi.lib()
    rng = np.random.default_rng(21 + bf16)
    n = 8 * 1024 + 5
    p, g, m, v = _adam_inputs(rng, n, bf16)
    tp, tm, tv = _adam_dev(nl, p, m, v, bf16)
    fn = lib.nl_adam_bf16 if bf16 else lib.nl_adam_f32
    for t in range(1, 13):
        gt = _cuda(g)
        cap.check(fn(n, cap.ptr(tp), cap.ptr(gt), cap.ptr(tm), cap.ptr(tv), HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], t,
                     cap.stream_ptr()))
        p, m, v = ER.adam_step(p, g, m, v, HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], t, bf16)
        for name, a, b in (("p", _host(tp), p), ("m", _host(tm), m), ("v", _host(tv), v)):
            assert _eq(a, b), (t, name, int((a != b).sum()))
        g = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 2, n)).astype(F32)
        g[:n // 8] = 0


@pytest.mark.parametrize("bf16", [False, True])
def test_adam_ctl_matches_host_constants(nl, bf16):
    """nl_adam_*_ctl evaluate the bias corrections per thread with the device's double pow; at each step they equal the
    host-constant kernel and adam_step bit for bit.  A set skip flag leaves p, m and v bit-identical."""
    import torch
    cap, lib = nl._capi, nl._capi.lib()
    rng = np.random.default_rng(5 + bf16)
    n = 4 * 1024 + 3
    host_fn, ctl_fn = (lib.nl_adam_bf16, lib.nl_adam_bf16_ctl) if bf16 else (lib.nl_adam_f32, lib.nl_adam_f32_ctl)
    for t in (1, 2, 3, 7, 100, 10 ** 3, 10 ** 4, 10 ** 6):
        p, g, m, v = _adam_inputs(rng, n, bf16)
        a, b = _adam_dev(nl, p, m, v, bf16), _adam_dev(nl, p, m, v, bf16)
        gt = _cuda(g)
        ctl = torch.zeros(cap.CTL_WORDS, dtype=torch.int32, device="cuda")
        ctl[cap.CTL_ADAM_STEP] = t
        cap.check(host_fn(n, *[cap.ptr(x) for x in (a[0], gt, a[1], a[2])], HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], t, cap.stream_ptr()))
        cap.check(ctl_fn(n, *[cap.ptr(x) for x in (b[0], gt, b[1], b[2])], HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], cap.ptr(ctl),
                         cap.stream_ptr()))
        ref = ER.adam_step(p, g, m, v, HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], t, bf16)
        for i, name in enumerate("pmv"):
            assert _eq(_host(a[i]), ref[i]), (t, name, "host constants vs adam_step")
            assert _eq(_host(b[i]), ref[i]), (t, name, "device constants vs adam_step")
        before = [x.clone() for x in b]
        ctl[cap.CTL_SKIP_NOW] = 1
        cap.check(ctl_fn(n, *[cap.ptr(x) for x in (b[0], gt, b[1], b[2])], HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], cap.ptr(ctl),
                         cap.stream_ptr()))
        assert all(torch.equal(x.view(torch.int16) if bf16 else x.view(torch.int32), y.view(torch.int16) if bf16 else y.view(torch.int32))
                   for x, y in zip(before, b)), t


if __name__ == "__main__":
    run_child(sys.argv[1], sys.argv[2])
