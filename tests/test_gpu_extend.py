"""slam.NeRFLOAM(..., base_map=...) on the GPU: a street drive A mapped and saved, then a later drive B that starts inside A (shifted
0.5 m and turned 10 degrees, no pose guess) and drives on past A's coverage, grown into A's map.  B's poses against the truth, what
stays frozen, the grown file on both octrees, a third drive C localised in the grown map from the saved ground into the new ground,
the grown mesh against a from-scratch map of the same drive, the refinement floor, a drive that cannot be placed, and
scripts/run_slam.py --base-map.  B is also mapped from scratch (an empty map, a new decoder, its first true pose given) as the
control for the pose drift and the mesh quality on ground the saved map never saw.

The street is synthetic.street_boxes with a longer `length`, so it reaches past B's last scan; A maps with the true poses (use_gt),
so the map frame is the scene's frame and B's tracked poses can be held to the true ones."""
import importlib
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from test_gpu_localise import MAX_DR, MAX_DT, SHIFT, TURN, MemoryStream, _buffers, _bytes, _same, config, errors

pytestmark = pytest.mark.gpu
share = importlib.import_module("nerf-loam_b200.share")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_A, SPACING_A = 12, 0.5              # drive A: x = 0 .. 5.5 m, as tests/test_gpu_localise.py
N_B, SPACING_B = 86, 1.0              # drive B: x = 0.3 .. 85.3 m
NEW_X = 58.0                          # B's scans from here on are new ground (asserted below: < 5 % of their rays hit map A)
NEW_HIT = 0.05
INSIDE_X = 40.0                       # B's scans up to here are held to MAX_DT; past it, tracking on new ground drifts like odometry
DRIFT = 0.01                          # m of translation error per m driven past INSIDE_X, on top of MAX_DT (measured 0.0045, DESIGN.md 11.6)
SCRATCH_RATIO = 1.5                   # B's worst translation error grown into A <= this x the same drive's from scratch
C_X = (30, 70)                        # drive C: 1 m apart from x = 30 (saved ground) to 69 (new ground)
# F-score at 0.1 m (percent) the grown map's mesh on B's new segment may lose against the from-scratch map's mesh on the same segment,
# each scored against B's points at its own estimated poses.  Measured on an H100 80GB HBM3 at 700 W: 89.3 grown against 88.9 from
# scratch (DESIGN.md section 11.6); the margin allows for run-to-run variation of the two tracked drives
MESH_MARGIN = 3.0


@pytest.fixture(scope="module")
def nl():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    sys.path.insert(0, ROOT)
    return importlib.import_module("nerfloam_b200")


def scan(nl, boxes, x, i, seed, shift=(0.0, 0.0, 0.0), turn=0.0):
    """A scan at x along the street with test_gpu_localise's weave in y and heading (index i), moved by `shift` and turned by
    `turn`; the pose without POSE_OFFSET, as loaders return it."""
    syn = nl.synthetic
    xyz = (x + shift[0], 0.05 * np.sin(0.7 * i) + shift[1], shift[2])
    pts, cos, pose = syn.make_street_scan(xyz, 0.01 * np.sin(0.5 * i) + turn, boxes=boxes, seed=seed)
    pose = pose.astype(np.float64)
    pose[:3, 3] -= syn.POSE_OFFSET
    return pts, cos, pose


def read_ply(path):
    """slam.write_ply's binary PLY -> (verts f32[V,3], faces i32[T,3])."""
    with open(path, "rb") as f:
        head = b""
        while not head.endswith(b"end_header\n"):
            head += f.readline()
        words = head.decode().split()
        nv, nf = int(words[words.index("vertex") + 1]), int(words[words.index("face") + 1])
        v = np.frombuffer(f.read(12 * nv), dtype="<f4").reshape(nv, 3)
        rec = np.frombuffer(f.read(13 * nf), dtype=[("n", "u1"), ("v", "<i4", (3,))])
    return v.copy(), rec["v"].copy()


def world_points(scans, lo, hi):
    """The scans' points at their true poses (without POSE_OFFSET), those with lo <= x <= hi."""
    out = []
    for pts, _, pose in scans:
        w = pts.astype(np.float64) @ pose[:3, :3].T + pose[:3, 3]
        out.append(w[(w[:, 0] >= lo) & (w[:, 0] <= hi)])
    return np.concatenate(out).astype(np.float32)


def hit_fractions(nl, saved, scans):
    """Localiser.score (deterministic score_poses on evenly spread rays) of each scan at its true pose in `saved`."""
    loc = nl.localise.Localiser(saved, MemoryStream(scans, False))
    out = []
    for i, (pts, cos, pose) in enumerate(scans):
        T = torch.as_tensor(pose.copy())
        T[:3, 3] += nl.frame.POSE_OFFSET
        f = nl.frame.LidarFrame(i, torch.from_numpy(pts), torch.from_numpy(cos), nl.se3pose.OptimizablePose.from_matrix(T.float()),
                                new_keyframe=True)
        out.append(loc.score(f)[1])
    return np.asarray(out)


@pytest.fixture(scope="module")
def run(nl, tmp_path_factory):
    tmp = tmp_path_factory.mktemp("extend")
    boxes = nl.synthetic.street_boxes(length=180.0)
    a = [scan(nl, boxes, SPACING_A * i, i, seed=2000 + i) for i in range(N_A)]
    sa = nl.slam.NeRFLOAM(config(), str(tmp / "A"), data_stream=MemoryStream(a, True))
    sa.run()
    torch.cuda.synchronize()
    path_a = tmp / "A.map"
    sa.save_map(path_a)
    b = [scan(nl, boxes, SPACING_B * i, i, seed=5000 + i, shift=SHIFT, turn=TURN) for i in range(N_B)]
    loaded = nl.slam.load_map(path_a)
    V0, n0 = int(loaded.map.n_rows), int(loaded.map.n_nodes)
    before = {"emb": _bytes(loaded.map.embeddings).clone(), "decoder": _bytes(share._flat_decoder_state(loaded.decoder)).clone(),
              "centres": _bytes(loaded.map._centres[:n0]).clone(), "vox2row": _bytes(loaded.map._vox2row[:n0]).clone()}
    cfg = config()
    cfg["data_specs"]["use_gt"] = False
    sb = nl.slam.NeRFLOAM(cfg, str(tmp / "B"), data_stream=MemoryStream(b, False), base_map=loaded)
    summary = sb.run()
    torch.cuda.synchronize()
    print("B summary:", json.dumps(summary))
    path_ab = tmp / "AB.map"
    sb.save_map(path_ab)
    scratch = nl.slam.NeRFLOAM(cfg, str(tmp / "scratch"), data_stream=FirstPose(b, False))
    scratch.run()
    torch.cuda.synchronize()
    return SimpleNamespace(boxes=boxes, a=a, b=b, slam_a=sa, slam_b=sb, path_a=path_a, path_ab=path_ab, tmp=tmp, V0=V0, n0=n0,
                           before=before, loaded=loaded, summary=summary)


class FirstPose(MemoryStream):
    """Scans without poses, but the first one's true pose as get_init_pose (the from-scratch control's starting point)."""

    def get_init_pose(self, i):
        return self.scans[i][2].copy()


def estimated(tmp, name):
    """frame_poses.txt of a run as f64[S,4,4] (without POSE_OFFSET)."""
    poses = np.loadtxt(tmp / name / "misc" / "frame_poses.txt", ndmin=2).reshape(-1, 3, 4)
    P = np.tile(np.eye(4), (poses.shape[0], 1, 1))
    P[:, :3, :] = poses
    return P


def points_at(scans, poses, lo, hi):
    """world_points with the scans placed at `poses` instead of their true ones."""
    return world_points([(s[0], s[1], p) for s, p in zip(scans, poses)], lo, hi)


def test_b_reaches_new_ground(nl, run):
    """B's scans past NEW_X, at their true poses, hit map A with fewer than 5 % of their rays: B really maps ground A never saw."""
    new = [s for i, s in enumerate(run.b) if SPACING_B * i >= NEW_X]
    hits = hit_fractions(nl, nl.slam.load_map(run.path_a), new)
    print("hit fraction in map A, new-ground scans:", np.round(hits, 4).tolist())
    assert len(new) >= 25 and float(hits.max()) < NEW_HIT


def test_b_poses_within_the_loop_bounds(nl, run):
    """Every B pose within MAX_DR of the truth, within MAX_DT up to INSIDE_X (the placed first scan included), and past it within
    MAX_DT + DRIFT per metre driven beyond INSIDE_X; frame_poses.txt holds them.  The same drive mapped from scratch drifts too: B's
    worst error grown into A is at most SCRATCH_RATIO x the from-scratch run's.  As a contrast, Localiser on map A alone scores B's
    last ten scans below its lost_hit_fraction."""
    P = estimated(run.tmp, "B")
    assert P.shape[0] == N_B
    dt, dr = errors(P, np.stack([s[2] for s in run.b]))
    st, sr = errors(estimated(run.tmp, "scratch"), np.stack([s[2] for s in run.b]))
    print("from scratch: translation error max", float(st.max()), "rotation error max", float(sr.max()))
    print("B translation error (m): max", float(dt.max()), "per scan", np.round(dt.numpy(), 4).tolist())
    print("B rotation error: max", float(dr.max()))
    x = SPACING_B * np.arange(N_B)
    inside = torch.from_numpy(x <= INSIDE_X)
    assert float(dt[inside].max()) < MAX_DT and float(dr.max()) < MAX_DR
    assert bool((dt[~inside] <= torch.from_numpy(MAX_DT + DRIFT * (x[~inside] - INSIDE_X))).all())
    assert float(dt.max()) <= SCRATCH_RATIO * float(st.max())
    assert run.summary["base"]["frozen_rows"] == run.V0 and run.summary["base"]["place_ms"]["search"] > 0
    first = [i for i in range(N_B) if SPACING_B * i >= NEW_X][0]
    loc = nl.localise.Localiser(str(run.path_a), MemoryStream(run.b, False), generator=torch.Generator().manual_seed(3))
    res = loc.run()
    lost = nl.localise.RECOVERY_SPECS["lost_hit_fraction"]
    print("Localiser on A alone, hit fraction of the new-ground scans:", np.round(res.hit_fraction[first:].numpy(), 3).tolist())
    assert float(res.hit_fraction[-10:].max()) < lost


def test_saved_rows_decoder_and_voxels_stay_frozen(nl, run):
    mu = run.slam_b.mapper.map
    assert mu is run.loaded.map and run.slam_b.mapper.decoder is run.loaded.decoder
    assert mu.n_rows > run.V0 and mu.n_nodes > run.n0
    torch.cuda.synchronize()
    assert torch.equal(_bytes(mu.embeddings[:run.V0]), run.before["emb"])
    assert torch.equal(_bytes(share._flat_decoder_state(run.loaded.decoder)), run.before["decoder"])
    # the saved leaf voxels (the nodes with embedding rows, which the sampler reads): centres and vox2row rows byte-identical
    v2r0 = run.before["vox2row"].view(torch.int32).reshape(run.n0, 8)
    leaf = (v2r0 >= 0).any(dim=1)
    c0 = run.before["centres"].view(torch.float32).reshape(run.n0, 3)
    same_c = (mu._centres[:run.n0].view(torch.int32) == c0.view(torch.int32)).all(dim=1)
    print(f"saved nodes {run.n0}, leaves {int(leaf.sum())}, centres changed: leaves {int((leaf & ~same_c).sum())}, "
          f"others {int((~leaf & ~same_c).sum())}")
    assert bool(same_c[leaf].all())
    # the others are corner (FEATURE) nodes, exported with a zero centre until a voxel inserted at their code makes them SURFACE
    assert bool((c0[~same_c] == 0).all())
    assert torch.equal(mu._vox2row[:run.n0][leaf], v2r0[leaf])
    print(f"rows {run.V0} -> {mu.n_rows}, nodes {run.n0} -> {mu.n_nodes}")


def test_grown_file_round_trips(nl, run):
    mu = run.slam_b.mapper.map
    want = _buffers(mu.map_states["_mapstate"], run.slam_b.mapper.decoder)
    saved_a = nl.slam.load_map(run.path_a)
    for octree in ("host", "device"):
        saved = nl.slam.load_map(run.path_ab, octree=octree)
        _same(_buffers(saved.map.map_states["_mapstate"], saved.decoder), want)
        assert saved.scan_ids.tolist() == list(range(N_A)) + list(range(N_B))
        assert torch.equal(saved.trajectory[:N_A], saved_a.trajectory)
        fp = np.loadtxt(run.tmp / "B" / "misc" / "frame_poses.txt", ndmin=2).reshape(-1, 3, 4)
        assert np.abs(saved.trajectory[N_A:, :3, :].numpy() - fp).max() < 1e-5


def test_third_drive_localised_from_saved_into_new_ground(nl, run):
    """Drive C (other scan noise, shifted 0.36 m and turned -6 degrees) from x = 30 m on the saved ground to 69 m on the new ground,
    localised by Localiser in the grown file with no pose guess.  On the new ground the map frame is where B put it, so C's poses are
    held to the truth carried into B's frame: E_k T_c, with E_k = P_k T_k^-1 the estimated-over-true pose of B's scan nearest in x."""
    c = [scan(nl, run.boxes, float(x), x, seed=9000 + x, shift=(0.2, -0.3, 0.0), turn=-np.radians(6.0)) for x in range(*C_X)]
    P, T = estimated(run.tmp, "B"), np.stack([s[2] for s in run.b])
    xb = SPACING_B * np.arange(N_B) + SHIFT[0]
    want = []
    for pts, _, Tc in c:
        k = int(np.abs(xb - Tc[0, 3]).argmin())
        want.append(P[k] @ np.linalg.inv(T[k]) @ Tc)
    loc = nl.localise.Localiser(str(run.path_ab), MemoryStream(c, False), generator=torch.Generator().manual_seed(5))
    res = loc.run()
    dt, dr = errors(res.poses, np.stack(want))
    tt, _ = errors(res.poses, np.stack([s[2] for s in c]))
    print("C against B's frame: translation", np.round(dt.numpy(), 4).tolist(), "rotation max", float(dr.max()))
    print("C against the truth: translation max", float(tt.max()), "hit", np.round(res.hit_fraction.numpy(), 3).tolist())
    assert float(dt.max()) < MAX_DT and float(dr.max()) < MAX_DR
    assert float(res.hit_fraction.min()) > 0.5


def test_grown_mesh_on_new_ground_matches_a_from_scratch_map(nl, run):
    """F-score at 0.1 m of the grown map's final_mesh.ply on B's new segment (the saved decoder, frozen) no worse than MESH_MARGIN
    below the from-scratch map's (a decoder trained on B), each scored against B's points at that run's own estimated poses, so
    pose drift does not count against either.  Map A's mesh on A's segment is printed beside them."""
    ev = nl.evaluate
    idx = [i for i in range(N_B) if SPACING_B * i >= NEW_X]
    new = [run.b[i] for i in idx]
    lo, hi = NEW_X - 5.0, SPACING_B * (N_B - 1) + 5.0
    score = {}
    for name in ("B", "scratch"):
        g = points_at(new, estimated(run.tmp, name)[idx], lo, hi)
        v, f = read_ply(run.tmp / name / "mesh" / "final_mesh.ply")
        score[name] = ev.eval_mesh(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(g).cuda())
    score["B_true_poses"] = ev.eval_mesh(*(torch.from_numpy(t).cuda() for t in read_ply(run.tmp / "B" / "mesh" / "final_mesh.ply")),
                                         torch.from_numpy(world_points(new, lo, hi)).cuda())
    xa = [SPACING_A * i for i in range(N_A)]
    va, fa = read_ply(run.tmp / "A" / "mesh" / "final_mesh.ply")
    score["A"] = ev.eval_mesh(torch.from_numpy(va).cuda(), torch.from_numpy(fa).cuda(),
                              torch.from_numpy(world_points(run.a, xa[0] - 5.0, xa[-1] + 5.0)).cuda())
    for k, m in score.items():
        print(f"mesh {k}:", json.dumps(m))
    assert score["B"]["fscore"] >= score["scratch"]["fscore"] - MESH_MARGIN


def test_global_placement_on_new_ground_diagnostic(nl, run):
    """Where the search with no pose guess puts a scan taken on the new ground, and the score (loss, hit fraction) of that placement
    against the score at the scan's pose in B's frame.  Reported, not asserted (DESIGN.md section 11.6)."""
    x = 60
    c = [scan(nl, run.boxes, float(x), x, seed=9000 + x, shift=(0.2, -0.3, 0.0), turn=-np.radians(6.0))]
    P, T = estimated(run.tmp, "B"), np.stack([s[2] for s in run.b])
    k = int(np.abs(SPACING_B * np.arange(N_B) + SHIFT[0] - c[0][2][0, 3]).argmin())
    want = P[k] @ np.linalg.inv(T[k]) @ c[0][2]
    loc = nl.localise.Localiser(str(run.path_ab), MemoryStream(c, False), generator=torch.Generator().manual_seed(5))
    try:
        res = loc.run()
    except nl._capi.NerfLoamError as e:
        print("no placement:", e)
        return
    dt, dr = errors(res.poses, want[None])
    Tw = torch.as_tensor(want.copy())
    Tw[:3, 3] += nl.frame.POSE_OFFSET
    f = nl.frame.LidarFrame(0, torch.from_numpy(c[0][0]), torch.from_numpy(c[0][1]), nl.se3pose.OptimizablePose.from_matrix(Tw.float()),
                            new_keyframe=True)
    print(f"placement {float(dt[0]):.3f} m / {float(dr[0]):.3f} from B's frame at x = {res.poses[0, 0, 3]:.2f}; score there "
          f"(loss, hit) = ({float(res.loss[0]):.5f}, {float(res.hit_fraction[0]):.3f}); at the pose in B's frame {loc.score(f)}; "
          f"search candidates {res.placement.diagnostics.n_placements}")


def test_refine_floor_holds_saved_rows(nl, run):
    """refine_map with frozen_rows = V0 leaves rows below V0 byte-identical while rows above move; frozen_rows = 0 gives the row
    list and the table of a call without the argument, bit for bit (deterministic sampling, so only the scatter's atomics could
    differ: the table is held to a tolerance, the kernel's own output to the bit in test_mark_rows_floor_zero_is_mark_rows)."""
    rh = nl.render_helpers
    m = run.slam_b.mapper
    kg = m.kg
    V0 = run.V0
    kw = dict(N_rays=1024, num_iterations=5, truncation=m.sdf_truncation, max_voxel_hit=m.max_voxel_hit, max_distance=m.max_distance,
              learning_rate=0.01, passes=3, deterministic=True)
    emb = m.map.embeddings
    keep = emb.clone()

    def call(**extra):
        emb.copy_(keep)
        rh.refine_map(kg, emb, m.map_state, m.decoder, m.loss_criteria, m.voxel_size, m.step_size, generator=torch.Generator().manual_seed(11),
                      **kw, **extra)
        torch.cuda.synchronize()
        g = rh._RefineGraph._cache["g"]
        listed = int(g.state[nl._capi.REFINE_PREV])
        return emb.clone(), sorted(g.rows[:listed].tolist())

    e_floor, rows_floor = call(frozen_rows=V0)
    assert torch.equal(_bytes(e_floor[:V0]), _bytes(keep[:V0]))
    assert not torch.equal(e_floor[V0:], keep[V0:]) and min(rows_floor) >= V0
    e_plain, rows_plain = call()
    e_zero, rows_zero = call(frozen_rows=0)
    assert rows_zero == rows_plain and min(rows_plain) < V0
    diff = float((e_zero.float() - e_plain.float()).abs().max())
    print("rows listed in the last pass:", len(rows_plain), "with the floor:", len(rows_floor), "table max |zero - plain|:", diff)
    assert torch.allclose(e_zero.float(), e_plain.float(), rtol=1e-2, atol=1e-4)
    emb.copy_(keep)


def test_mark_rows_floor_zero_is_mark_rows(nl):
    """nl_mark_rows_floor with floor 0 gives nl_mark_rows' flag bits and count, and the same rows; with a floor, exactly the rows at
    or above it."""
    lib, cap = nl._capi.lib(), nl._capi
    g = torch.Generator().manual_seed(0)
    n_rows, n_vox, M = 5000, 3000, 20000
    vox2row = torch.randint(-1, n_rows, (n_vox, 8), generator=g, dtype=torch.int32).cuda()
    vox = torch.randint(0, n_vox, (M,), generator=g, dtype=torch.int32).cuda()

    def mark(floor):
        bits = torch.zeros((n_rows + 31) // 32, dtype=torch.int32, device="cuda")
        rows = torch.full((n_rows,), -7, dtype=torch.int32, device="cuda")
        state = torch.zeros(cap.REFINE_STATE_WORDS, dtype=torch.int32, device="cuda")
        args = (M, None, cap.ptr(vox), cap.ptr(vox2row), n_rows)
        tail = (cap.ptr(bits), cap.ptr(rows), cap.ptr(state), cap.stream_ptr())
        cap.check(lib.nl_mark_rows(*args, *tail) if floor is None else lib.nl_mark_rows_floor(*args, floor, *tail), "mark")
        torch.cuda.synchronize()
        n = int(state[cap.REFINE_LISTED])
        return bits.cpu(), n, sorted(rows[:n].tolist()), state.cpu()

    want = sorted(set(v for v in vox2row[vox.long()].reshape(-1).tolist() if v >= 0))
    b0, n0, r0, s0 = mark(None)
    b1, n1, r1, s1 = mark(0)
    assert r0 == want and torch.equal(b0, b1) and n0 == n1 and r0 == r1 and torch.equal(s0, s1)
    b2, n2, r2, _ = mark(2500)
    assert r2 == [v for v in want if v >= 2500] and n2 == len(r2)
    assert lib.nl_mark_rows_floor(M, None, cap.ptr(vox), cap.ptr(vox2row), n_rows, n_rows + 1, cap.ptr(vox), cap.ptr(vox), cap.ptr(vox),
                                  None) != 0


def test_drive_outside_the_map_raises_and_writes_no_map(nl, run, tmp_path):
    """A drive whose returns all lie 20-30 m away at 70-85 degrees of elevation (test_gpu_localise's unexplainable scan): no
    placement near the saved trajectory reaches the map, so run() raises and writes no file."""
    rng = np.random.default_rng(0)
    n = 6000
    el, az, r = np.deg2rad(rng.uniform(70, 85, n)), rng.uniform(-np.pi, np.pi, n), rng.uniform(20, 30, n)
    pts = (np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1) * r[:, None]).astype(np.float32)
    far = [(pts, np.ones(n, np.float32), np.eye(4))] * 3
    cfg = config()
    cfg["data_specs"]["use_gt"] = False
    s = nl.slam.NeRFLOAM(cfg, str(tmp_path / "far"), data_stream=MemoryStream(far, False), base_map=str(run.path_a))
    with pytest.raises(nl._capi.NerfLoamError, match="could not be placed"):
        s.run()
    assert [f for _, _, fs in os.walk(tmp_path) for f in fs] == []


def test_run_slam_script_with_base_map(nl, run):
    seq = run.tmp / "seq"
    os.makedirs(seq / "velodyne", exist_ok=True)
    for i, (pts, _, _) in enumerate(run.b[:8]):
        np.concatenate([pts, np.zeros((pts.shape[0], 1), np.float32)], 1).astype(np.float32).tofile(str(seq / "velodyne" / f"{i:06d}.bin"))
    cfg = config()
    cfg["data_specs"].update(use_gt=False, data_path=str(seq))
    import yaml
    with open(run.tmp / "b.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    out_map = run.tmp / "script.map"
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "run_slam.py"), str(run.tmp / "b.yaml"), "--base-map", str(run.path_a),
                          "--save-map", str(out_map), "--out", str(run.tmp / "script")], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    summary = json.loads(out.stdout.strip().splitlines()[-1])
    print(summary)
    assert summary["scans"] == 8 and summary["base"]["frozen_rows"] == run.V0 and summary["map_file"] == str(out_map)
    grown = nl.slam.load_map(out_map)
    assert grown.scan_ids.tolist() == list(range(N_A)) + list(range(8)) and grown.map.n_rows > run.V0
