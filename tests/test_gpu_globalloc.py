"""Global localisation on the GPU: the occupied set against the host tree's leaf voxels, the cell table, matrices, coarse counts and
selection against the NumPy restatement (tests/globalloc_ref.py), determinism and chunking, the argument errors, and
relocalise_global placing held-out scans of the street scene with no guess."""
import math
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import globalloc_ref as ref

pytestmark = pytest.mark.gpu

VS, MD, TRUNC = 0.3, 40.0, 0.3
SPACING = 3.0
HELD_OUT = [((4.4, 0.6, 0.0), math.pi + 0.03), ((10.7, -0.8, 0.0), 0.6), ((16.2, 0.4, 0.0), -1.9)]
TRACK = dict(step_size=0.06, truncation=0.3, max_voxel_hit=20, max_distance=40.0)
RELOC = dict(N_rays=1024, refine_iterations=150, learning_rate=0.03, **TRACK)


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


@pytest.fixture(scope="module")
def street(nl):
    """Ten street scans mapped at their true poses (MapUpdater + bundle_adjust_frames, as test_gpu_score_poses.py's slam_map)."""
    dev = torch.device("cuda")
    syn, rh = nl.synthetic, nl.render_helpers
    crit = nl.criterion.Criterion(SimpleNamespace(criteria={"eiko_weight": 0.1, "sdf_weight": 10000.0, "fs_weight": 1.0, "sdf_truncation": TRUNC},
                                                  data_specs={"max_depth": MD}))
    torch.manual_seed(777)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).to(dev)
    mu = nl.mapping.MapUpdater(VS, device=dev, reserve_nodes=600_000, reserve_rows=600_000)
    scans = [syn.make_street_scan((SPACING * i, 0.05 * np.sin(0.7 * i), 0.0), 0.01 * np.sin(0.5 * i), seed=2000 + i) for i in range(10)]
    gt = [torch.from_numpy(s[2]).float() for s in scans]
    frames = [nl.frame.LidarFrame(i, torch.from_numpy(scans[i][0]), torch.from_numpy(scans[i][1]),
                                  nl.se3pose.OptimizablePose.from_matrix(gt[i].clone()), new_keyframe=True) for i in range(10)]
    ms = None
    for i in range(10):
        ms = mu.create_voxels(scans[i][0], gt[i].double())
        for _ in range(6 if i else 12):
            rh.bundle_adjust_frames(frames[max(0, i - 3):i + 1], mu.embeddings, ms, dec, crit, VS, 0.5 * VS, N_rays=2048, num_iterations=25,
                                    truncation=TRUNC, max_voxel_hit=20, max_distance=MD, learning_rate=[0.01, 0.005, 0.001],
                                    update_pose=False, update_decoder=True)
    anchors = torch.stack(gt).double()
    return SimpleNamespace(mu=mu, ms=ms, dec=dec, crit=crit, anchors=anchors, frames=frames)


def _keys(occ):
    s = occ.slots.cpu().numpy()
    return np.sort(s[s != -1])


def test_occupied_set_equals_leaf_voxels(nl, street):
    occ = nl.globalloc.occupied_set(street.ms, VS)
    want = ref.leaf_keys(street.mu.svo.get_leaf_voxels().numpy())
    got = _keys(occ)
    assert occ.n_leaves == want.size and np.array_equal(got, want)
    assert occ.slots.numel() >= 2 * want.size and occ.slots.numel() & (occ.slots.numel() - 1) == 0
    assert nl.globalloc.occupied_set(street.ms, VS) is occ                  # built once per map


def test_cells_and_matrices_equal_restatement(nl, street):
    A12 = street.anchors[:, :3, :4].reshape(-1, 12).numpy()
    for radius, step in ((5.0, 1.0), (4.0, 0.5), (0.0, 1.0), (7.5, 0.77)):
        pl = nl.globalloc.placements(street.anchors, radius, step, 72)
        want = ref.cells(A12, radius, step)
        if want.shape[0] == 0:
            continue
        assert np.array_equal(pl.cells.cpu().numpy().astype(np.int64), want), (radius, step)
        ids = np.arange(pl.n_placements)
        T = nl.globalloc.placement_matrices(pl, ids).cpu().numpy()
        got = np.concatenate([T[:, :3, :3].reshape(-1, 9), T[:, :3, 3]], 1)
        assert np.abs(got - ref.matrices(want, A12, 72, step, ids)).max() <= 1e-6


def _snapped_points(occ, Rt0):
    """Points whose world point under matrix Rt0 (a pure translation) lies on an occupied voxel's lower faces, and one ulp either side."""
    keys = _keys(occ)[::max(1, occ.n_leaves // 40)][:40]
    corner = np.stack([(keys >> 36) & 0x3FFFF, (keys >> 18) & 0x3FFFF, keys & 0x3FFFF], 1).astype(np.float64)
    p = (corner * VS - Rt0[9:12].astype(np.float64)).astype(np.float32)
    return np.concatenate([p, np.nextafter(p, np.float32(np.inf)), np.nextafter(p, np.float32(-np.inf))])


def test_counts_and_selection_equal_restatement(nl, street):
    """At least 10^5 placements, with scan points plus points snapped onto voxel faces: exact counts, exact selection."""
    dev = torch.device("cuda")
    anchors = street.anchors.clone()
    anchors[0, :3, :3] = torch.eye(3, dtype=torch.float64)                   # placement 0 (k = 0 at anchor 0's cell) is a pure translation
    pl = nl.globalloc.placements(anchors, 5.0, 0.45, 72)
    assert pl.n_placements >= 100_000
    occ = nl.globalloc.occupied_set(street.ms, VS)
    torch.manual_seed(5)
    pts, _ = nl.globalloc.scan_points(street.frames[3], 512)
    cells = pl.cells.cpu().numpy()
    c0 = int(np.nonzero(cells[:, 2] == 0)[0][0])
    T0 = nl.globalloc.placement_matrices(pl, [c0 * 72]).cpu().numpy()[0]
    assert np.array_equal(T0[:3, :3], np.eye(3, dtype=np.float32))
    Rt0 = np.concatenate([T0[:3, :3].reshape(-1), T0[:3, 3]])
    pts = torch.cat([pts, torch.from_numpy(_snapped_points(occ, Rt0)).to(dev)]).contiguous()
    counts = nl.globalloc.coarse_scores(pl, occ, pts)
    T = nl.globalloc.placement_matrices(pl, np.arange(pl.n_placements)).cpu().numpy()
    Rt = np.concatenate([T[:, :3, :3].reshape(-1, 9), T[:, :3, 3]], 1)
    want = ref.counts(Rt, pts.cpu().numpy(), _keys(occ), VS, 1 << 18)
    got = counts.cpu().numpy()
    assert np.array_equal(got, want)
    assert got[c0 * 72] > 0
    M = pts.shape[0]
    for n in (1, 100, 4096, pl.n_placements):
        ids, sel = nl.globalloc.top_placements(counts, M, n)
        wi, wc = ref.select(want, n)
        assert np.array_equal(ids.cpu().numpy(), wi) and np.array_equal(sel.cpu().numpy(), wc), n


def test_two_calls_identical_and_chunk_independent(nl, street):
    occ = nl.globalloc.occupied_set(street.ms, VS)
    pl1 = nl.globalloc.placements(street.anchors, 5.0, 1.0, 72)
    pl2 = nl.globalloc.placements(street.anchors, 5.0, 1.0, 72)
    assert torch.equal(pl1.cells, pl2.cells)
    torch.manual_seed(9)
    pts, pid = nl.globalloc.scan_points(street.frames[5], 512)
    torch.manual_seed(9)
    pts2, pid2 = nl.globalloc.scan_points(street.frames[5], 512)
    assert torch.equal(pid, pid2) and torch.equal(pts, pts2)
    cos = street.frames[5].pointsCos[pid.cpu().long()]
    assert bool((cos == 1).all())                                          # non-ground rows only
    a = nl.globalloc.coarse_scores(pl1, occ, pts)
    b = nl.globalloc.coarse_scores(pl2, occ, pts)
    c = nl.globalloc.coarse_scores(pl1, occ, pts, chunk=997)
    assert torch.equal(a, b) and torch.equal(a, c)
    s1, s2 = nl.globalloc.top_placements(a, 512, 777), nl.globalloc.top_placements(c, 512, 777)
    assert torch.equal(s1[0], s2[0]) and torch.equal(s1[1], s2[1])


def test_bad_inputs_raise(nl, street):
    g = nl.globalloc
    frame = street.frames[0]
    kw = dict(anchors=street.anchors, radius=5.0, xy_step=1.0, yaw_steps=72)
    bad = [dict(anchors=street.anchors[:0]), dict(radius=-1.0), dict(xy_step=0.0), dict(radius=float("inf")), dict(yaw_steps=0),
           dict(n_points=0), dict(yaw_steps=2 ** 30)]
    nan = street.anchors.clone()
    nan[2, 0, 3] = float("nan")
    bad.append(dict(anchors=nan))
    for b in bad:
        with pytest.raises(ValueError):
            g.relocalise_global(frame, street.ms, street.dec, street.crit, VS, **dict(kw, **b))
    empty = nl.engine.MapState(torch.zeros((0, 3)), torch.zeros((0, 9), dtype=torch.int32), torch.zeros((0, 8), dtype=torch.int32),
                               torch.zeros((1, 16)))
    with pytest.raises(ValueError):
        g.relocalise_global(frame, empty, street.dec, street.crit, VS, **kw)
    with pytest.raises(ValueError):
        g.occupied_set(empty, VS)


def _pose_error(nl, p, T_true):
    T = nl.se3pose.OptimizablePose(p.data.detach().cpu().float().clone()).matrix().detach().double()
    dt = float((T[:3, 3] - T_true[:3, 3]).norm())
    c = float(((T[:3, :3].T @ T_true[:3, :3]).trace() - 1.0) / 2.0)
    return dt, math.degrees(math.acos(max(-1.0, min(1.0, c))))


def test_relocalise_global_places_held_out_scans(nl, street):
    """Scans between the anchors, one turned 180 degrees from the driving direction and the others at headings off the 5-degree lattice,
    localised with no guess within 0.10 m and 1 degree."""
    syn = nl.synthetic
    for n, (xyz, yaw) in enumerate(HELD_OUT):
        pts, cos, pose = syn.make_street_scan(xyz, yaw, seed=3000 + n)
        T_true = torch.from_numpy(pose).double()
        frame = nl.frame.LidarFrame(100 + n, torch.from_numpy(pts), torch.from_numpy(cos), nl.se3pose.OptimizablePose(torch.zeros(6)),
                                    new_keyframe=True)
        torch.manual_seed(11 + n)
        t0 = time.perf_counter()
        res = nl.relocalise_global(frame, street.ms, street.dec, street.crit, VS, anchors=street.anchors, **RELOC)
        wall = time.perf_counter() - t0
        dt, dr = _pose_error(nl, res.pose, T_true)
        d = res.diagnostics
        ids = d.ids.cpu().numpy()
        pl = nl.globalloc.placements(street.anchors, 5.0, 1.0, 72)
        cells = pl.cells.cpu().numpy()
        q = np.round((T_true[:2, 3].numpy()) / 1.0).astype(np.int64)
        true_cell = np.nonzero((cells[:, 0] == q[0]) & (cells[:, 1] == q[1]))[0]
        k_true = int(round((yaw % (2 * math.pi)) / (2 * math.pi / 72))) % 72
        rank_cell = np.nonzero(np.isin(ids // 72, true_cell))[0]
        rank_pl = np.nonzero(ids == (true_cell[0] * 72 + k_true if true_cell.size else -1))[0]
        print(f"scan {n} at {xyz}, yaw {math.degrees(yaw):.1f} deg: {dt:.3f} m, {dr:.2f} deg; loss {res.loss:.4g}; "
              f"{d.n_placements} placements; true cell first at coarse rank {rank_cell[:1].tolist()}, true placement at "
              f"{rank_pl[:1].tolist()}; seeds {d.seeds}; stages {', '.join(f'{k} {v * 1e3:.0f} ms' for k, v in d.times.items())}; "
              f"total {wall:.2f} s")
        assert res.hit_mask is not None and math.isfinite(res.loss)
        assert dt < 0.10 and dr < 1.0, (n, dt, dr)


def test_out_of_range_counts_and_ids_are_guarded(nl, street):
    """Counts outside [0, n_points] are never selected (the rest of the output is -1); device ids outside the lattice give NaN
    matrices and host ids raise."""
    dev = torch.device("cuda")
    g = nl.globalloc
    c = torch.tensor([5, 900, -3, 2, 7, 5, 513, 0], dtype=torch.int32, device=dev)
    ids, sel = g.top_placements(c, 512, 8)
    valid = np.array([5, -1, -1, 2, 7, 5, -1, 0])
    order = [h for h in np.lexsort((np.arange(8), -valid)) if valid[h] >= 0]
    assert ids.cpu().tolist() == order + [-1] * 3 and sel.cpu().tolist() == [int(valid[h]) for h in order] + [-1] * 3
    ids, sel = g.top_placements(c, 512, 2)
    assert ids.cpu().tolist() == [4, 0] and sel.cpu().tolist() == [7, 5]
    pl = g.placements(street.anchors, 5.0, 1.0, 72)
    T = g.placement_matrices(pl, torch.tensor([0, -1, pl.n_placements, 2 ** 40, pl.n_placements - 1], device=dev)).cpu()
    assert bool(torch.isfinite(T[[0, 4]]).all()) and bool(torch.isnan(T[1:4, :3, :]).all())
    for bad in ([-1], [pl.n_placements], [2 ** 40]):
        with pytest.raises(ValueError):
            g.placement_matrices(pl, bad)
