"""Change detection on the GPU (changes.ChangeDetector, localise.Localiser's "change_specs"; DESIGN.md §11.7).

A street map A is built as test_gpu_localise.py builds it (synthetic.street_boxes, true poses) and saved.  Drive B goes over the
same street with two kerbside boxes and one building taken out of the box list and two new boxes put in, shifted 0.5 m and turned 10
degrees, and is localised in A's file with no pose guess.  Checked: the kernels' integers against change_ref.py on the engine's own
sample arrays (several scans, chunk boundaries, forced capacity redos of the sample list and the added table, the file restored onto
both octrees); the flagged voxels against the boxes that changed; drive B over the unchanged street as a control; the option's
off switch; scripts/localise.py --changes."""
import json
import math
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import change_ref as ref
from test_gpu_localise import N_MAP, ROOT, SHIFT, SPACING, TURN, MemoryStream, _buffers, _same, config, errors

pytestmark = pytest.mark.gpu
N_B = 8
NEAR = 1.0 + math.sqrt(3.0) / 2.0        # a voxel "near" a box face: its centre within one voxel plus half a diagonal of the face


@pytest.fixture(scope="module")
def nl():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    sys.path.insert(0, ROOT)
    import nerfloam_b200
    return nerfloam_b200


def scan(nl, i, seed, boxes, shift=(0.0, 0.0, 0.0), turn=0.0):
    """test_gpu_localise.street over an explicit box list."""
    syn = nl.synthetic
    xyz = (SPACING * i + shift[0], 0.05 * np.sin(0.7 * i) + shift[1], shift[2])
    pts, cos, pose = syn.make_street_scan(xyz, 0.01 * np.sin(0.5 * i) + turn, boxes=boxes, seed=seed)
    pose = pose.astype(np.float64)
    pose[:3, 3] -= syn.POSE_OFFSET
    return pts, cos, pose


def scene(nl):
    """(A's boxes, B's boxes, removed boxes, new boxes)."""
    boxes = nl.synthetic.street_boxes()
    mid = SPACING * (N_MAP - 1) / 2
    inner = np.minimum(np.abs(boxes[:, 1]), np.abs(boxes[:, 4]))
    dist = np.abs((boxes[:, 0] + boxes[:, 3]) / 2 - mid)
    kerb = [int(i) for i in np.argsort(dist) if inner[i] < 5.5][:2]
    building = [int(i) for i in np.argsort(dist) if inner[i] >= 5.5][:1]
    gone = kerb + building
    new = np.array([[mid - 1.0, 3.6, -1.73, mid + 0.2, 4.4, -0.2], [mid + 2.5, -4.6, -1.73, mid + 3.5, -3.7, -0.5]])
    keep = np.array([i not in gone for i in range(len(boxes))])
    return boxes, np.concatenate([boxes[keep], new]), boxes[gone], new


def face_distance(p, box):
    """Distance of points p [n,3] to the surface of an axis-aligned box (min xyz, max xyz)."""
    lo, hi = box[:3], box[3:]
    out = np.linalg.norm(np.maximum(np.maximum(lo - p, p - hi), 0.0), axis=1)
    inside = np.min(np.minimum(p - lo, hi - p), axis=1)
    return np.where(out > 0, out, np.abs(inside))


@pytest.fixture(scope="module")
def run(nl, tmp_path_factory):
    tmp = tmp_path_factory.mktemp("changes")
    a_boxes, b_boxes, gone, new = scene(nl)
    scans = [scan(nl, i, 2000 + i, a_boxes) for i in range(N_MAP)]
    s = nl.slam.NeRFLOAM(config(), str(tmp / "run"), data_stream=MemoryStream(scans, True))
    s.run()
    torch.cuda.synchronize()
    path = tmp / "run.map"
    s.save_map(path)
    b = [scan(nl, i, 5000 + i, b_boxes, SHIFT, TURN) for i in range(N_B)]
    same = [scan(nl, i, 5000 + i, a_boxes, SHIFT, TURN) for i in range(N_B)]
    return SimpleNamespace(path=path, tmp=tmp, b=b, same=same, gone=gone, new=new, a_boxes=a_boxes, b_boxes=b_boxes)


def _detector(nl, saved, **kw):
    cfg = saved.config
    vs = float(cfg["voxel_size"])
    tk = {"step_size": cfg["tracker_specs"]["step_size"] * vs, "max_distance": cfg["data_specs"]["max_depth"]}
    return nl.changes.ChangeDetector(saved.map.map_states["_mapstate"], saved.decoder, vs, cfg["criteria"], tk, {}, **kw)


def _frame(nl, pts, cos, pose):
    T = torch.as_tensor(pose, dtype=torch.float64).clone()
    T[:3, 3] += nl.frame.POSE_OFFSET
    return nl.frame.LidarFrame(0, torch.from_numpy(pts), torch.from_numpy(cos), nl.se3pose.OptimizablePose.from_matrix(T.float()),
                               new_keyframe=True)


def _spy(det):
    """Records, per render call whose sample list fit, the arrays nl_change_votes read, and per added call the posed points."""
    calls, added = [], []
    votes, add = det._votes, det._added

    def v(m, bufs, dirs, gt, r0, R, status):
        votes(m, bufs, dirs, gt, r0, R, status)
        st = det.eng.read_stats()
        if not st.error & 6:
            e, M = det.eng, st.n_samples
            calls.append(tuple(t[:M].cpu().numpy() for t in (e.s_ray, e.s_vox, e.s_depth, e.sdf)) + (gt[r0:r0 + R].cpu().numpy(),))

    def a(pts, scan_id):
        add(pts, scan_id)
        added.append((scan_id, pts.cpu().numpy(), det.Rt12.cpu().numpy()))
    det._votes, det._added = v, a
    return calls, added


def _check_exact(nl, det, calls, added):
    m = det.m
    n = m.n_nodes
    want = np.zeros((n, 2), np.int64)
    for s_ray, s_vox, s_depth, sdf, gt in calls:
        want += ref.votes(s_ray, s_vox, s_depth, sdf, gt, n, det.truncation, det.through)
    got = det.votes.cpu().numpy().astype(np.int64) & 0xffffffff
    assert np.array_equal(got, want), int(np.abs(got - want).sum())
    occ = ref.leaf_keys(m.centres.cpu().numpy(), m.structure.cpu().numpy(), det.vs)
    last = {}
    for scan_id, pts, Rt in added:                          # a redone insert replaces the overflowed one (which inserted nothing)
        last[scan_id] = (pts, Rt)
    table = ref.added([last[k] for k in sorted(last)], occ, det.vs)
    keys = det.keys.cpu().numpy().view(np.uint64)
    vals = det.vals.cpu().numpy().view(np.uint32)
    used = keys != np.uint64(ref.EMPTY)
    got_table = {int(k): [int(v[0]), int(v[1])] for k, v in zip(keys[used], vals[used])}
    assert got_table == table
    ch = det.result()
    sp = det.specs
    ids, conf, rem, unobs = ref.classify(want, m.structure.cpu().numpy(), sp["min_votes"], sp["ratio"])
    assert ch.removed_ids.tolist() == ids.tolist() and (ch.n_confirmed, ch.n_removed, ch.n_unobserved) == (conf, rem, unobs)
    assert np.array_equal(ch.through, want[ids, 0]) and np.array_equal(ch.surface, want[ids, 1])
    k, p, s = ref.select_added(table, sp["min_points"], sp["min_scans"])
    vs = det.vs
    cen = (np.stack([(k >> np.uint64(36)) & np.uint64(0x3ffff), (k >> np.uint64(18)) & np.uint64(0x3ffff), k & np.uint64(0x3ffff)], -1)
           .astype(np.float64) + 0.5) * vs - nl.frame.POSE_OFFSET
    assert np.array_equal(ch.added_points, p) and np.array_equal(ch.added_scans, s) and np.array_equal(ch.added_centres, cen.reshape(-1, 3))
    return want, table, ch


def test_exact_against_restatement(nl, run):
    """Three scans of B at their true poses: small chunks (a chunk boundary inside every scan), a sample list too small for any chunk
    and a 1024-slot added table, so both redo; then the default sizes.  Both equal the restatement on their own sample arrays."""
    saved = nl.slam.load_map(str(run.path))
    frames = [_frame(nl, *run.b[i]) for i in (0, 3, 7)]
    small = _detector(nl, saved, chunk_rays=20000, samples_per_ray=2, added_slots=1024)
    calls, added = _spy(small)
    for f in frames:
        small.add_scan(f, f.pose)
    print("redos:", small.redos, "render calls:", len(calls))
    assert small.redos["samples"] >= 1 and small.redos["added"] >= 1 and len(calls) >= 2 * len(frames)
    want, table, ch = _check_exact(nl, small, calls, added)
    assert want[:, 0].sum() > 0 and want[:, 1].sum() > 0 and len(table) > 0
    big = _detector(nl, saved)
    c2, a2 = _spy(big)
    for f in frames:
        big.add_scan(f, f.pose)
    assert big.redos == {"samples": 0, "added": 0}
    want2, table2, _ = _check_exact(nl, big, c2, a2)
    # the sampler's strata depend on the rays rendered together (render_rays' batch quirks), so the votes depend on chunk_rays, while
    # the added table does not
    print("votes differing between chunk sizes:", int(np.abs(want - want2).sum()), "of", int(want.sum()))
    assert table == table2


@pytest.mark.parametrize("octree", ["host", "device"])
def test_exact_on_restored_map(nl, run, octree):
    saved = nl.slam.load_map(str(run.path), octree=octree)
    det = _detector(nl, saved)
    calls, added = _spy(det)
    for i in (1, 5):
        f = _frame(nl, *run.b[i])
        det.add_scan(f, f.pose)
    want, _, _ = _check_exact(nl, det, calls, added)
    host = _detector(nl, nl.slam.load_map(str(run.path), octree="host"))
    for i in (1, 5):
        f = _frame(nl, *run.b[i])
        host.add_scan(f, f.pose)
    assert np.array_equal(host.votes.cpu().numpy(), det.votes.cpu().numpy())


def _localise(nl, run, drive, config, seed=1, out=None):
    gen = torch.Generator().manual_seed(seed)
    loc = nl.localise.Localiser(str(run.path), MemoryStream(drive, False), config=config, generator=gen, out_dir=out)
    res = loc.run()
    return loc, res, gen.get_state()


@pytest.fixture(scope="module")
def located(nl, run):
    out = {}
    out["b"] = _localise(nl, run, run.b, {"change_specs": {}, "recovery_specs": {}}, out=str(run.tmp / "b"))
    out["same"] = _localise(nl, run, run.same, {"change_specs": {}, "recovery_specs": {}})
    return out


def test_scenario(nl, run, located):
    loc, res, _ = located["b"]
    ch = res.changes
    truth = np.stack([p[2] for p in run.b])
    dt, dr = errors(res.poses, truth)
    assert float(dt.max()) < 0.10 and float(dr.max()) < 0.01 and all(s != "lost" for s in res.status)
    vs = loc.tracker.voxel_size
    m = loc.map_state
    leaves = m.centres[m.structure[:, 8] == 1].double().cpu().numpy() - nl.frame.POSE_OFFSET
    path_xy = truth[:, :2, 3]
    near_rm = np.stack([face_distance(ch.removed_centres, b) <= NEAR * vs for b in run.gone]) if len(ch.removed_centres) else \
        np.zeros((len(run.gone), 0), bool)
    near_add = np.stack([face_distance(ch.added_centres, b) <= NEAR * vs for b in run.new]) if len(ch.added_centres) else \
        np.zeros((len(run.new), 0), bool)
    prec_rm = float(near_rm.any(0).mean()) if near_rm.shape[1] else float("nan")
    prec_add = float(near_add.any(0).mean()) if near_add.shape[1] else float("nan")
    summary = loc.summary(res)
    print("changes:", json.dumps(summary["changes"]))
    print("removed: per box", near_rm.sum(1).tolist(), "precision", prec_rm, " added: per box", near_add.sum(1).tolist(), "precision", prec_add)
    for b, hits in zip(run.gone, near_rm):
        # a removed box B's rays reach: A's map held its faces, and B's path passes within 15 m of it
        held = int((face_distance(leaves, b) <= NEAR * vs).sum())
        reach = float(np.min(np.linalg.norm(path_xy - np.clip(path_xy, b[:2], b[3:5]), axis=1)))
        print("removed box", np.round(b, 2).tolist(), "saved leaves at its faces", held, "path distance", round(reach, 2), "flagged", int(hits.sum()))
        if held >= 10 and reach < 15.0:
            assert hits.sum() > 0
    for b, hits in zip(run.new, near_add):
        assert hits.sum() > 0, b
    # surfaces B sees and A never did (behind the removed boxes, at the edge of A's coverage) are added too: DESIGN.md §11.7 gives
    # the measured share of added voxels at the new boxes (0.10), which is reported here, not held to the removed side's 0.9
    faces = np.stack([face_distance(ch.added_centres, b) <= NEAR * vs for b in run.b_boxes]).any(0) if len(ch.added_centres) else []
    ground = np.abs(ch.added_centres[:, 2] + 1.73) <= NEAR * vs if len(ch.added_centres) else []
    print("added voxels at any face of B's boxes:", float(np.mean(faces)), " on the ground:", float(np.mean(ground)))
    assert prec_rm >= 0.9 and prec_add > 0.0
    for name in ("changes_removed.ply", "changes_added.ply", "changes.txt"):
        assert (run.tmp / "b" / name).exists()


def test_control(nl, run, located):
    loc, res, _ = located["same"]
    ch = res.changes
    m = loc.map_state
    n_leaves = int((m.structure[:, 8] == 1).sum())
    observed = n_leaves - ch.n_unobserved
    frac = ch.n_removed / max(observed, 1)
    print("control: removed", ch.n_removed, "of", observed, "observed voxels:", frac, " added", len(ch.added_centres))
    # measured 0.091 % (DESIGN.md §11.7); the bound leaves room for the last-bit spread of tracked poses (fp32 pose atomics)
    assert observed > 0 and frac < 2e-3


def test_off_switch(nl, run, located):
    """The same drive with change_specs off, twice: the same generator state and statuses as with it on, poses within 1 cm and 1e-3
    (bit-identical whenever the two runs without it are), the map's device buffers untouched by a run with it on."""
    saved = nl.slam.load_map(str(run.path))
    before = {k: v.clone() for k, v in _buffers(saved.map.map_states["_mapstate"], saved.decoder).items()}
    gen = torch.Generator().manual_seed(1)
    loc = nl.localise.Localiser(saved, MemoryStream(run.b, False), config={"change_specs": {}, "recovery_specs": {}}, generator=gen)
    on = loc.run()
    on_state = gen.get_state()
    _same(_buffers(saved.map.map_states["_mapstate"], saved.decoder), before)
    _, off, off_state = _localise(nl, run, run.b, {"recovery_specs": {}})
    _, again, _ = _localise(nl, run, run.b, {"recovery_specs": {}})
    assert torch.equal(on_state, off_state) and on.status == off.status and off.changes is None
    bits = {f: torch.equal(getattr(on, f), getattr(off, f)) for f in ("poses", "loss", "hit_fraction")}
    bits_again = {f: torch.equal(getattr(again, f), getattr(off, f)) for f in ("poses", "loss", "hit_fraction")}
    print("bit-identical, on vs off:", bits, " off vs off:", bits_again)
    if all(bits_again.values()):
        assert all(bits.values())
    dt, dr = errors(on.poses, off.poses)
    assert float(dt.max()) < 0.01 and float(dr.max()) < 1e-3


def test_localise_script_changes(nl, run):
    seq = run.tmp / "seq"
    os.makedirs(seq / "velodyne", exist_ok=True)
    for i, (pts, _, _) in enumerate(run.b[:5]):
        np.concatenate([pts, np.zeros((pts.shape[0], 1), np.float32)], 1).astype(np.float32).tofile(str(seq / "velodyne" / f"{i:06d}.bin"))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "localise.py"), str(run.path), "--data", str(seq), "--out",
                          str(run.tmp / "script"), "--changes"], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    summary = json.loads(out.stdout.strip().splitlines()[-1])
    print(summary)
    assert summary["changes"]["scans"] == 5
    for name in ("changes_removed.ply", "changes_added.ply", "changes.txt"):
        assert (run.tmp / "script" / name).exists()
    bad = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "localise.py"), str(run.path), "--data", str(seq),
                          "--change-specs", '{"ratio": 2}'], capture_output=True, text=True, timeout=900)
    assert bad.returncode != 0 and "ratio" in bad.stderr
