"""Change detection without a GPU: the NumPy restatement (change_ref.py) on hand-built sample lists, the added count with min_scans,
change_specs validation, the PLY and text writers, and the Localiser's wiring with tracking, scoring and the detector stubbed."""
import importlib
import json

import numpy as np
import pytest
import torch

import change_ref as ref
from test_localise_cpu import _saved, _Stream
from test_localise_recovery_cpu import TRUTH, WANT, _Drive

changes = importlib.import_module("nerf-loam_b200.changes")
localise = importlib.import_module("nerf-loam_b200.localise")

T, THROUGH = 0.3, 0.6                 # truncation; truncation + one 0.3 m voxel of margin


def _votes(rows, gt, n_nodes=4):
    """rows: (ray, voxel, depth, sdf) per sample in list order."""
    r, v, d, s = (np.array(c) for c in zip(*rows))
    return ref.votes(r, v, np.float32(d), np.float32(s), np.float32(gt), n_nodes, T, THROUGH)


# -- the run rule ---------------------------------------------------------------------------------------------------------------
def test_run_in_front_that_crosses_zero_is_through():
    got = _votes([(0, 1, 5.0, 0.4), (0, 1, 5.2, -0.1), (0, 1, 5.4, -0.3)], [10.0])
    assert got[1].tolist() == [1, 0] and got.sum() == 1


def test_run_in_front_with_positive_sdf_gives_nothing():
    assert _votes([(0, 1, 5.0, 0.4), (0, 1, 5.2, 0.1), (0, 1, 5.4, 0.05)], [10.0]).sum() == 0


def test_run_that_straddles_the_return_is_surface():
    got = _votes([(0, 2, 9.6, 0.2), (0, 2, 9.9, 0.0), (0, 2, 10.2, -0.2)], [10.0])
    assert got[2].tolist() == [0, 1] and got.sum() == 1


def test_run_within_the_margin_is_neither():
    # d = 0.5: beyond the truncation but inside truncation + margin: no through vote even though the sdf crosses zero
    assert _votes([(0, 1, 9.5, -0.2)], [10.0]).sum() == 0


def test_one_vote_per_ray_and_voxel():
    # voxel 1 appears in two runs of ray 0 (voxel 3 between them); the union decides: every sample in front and a crossing
    rows = [(0, 1, 5.0, 0.4), (0, 3, 5.5, 0.5), (0, 1, 6.0, -0.2), (1, 1, 5.0, -0.1)]
    got = _votes(rows, [10.0, 10.0])
    assert got[1].tolist() == [2, 0] and got[3].tolist() == [0, 0]
    # a surface sample in the second run turns the union into one surface vote
    rows = [(0, 1, 5.0, -0.4), (0, 3, 5.5, 0.5), (0, 1, 9.9, 0.0)]
    assert _votes(rows, [10.0])[1].tolist() == [0, 1]


def test_nan_sdf_is_not_a_crossing():
    assert _votes([(0, 1, 5.0, np.nan), (0, 1, 5.2, np.nan)], [10.0]).sum() == 0
    assert _votes([(0, 1, 5.0, np.nan), (0, 1, 5.2, -0.1)], [10.0])[1].tolist() == [1, 0]


@pytest.mark.parametrize("t,s,removed", [(3, 0, True), (2, 0, False), (4, 1, True), (3, 1, False), (8, 2, True), (7, 2, False)])
def test_classification_boundaries(t, s, removed):
    """min_votes 3, ratio 0.8: through >= 3 and through >= 0.8 (through + surface)."""
    counts = np.array([[t, s], [0, 0], [0, 5], [9, 9]])
    structure = np.zeros((4, 9), np.int32)
    structure[:, 8] = [1, 1, 1, 2]                      # node 3 is not a leaf: never classified
    ids, conf, rem, unobs = ref.classify(counts, structure, 3, 0.8)
    assert ids.tolist() == ([0] if removed else []) and rem == int(removed)
    assert conf == 1 + int(not removed and s > 0) and unobs == 1


def test_ratio_one_needs_only_through_votes():
    counts = np.array([[5, 0], [5, 1]])
    structure = np.ones((2, 9), np.int32)
    assert ref.classify(counts, structure, 1, 1.0)[0].tolist() == [0]


# -- added -------------------------------------------------------------------------------------------------------------------
def test_added_counts_points_and_distinct_scans():
    vs = 0.5
    I = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32)
    occupied = {int(ref.voxel_keys(np.array([[0.1, 0.1, 0.1]], np.float32), I, vs)[0][0])}
    a = np.array([[0.1, 0.1, 0.1], [1.1, 0.1, 0.1], [1.2, 0.2, 0.2], [2.1, 0.1, 0.1]], np.float32)
    shifted = I.copy()
    shifted[9] = 1.0                                          # one metre along x: [0.1 ..] lands in the voxel of [1.1 ..]
    table = ref.added([(a, I), (a[1:2], I), (a[:1], shifted)], occupied, vs)
    k2 = int(ref.voxel_keys(a[1:2], I, vs)[0][0])
    k4 = int(ref.voxel_keys(a[3:4], I, vs)[0][0])
    assert table == {k2: [4, 3], k4: [1, 1]}                         # the occupied voxel of [0.1 ..] counts nothing
    keys, pts, scans = ref.select_added(table, 1, 1)
    assert keys.tolist() == [k2, k4] and pts.tolist() == [4, 1] and scans.tolist() == [3, 1]
    assert ref.select_added(table, 1, 2)[0].tolist() == [k2]           # min_scans
    assert ref.select_added(table, 1, 4)[0].size == 0 and ref.select_added(table, 5, 1)[0].size == 0
    # negative coordinates have no key
    assert not ref.voxel_keys(np.array([[-1.0, 0.0, 0.0]], np.float32), I, vs)[1][0]


# -- settings ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("specs,match", [
    ({"margn": 1.0}, "margn"),
    ({"margin": float("nan")}, "margin"),
    ({"margin": -0.5}, "margin"),
    ({"ratio": 0.0}, "ratio"),
    ({"ratio": 1.01}, "ratio"),
    ({"ratio": "0.5"}, "ratio"),
    ({"min_votes": 0}, "min_votes"),
    ({"min_points": 2.5}, "min_points"),
    ({"min_scans": True}, "min_scans"),
    ({"min_scans": None}, "min_scans"),
    ({"min_votes": float("inf")}, "min_votes"),
])
def test_change_specs_rejected(specs, match):
    with pytest.raises(ValueError, match=match):
        changes.change_specs(specs)
    with pytest.raises(ValueError, match=match):
        localise.Localiser(_saved(), _Stream(2), config={"change_specs": specs})


def test_change_specs_accepted():
    assert changes.change_specs({}) == changes.CHANGE_SPECS
    got = changes.change_specs({"min_votes": np.int64(4), "ratio": 1, "margin": 0})
    assert got == dict(changes.CHANGE_SPECS, min_votes=4, ratio=1.0, margin=0.0) and type(got["min_votes"]) is int
    assert localise.Localiser(_saved(), _Stream(2)).change_specs is None
    assert localise.Localiser(_saved(), _Stream(2), config={"change_specs": {}}).change_specs == changes.CHANGE_SPECS
    with pytest.raises(ValueError, match="dict"):
        changes.change_specs([])


# -- writers -------------------------------------------------------------------------------------------------------------------
def _read_ply(path):
    data = path.read_bytes()
    head, body = data.split(b"end_header\n", 1)
    lines = head.decode().splitlines()
    nv = int(next(l for l in lines if l.startswith("element vertex")).split()[-1])
    nf = int(next(l for l in lines if l.startswith("element face")).split()[-1])
    assert nf == 0 and len(body) == 12 * nv
    return np.frombuffer(body, "<f4").reshape(nv, 3)


def test_writers(tmp_path):
    ch = changes.Changes(np.array([[1.0, 2.0, 3.0], [4.0, 5.0, 6.5]]), np.array([7, 9]), np.array([5, 6]), np.array([0, 1]), 10, 2, 30,
                         np.array([[0.15, -0.45, 1.05]]), np.array([12]), np.array([3]), 4)
    changes.write_changes(str(tmp_path / "out"), ch)
    assert np.array_equal(_read_ply(tmp_path / "out" / "changes_removed.ply"), np.float32(ch.removed_centres))
    assert np.array_equal(_read_ply(tmp_path / "out" / "changes_added.ply"), np.float32(ch.added_centres))
    lines = (tmp_path / "out" / "changes.txt").read_text().splitlines()
    assert lines[:5] == ["scans 4", "confirmed 10", "removed 2", "unobserved 30", "added 1"]
    assert lines[5:] == ["removed 1.0000 2.0000 3.0000 5 0", "removed 4.0000 5.0000 6.5000 6 1", "added 0.1500 -0.4500 1.0500 12 3"]
    empty = changes.Changes(np.zeros((0, 3)), np.zeros(0, np.int64), np.zeros(0), np.zeros(0), 0, 0, 0, np.zeros((0, 3)), np.zeros(0),
                            np.zeros(0), 0)
    changes.write_changes(str(tmp_path / "empty"), empty)
    assert _read_ply(tmp_path / "empty" / "changes_added.ply").shape == (0, 3)


# -- the Localiser's wiring ------------------------------------------------------------------------------------------------------
class _Detector:
    built = []

    def __init__(self, map_state, decoder, voxel_size, criteria, tracking_kw, specs):
        self.scans = []
        self.specs = specs
        _Detector.built.append(self)

    def add_scan(self, frame, pose):
        self.scans.append((frame.index, float(pose.data.reshape(-1)[0])))

    def result(self):
        return changes.Changes(np.zeros((1, 3)), np.array([3]), np.array([4]), np.array([0]), 5, 1, 6, np.zeros((2, 3)), np.array([5, 6]),
                               np.array([2, 2]), len(self.scans))


def _run(monkeypatch, tmp_path, config):
    _Drive(monkeypatch)
    _Detector.built = []
    monkeypatch.setattr(localise, "ChangeDetector", _Detector)
    loc = localise.Localiser(_saved(), _Stream(len(TRUTH)), config={"tracker_specs": {"num_iterations": 7}, **config}, out_dir=str(tmp_path))
    return loc, loc.run(init_pose=np.eye(4))


def test_lost_scans_are_not_added(monkeypatch, tmp_path):
    loc, res = _run(monkeypatch, tmp_path, {"recovery_specs": {"global_interval": 2}, "change_specs": {"min_votes": 4}})
    assert res.status == WANT and len(_Detector.built) == 1
    det = _Detector.built[0]
    assert det.specs == dict(changes.CHANGE_SPECS, min_votes=4)
    assert [i for i, _ in det.scans] == [i for i, s in enumerate(WANT) if s != "lost"]
    # at the final pose: what run() reports for that scan
    for i, x in det.scans:
        assert x - localise.POSE_OFFSET == pytest.approx(float(res.poses[i, 0, 3]), abs=1e-3)
    assert res.changes.n_removed == 1 and res.changes.n_scans == 7
    sm = loc.summary(res)
    json.dumps(sm)
    assert sm["changes"]["removed"] == 1 and sm["changes"]["added"] == 2 and sm["changes"]["scans"] == 7
    assert sm["changes"]["ms_per_scan"] >= 0
    assert {"changes_removed.ply", "changes_added.ply", "changes.txt"} <= {p.name for p in tmp_path.iterdir()}


def test_without_recovery_every_scan_is_added(monkeypatch, tmp_path):
    _, res = _run(monkeypatch, tmp_path, {"change_specs": {}})
    assert [i for i, _ in _Detector.built[0].scans] == list(range(len(TRUTH)))
    assert res.status is None and res.changes is not None


def test_off_builds_no_detector(monkeypatch, tmp_path):
    loc, res = _run(monkeypatch, tmp_path, {})
    assert _Detector.built == [] and res.changes is None
    assert "changes" not in loc.summary(res)
    assert not (tmp_path / "changes.txt").exists() and (tmp_path / "frame_poses.txt").exists()
    assert res._fields[-1] == "changes" and res._fields[:-1] == ("scan_ids", "poses", "loss", "hit_fraction", "placement", "status")
