"""Global localisation without a GPU: the NumPy restatement against brute-force loops, the exported C ABI, and argument checks that
raise ValueError before any device work."""
import math

import numpy as np
import pytest
import torch

import globalloc_ref as ref


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


def _anchors(rng, A):
    out = np.zeros((A, 12))
    for a in range(A):
        yaw, roll = rng.uniform(-np.pi, np.pi), rng.uniform(-0.05, 0.05)
        cz, sz, cr, sr = np.cos(yaw), np.sin(yaw), np.cos(roll), np.sin(roll)
        R = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1.0]]) @ np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
        out[a].reshape(3, 4)[:, :3] = R
        out[a].reshape(3, 4)[:, 3] = [rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-1, 1)]
    return out


def test_cells_equal_brute_force():
    rng = np.random.default_rng(3)
    for A, r, step in ((1, 2.0, 1.0), (3, 1.5, 0.5), (5, 2.5, 0.7), (4, 0.0, 1.0)):
        An = _anchors(rng, A)
        An[-1, 3], An[-1, 7] = 1.0, -2.0                     # a lattice point exactly on one anchor
        got = ref.cells(An, r, step)
        want = []
        for i in range(-40, 41):
            for j in range(-40, 41):
                d = [math.sqrt((i * step - a[3]) ** 2 + (j * step - a[7]) ** 2) for a in An]
                inside = [(np.float32(x).view(np.uint32), k) for k, x in enumerate(d) if x <= r]
                if inside:
                    want.append((i, j, min(inside)[1]))
        assert np.array_equal(got, np.array(want, dtype=np.int64).reshape(-1, 3)), (A, r, step)


def test_matrices_counts_and_selection_equal_loops():
    rng = np.random.default_rng(4)
    An = _anchors(rng, 3)
    cells = ref.cells(An, 2.0, 1.0)
    Y, step, vs, gd = 8, 1.0, 0.5, 64
    ids = np.arange(cells.shape[0] * Y)
    M = ref.matrices(cells, An, Y, step, ids)
    for h in rng.choice(ids, 20, replace=False):
        i, j, a = cells[h // Y]
        Ra = An[a].reshape(3, 4)
        psi = math.atan2(Ra[1, 0], Ra[0, 0])
        th = 2 * math.pi * (h % Y) / Y - psi
        Rz = np.array([[math.cos(th), -math.sin(th), 0], [math.sin(th), math.cos(th), 0], [0, 0, 1.0]])
        want = np.concatenate([(Rz @ Ra[:, :3]).reshape(-1), [i * step, j * step, Ra[2, 3]]])
        assert np.allclose(M[h], want, atol=1e-6)
    pts = rng.uniform(-6, 6, (40, 3)).astype(np.float32)
    pts[0] = np.nan
    pts[1] = [1e6, 0, 0]
    occ_v = rng.integers(0, 20, (300, 3))
    occ = ref.leaf_keys(occ_v)
    occ_set = {tuple(v) for v in occ_v}
    got = ref.counts(M + np.float32(4.0) * np.array([0] * 9 + [1, 1, 1], np.float32), pts, occ, vs, gd, block=7)
    for h in range(0, ids.size, 5):
        Rt = (M[h] + np.float32(4.0) * np.array([0] * 9 + [1, 1, 1], np.float32)).astype(np.float64)
        n = 0
        for p in pts.astype(np.float64):
            w = [((Rt[3 * c] * p[0] + Rt[3 * c + 1] * p[1]) + Rt[3 * c + 2] * p[2]) + Rt[9 + c] for c in range(3)]
            if not all(np.isfinite(w)):
                continue
            v = tuple(int(math.floor(x / vs)) for x in w)
            n += all(0 <= x < gd for x in v) and v in occ_set
        assert got[h] == n, h
    c = rng.integers(0, 5, 200)
    for n in (1, 7, 50, 200):
        ids_s, cnt = ref.select(c, n)
        want = sorted(range(200), key=lambda h: (-c[h], h))[:n]
        assert list(ids_s) == want and list(cnt) == [c[h] for h in want]


def test_c_abi_symbols_exported(nl):
    names = ("nl_abi_sizes_globalloc", "nl_globalloc_count_leaves", "nl_globalloc_occupied_slots", "nl_globalloc_occupied",
             "nl_globalloc_cells_workspace_bytes", "nl_globalloc_cells", "nl_globalloc_cells_finish", "nl_globalloc_matrices",
             "nl_globalloc_score", "nl_globalloc_select_workspace_bytes", "nl_globalloc_select")
    L = nl._capi.lib()
    for n in names:
        assert n in nl._capi.EXPORTED_SYMBOLS and hasattr(L, n), n
    assert "relocalise_global" in nl.__all__ and nl.relocalise_global is nl.globalloc.relocalise_global


def test_c_abi_rejects_bad_arguments(nl):
    L = nl._capi.lib()
    a = np.eye(4)[:3].reshape(1, 12).copy()
    ok = L.nl_globalloc_cells_workspace_bytes(1, a.ctypes.data, 5.0, 1.0)
    assert ok > 0
    assert L.nl_globalloc_cells_workspace_bytes(0, a.ctypes.data, 5.0, 1.0) < 0
    assert L.nl_globalloc_cells_workspace_bytes(1, a.ctypes.data, -1.0, 1.0) < 0
    assert L.nl_globalloc_cells_workspace_bytes(1, a.ctypes.data, 5.0, 0.0) < 0
    assert L.nl_globalloc_cells_workspace_bytes(1, a.ctypes.data, float("inf"), 1.0) < 0
    assert L.nl_globalloc_cells_workspace_bytes(1, a.ctypes.data, 1e6, 1e-3) < 0           # lattice too large
    bad = a.copy()
    bad[0, 5] = float("nan")
    assert L.nl_globalloc_cells_workspace_bytes(1, bad.ctypes.data, 5.0, 1.0) < 0
    assert L.nl_globalloc_occupied_slots(0) < 0                                             # an empty map
    assert L.nl_globalloc_occupied_slots(1000) == 2048
    assert L.nl_globalloc_select_workspace_bytes(100, 0, 10) < 0                            # M < 1
    assert L.nl_globalloc_select_workspace_bytes(100, 512, 101) < 0
    assert L.nl_globalloc_select_workspace_bytes(2 ** 31, 512, 10) < 0                      # ids are int32
    assert L.nl_globalloc_matrices(1, None, 10, None, None, 0, 1.0, None, None) != 0        # Y < 1
    assert L.nl_globalloc_matrices(1, None, 2 ** 28, None, None, 16, 1.0, None, None) != 0  # cells x Y >= 2^31
    assert L.nl_globalloc_score(0, 1, 10, None, None, 4, 1.0, 0, None, None, 1024, 0.3, 1 << 18, None, None) != 0   # M < 1


def _frame(nl, n=2000):
    pts = torch.randn(n, 3) * 10
    return nl.frame.LidarFrame(0, pts, torch.ones(n), nl.se3pose.OptimizablePose(torch.zeros(6)), new_keyframe=True)


@pytest.mark.parametrize("bad", [dict(anchors=np.zeros((0, 4, 4))), dict(radius=-1.0), dict(xy_step=0.0), dict(xy_step=-1.0),
                                 dict(radius=float("nan")), dict(anchors="nan"), dict(yaw_steps=0), dict(n_points=0),
                                 dict(n_points=8193), dict(n_candidates=0), dict(n_candidates=65536), dict(n_seeds=0),
                                 dict(seed_separation=-1.0), dict(grid_dim=3), dict(voxel_size=0.0), dict(anchors=np.zeros((2, 2, 4))),
                                 dict(radius=1e5, xy_step=1e-2), dict(chunk=0)])
def test_relocalise_global_rejects_bad_arguments_before_device_work(nl, bad, monkeypatch):
    """Every check runs on the host: a CUDA call would fail the test here, with or without a GPU."""
    def no_device(*a, **k):
        raise AssertionError("device work before argument validation")
    monkeypatch.setattr(nl.globalloc, "_map_state", no_device)
    kw = dict(anchors=np.eye(4)[None].repeat(2, 0), radius=5.0, xy_step=1.0, yaw_steps=72, n_points=512, n_candidates=4096, n_seeds=4,
              seed_separation=2.0)
    kw.update(bad)
    if isinstance(kw["anchors"], str):
        kw["anchors"] = np.eye(4)[None].repeat(2, 0)
        kw["anchors"][1, 0, 3] = float("nan")
    vs = kw.pop("voxel_size", 0.3)
    with pytest.raises(ValueError):
        nl.relocalise_global(_frame(nl), None, None, None, vs, **kw)
