"""score_poses / relocalise pieces that need no GPU: argument checks, the yaw x translation lattice, the batched from_matrix and the
hit-fraction filter."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


def _frame(points=100):
    return SimpleNamespace(points=torch.zeros(points, 3), index=5)


def test_arguments_are_checked(nl):
    assert nl._capi.SCORE_MAX_PROBLEMS == 65535
    f = _frame()
    for K in (0, 65536):
        with pytest.raises(ValueError, match="number of poses"):
            nl.score_poses(torch.zeros(K, 6), f, None, None, None, 0.3, N_rays=10)
    with pytest.raises(ValueError, match=r"\[K,6\]"):
        nl.render_helpers.score_poses(torch.zeros(4, 7), f, None, None, None, 0.3, N_rays=10)
    with pytest.raises(ValueError, match=r"\[K,6\]"):
        nl.score_poses(torch.zeros(6), f, None, None, None, 0.3, N_rays=10)
    with pytest.raises(ValueError, match="N_rays"):
        nl.score_poses(torch.zeros(3, 6), f, None, None, None, 0.3, N_rays=101)
    for bad in (0, -5, 2.5, True, "1024"):
        with pytest.raises(ValueError, match="chunk_rays"):
            nl.score_poses(torch.zeros(3, 6), f, None, None, None, 0.3, N_rays=10, chunk_rays=bad)
    with pytest.raises(ValueError, match="at least one hypothesis"):
        nl.score_poses(torch.zeros(3, 6), f, None, None, None, 0.3, N_rays=10, chunk_rays=9)
    guess = nl.se3pose.OptimizablePose(torch.zeros(6))
    with pytest.raises(ValueError, match="top_k"):
        nl.relocalise(f, guess, None, None, None, 0.3, top_k=32)
    with pytest.raises(ValueError, match="top_k"):
        nl.render_helpers.relocalise(f, guess, None, None, None, 0.3, top_k=0)
    with pytest.raises(ValueError, match="min_hit_fraction"):
        nl.relocalise(f, guess, None, None, None, 0.3, min_hit_fraction=1.5)


def _guess(nl):
    return nl.se3pose.OptimizablePose(torch.tensor([3.0, -1.0, 0.4, 0.02, -0.03, 0.7]))


@pytest.mark.parametrize("yaw_steps,xy_steps", [(31, 9), (4, 3), (1, 1), (5, 2)])
def test_lattice_count_and_guess_first(nl, yaw_steps, xy_steps):
    g = _guess(nl)
    lat = nl.score.yaw_lattice(g, np.pi / 6, yaw_steps, 2.0, xy_steps)
    both_odd = yaw_steps % 2 == 1 and xy_steps % 2 == 1
    assert lat.shape == (yaw_steps * xy_steps ** 2 + (0 if both_odd else 1), 6) and lat.dtype == torch.float32
    assert torch.equal(lat[0], g.data.detach()) and not lat.requires_grad
    # every hypothesis: the guess turned about world z through its position and moved in x / y; z, roll and pitch unchanged
    Tg = g.matrix().detach().double()
    ez = Tg[:3, :3].T @ torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)     # world z in the sensor frame
    yaws = set()
    for p in lat[1:]:
        T = nl.se3pose.OptimizablePose(p.clone()).matrix().detach().double()
        assert abs(float(T[2, 3] - Tg[2, 3])) < 1e-6
        torch.testing.assert_close(T[:3, :3].T @ torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64), ez, atol=1e-5, rtol=0)
        d = T[:3, :3] @ Tg[:3, :3].T
        yaw = math.atan2(float(d[1, 0]), float(d[0, 0]))
        assert abs(yaw) <= np.pi / 6 + 1e-5
        assert abs(float(T[0, 3] - Tg[0, 3])) <= 2.0 + 1e-5 and abs(float(T[1, 3] - Tg[1, 3])) <= 2.0 + 1e-5
        yaws.add(round(yaw, 4))
    assert len(yaws) == yaw_steps or (yaw_steps == 1 and len(lat) == 1)


def test_batched_from_matrix(nl):
    gen = torch.Generator().manual_seed(5)
    Rt = []
    for _ in range(64):
        w = (torch.rand(3, generator=gen) - 0.5) * 3.0
        t = (torch.rand(3, generator=gen) - 0.5) * 20.0
        Rt.append(nl.se3pose.OptimizablePose(torch.cat([t, w])).matrix())
    Rt = torch.stack(Rt)
    batched = nl.score.poses_from_matrices(Rt)
    for k in range(Rt.shape[0]):
        one = nl.se3pose.OptimizablePose.from_matrix(Rt[k]).data.detach()
        torch.testing.assert_close(batched[k], one, atol=1e-6, rtol=0)


def test_hit_fraction_filter(nl):
    nan = float("nan")
    loss = torch.tensor([0.50, 0.01, 0.20, nan, 0.30, 0.05, 0.10])
    hits = torch.tensor([400, 3, 390, 0, 100, 250, 199], dtype=torch.int32)
    sel = nl.score.select_hypotheses(loss, hits, 16, 0.5)
    assert sel.tolist() == [5, 2, 0]                  # 3 hits (1) and 100 / 199 hits (4, 6) fall below half of 400
    assert nl.score.select_hypotheses(loss, hits, 2, 0.5).tolist() == [5, 2]
    assert nl.score.select_hypotheses(loss, hits, 16, 0.0).tolist() == [1, 5, 6, 2, 4, 0]
    assert nl.score.select_hypotheses(torch.full((3,), nan), hits[:3], 4, 0.5).numel() == 0
