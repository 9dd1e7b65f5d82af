"""track_frames argument checks that need no GPU: the problem count bound, one pose per frame, enough points per scan."""
from types import SimpleNamespace

import pytest
import torch


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


def _frames(n, points=100):
    return [SimpleNamespace(points=torch.zeros(points, 3), index=5) for _ in range(n)]


def test_problem_count_is_bounded(nl):
    assert nl._capi.BATCH_MAX_PROBLEMS == 31
    for K in (0, 32):
        with pytest.raises(ValueError, match="number of problems"):
            nl.track_frames([None] * K, _frames(K), None, None, None, 0.3, N_rays=10)


def test_mismatched_or_short_inputs_are_refused(nl):
    with pytest.raises(ValueError, match="one starting pose per frame"):
        nl.render_helpers.track_frames([None], _frames(2), None, None, None, 0.3, N_rays=10)
    with pytest.raises(ValueError, match="at least N_rays points"):
        nl.track_frames([None, None], _frames(2, points=5), None, None, None, 0.3, N_rays=10)
    with pytest.raises(ValueError, match="ray_selection"):
        nl.track_frames([None], _frames(1), None, None, None, 0.3, N_rays=10, ray_selection="cpu")
