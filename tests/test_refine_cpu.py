"""Key-scan map refinement without a GPU: the up-front schedule against the mapper loop's own draws, the exactness argument of the
row-list Adam on the bf16 arithmetic (tests/embedding_ref.py), and the argument checks of the C ABI and of refine_map that run before
any device work."""
import ctypes
import random

import numpy as np
import pytest
import torch

import embedding_ref as ER


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    return nl


def _graph(nl, K, W=4, n_rays=8, n_points=40):
    kg = nl.keyframes.KeyframeGraph(window_size=W, keyframe_gap=1.0, key_distance=50.0, n_rays=n_rays, voxel_size=0.3)
    g = torch.Generator().manual_seed(K)
    for i in range(K):
        pts = torch.rand((n_points, 3), generator=g) * 10.0 - 5.0
        kg.insert_keyframe(nl.frame.LidarFrame(2 * i, pts, torch.ones(n_points), nl.se3pose.OptimizablePose(torch.zeros(6)),
                                               new_keyframe=True))
    return kg


@pytest.mark.parametrize("K,P", [(9, 10), (26, 27), (5, 3)])
def test_schedule_draws_the_loops_windows(nl, K, P):
    kg = _graph(nl, K)
    random.seed(123)
    want = [[kg.keyframe_graph.index(f) for f in kg.select_optimize_targets(None, "random")] for _ in range(P)]
    random.seed(123)
    windows, noise, sel = nl.render_helpers.refine_schedule(kg, P, deterministic=True, device="cpu")
    assert windows == want
    assert len(set(map(tuple, windows))) > 1
    assert all(len(w) == 4 and len(set(w)) == 4 for w in windows)
    assert noise == [0] * P and len(sel) == P


def test_schedule_noise_and_selection_seeds_follow_the_generators(nl):
    kg = _graph(nl, 6)
    torch.manual_seed(7)
    want_noise, want_sel = [], []
    for _ in range(3):                                  # bundle_adjust_frames: the noise seed, then the selection seed, per call
        want_noise.append(int(torch.randint(1, 2 ** 31 - 1, (1,)).item()))
        want_sel.append(int(torch.randint(1, 2 ** 31 - 1, (1,), dtype=torch.int32).item()))
    torch.manual_seed(7)
    _, noise, sel = nl.render_helpers.refine_schedule(kg, 3, device="cpu")
    assert noise == want_noise and [int(s.item()) for s in sel] == want_sel


@pytest.mark.parametrize("K", [1, 3, 4])
def test_small_graph_gives_every_keyframe_in_graph_order(nl, K):
    kg = _graph(nl, K)
    state = random.getstate()
    windows, _, _ = nl.render_helpers.refine_schedule(kg, K + 1, deterministic=True, device="cpu")
    assert windows == [list(range(K))] * (K + 1)
    assert random.getstate() == state                   # no window was drawn


def _bf16_specials():
    bits = np.array([0x0000, 0x8000, 0x0001, 0x8001, 0x007F, 0x807F, 0x0080, 0x8080, 0x7F7F, 0xFF7F, 0x3F80, 0xBF80, 0x3DCD, 0x4049],
                    np.uint16)
    rnd = np.random.default_rng(0).integers(0, 1 << 16, 4096, dtype=np.uint32).astype(np.uint16)
    rnd = rnd[(rnd & 0x7F80) != 0x7F80]                  # finite values only
    return np.concatenate([bits, rnd])


@pytest.mark.parametrize("t", [1, 2, 3, 10, 25, 1000])
@pytest.mark.parametrize("lr", [1e-2, 2e-3])
def test_zero_gradient_and_moments_leave_bf16_bits_unchanged(t, lr):
    bits = _bf16_specials()
    p = ER.bf16_to_f32(bits)
    z = np.zeros_like(p)
    p1, m1, v1 = ER.adam_step(p, z, z, z, lr, 0.9, 0.999, 1e-8, t, True)
    assert np.array_equal(ER.bf16_bits(p1), bits)       # bitwise: -0.0 stays -0.0, subnormals and the largest finite values stay
    assert np.array_equal(ER.bf16_bits(m1), np.zeros_like(bits)) and np.array_equal(ER.bf16_bits(v1), np.zeros_like(bits))


def test_c_abi_exports_and_rejects_bad_arguments(nl):
    L = nl._capi.lib()
    for name in ("nl_refine_pass_begin", "nl_mark_rows", "nl_adam_bf16_rows_ctl", "nl_refine_iter_end"):
        assert name in nl._capi.EXPORTED_SYMBOLS and getattr(L, name) is not None
    err = lambda: L.nl_last_error().decode()
    a = [ctypes.c_void_p(256 * k) for k in range(1, 25)]                  # never dereferenced: every call below fails its checks
    names = ("state", "win", "kfa", "kfn", "kfp", "ss", "ns", "dirs", "gt", "cos", "n", "pose", "sel", "noise", "ctl", "rows", "bits", "m", "v")
    ptrs = dict(zip(names, a))

    def begin(**kw):
        s = dict(F=4, cap=1 << 17, K=6, iters=3, P=7, n_rows=1000, **ptrs)
        s.update(kw)
        return L.nl_refine_pass_begin(s["F"], s["cap"], s["K"], s["iters"], s["P"], *[s[k] for k in names[:15]], s["n_rows"],
                                      *[s[k] for k in names[15:]], None)
    for k, bad in (("F", 0), ("cap", 0), ("K", 0), ("iters", 0), ("P", -1), ("n_rows", 0), ("n_rows", 1 << 31)):
        assert begin(**{k: bad}) != 0 and "sizes" in err(), k
    for k in names:
        if k in ("ss", "ns", "sel", "noise"):
            continue
        assert begin(**{k: None}) != 0 and "null" in err(), k
    assert begin(sel=None) != 0 and "seed" in err()
    assert begin(ns=None) != 0 and "seed" in err()     # a noise seed without its per-pass array
    mark = lambda M=10, n_rows=1000, **kw: L.nl_mark_rows(M, None, *[kw.get(k, ptrs[k]) for k in ("win", "kfa")], n_rows,
                                                           *[kw.get(k, ptrs[k]) for k in ("bits", "rows", "state")], None)
    assert mark(M=-1) != 0 and "sizes" in err()
    assert mark(n_rows=0) != 0 and "sizes" in err()
    for k in ("win", "kfa", "bits", "rows", "state"):
        assert mark(**{k: None}) != 0 and "null" in err(), k
    assert mark(M=0) == 0                                                  # nothing to launch
    rows = lambda n=10, **kw: L.nl_adam_bf16_rows_ctl(n, *[kw.get(k, ptrs[k]) for k in ("rows", "state", "m", "v", "gt", "cos")], 1e-2, 0.9,
                                                       0.999, 1e-8, kw.get("ctl", ptrs["ctl"]), None)
    assert rows(n=-1) != 0 and "bad" in err()
    for k in ("rows", "state", "m", "v", "gt", "cos", "ctl"):
        assert rows(**{k: None}) != 0 and "null" in err(), k
    assert rows(n=0) == 0
    assert L.nl_refine_iter_end(0, ptrs["state"], None, 0, None, 0, None) != 0 and "iters" in err()
    assert L.nl_refine_iter_end(3, None, None, 0, None, 0, None) != 0 and "null" in err()


def test_refine_map_checks_arguments_before_device_work(nl, monkeypatch):
    rh = nl.render_helpers
    monkeypatch.setattr(rh, "_seed_from_cuda", lambda dev: pytest.fail("a seed was drawn"))
    monkeypatch.setattr(rh.MapState, "from_map_states", classmethod(lambda *a, **k: pytest.fail("the map was touched")))
    emb = torch.zeros((100, 16), dtype=torch.bfloat16)
    kw = dict(map_states={}, sdf_network=None, loss_criteria=None, voxel_size=0.3, step_size=0.15)
    with pytest.raises(ValueError, match="empty"):
        rh.refine_map(_graph(nl, 0), emb, **kw)
    with pytest.raises(ValueError, match="fewer than N_rays"):
        rh.refine_map(_graph(nl, 3, n_points=40), emb, N_rays=64, **kw)
    with pytest.raises(ValueError, match="CUDA"):
        rh.refine_map(_graph(nl, 3), emb, N_rays=16, **kw)
    for bad in (dict(N_rays=0), dict(num_iterations=-1), dict(passes=-2)):
        with pytest.raises(ValueError):
            rh.refine_map(_graph(nl, 3), emb, **{**dict(N_rays=16), **bad}, **kw)
    assert nl.refine_map is rh.refine_map
