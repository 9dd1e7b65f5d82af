"""Key-scan map refinement on the GPU (render_helpers.refine_map, csrc/refine.cu): against the mapper's loop of bundle_adjust_frames
calls under the same seeds, the row-list Adam against the dense one bit for bit, the capacity-overflow redo, the loss it lowers, and
the demo's --final-iter."""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from util import ROOT

pytestmark = pytest.mark.gpu

VS, TR, MD = 0.3, 0.3, 40.0
KW = dict(voxel_size=VS, step_size=0.15, N_rays=512, num_iterations=3, truncation=TR, max_voxel_hit=20, max_distance=MD)
LR = 0.01


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


class _Args:
    criteria = {"eiko_weight": 0.1, "sdf_weight": 10000.0, "fs_weight": 1.0, "sdf_truncation": TR}
    data_specs = {"max_depth": MD}


def _setup(nl, n_kf=6, train_calls=0):
    """n_kf synthetic keyframes along a line on a MapUpdater map, a seeded decoder; optionally a briefly trained map."""
    mu = nl.mapping.MapUpdater(VS, init_std=0.01, seed=3, reserve_nodes=200_000, reserve_rows=200_000)
    torch.manual_seed(5)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    crit = nl.criterion.Criterion(_Args())
    kg = nl.keyframes.KeyframeGraph(window_size=4, keyframe_gap=0.5, key_distance=MD, n_rays=512, voxel_size=VS)
    ms = None
    for i in range(n_kf):
        xyz, yaw = nl.synthetic.path_pose(i, n_kf, 1.0, "line")
        pts, cos, pose = nl.synthetic.make_scan(seed=1000 + i, sensor_xyz=xyz, yaw=yaw)
        f = nl.frame.LidarFrame(i, torch.from_numpy(pts), torch.from_numpy(cos), nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose)),
                                new_keyframe=True)
        ms = mu.create_voxels(f.points, f.get_pose().detach())
        kg.insert_keyframe(f)
    for c in range(train_calls):
        nl.render_helpers.bundle_adjust_frames(kg.keyframe_graph[c % n_kf:][:4], mu.embeddings, ms, dec, crit, learning_rate=[LR, 0.005, 0.0],
                                               update_pose=False, update_decoder=True, deterministic=True, **{**KW, "num_iterations": 10})
    return mu, dec, crit, kg, ms


def _loop(nl, mu, dec, crit, kg, ms, passes, deterministic):
    for _ in range(passes):
        nl.render_helpers.bundle_adjust_frames(kg.select_optimize_targets(None, "random"), mu.embeddings, ms, dec, crit,
                                               learning_rate=[LR, 0.005, 0.001], update_pose=False, update_decoder=False,
                                               deterministic=deterministic, **KW)


def _frozen(dec, kg):
    return [p.detach().clone() for p in dec.parameters()], [f.pose.data.detach().clone() for f in kg.keyframe_graph]


def _assert_frozen(dec, kg, before):
    for a, b in zip(dec.parameters(), before[0]):
        assert torch.equal(a.detach(), b)
    for f, b in zip(kg.keyframe_graph, before[1]):
        assert torch.equal(f.pose.data.detach(), b)


def _agree(e0, e_r, e_p):
    """The criteria of test_gpu_dropin_reference's embedding check, plus: the same rows left bitwise unchanged."""
    same_r = (e_r.view(torch.int16) == e0.view(torch.int16)).all(1)
    same_p = (e_p.view(torch.int16) == e0.view(torch.int16)).all(1)
    assert torch.equal(same_r, same_p), int((same_r != same_p).sum())
    e0, e_r, e_p = e0.float(), e_r.float(), e_p.float()
    u_r, u_p = e_r - e0, e_p - e0
    stats = dict(moved=float((u_r.abs() > 1e-3).float().mean()), update_rel=float((u_p - u_r).norm() / u_r.norm()),
                 frac_gt_fifth=float(((e_p - e_r).abs() > LR / 5).float().mean()))
    print("refine_map vs the loop:", stats)
    assert stats["moved"] > 1e-3
    assert stats["update_rel"] < 0.05, stats
    assert stats["frac_gt_fifth"] < 5e-3, stats
    return stats


@pytest.mark.parametrize("deterministic", [True, False])
def test_refine_map_computes_the_mappers_loop(nl, deterministic):
    mu, dec, crit, kg, ms = _setup(nl)
    table = mu._emb_buf                                   # the capacity-sized table both optimise
    e0 = table.clone()
    before = _frozen(dec, kg)
    random.seed(21); torch.manual_seed(22)
    _loop(nl, mu, dec, crit, kg, ms, 7, deterministic)
    e_loop = table.clone()
    rng_after = (random.getstate(), torch.get_rng_state())
    _assert_frozen(dec, kg, before)
    table.copy_(e0)
    random.seed(21); torch.manual_seed(22)
    assert nl.refine_map(kg, mu.embeddings, ms, dec, crit, learning_rate=LR, passes=7, deterministic=deterministic, **KW) is None
    torch.cuda.synchronize()
    _assert_frozen(dec, kg, before)
    assert random.getstate() == rng_after[0] and torch.equal(torch.get_rng_state(), rng_after[1])
    _agree(e0, e_loop, table.clone())
    # a second call on the same captured graph starts from fresh moments again: it equals a loop from the refined table
    g = nl.render_helpers._RefineGraph._cache["g"]
    e1 = table.clone()
    random.seed(5); torch.manual_seed(6)
    nl.refine_map(kg, mu.embeddings, ms, dec, crit, learning_rate=LR, passes=7, deterministic=deterministic, **KW)
    assert nl.render_helpers._RefineGraph._cache["g"] is g
    e_again = table.clone()
    table.copy_(e1)
    random.seed(5); torch.manual_seed(6)
    _loop(nl, mu, dec, crit, kg, ms, 7, deterministic)
    _agree(e1, table.clone(), e_again)


def _bf16_table(gen, V):
    p = (torch.randn((V, 16), generator=gen) * 0.05).to(torch.bfloat16)
    z = torch.rand((V, 16), generator=gen) < 0.05
    p[z] = 0.0
    p[z & (torch.rand((V, 16), generator=gen) < 0.5)] = -0.0
    return p


def test_row_list_adam_equals_the_dense_step_bitwise(nl):
    L, cap = nl._capi.lib(), nl._capi
    gen = torch.Generator().manual_seed(0)
    V = 20_000
    p = _bf16_table(gen, V)
    listed = torch.randperm(V, generator=gen)[:6000]
    moved = listed[:4000]                                  # rows with moments; the other listed rows have g = m = v = 0
    m = torch.zeros((V, 16), dtype=torch.bfloat16)
    v = torch.zeros((V, 16), dtype=torch.bfloat16)
    m[moved] = (torch.randn((len(moved), 16), generator=gen) * 1e-3).to(torch.bfloat16)
    v[moved] = (torch.rand((len(moved), 16), generator=gen) * 1e-6).to(torch.bfloat16)
    dense = [t.cuda() for t in (p, m, v)]
    rows = [t.cuda() for t in (p, m, v)]
    buf = torch.randperm(V, generator=gen).to(torch.int32)            # entries past the count name unlisted rows: never touched
    buf[:len(listed)] = listed[torch.randperm(len(listed), generator=gen)].to(torch.int32)
    buf, n_listed = buf.cuda(), torch.tensor([len(listed)], dtype=torch.int32, device="cuda")
    unlisted = torch.ones(V, dtype=torch.bool)
    unlisted[listed] = False
    ctl = torch.zeros(cap.CTL_WORDS, dtype=torch.int32, device="cuda")
    for t, skip in ((1, 0), (2, 0), (2, 1), (3, 0), (4, 0)):
        g = torch.zeros((V, 16))
        with_grad = moved[torch.rand(len(moved), generator=gen) < 0.7]      # some moved rows get a zero gradient this step
        g[with_grad] = torch.randn((len(with_grad), 16), generator=gen) * 1e-2
        g_dense = g.cuda()
        g_rows = g.clone()
        g_rows[unlisted] = 7.0                              # never read, never written
        g_rows = g_rows.cuda()
        ctl[cap.CTL_ADAM_STEP], ctl[cap.CTL_SKIP_NOW] = t, skip
        cap.check(L.nl_adam_bf16_ctl(V * 16, cap.ptr(dense[0]), cap.ptr(g_dense), cap.ptr(dense[1]), cap.ptr(dense[2]), LR, 0.9, 0.999, 1e-8,
                                     cap.ptr(ctl), cap.stream_ptr()))
        cap.check(L.nl_adam_bf16_rows_ctl(V, cap.ptr(buf), cap.ptr(n_listed), cap.ptr(rows[0]), cap.ptr(g_rows), cap.ptr(rows[1]), cap.ptr(rows[2]),
                                          LR, 0.9, 0.999, 1e-8, cap.ptr(ctl), cap.stream_ptr()))
        for a, b in zip(dense, rows):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (t, skip)
        gr = g_rows.cpu()
        assert (gr[listed] == 0).all() and (gr[unlisted] == 7.0).all()
    assert not torch.equal(dense[0].cpu().view(torch.int16), p.view(torch.int16))
    untouched = torch.ones(V, dtype=torch.bool)
    untouched[moved] = False
    assert torch.equal(rows[0].cpu()[untouched].view(torch.int16), p[untouched].view(torch.int16))     # +-0 bits included


def test_capacity_overflow_is_redone(nl, monkeypatch, capsys):
    mu, dec, crit, kg, ms = _setup(nl)
    table = mu._emb_buf
    e0 = table.clone()
    random.seed(3); torch.manual_seed(4)
    nl.refine_map(kg, mu.embeddings, ms, dec, crit, learning_rate=LR, passes=5, deterministic=True, **KW)
    e_ok = table.clone()
    table.copy_(e0)
    monkeypatch.setattr(nl.render_helpers, "SAMPLES_PER_RAY_MAP", 1)
    random.seed(3); torch.manual_seed(4)
    nl.refine_map(kg, mu.embeddings, ms, dec, crit, learning_rate=LR, passes=5, deterministic=True, **KW)
    g = nl.render_helpers._RefineGraph._cache["g"]
    assert g.eng.max_samples > 4 * 512 * 2                 # redone on a grown capacity
    _agree(e0, e_ok, table.clone())


def _keyframe_loss(nl, kg, ms, dec, crit):
    total = 0.0
    for f in kg.keyframe_graph:
        torch.manual_seed(99)
        r = nl.score_poses(f.pose.data.detach().reshape(1, 6), f, ms, dec, crit, VS, N_rays=2048, step_size=0.15, max_distance=MD,
                           deterministic=True)
        total += float(r.loss[0])
    return total


def test_refinement_lowers_the_keyframe_loss(nl):
    mu, dec, crit, kg, ms = _setup(nl, train_calls=4)
    before = _keyframe_loss(nl, kg, ms, dec, crit)
    random.seed(1)
    nl.refine_map(kg, mu.embeddings, ms, dec, crit, learning_rate=LR, deterministic=True, **{**KW, "num_iterations": 10, "N_rays": 1024})
    after = _keyframe_loss(nl, kg, ms, dec, crit)
    print("sum of keyframe losses before / after refinement:", before, after)
    assert np.isfinite(before) and after < before


def test_demo_final_iter(tmp_path):
    out = tmp_path / "demo.json"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "demo_slam.py"), "--scans", "6", "--final-iter", "--json", str(out)],
                       cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(out.read_text())
    for k in ("reconstruction", "reconstruction_before_refine"):
        assert np.isfinite(res[k]["chamfer_l1"]) and 0.0 < res[k]["fscore"] <= 100.0, k          # F-score in percent
    print("reconstruction before / after refinement:", {k: {q: res[k][q] for q in ("chamfer_l1", "fscore")}
                                                        for k in ("reconstruction_before_refine", "reconstruction")})
    assert res["refine_ms"] > 0 and res["refine_passes"] == 4
