"""The oracle (oracle/) against the golden vectors produced by executing the reference
(tests/golden/make_golden.py).  CPU only.  This is what pins the oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import chain as C
from oracle import kernels as K
from util import golden

G = os.path.join(os.path.dirname(__file__), "golden")


def bf16_from_bits(a):
    return torch.from_numpy(a.copy()).view(torch.bfloat16)


def vertex_rows(features, id2emb):
    f = features.astype(np.int64)
    rows = np.where(f >= 0, id2emb.reshape(-1)[np.clip(f, 0, None)], -1)
    return rows.astype(np.int64)


def build_oracle_map(vox, voxel_size, id2emb=None, grid_dim=256 * 256 * 4):
    o = K.Octree()
    o.init(grid_dim, 16, voxel_size)
    o.insert(vox)
    voxels, children, features = o.get_centres_and_children()
    centres, structure, feats = K.map_arrays(voxels, children, features, voxel_size)
    m = {"centres": centres, "structure": structure, "features": feats}
    if id2emb is not None:
        m["vertex_rows"] = vertex_rows(feats, id2emb)
    return m


def test_octree_bit_exact_vs_reference_svo():
    z = np.load(os.path.join(G, "octree.npz"))
    o = K.Octree()
    o.init(256 * 256 * 4, 16, 0.3)
    o.insert(z["v1"])
    v, c, f = o.get_centres_and_children()
    assert np.array_equal(v, z["voxels1"]) and np.array_equal(c, z["children1"]) and np.array_equal(f, z["features1"])
    assert [o.count_nodes(), o.count_leaf_nodes()] == list(z["count1"])
    o.insert(z["v2"])
    v, c, f = o.get_centres_and_children()
    assert np.array_equal(v, z["voxels2"]) and np.array_equal(c, z["children2"]) and np.array_equal(f, z["features2"])
    assert [o.count_nodes(), o.count_leaf_nodes()] == list(z["count2"])


def test_octree_8cubed_config0():
    z = np.load(os.path.join(G, "octree_8.npz"))
    o = K.Octree()
    o.init(8, 16, 1.0)
    o.insert(z["v0"])
    v, c, f = o.get_centres_and_children()
    assert np.array_equal(v, z["voxels"]) and np.array_equal(c, z["children"]) and np.array_equal(f, z["features"])


def test_pose_known_answer():
    z = np.load(os.path.join(G, "pose.npz"))
    data = C.pose_from_matrix(torch.from_numpy(z["before"]))
    np.testing.assert_allclose(data.numpy(), z["data"], rtol=0, atol=1e-7)
    R = C.pose_rotation(torch.from_numpy(z["data"]))
    np.testing.assert_allclose(R.numpy(), z["R"], rtol=0, atol=1e-7)
    # the reference's only self-check (se3pose.py:95-105): round trip reproduces the translation
    np.testing.assert_allclose(z["after"][:3, 3], z["before"][:3, 3], atol=1e-6)
    Gm = torch.from_numpy(z["G"])
    for d, Rref, gref in zip(z["datas"], z["Rs"], z["grads"]):
        dd = torch.from_numpy(d).requires_grad_()
        Rm = C.pose_rotation(dd)
        np.testing.assert_allclose(Rm.detach().numpy(), Rref, atol=1e-6)
        g = torch.autograd.grad((Rm * Gm).sum(), dd)[0]
        np.testing.assert_allclose(g.numpy(), gref, atol=2e-5, rtol=1e-5)


@pytest.mark.parametrize("width", [256, 32])
def test_chain_embeddings_decoder(width):
    z = np.load(os.path.join(G, "chain.npz"))
    xyz = torch.from_numpy(z["xyz"]).requires_grad_()
    feats = bf16_from_bits(z["feats_bf16"]).requires_grad_()
    emb = C.get_embeddings(xyz, torch.from_numpy(z["centre"]), feats, float(z["voxel_size"]))
    np.testing.assert_allclose(emb.detach().numpy(), z[f"w{width}_emb"], atol=1e-7)
    dec = C.Decoder(depth=2, width=width, in_dim=16)
    dec.load_state_dict({k[len(f"w{width}_p_"):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(f"w{width}_p_")})
    sdf = dec(emb)["sdf"]
    np.testing.assert_allclose(sdf.detach().numpy(), z[f"w{width}_sdf"], atol=1e-6)
    grads = torch.autograd.grad((sdf * torch.from_numpy(z[f"w{width}_gout"])).sum(), [xyz, feats] + list(dec.parameters()))
    np.testing.assert_allclose(grads[0].numpy(), z[f"w{width}_dxyz"], atol=1e-5, rtol=1e-5)
    np.testing.assert_allclose(grads[1].float().numpy(), z[f"w{width}_dfeats"], atol=1e-6, rtol=1e-2)
    for (k, _), g in zip(dec.state_dict().items(), grads[2:]):
        np.testing.assert_allclose(g.numpy(), z[f"w{width}_g_{k}"], atol=1e-5, rtol=1e-5)


def test_criterion():
    z = np.load(os.path.join(G, "criterion.npz"))
    rm = torch.from_numpy(z["ray_mask"])[0]
    pts = torch.from_numpy(z["points"])[0][rm]
    cos = torch.from_numpy(z["cos"])[0][rm].view(-1)
    valid = torch.from_numpy(z["valid"])
    sv = torch.from_numpy(z["sdf_valid"]).requires_grad_()
    sdf = torch.ones(valid.shape).masked_scatter(valid, sv)
    loss, parts = C.sdf_loss(torch.from_numpy(z["z"]), sdf, valid, pts, cos, 0.3, 40.0, 1, 10000.0)
    np.testing.assert_allclose(float(loss), float(z["loss"]), rtol=1e-6)
    np.testing.assert_allclose(float(parts["fs_loss"]), float(z["fs_loss"]), rtol=1e-6)
    np.testing.assert_allclose(float(parts["sdf_loss"]), float(z["sdf_loss"]), rtol=1e-6)
    g = torch.autograd.grad(loss, sv)[0]
    np.testing.assert_allclose(g.numpy(), z["grad_sdf"], rtol=1e-5, atol=1e-7)


def test_ray_intersect_and_sample_wrappers():
    """numpy restatement of voxel_helpers.ray_intersect / ray_sample / InverseCDFRaySampling vs the
    reference's own Python wrappers run over the same kernel restatement."""
    z = golden("render.npz")
    vs, md, step = float(z["voxel_size"]), float(z["max_distance"]), float(z["step"])
    m = build_oracle_map(z["vox"], vs, z["id2emb"])
    inter, hits = K.ray_intersect(z["rays_o"], z["rays_d"], m["centres"], m["structure"], vs, 20, md)
    assert np.array_equal(hits, z["hits"])
    assert np.array_equal(inter["intersected_voxel_idx"], z["hit_idx"])
    assert np.array_equal(inter["min_depth"], z["hit_min"]) and np.array_equal(inter["max_depth"], z["hit_max"])
    ih = {k: v[hits] for k, v in inter.items()}
    # torch's reduction order for dists.sum(-1) (reference) vs sequential: compare to 1 ulp-level tolerance,
    # voxel ids exactly
    s = K.ray_sample(dict(ih), step_size=step, fixed=False, noise=z["noise"], sequential_sum=False)
    assert np.array_equal(s["sampled_point_voxel_idx"], z["s_idx"])
    np.testing.assert_allclose(s["sampled_point_depth"], z["s_depth"], rtol=2e-6)
    sd = K.ray_sample(dict(ih), step_size=step, fixed=True, sequential_sum=False)
    assert np.array_equal(sd["sampled_point_voxel_idx"], z["sd_idx"])
    np.testing.assert_allclose(sd["sampled_point_depth"], z["sd_depth"], rtol=2e-6)
    np.testing.assert_allclose(sd["sampled_point_distance"], z["sd_dists"], rtol=1e-3, atol=2e-6)


def test_render_rays_vs_reference():
    z = golden("render.npz")
    vs, md, step = float(z["voxel_size"]), float(z["max_distance"]), float(z["step"])
    m = build_oracle_map(z["vox"], vs, z["id2emb"])
    dec = C.Decoder(depth=2, width=256, in_dim=16)
    dec.load_state_dict({k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("dec_")})
    out = C.render_rays(torch.from_numpy(z["rays_o"]), torch.from_numpy(z["rays_d"]), m, bf16_from_bits(z["emb_bf16"]),
                        dec, step, vs, md, deterministic=False, noise=z["noise"])
    assert np.array_equal(out["valid_mask"].numpy(), z["out_valid"])
    np.testing.assert_allclose(out["z_vals"].numpy(), z["out_z"], rtol=2e-6)
    np.testing.assert_allclose(out["sdf"].detach().numpy(), z["out_sdf"], atol=1e-5)


def _load_mt():
    return golden("mapping_tracking.npz")


@pytest.mark.parametrize("name,upd_dec", [("map", True), ("mapfrozen", False)])
def test_mapping_iterations_vs_reference(name, upd_dec):
    """3 iterations of bundle_adjust_frames: losses, and parameters after Adam, vs the reference run."""
    z = _load_mt()
    vs, md = float(z["voxel_size"]), float(z["max_distance"])
    m = build_oracle_map(z["vox"], vs, z["id2emb"])
    emb = bf16_from_bits(z["emb_bf16"]).clone().requires_grad_()
    dec = C.Decoder(depth=2, width=256, in_dim=16)
    dec.load_state_dict({k[len(name) + 6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(f"{name}_dec0_")})
    poses = [torch.nn.Parameter(torch.from_numpy(p.copy())) for p in z[f"{name}_pose0"]]
    groups = [{"params": [emb], "lr": 0.01}]
    if upd_dec:
        groups.append({"params": list(dec.parameters()), "lr": 0.005})
    for i, p in enumerate(poses):
        if i != 0:
            groups.append({"params": [p], "lr": 0.001})
    opt = torch.optim.Adam(groups)
    cfg = dict(step_size=0.5 * vs, voxel_size=vs, max_distance=md, truncation=0.3, max_depth=40.0, fs_weight=1,
               sdf_weight=10000.0)
    losses = []
    for it in range(3):
        frames = []
        for f in range(3):
            pts = torch.from_numpy(z[f"scan{f}_pts"])
            mask = torch.from_numpy(np.unpackbits(z[f"{name}_mask_it{it}_f{f}"])[:pts.shape[0]].astype(bool))
            dirs = pts / (pts.norm(dim=-1, keepdim=True) + 1e-8)
            frames.append(dict(pose=poses[f], dirs=dirs[mask], points=pts[mask], cos=torch.from_numpy(z[f"scan{f}_cos"])[mask]))
        loss, out = C.mapping_iteration(frames, m, emb, dec, cfg, deterministic=False, noise=z[f"{name}_noise{it}"])
        losses.append(float(loss))
        opt.zero_grad()
        loss.backward()
        opt.step()
    np.testing.assert_allclose(losses, z[f"{name}_loss"], rtol=2e-4)
    np.testing.assert_allclose(np.stack([p.detach().numpy() for p in poses]), z[f"{name}_pose_after"], atol=2e-5)
    e_ref = bf16_from_bits(z[f"{name}_emb_after_bf16"]).float().numpy()
    assert np.mean(np.abs(emb.detach().float().numpy() - e_ref) > 1e-3) < 1e-3
    for k, v in dec.state_dict().items():
        np.testing.assert_allclose(v.numpy(), z[f"{name}_dec_after_{k}"], atol=2e-4)


def test_config0_plumbing_on_cpu():
    """BASELINE.json configs[0]: a 1k-point scan, an 8^3 octree and a 2x32 decoder, entirely on the CPU through the oracle: the chain
    runs end to end, the loss is finite, and its gradient w.r.t. the pose agrees with central finite differences."""
    import torch
    from oracle import chain as OC
    from oracle import kernels as OK
    rng = np.random.default_rng(7)
    n = 1000
    world = np.stack([rng.uniform(1.0, 6.0, n), rng.uniform(1.0, 6.0, n), np.full(n, 2.3) + rng.normal(0, 0.02, n)], -1)
    sensor = np.array([3.5, 3.5, 5.8])
    pts = torch.from_numpy((world - sensor).astype(np.float32))
    vox = np.floor(world.astype(np.float32) / np.float32(1.0)).astype(np.int32)
    tree = OK.Octree()
    tree.init(8, 16, 1.0)
    tree.insert(vox)
    v, c, f = tree.get_centres_and_children()
    centres, structure, vertex = OK.map_arrays(v, c, f, 1.0)
    assert structure[0, 8] == 8 and (structure[:, 8] == 1).sum() == tree.count_leaf_nodes() > 0
    ids = np.unique(vertex[vertex >= 0])
    remap = np.full(int(vertex.max()) + 1, -1, np.int64)
    remap[ids] = np.arange(ids.shape[0])
    rows = np.where(vertex >= 0, remap[np.clip(vertex, 0, None)], -1)
    torch.manual_seed(0)
    emb = (torch.randn(ids.shape[0], 16) * 0.05).requires_grad_()
    dec = OC.Decoder(depth=2, width=32, in_dim=16)
    map_np = {"centres": centres, "structure": structure, "vertex_rows": rows}
    cfg = dict(step_size=0.5, voxel_size=1.0, max_distance=40.0, truncation=0.3, max_depth=40.0, fs_weight=1.0, sdf_weight=10000.0)
    dirs = pts / pts.norm(dim=-1, keepdim=True)
    cos = torch.ones(n)

    def loss_at(p6):
        loss, out = OC.mapping_iteration([dict(pose=p6, dirs=dirs, points=pts, cos=cos)], map_np, emb, dec, cfg, deterministic=True)
        return loss, out
    pose = torch.tensor([3.5, 3.5, 5.8, 0.0, 0.0, 0.0], requires_grad=True)
    loss, out = loss_at(pose)
    assert out is not None and torch.isfinite(loss) and int(out["ray_mask"].sum()) > 0.9 * n
    loss.backward()
    assert emb.grad is not None and torch.isfinite(emb.grad).all() and float(emb.grad.abs().max()) > 0
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in dec.parameters())
    assert pose.grad is not None and torch.isfinite(pose.grad).all() and float(pose.grad.abs().max()) > 0
    # Finite differences against autograd where the chain is differentiable: the embedding table (the ray/voxel intersection and
    # the sampler run without gradient in the reference, voxel_helpers.py:92-137 / :262-344, so d loss / d pose deliberately ignores
    # how the sample depths move with the pose and cannot be checked this way).
    ge = emb.grad.clone()
    flat = ge.abs().flatten()
    for idx in torch.topk(flat, 3).indices.tolist():
        r, cidx = divmod(idx, 16)
        h = 1e-2
        with torch.no_grad():
            emb[r, cidx] += h
            lp, _ = loss_at(pose.detach())
            emb[r, cidx] -= 2 * h
            lm, _ = loss_at(pose.detach())
            emb[r, cidx] += h
        fd = float(lp - lm) / (2 * h)
        assert abs(fd - float(ge[r, cidx])) <= 0.05 * abs(float(ge[r, cidx])) + 1e-3, (r, cidx, fd, float(ge[r, cidx]))
