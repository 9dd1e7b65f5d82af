"""Generate tests/golden/*.npz by EXECUTING THE REFERENCE in this container (CPU only).

What runs here is the reference's own code, imported / compiled from /root/reference:
  * the compiled, unmodified `svo` octree (oracle/_ref/svo, see oracle/build_ref.py);
  * the reference Python: variations.render_helpers (render_rays, bundle_adjust_frames, track_frame,
    get_embeddings ...), variations.voxel_helpers (ray_intersect, ray_sample and the autograd.Function
    wrappers), variations.lidar.Decoder, criterion.Criterion, se3pose.OptimizablePose,
    lidarFrame.LidarFrame, utils.sample_util.
Two things are substituted, because the reference needs a GPU for them:
  * the `grid` CUDA extension is replaced by a stub that forwards the two live kernels
    (svo_intersect, inverse_cdf_sampling) to oracle/nl_oracle.c -- the kernel restatement that is
    separately pinned against the real compiled `grid` on the GPU box;
  * torch.Tensor.cuda / Module.cuda are made no-ops so the reference's hard-coded .cuda() calls run on CPU;
  * Tensor.sort is forced to stable=True (the reference's tie order among equal min_depth is unspecified).
Everything else -- batching/padding wrappers, sorting, masking, trilinear interpolation, decoder,
loss, autograd, torch.optim.Adam -- is the reference itself.

Run:  python tests/golden/make_golden.py        (needs /root/reference; writes tests/golden/*.npz)
"""
import importlib
import os
import sys
import types
from copy import deepcopy

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("NERFLOAM_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(REF, "src"))

from oracle import kernels as OK  # noqa: E402

sys.path.insert(0, os.path.dirname(HERE))
from util import save_golden  # noqa: E402

syn = importlib.import_module("nerf-loam_b200.synthetic")

# ---------------------------------------------------------------- substitutions
RECORD = {"noise": [], "loss": [], "sample_mask": []}


def _svo_intersect(ray_start, ray_dir, points, children, voxelsize, n_max):
    B, Kr = ray_start.shape[:2]
    idx, mn, mx = OK.svo_intersect(ray_start.reshape(-1, 3).numpy(), ray_dir.reshape(-1, 3).numpy(),
                                   points[0].numpy(), children[0].numpy(), voxelsize, n_max)
    f = lambda a: torch.from_numpy(a).reshape(B, Kr, n_max)
    return f(idx), f(mn), f(mx)


def _inverse_cdf_sampling(pts_idx, min_depth, max_depth, noise, probs, steps, fixed_step_size):
    RECORD["noise"].append(noise.numpy().copy())
    b, nr, P = pts_idx.shape
    S = noise.shape[-1]
    si = np.empty((b, nr, S), np.int32)
    sd = np.empty((b, nr, S), np.float32)
    sl = np.empty((b, nr, S), np.float32)
    a = [np.ascontiguousarray(x.numpy()) for x in (pts_idx, min_depth, max_depth, noise, probs, steps)]
    OK.lib().nlo_inverse_cdf_sampling(b, nr, P, S, float(fixed_step_size), OK._p(a[0]), OK._p(a[1]), OK._p(a[2]),
                                      OK._p(a[3]), OK._p(a[4]), OK._p(a[5]), OK._p(si), OK._p(sd), OK._p(sl))
    return torch.from_numpy(si), torch.from_numpy(sd), torch.from_numpy(sl)


grid_stub = types.ModuleType("grid")
grid_stub.svo_intersect = _svo_intersect
grid_stub.inverse_cdf_sampling = _inverse_cdf_sampling
sys.modules["grid"] = grid_stub
torch.Tensor.cuda = lambda self, *a, **k: self
torch.nn.Module.cuda = lambda self, *a, **k: self
torch.cuda.empty_cache = lambda: None
# voxel_helpers.py:546 sorts hits by min_depth with torch.sort's default (unstable) algorithm.  Rays that
# graze a voxel edge enter several voxels at bit-identical depths, so the reference's own order of those
# ties depends on the torch version/device.  The goldens pin the stable order (ties keep DFS emission order).
_orig_sort = torch.Tensor.sort
torch.Tensor.sort = lambda self, dim=-1, descending=False: _orig_sort(self, stable=True, dim=dim, descending=descending)

from variations import render_helpers as RH  # noqa: E402
from variations import voxel_helpers as VH  # noqa: E402
from variations.lidar import Decoder  # noqa: E402
from criterion import Criterion  # noqa: E402
from se3pose import OptimizablePose  # noqa: E402
from lidarFrame import LidarFrame  # noqa: E402

SVO_SO = os.path.join(ROOT, "oracle", "_ref", "svo", "svo_ref.so")


def run_ref_svo(inserts, grid_dim, voxel_size, emb_dim=16):
    """Run the compiled reference `svo` in a FRESH process (its node counter Octant::next_index_ is a
    process-global, octree.h:62, so only one octree per process gives valid indices).
    Returns a list with (voxels, children, features, count_nodes, count_leaf_nodes) after each insert."""
    import subprocess
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        fi, fo = os.path.join(td, "in.npz"), os.path.join(td, "out.npz")
        np.savez(fi, grid_dim=grid_dim, voxel_size=voxel_size, emb_dim=emb_dim, **{f"ins{i}": v for i, v in enumerate(inserts)})
        subprocess.check_call([sys.executable, os.path.abspath(__file__), "--svo-worker", fi, fo])
        z = np.load(fo)
        return [(z[f"voxels{i}"], z[f"children{i}"], z[f"features{i}"], int(z[f"count{i}"][0]), int(z[f"count{i}"][1]))
                for i in range(len(inserts))]


def _svo_worker(fi, fo):
    torch.classes.load_library(SVO_SO)
    z = np.load(fi)
    svo = torch.classes.svo.Octree()
    svo.init(int(z["grid_dim"]), int(z["emb_dim"]), float(z["voxel_size"]))
    out = {}
    i = 0
    while f"ins{i}" in z:
        svo.insert(torch.from_numpy(z[f"ins{i}"]))
        a = [t.numpy().copy() for t in svo.get_centres_and_children()]
        out[f"voxels{i}"], out[f"children{i}"], out[f"features{i}"] = a
        out[f"count{i}"] = np.array([svo.count_nodes(), svo.count_leaf_nodes()])
        i += 1
    np.savez(fo, **out)


def bf16_bits(t):
    return t.detach().contiguous().view(torch.int16).numpy().copy()


def build_map(voxel_coords, voxel_size, grid_dim=256 * 256 * 4, emb_dim=16, seed=0):
    """reference svo + mapping.py:294-339 glue (mapping.py itself needs open3d, so its few lines of
    tensor glue are reproduced here; rows are allocated once per distinct vertex, see SURVEY A.1)."""
    voxels, children, features = [torch.from_numpy(a) for a in run_ref_svo([voxel_coords], grid_dim, voxel_size)[0][:3]]
    centres = ((voxels[:, :3] + voxels[:, -1:] / 2) * voxel_size).float()
    structure = torch.cat([children, voxels[:, -1:]], -1).int()
    flat = features.reshape(-1).long()
    valid = flat[flat.ne(-1)]
    uniq, first = np.unique(valid.numpy(), return_index=True)
    order = uniq[np.argsort(first)]                      # first-appearance order
    id2emb = -torch.ones((voxels.shape[0], 1), dtype=torch.int)
    id2emb[torch.from_numpy(order)] = torch.arange(len(order), dtype=torch.int).view(-1, 1)
    g = torch.Generator().manual_seed(seed)
    emb = (torch.randn(len(order), emb_dim, generator=g) * 0.01).to(torch.bfloat16)
    return dict(voxels=voxels, children=children, features=features, centres=centres, structure=structure,
                id2emb=id2emb, emb=emb)


def golden_octree():
    pts, cos, pose = syn.make_scan(n_beams=16, n_az=128, seed=777)
    v1 = syn.voxelize(pts, pose, 0.3)
    pts2, _, pose2 = syn.make_scan(n_beams=16, n_az=128, seed=778, sensor_xyz=(1.0, 0.2, 0.0))
    v2 = syn.voxelize(pts2, pose2, 0.3)
    (a0, a1, a2, n1, l1), (b0, b1, b2, n2, l2) = run_ref_svo([v1, v2], 256 * 256 * 4, 0.3)
    np.savez_compressed(os.path.join(HERE, "octree.npz"), v1=v1, v2=v2, voxels1=a0, children1=a1, features1=a2,
                        voxels2=b0, children2=b1, features2=b2, count1=np.array([n1, l1]), count2=np.array([n2, l2]))
    print("octree.npz", a0.shape, b0.shape)


def golden_octree_small():
    """8^3 octree (config 0).  Must run in a process where Octant::next_index_ is still 0 -> called first."""
    rng = np.random.default_rng(5)
    v0 = rng.integers(0, 7, size=(40, 3)).astype(np.int32)
    (a0, a1, a2, n, l), = run_ref_svo([v0], 8, 1.0)
    np.savez_compressed(os.path.join(HERE, "octree_8.npz"), v0=v0, voxels=a0, children=a1, features=a2, count=np.array([n, l]))
    print("octree_8.npz", a0.shape)


def golden_pose():
    before = torch.tensor([[-0.955421, 0.119616, - 0.269932, 2.655830],
                           [0.295248, 0.388339, - 0.872939, 2.981598],
                           [0.000408, - 0.913720, - 0.406343, 1.368648],
                           [0.000000, 0.000000, 0.000000, 1.000000]])   # se3pose.py:96-99
    pose = OptimizablePose.from_matrix(before)
    R = pose.rotation()
    after = pose.matrix()
    # gradient of a fixed linear functional of R,t w.r.t. the 6-vector
    g = torch.Generator().manual_seed(3)
    G = torch.randn(3, 3, generator=g)
    gt = torch.randn(3, generator=g)
    val = (pose.rotation() * G).sum() + (pose.translation() * gt).sum()
    grad = torch.autograd.grad(val, pose.data)[0]
    datas = torch.randn(8, 6, generator=g) * torch.tensor([10, 10, 10, 0.5, 0.5, 0.5])
    Rs, grads = [], []
    for d in datas:
        p = OptimizablePose(d.clone())
        Rs.append(p.rotation().detach().numpy())
        grads.append(torch.autograd.grad((p.rotation() * G).sum(), p.data)[0].numpy())
    np.savez_compressed(os.path.join(HERE, "pose.npz"), before=before.numpy(), data=pose.data.detach().numpy(),
                        R=R.detach().numpy(), after=after.detach().numpy(), G=G.numpy(), gt=gt.numpy(),
                        grad=grad.numpy(), datas=datas.numpy(), Rs=np.stack(Rs), grads=np.stack(grads))
    print("pose.npz")


def golden_chain():
    """get_embeddings + Decoder forward/backward on seeded inputs (reference functions, CPU)."""
    g = torch.Generator().manual_seed(11)
    M, E = 300, 16
    voxel_size = 0.3
    centre = (torch.randint(6000, 7000, (M, 3), generator=g).float() + 0.5) * voxel_size
    xyz = (centre + (torch.rand(M, 3, generator=g) - 0.5) * voxel_size).requires_grad_()
    feats = (torch.randn(M, 8 * E, generator=g) * 0.05).to(torch.bfloat16).requires_grad_()
    out = {}
    for width in (256, 32):
        torch.manual_seed(777)
        dec = Decoder(depth=2, width=width, in_dim=E, skips=[], embedder="none", multires=0)
        emb = RH.get_embeddings(xyz, centre, feats, voxel_size)
        sdf = dec(emb)["sdf"]
        gout = torch.randn(M, 1, generator=torch.Generator().manual_seed(5))
        params = list(dec.parameters())
        grads = torch.autograd.grad((sdf * gout).sum(), [xyz, feats] + params)
        out[f"w{width}_emb"] = emb.detach().numpy()
        out[f"w{width}_sdf"] = sdf.detach().numpy()
        out[f"w{width}_gout"] = gout.numpy()
        out[f"w{width}_dxyz"] = grads[0].numpy()
        out[f"w{width}_dfeats"] = grads[1].float().numpy()
        for (k, v), gr in zip(dec.state_dict().items(), grads[2:]):
            out[f"w{width}_p_{k}"] = v.numpy()
            out[f"w{width}_g_{k}"] = gr.numpy()
    np.savez_compressed(os.path.join(HERE, "chain.npz"), centre=centre.numpy(), xyz=xyz.detach().numpy(),
                        feats_bf16=bf16_bits(feats), voxel_size=np.float32(voxel_size), **out)
    print("chain.npz")


def make_args(voxel_size=0.3, max_depth=40.0, trunc=0.3):
    a = types.SimpleNamespace()
    a.criteria = {"eiko_weight": 0.1, "sdf_weight": 10000.0, "fs_weight": 1, "sdf_truncation": trunc}
    a.data_specs = {"max_depth": max_depth}
    return a


def golden_criterion():
    g = torch.Generator().manual_seed(21)
    R, Rh, S = 300, 260, 14
    ray_mask = torch.zeros(1, R, dtype=torch.bool)
    ray_mask[0, torch.randperm(R, generator=g)[:Rh]] = True
    points = torch.randn(1, R, 3, generator=g) * torch.tensor([10.0, 6.0, 1.0])
    cos = torch.rand(1, R, 1, generator=g).clamp(min=0.05)
    cos[0, ::3] = 1.0
    depth = points[ray_mask].norm(dim=-1)
    z = (depth[:, None] + (torch.rand(Rh, S, generator=g) - 0.6) * 2.0)
    nvalid = torch.randint(1, S + 1, (Rh,), generator=g)
    nvalid[0] = S
    valid = torch.arange(S)[None, :] < nvalid[:, None]
    z = torch.where(valid, z, torch.full_like(z, 80.0))
    sdf_v = (torch.randn(int(valid.sum()), generator=g) * 0.3).requires_grad_()
    sdf = torch.ones(Rh, S).masked_scatter(valid, sdf_v)
    crit = Criterion(make_args())
    loss, ld = crit({"sdf": sdf, "z_vals": z, "ray_mask": ray_mask, "valid_mask": valid, "sampled_xyz": None},
                    points, cos)
    gsdf = torch.autograd.grad(loss, sdf_v)[0]
    np.savez_compressed(os.path.join(HERE, "criterion.npz"), ray_mask=ray_mask.numpy(), points=points.numpy(),
                        cos=cos.numpy(), z=z.numpy(), valid=valid.numpy(), sdf_valid=sdf_v.detach().numpy(),
                        loss=loss.detach().numpy(), fs_loss=np.float32(ld["fs_loss"]), sdf_loss=np.float32(ld["sdf_loss"]),
                        grad_sdf=gsdf.numpy())
    print("criterion.npz", float(loss))


def small_scene(voxel_size=0.3):
    pts, cos, pose = syn.make_scan(n_beams=24, n_az=160, seed=777)
    vox = syn.voxelize(pts, pose, voxel_size)
    return pts, cos, pose, vox


def golden_render():
    """ray_intersect / ray_sample (reference wrappers over the stubbed kernels) and render_rays."""
    voxel_size, max_distance, step = 0.3, 40.0, 0.5 * 0.3
    pts, cos, pose, vox = small_scene(voxel_size)
    m = build_map(vox, voxel_size)
    torch.manual_seed(777)
    dec = Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0)
    P = torch.from_numpy(pts)
    dirs = P / (P.norm(dim=-1, keepdim=True) + 1e-8)
    Rm = torch.from_numpy(pose[:3, :3])
    rays_d = (dirs @ Rm.T)[None].contiguous()
    rays_o = torch.from_numpy(pose[:3, 3]).reshape(1, 1, 3).expand_as(rays_d).contiguous()
    inter, hits = VH.ray_intersect(rays_o, rays_d, m["centres"], m["structure"], voxel_size, 20, max_distance)
    inter_h = {k: v[hits.view(1, -1)].reshape(-1, v.size(-1)) for k, v in inter.items()}
    RECORD["noise"].clear()
    torch.manual_seed(123)
    samples = VH.ray_sample(dict(inter_h), step_size=step)          # stochastic (fixed=False)
    noise = RECORD["noise"][0].copy()
    assert len(RECORD["noise"]) == 1
    samples_det = VH.ray_sample(dict(inter_h), step_size=step, fixed=True)
    map_states = {"voxel_vertex_idx": m["features"], "voxel_center_xyz": m["centres"], "voxel_structure": m["structure"],
                  "voxel_vertex_emb": m["emb"], "voxel_id2embedding_id": m["id2emb"]}
    RECORD["noise"].clear()
    torch.manual_seed(123)
    out = RH.render_rays(rays_o, rays_d, map_states, dec, step, voxel_size, 0.3, 20, max_distance, chunk_size=-1)
    assert np.array_equal(RECORD["noise"][0], noise)
    save_golden(
        os.path.join(HERE, "render.npz"), vox=vox, pts=pts, cos=cos, pose=pose, voxel_size=np.float32(voxel_size),
        max_distance=np.float32(max_distance), step=np.float32(step), emb_bf16=bf16_bits(m["emb"]),
        id2emb=m["id2emb"].numpy(), rays_o=rays_o[0].numpy(), rays_d=rays_d[0].numpy(),
        hit_idx=inter["intersected_voxel_idx"][0].numpy(), hit_min=inter["min_depth"][0].numpy(),
        hit_max=inter["max_depth"][0].numpy(), hits=hits[0].numpy(), noise=noise,
        s_idx=samples["sampled_point_voxel_idx"].numpy(), s_depth=samples["sampled_point_depth"].numpy(),
        s_dists=samples["sampled_point_distance"].numpy(), sd_idx=samples_det["sampled_point_voxel_idx"].numpy(),
        sd_depth=samples_det["sampled_point_depth"].numpy(), sd_dists=samples_det["sampled_point_distance"].numpy(),
        probs=inter_h["probs"].numpy() if "probs" in inter_h else np.zeros(0), out_z=out["z_vals"].numpy(),
        out_sdf=out["sdf"].detach().numpy(), out_valid=out["valid_mask"].numpy(), out_ray_mask=out["ray_mask"].numpy(),
        **{"dec_" + k: v.numpy() for k, v in dec.state_dict().items()})
    print("render.npz rays", rays_d.shape, "hits", int(hits.sum()), "z", tuple(out["z_vals"].shape))


class RecCriterion(Criterion):
    def forward(self, *a, **k):
        loss, d = super().forward(*a, **k)
        RECORD["loss"].append(float(loss))
        return loss, d


def _patch_frame_sampling():
    orig = LidarFrame.sample_rays

    def rec(self, N_rays, track=False):
        orig(self, N_rays, track)
        RECORD["sample_mask"].append(self.sample_mask.numpy().copy())
    LidarFrame.sample_rays = rec


def golden_mapping_tracking():
    voxel_size, max_distance = 0.3, 40.0
    _patch_frame_sampling()
    scans = []
    for i in range(3):
        pts, cos, pose = syn.make_scan(n_beams=24, n_az=160, seed=777 + i, sensor_xyz=(0.8 * i, 0.05 * i, 0.0),
                                       yaw=0.01 * i)
        scans.append((pts, cos, pose))
    vox = np.concatenate([syn.voxelize(p, T, voxel_size) for p, c, T in scans])
    m = build_map(vox, voxel_size, seed=4)
    crit = RecCriterion(make_args())
    out = {}
    for name, upd_dec in (("map", True), ("mapfrozen", False)):
        torch.manual_seed(777)
        dec = Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0)
        dec0 = {k: v.numpy().copy() for k, v in dec.state_dict().items()}
        emb = m["emb"].clone().requires_grad_()
        map_states = {"voxel_vertex_idx": m["features"], "voxel_center_xyz": m["centres"],
                      "voxel_structure": m["structure"], "voxel_vertex_emb": emb, "voxel_id2embedding_id": m["id2emb"]}
        frames = []
        for i, (pts, cos, pose) in enumerate(scans):
            T = pose.copy().astype(np.float64)
            T[:3, 3] -= 2000.0                                    # LidarFrame adds the offset back (lidarFrame.py:18)
            T[:3, 3] += np.array([0.05, -0.03, 0.02]) * i        # perturb so pose gradients are non-trivial
            frames.append(LidarFrame(i, torch.from_numpy(pts), torch.from_numpy(cos), T))
        pose0 = np.stack([f.pose.data.detach().numpy().copy() for f in frames])
        for k in RECORD:
            RECORD[k].clear()
        torch.manual_seed(2024)
        n_it = 3
        RH.bundle_adjust_frames(frames, emb, map_states, dec, crit, voxel_size, 0.5 * voxel_size, N_rays=256,
                                num_iterations=n_it, truncation=0.3, max_voxel_hit=20, max_distance=max_distance,
                                learning_rate=[0.01, 0.005, 0.001], update_pose=True, update_decoder=upd_dec)
        out.update({f"{name}_loss": np.array(RECORD["loss"], np.float64),
                    f"{name}_emb_after_bf16": bf16_bits(emb), f"{name}_pose0": pose0,
                    f"{name}_pose_after": np.stack([f.pose.data.detach().numpy() for f in frames])})
        for i, nz in enumerate(RECORD["noise"]):
            out[f"{name}_noise{i}"] = nz
        assert len(RECORD["sample_mask"]) == n_it * len(frames)
        for i, mk in enumerate(RECORD["sample_mask"]):          # order: iteration-major, frame-minor
            out[f"{name}_mask_it{i // len(frames)}_f{i % len(frames)}"] = np.packbits(mk.reshape(-1))
        for k, v in dec.state_dict().items():
            out[f"{name}_dec0_{k}"] = dec0[k]
            out[f"{name}_dec_after_{k}"] = v.numpy().copy()
        assert len(RECORD["noise"]) == n_it, len(RECORD["noise"])
        print(name, "losses", RECORD["loss"])

    # ---- tracking: 3 iterations of track_frame on scan 1 with a perturbed initial pose
    torch.manual_seed(777)
    dec = Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0)
    pts, cos, pose = scans[1]
    T = pose.copy().astype(np.float64)
    T[:3, 3] -= 2000.0
    T[:3, 3] += np.array([0.06, -0.04, 0.01])
    frame = LidarFrame(1, torch.from_numpy(pts), torch.from_numpy(cos), T)
    map_states = {"voxel_vertex_idx": m["features"], "voxel_center_xyz": m["centres"], "voxel_structure": m["structure"],
                  "voxel_vertex_emb": m["emb"].clone(), "voxel_id2embedding_id": m["id2emb"]}
    for k in RECORD:
        RECORD[k].clear()
    torch.manual_seed(99)
    pose_in = deepcopy(frame.pose)
    pose_out, hit_mask = RH.track_frame(pose_in, frame, map_states, dec, crit, voxel_size, N_rays=256,
                                        step_size=0.2 * voxel_size, num_iterations=3, truncation=0.3,
                                        learning_rate=0.06, max_voxel_hit=20, max_distance=max_distance)
    out.update(track_loss=np.array(RECORD["loss"], np.float64), track_masks=np.stack([np.packbits(mk.reshape(-1)) for mk in RECORD["sample_mask"]]),
               track_pose0=frame.pose.data.detach().numpy().copy(), track_pose_after=pose_out.data.detach().numpy(),
               track_hit_mask=hit_mask.numpy())
    for i, nz in enumerate(RECORD["noise"]):
        out[f"track_noise{i}"] = nz
    print("track losses", RECORD["loss"])
    save_golden(
        os.path.join(HERE, "mapping_tracking.npz"), vox=vox, voxel_size=np.float32(voxel_size),
        max_distance=np.float32(max_distance), emb_bf16=bf16_bits(m["emb"]), id2emb=m["id2emb"].numpy(),
        **{f"scan{i}_pts": s[0] for i, s in enumerate(scans)}, **{f"scan{i}_cos": s[1] for i, s in enumerate(scans)},
        **{f"scan{i}_pose": s[2] for i, s in enumerate(scans)}, **out)
    print("mapping_tracking.npz")


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--svo-worker":
        _svo_worker(sys.argv[2], sys.argv[3])
        sys.exit(0)
    which = sys.argv[1:] or ["octree8", "octree", "pose", "chain", "criterion", "render", "maptrack"]
    if "octree8" in which:
        golden_octree_small()
    if "octree" in which:
        golden_octree()
    if "pose" in which:
        golden_pose()
    if "chain" in which:
        golden_chain()
    if "criterion" in which:
        golden_criterion()
    if "render" in which:
        golden_render()
    if "maptrack" in which:
        golden_mapping_tracking()
