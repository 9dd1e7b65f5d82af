"""Generate the goldens that need the reference ON THE GPU, by running it there:
  * tests/golden/reference_grid.*.npz   -- its compiled `grid` kernels (svo_intersect, inverse_cdf_sampling) on the inputs of
                                           tests/test_gpu_ops.py;
  * tests/golden/dropin_reference.*.npz -- its bundle_adjust_frames / track_frame / render_rays on the inputs of
                                           tests/test_gpu_dropin_reference.py (the initial decoder is stored too).

What runs is the reference itself as oracle/build_ref.py stages it into oracle/_ref/: its compiled `grid` CUDA extension and
its hot-path Python (render_helpers, Criterion, LidarFrame, OptimizablePose, Decoder), with the sampler noise and sort ties
pinned like every golden (oracle/ref_harness.py:pinned).

Run:  python tests/golden/make_golden_gpu.py      (needs a GPU and oracle/_ref, i.e. a build() where the reference exists;
                                                    NL_GOLDEN_OUT=<dir> writes elsewhere)
"""
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import test_gpu_dropin_reference as T  # noqa: E402
import test_gpu_ops as O  # noqa: E402
from oracle import ref_harness as H  # noqa: E402
from util import golden, product_map, ref_grid, save_golden  # noqa: E402


def grid_outputs():
    g = ref_grid()
    z = golden("render.npz")
    m = product_map(z["vox"], float(z["voxel_size"]), z["id2emb"], z["emb_bf16"])
    vs = float(z["voxel_size"])
    ro, rd, pts, ch = O.scene_rays(z, m)
    out = {}
    for tag, args in (("svo", (ro, rd, pts, ch)), ("svo4", O.batched4(ro, rd, pts, ch))):
        i, a, b = g.svo_intersect(*args, vs, 20)
        out.update({f"{tag}_idx": i.cpu().numpy(), f"{tag}_min": a.cpu().numpy(), f"{tag}_max": b.cpu().numpy()})
    i, d, s = g.inverse_cdf_sampling(*O.icdf_args(z), -1.0)
    out.update(icdf_idx=i.cpu().numpy(), icdf_depth=d.cpu().numpy(), icdf_dist=s.cpu().numpy())
    return out


def dropin_outputs(nl):
    ref = H.load()
    crit = ref.Criterion(H.args(T.MD, T.TR))
    out = {}

    scans, ms0, dec0 = T.state(ref, nl, table_rows=4_000_000)
    out.update({f"dec0_{k}": v.detach().cpu().numpy() for k, v in dec0.state_dict().items()})
    for upd in (True, False):
        ms_r, dec_r, fr_r = T.clone_ms(ms0), copy.deepcopy(dec0), T.make_frames(ref, scans)
        torch.manual_seed(11)
        with H.pinned(ref):
            ref.orig["bundle_adjust_frames"](fr_r, ms_r["voxel_vertex_emb"], ms_r, dec_r, crit, update_decoder=upd, **T.BA_KW)
        torch.cuda.synchronize()
        tag = f"ba{int(upd)}_"
        out[tag + "poses"] = torch.stack([f.pose.data.detach().cpu() for f in fr_r]).numpy()
        out[tag + "emb_bf16"] = T.vertex_emb(ms_r).to(torch.bfloat16).view(torch.int16).numpy()
        if upd:
            out.update({f"{tag}dec_{k}": v.detach().cpu().numpy() for k, v in dec_r.state_dict().items()})
        else:
            assert all(torch.equal(a, b) for a, b in zip(dec_r.state_dict().values(), dec0.state_dict().values()))

    scans, ms0, dec0 = T.state(ref, nl)
    f_r = T.track_input(ref, scans)
    torch.manual_seed(21)
    with H.pinned(ref):
        pose_r, hit_r = ref.orig["track_frame"](copy.deepcopy(f_r.pose), f_r, T.clone_ms(ms0), copy.deepcopy(dec0), crit, **T.TRACK_KW)
    torch.cuda.synchronize()
    out["track_pose"] = pose_r.data.detach().cpu().numpy()
    out["track_hit"] = hit_r.cpu().numpy()

    ro, rd, P, Cn = T.render_input(scans)
    with H.pinned(ref):
        o = ref.orig["render_rays"](ro, rd, T.clone_ms(ms0), copy.deepcopy(dec0), *T.RENDER_ARGS, chunk_size=-1)
        loss, _ = crit(o, P[None], Cn[None, :, None])
    out.update(render_ray_mask=o["ray_mask"].view(-1).cpu().numpy(), render_valid_mask=o["valid_mask"].cpu().numpy(),
               render_z_vals=o["z_vals"].detach().cpu().numpy(), render_sdf=o["sdf"].detach().cpu().numpy(),
               render_loss=np.float64(float(loss)))
    return out


def main():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available() and H.available(), "needs a GPU and the staged reference (oracle/_ref)"
    path = os.environ.get("NL_GOLDEN_OUT", HERE)
    os.makedirs(path, exist_ok=True)
    save_golden(os.path.join(path, "reference_grid.npz"), **grid_outputs())
    save_golden(os.path.join(path, "dropin_reference.npz"), **dropin_outputs(nl))
    print("written to", path)


if __name__ == "__main__":
    main()
