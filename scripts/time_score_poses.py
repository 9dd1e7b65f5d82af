"""score_poses with K = 64, 256, 1024, 4096 hypotheses x 512 rays of the KITTI-shape synthetic scan, against the two other ways of
getting the same losses: ceil(K / 31) one-iteration track_frames calls, and K solo render_rays + Criterion.forward calls.  Whole calls
are timed with a host clock around work that ends in a device synchronise, warmed up first and alternated over repeats.  Then the
decoder alone on the samples of the largest score call: the score kernel (nl_mlp_tc_score_batch) against nl_mlp_tc_train_batch, CUDA
events over many launches, alternated.  Prints the card and its power limit, then one JSON line per K and one for the decoder.

    python scripts/time_score_poses.py [--repeats 5] [--ks 64,256,1024,4096] [--solo-max 4096] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nerfloam_b200 as nl  # noqa: E402
from nerfloam_b200.criterion import Criterion  # noqa: E402
from time_track_batch import _Args, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--ks", default="64,256,1024,4096")
    ap.add_argument("--rays", type=int, default=512)
    ap.add_argument("--solo-max", type=int, default=4096, help="largest K also timed as K solo render_rays calls")
    ap.add_argument("--kernel-reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_score_poses.py measures on the GPU; none found")
    dev = torch.device("cuda")
    syn = nl.synthetic
    pts, cos, pose = syn.make_scan()                     # KITTI shape: 64 beams x 1563 azimuths
    mu = nl.mapping.MapUpdater(0.3, init_std=0.02, seed=1)
    ms = mu.insert_voxels(torch.from_numpy(syn.voxelize(pts, pose, 0.3)))
    torch.manual_seed(0)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    crit = Criterion(_Args())
    guess = nl.se3pose.OptimizablePose.from_matrix(torch.from_numpy(pose).float())
    fr = nl.frame.LidarFrame(5, torch.from_numpy(pts), torch.from_numpy(cos), nl.se3pose.OptimizablePose(guess.data.detach().clone()),
                             new_keyframe=True)
    N = a.rays
    ids = torch.randperm(pts.shape[0])[:N].sort().values
    kw = dict(step_size=0.15, max_distance=40.0)
    lattice = nl.score.yaw_lattice(guess, 3.14159 / 6, 64, 2.0, 8)            # 4097 hypotheses around the true pose
    dirs = nl.render_helpers._frame_arrays(fr, dev)[0][ids.to(dev)].contiguous()
    obs, pcos = fr.points[ids].to(dev).view(1, -1, 3), fr.pointsCos[ids].to(dev).view(1, -1)

    def score(K):
        return nl.score_poses(lattice[:K], fr, ms, dec, crit, 0.3, N, ray_ids=ids, **kw)

    def track(K):
        for k0 in range(0, K, 31):
            starts = [nl.se3pose.OptimizablePose(lattice[k].clone()) for k in range(k0, min(K, k0 + 31))]
            nl.track_frames(starts, [fr] * len(starts), ms, dec, crit, 0.3, N_rays=N, num_iterations=1, truncation=0.3, learning_rate=0.01,
                            max_voxel_hit=20, **kw)

    def solo(K):
        p6 = lattice[:K].to(dev)
        for k in range(K):
            ro, rd = nl.score.rays_of_poses(p6[k:k + 1], dirs)
            out = nl.render_helpers.render_rays(ro[None], rd[None], ms, dec, 0.15, 0.3, 0.3, 20, 40.0)
            if out is not None:
                crit(out, obs, pcos)

    dev_card = card()
    print("card:", dev_card, flush=True)
    rows = []
    for K in [int(x) for x in a.ks.split(",")]:
        variants = {"score": lambda: score(K), "track_frames": lambda: track(K)}
        if K <= a.solo_max:
            variants["solo"] = lambda: solo(K)
        for f in variants.values():              # warm-up: engines, captures, frame uploads
            f()
        times = {n: [] for n in variants}
        for _ in range(a.repeats if K <= 1024 else max(1, a.repeats // 2)):
            for n, f in variants.items():        # alternated
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                f()
                torch.cuda.synchronize()
                times[n].append((time.perf_counter() - t0) * 1e3)
        row = dict(K=K, rays=N, card=dev_card)
        for n, t in times.items():
            row[n + "_ms"] = round(statistics.median(t), 3)
            row[n + "_min_max_ms"] = [round(min(t), 3), round(max(t), 3)]
        row["speedup_vs_track_frames"] = round(row["track_frames_ms"] / row["score_ms"], 2)
        if "solo_ms" in row:
            row["speedup_vs_solo"] = round(row["solo_ms"] / row["score_ms"], 2)
        print(json.dumps(row), flush=True)
        rows.append(row)

    # ---- the decoder alone, on the samples the last score call left in its engine (its last chunk) ----
    res = score(max(int(x) for x in a.ks.split(",")))
    eng = nl.score._ENGINES[str(dev)]
    st = eng.read_stats()
    bufs = nl.engine.DecoderBuffers.of(dec, dev)
    bufs.refresh_transposes()
    lib, sp, ptr = nl._capi.lib(), nl._capi.stream_ptr(), nl._capi.ptr
    p = bufs.params
    R = eng.max_rays
    gt_r = torch.ones(R, device=dev)
    cos_r = torch.ones(R, device=dev)
    K_last = int(res.loss.shape[0])
    pst = torch.zeros((K_last, nl.engine.STATS_BYTES), dtype=torch.uint8, device=dev)
    M = st.n_samples

    def k_score():
        nl._capi.check(lib.nl_mlp_tc_score_batch(M, None, ptr(eng.feats), ptr(bufs.tc_panels), ptr(p[1]), ptr(p[3]), ptr(p[4]), ptr(p[5]),
                                                 ptr(eng.s_flag), ptr(eng.s_depth), ptr(eng.s_ray), ptr(cos_r), ptr(gt_r), ptr(pst), N, 0.3,
                                                 ptr(eng.sdf), sp), "nl_mlp_tc_score_batch")

    def k_train():
        nl._capi.check(lib.nl_mlp_tc_train_batch(M, None, ptr(eng.feats), ptr(bufs.tc_panels), ptr(p[1]), ptr(p[3]), ptr(p[4]), ptr(p[5]),
                                                 ptr(eng.s_flag), ptr(eng.s_depth), ptr(eng.s_ray), ptr(cos_r), ptr(gt_r), ptr(pst), N, 0.3,
                                                 ptr(eng.sdf), ptr(eng.dfeats), sp), "nl_mlp_tc_train_batch")
    kern = {"score_kernel": k_score, "train_batch_kernel": k_train}
    for f in kern.values():
        f(); f()
    ktimes = {n: [] for n in kern}
    for _ in range(5):
        for n, f in kern.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.kernel_reps):
                f()
            e1.record()
            torch.cuda.synchronize()
            ktimes[n].append(e0.elapsed_time(e1) / a.kernel_reps * 1e3)
    krow = dict(decoder_samples=int(M), card=dev_card)
    for n, t in ktimes.items():
        krow[n + "_us"] = round(statistics.median(t), 1)
        krow[n + "_min_max_us"] = [round(min(t), 1), round(max(t), 1)]
    krow["score_kernel_speedup"] = round(krow["train_batch_kernel_us"] / krow["score_kernel_us"], 2)
    print(json.dumps(krow), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_score_poses.json"), "w") as fh:
            json.dump({"calls": rows, "decoder": krow}, fh, indent=1)


if __name__ == "__main__":
    main()
