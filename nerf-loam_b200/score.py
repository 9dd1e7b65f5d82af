"""score_poses: the tracking loss of K pose hypotheses of ONE scan against a frozen map and decoder, forward only, in one launch chain
per chunk of hypotheses; relocalise: a yaw x translation search around a guess, scored here and refined with track_frames.

A lost scan (track_frame hits nothing or converges to a wrong pose) is never recovered by the reference: it prints "Restarting!!" and
keeps the constant-velocity guess (src/tracking.py:136-137).  The same gap appears when a scan is localised against a saved map with only
a rough prior.  A useful search scores hundreds to thousands of poses; track_frames takes at most 31 and runs full optimisations.  Here
hypothesis k owns rays [k N, (k+1) N) of a chunk, exactly as a track_frames problem does (include/nerfloam_b200.h section 3b), and every
hypothesis uses the same N rays and the same sampling noise, so scores differ only because the poses differ.
"""
import ctypes as C
from collections import namedtuple

import numpy as np
import torch

from . import _capi
from . import render_helpers as rh
from ._capi import BatchArgs, RenderStats
from .engine import STATS_BYTES, DecoderBuffers, MapState, SDFEngine, mlp_impl
from .se3pose import OptimizablePose

# initial sample capacity per ray; a chunk that exceeds it is redone on a larger engine
SAMPLES_PER_RAY_SCORE = 32
_HIT_WORD, _NSAMP_WORD = RenderStats.n_hit_rays.offset // 4, RenderStats.n_samples.offset // 4

ScoreResult = namedtuple("ScoreResult", ["loss", "hit_rays", "n_samples", "ray_ids"])
ScoreResult.__doc__ = """score_poses' result, all on the device: loss f32[K] (NaN where render_rays would return None), hit_rays i32[K],
n_samples i32[K], ray_ids i32[N] (the scan points every hypothesis used)."""

_ENGINES = {}


def _engine(R, cap, dev):
    """One engine per device, replaced by a larger one when a call needs more rays or samples."""
    e = _ENGINES.get(str(dev))
    if e is None or e.max_rays < R or e.max_samples < cap:
        _ENGINES.pop(str(dev), None)
        e = _ENGINES[str(dev)] = SDFEngine(R, cap, dev)
    return e


def _pose_tensor(frame_poses):
    if isinstance(frame_poses, torch.Tensor):
        p = frame_poses
    else:
        p = [fp.data.detach().reshape(-1) if isinstance(fp, OptimizablePose) else torch.as_tensor(fp).reshape(-1) for fp in frame_poses]
        p = torch.stack([x.float().cpu() for x in p]) if p else torch.zeros((0, 6))
    if p.dim() != 2 or p.shape[1] != 6:
        raise ValueError(f"score_poses: frame_poses must be [K,6] or a list of OptimizablePose, got shape {tuple(p.shape)}")
    K = p.shape[0]
    if not 1 <= K <= _capi.SCORE_MAX_PROBLEMS:
        raise ValueError(f"score_poses: 1 <= number of poses <= {_capi.SCORE_MAX_PROBLEMS}, got {K}")
    return p


def _decoder(eng, bufs, cfg, gt, cos, pstats_ptr, N):
    """Sdf of every sample and each hypothesis' squared-error sums (no weight gradients)."""
    lib, st = _capi.lib(), _capi.stream_ptr()
    if mlp_impl(bufs.width) == "tc":
        p = bufs.params
        _capi.check(lib.nl_mlp_tc_score_batch(eng.max_samples, eng.n_samples_dev, _capi.ptr(eng.feats), _capi.ptr(bufs.tc_panels), _capi.ptr(p[1]),
                                              _capi.ptr(p[3]), _capi.ptr(p[4]), _capi.ptr(p[5]), _capi.ptr(eng.s_flag), _capi.ptr(eng.s_depth),
                                              _capi.ptr(eng.s_ray), _capi.ptr(cos), _capi.ptr(gt), pstats_ptr, N, float(cfg["truncation"]),
                                              _capi.ptr(eng.sdf), st), "nl_mlp_tc_score_batch")
    else:                                  # the CUDA-core kernel; its d feats go to the engine's scratch
        w = bufs.weights_struct()
        _capi.check(lib.nl_mlp_train_batch(eng.max_samples, eng.n_samples_dev, _capi.ptr(eng.feats), C.byref(w), _capi.ptr(eng.s_flag),
                                           _capi.ptr(eng.s_depth), _capi.ptr(eng.s_ray), _capi.ptr(cos), _capi.ptr(gt), pstats_ptr, N,
                                           float(cfg["truncation"]), _capi.ptr(eng.sdf), _capi.ptr(eng.dfeats), st), "nl_mlp_train_batch")
    _capi.LAUNCHES += 1


def _select(frame, N_rays, ray_ids, dev):
    """The scan's rays used by every hypothesis: ray_ids, or one nl_select_rays draw (CUDA generator) -> (ids, dirs, gt, cos)."""
    dirs_all, cos_all, gt_all = rh._frame_arrays(frame, dev)
    n_pts = dirs_all.shape[0]
    if ray_ids is not None:
        ids = torch.as_tensor(ray_ids).to(dev, torch.int32).reshape(-1).contiguous()
        if ids.numel() == 0 or int(ids.min()) < 0 or int(ids.max()) >= n_pts:
            raise ValueError(f"score_poses: ray_ids must be non-empty indices into the scan's {n_pts} points")
        il = ids.long()
        return ids, dirs_all[il].contiguous(), gt_all[il].contiguous(), cos_all[il].contiguous()
    N = int(N_rays)
    ids = torch.empty(N, dtype=torch.int32, device=dev)
    dirs, gt, cos = (torch.empty((N, 3), device=dev), torch.empty(N, device=dev), torch.empty(N, device=dev))
    n_dev = torch.full((1,), n_pts, dtype=torch.int64, device=dev)
    _capi.check(_capi.lib().nl_select_rays(1, n_pts, N, _capi.ptr(n_dev), _capi.ptr(rh._seed_from_cuda(dev)), 0, _capi.ptr(dirs_all),
                                           _capi.ptr(gt_all), _capi.ptr(cos_all), _capi.ptr(dirs), _capi.ptr(gt), _capi.ptr(cos), _capi.ptr(ids),
                                           _capi.stream_ptr()), "nl_select_rays")
    _capi.LAUNCHES += 1
    return ids, dirs, gt, cos


def rays_of_poses(pose6, dirs, out_o=None, out_d=None, Rt12=None):
    """Ray origins and directions of every hypothesis: ray r of the result is dirs[r % N] seen from pose6[r // N]
    (nl_pose_matrices, then nl_rays_from_poses).  This is the ray arithmetic score_poses uses."""
    K, N, dev = pose6.shape[0], dirs.shape[0], pose6.device
    R = K * N
    rep = dirs.repeat(K, 1).contiguous()
    frame = torch.div(torch.arange(R, device=dev, dtype=torch.int32), N, rounding_mode="floor")
    out_o = torch.empty((R, 3), device=dev) if out_o is None else out_o
    out_d = torch.empty((R, 3), device=dev) if out_d is None else out_d
    Rt12 = torch.empty((K, 12), device=dev) if Rt12 is None else Rt12
    lib, st = _capi.lib(), _capi.stream_ptr()
    _capi.check(lib.nl_pose_matrices(K, _capi.ptr(pose6), _capi.ptr(Rt12), st), "nl_pose_matrices")
    _capi.check(lib.nl_rays_from_poses(R, _capi.ptr(rep), _capi.ptr(frame), _capi.ptr(Rt12), _capi.ptr(out_o), _capi.ptr(out_d), st),
                "nl_rays_from_poses")
    _capi.LAUNCHES += 2
    return out_o, out_d


@torch.no_grad()
def score_poses(frame_poses, frame, map_states, sdf_network, loss_criteria, voxel_size, N_rays=512, step_size=0.05, max_distance=10, *,
                deterministic=False, noise=None, ray_ids=None, chunk_rays=1 << 20):
    """The loss of K poses of one scan, forward only: loss[k] is what Criterion.forward(render_rays(o_k, d_k, ...), gt, cos) gives for
    pose k on the shared rays and noise (the first loss_log entry of a one-iteration track_frame), NaN where render_rays returns None.

    frame_poses: f32[K,6] or a list of OptimizablePose, 1 <= K <= NL_SCORE_MAX_PROBLEMS (65 535).  Every hypothesis uses the same N rays
    (one device draw, or ray_ids) and the same noise: one seed for all (deterministic: the constant 0.5; noise: f32[rows >= N, stride]
    in render_rays' layout).  The hypotheses run in chunks of at most chunk_rays rays (>= N); a chunk that exceeds the sample capacity
    is redone on a larger engine, and results do not depend on the chunk size.  One host read-back per chunk.  Returns ScoreResult."""
    pose6 = _pose_tensor(frame_poses)
    K = pose6.shape[0]
    if isinstance(chunk_rays, bool) or not isinstance(chunk_rays, (int, np.integer)) or chunk_rays <= 0:
        raise ValueError(f"score_poses: chunk_rays must be a positive int, got {chunk_rays!r}")
    n_pts = int(frame.points.shape[0])
    N = int(N_rays) if ray_ids is None else int(torch.as_tensor(ray_ids).numel())
    if ray_ids is None and not 1 <= N <= n_pts:
        raise ValueError(f"score_poses: need 1 <= N_rays <= the scan's {n_pts} points, got {N}")
    if chunk_rays < N:
        raise ValueError(f"score_poses: chunk_rays ({chunk_rays}) must hold at least one hypothesis ({N} rays)")
    dev = torch.device("cuda")
    pose6 = pose6.to(dev, torch.float32).contiguous()
    ids, dirs, gt, cos = _select(frame, N, ray_ids, dev)
    if noise is not None:
        if not (noise.is_cuda and noise.dtype == torch.float32 and noise.dim() == 2 and noise.shape[0] >= N):
            raise ValueError("score_poses: noise must be a CUDA f32[rows >= N, stride] tensor (rows by hit rank, as render_rays)")
        noise = noise.contiguous()
    m = map_states if isinstance(map_states, MapState) else MapState.from_map_states(map_states, dev)
    cfg = rh._cfg(step_size, voxel_size, max_distance, loss_criteria)
    P = min(K, int(chunk_rays) // N)                        # hypotheses per chunk
    seed = 0 if (deterministic or noise is not None) else rh._seed_from_torch()
    seeds = torch.full((P,), seed, dtype=torch.int32, device=dev) if seed else None
    gt_rep, cos_rep = gt.repeat(P).contiguous(), cos.repeat(P).contiguous()
    noise_rep = noise.repeat(P, 1).contiguous() if noise is not None else None
    bufs = DecoderBuffers.of(sdf_network, dev)
    bufs.refresh_transposes()
    pstats = torch.zeros((K, STATS_BYTES), dtype=torch.uint8, device=dev)
    base = torch.empty(P, dtype=torch.int32, device=dev)
    Rt12 = torch.empty((P, 12), device=dev)
    b = BatchArgs()
    cap = P * N * SAMPLES_PER_RAY_SCORE
    for k0 in range(0, K, P):
        Kc = min(P, K - k0)
        R = Kc * N
        while True:
            eng = _engine(P * N, cap, dev)
            rays_of_poses(pose6[k0:k0 + Kc], dirs, eng.ray_o[:R], eng.ray_d[:R], Rt12)
            b.n_problems, b.noise_rows = Kc, N if noise is None else noise.shape[0]
            b.d_problem_stats, b.d_problem_base = pstats[k0].data_ptr(), base.data_ptr()
            b.d_problem_seeds = seeds.data_ptr() if seeds is not None else None
            eng.render_samples(m, R, cfg, None, None, gt_rep, cos_rep, noise_rep, 0, True, None, batch=b)
            eng._vs = cfg["voxel_size"]
            eng.gather_forward(m)
            _decoder(eng, bufs, cfg, gt_rep, cos_rep, C.c_void_p(pstats[k0].data_ptr()), N)
            st = eng.read_stats()               # the chunk's one read-back: capacity and traversal errors
            if st.error & 4:
                rh._check_ctl([4], "score_poses")
            if not (st.error & 2):
                break
            rh._check_sample_total(st.n_samples, "score_poses")
            cap = max(2 * cap, int(st.n_samples * 1.25) + 1024)
    loss = torch.empty(K, dtype=torch.float32, device=dev)
    _capi.check(_capi.lib().nl_loss_finalize_batch(K, _capi.ptr(pstats), float(cfg["fs_weight"]), float(cfg["sdf_weight"]), _capi.ptr(loss),
                                                   _capi.stream_ptr()), "nl_loss_finalize_batch")
    _capi.LAUNCHES += 1
    words = pstats.view(torch.int32)
    return ScoreResult(loss, words[:, _HIT_WORD].clone(), words[:, _NSAMP_WORD].clone(), ids)


# ------------------------------------------------------------------------------------------------ relocalise
def poses_from_matrices(Rt):
    """OptimizablePose.from_matrix for a batch: [..., 4, 4] (or [..., 3, 4]) -> [..., 6] = [t, log R]."""
    return torch.cat([Rt[..., :3, 3], OptimizablePose.log(Rt[..., :3, :3])], dim=-1)


def _steps(half_range, n):
    """n values symmetric about 0 spanning [-half_range, half_range]; the middle one is exactly 0 when n is odd."""
    if n == 1:
        return np.zeros(1)
    return half_range * (np.arange(n) - (n - 1) / 2) / ((n - 1) / 2)


def yaw_lattice(guess_pose, yaw_range=np.pi / 6, yaw_steps=31, xy_range=2.0, xy_steps=9):
    """Pose hypotheses around a guess for a ground vehicle: a yaw about the world z axis through the guess's position, then an x/y
    offset; roll, pitch and z stay the guess's.  f32[K,6] on the CPU; row 0 is the guess itself, the lattice point without yaw or
    offset is not repeated, so K = yaw_steps * xy_steps^2 when both are odd, one more otherwise."""
    if int(yaw_steps) < 1 or int(xy_steps) < 1:
        raise ValueError("relocalise: yaw_steps and xy_steps must be >= 1")
    g6 = (guess_pose.data if isinstance(guess_pose, OptimizablePose) else torch.as_tensor(guess_pose)).detach().reshape(6).float().cpu()
    Tg = OptimizablePose(g6.clone()).matrix().detach().double()
    yaw, dx, dy = np.meshgrid(_steps(yaw_range, int(yaw_steps)), _steps(xy_range, int(xy_steps)), _steps(xy_range, int(xy_steps)), indexing="ij")
    yaw, dx, dy = (torch.from_numpy(a.reshape(-1)) for a in (yaw, dx, dy))
    keep = (yaw != 0) | (dx != 0) | (dy != 0)
    yaw, dx, dy = yaw[keep], dx[keep], dy[keep]
    c, s = torch.cos(yaw), torch.sin(yaw)
    Rz = torch.zeros((yaw.shape[0], 3, 3), dtype=torch.float64)
    Rz[:, 0, 0], Rz[:, 0, 1], Rz[:, 1, 0], Rz[:, 1, 1], Rz[:, 2, 2] = c, -s, s, c, 1.0
    Rt = torch.zeros((yaw.shape[0], 3, 4), dtype=torch.float64)
    Rt[:, :, :3] = Rz @ Tg[:3, :3]
    Rt[:, :, 3] = Tg[:3, 3] + torch.stack([dx, dy, torch.zeros_like(dx)], -1)
    return torch.cat([g6[None], poses_from_matrices(Rt.float())]).contiguous()


def select_hypotheses(loss, hit_rays, top_k, min_hit_fraction=0.5):
    """Indices of the top_k lowest finite losses among the hypotheses with hit_rays >= min_hit_fraction x the best hit_rays (without
    that filter a pose that hits three rays well would win), lowest loss first."""
    loss, hit = loss.detach().float().cpu(), hit_rays.detach().cpu().long()
    finite = torch.isfinite(loss)
    if not bool(finite.any()):
        return torch.zeros(0, dtype=torch.long)
    keep = finite & (hit.double() >= float(min_hit_fraction) * float(hit[finite].max()))
    idx = keep.nonzero().view(-1)
    return idx[torch.argsort(loss[idx], stable=True)[:int(top_k)]]


def relocalise(frame, guess_pose, map_states, sdf_network, loss_criteria, voxel_size, *, yaw_range=np.pi / 6, yaw_steps=31, xy_range=2.0,
               xy_steps=9, top_k=16, min_hit_fraction=0.5, N_rays=512, refine_iterations=25, **track_kw):
    """Recover the pose of a scan from a rough guess: score a yaw x x/y lattice around it (yaw_lattice, score_poses), keep the top_k
    lowest losses among the hypotheses that hit at least min_hit_fraction of the best hit count, refine them with one track_frames call
    (refine_iterations iterations; track_kw are track_frames' keywords) and return (pose, hit_mask, ScoreResult) of the refined pose
    with the lowest final loss.  If no hypothesis hits the map: (a copy of the guess, None, ScoreResult)."""
    if not 1 <= int(top_k) <= _capi.BATCH_MAX_PROBLEMS:
        raise ValueError(f"relocalise: 1 <= top_k <= {_capi.BATCH_MAX_PROBLEMS}, got {top_k}")
    if not 0.0 <= float(min_hit_fraction) <= 1.0:
        raise ValueError(f"relocalise: 0 <= min_hit_fraction <= 1, got {min_hit_fraction}")
    from .track_batch import track_frames
    lattice = yaw_lattice(guess_pose, yaw_range, yaw_steps, xy_range, xy_steps)
    score_kw = {k: track_kw[k] for k in ("step_size", "max_distance", "deterministic") if k in track_kw}
    sc = score_poses(lattice, frame, map_states, sdf_network, loss_criteria, voxel_size, N_rays, **score_kw)
    idx = select_hypotheses(sc.loss, sc.hit_rays, top_k, min_hit_fraction)
    if idx.numel() == 0:
        return OptimizablePose(lattice[0].clone()).cuda(), None, sc
    starts = [OptimizablePose(lattice[int(i)].clone()) for i in idx]
    res = track_frames(starts, [frame] * len(starts), map_states, sdf_network, loss_criteria, voxel_size, N_rays=N_rays,
                       num_iterations=refine_iterations, **track_kw)
    ok = [k for k in range(len(res)) if res[k][1] is not None and bool(torch.isfinite(res.loss[k]))]
    if not ok:
        return OptimizablePose(lattice[0].clone()).cuda(), None, sc
    best = min(ok, key=lambda k: float(res.loss[k]))
    return res[best][0], res[best][1], sc
