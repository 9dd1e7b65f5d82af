"""track_frames: K independent pose optimisations against one frozen map and decoder, each what render_helpers.track_frame computes
alone, run as ONE launch chain over a K x N_rays ray batch instead of K calls one after the other.

A tracking iteration at the reference's size (2048 rays, ~40 k samples) is a chain of latency-bound launches that fills a small part
of an H100 (DESIGN.md section 12).  Here the K problems share every launch, and everything that defines one problem's loss -- R_hit,
P, S_max and the hit ranks the sampler keys its quirks by, the loss-mask counts and class weights, the R_hit * S_max normalisation,
the skip flag and Adam's step count -- is kept per problem on the device (include/nerfloam_b200.h section 3b).  Uses: several
starting poses for one scan (keep the lowest final loss), re-localisation, localising a sequence offline against a saved map.
"""
import ctypes as C
import os
from copy import deepcopy

import torch

from . import _capi
from . import render_helpers as rh
from .engine import STATS_BYTES, DecoderBuffers, MapState, SDFEngine, mlp_impl
from ._capi import RenderStats

SEED_INC_SELECT, SEED_INC_NOISE = 0x632BE5, 0x3779B1     # the per-iteration seed advances of the captured track_frame


class TrackFramesResult(list):
    """The K (pose, hit_mask) pairs of track_frames in problem order; `loss` f32[K] (CPU): each problem's loss in its last iteration
    that was not skipped (NaN if there was none)."""

    def __init__(self, items, loss):
        super().__init__(items)
        self.loss = loss


class BatchTracker:
    """Device state of a K-problem tracking chain: a private SDFEngine for K * N rays (problem k owns rays [k N, (k+1) N)), K
    statistics blocks, K control blocks, and each problem's Adam moments, rate and seeds."""

    def __init__(self, K, N, max_samples, device):
        if not 1 <= K <= _capi.BATCH_MAX_PROBLEMS:
            raise ValueError(f"track_frames: 1 <= number of problems <= {_capi.BATCH_MAX_PROBLEMS}, got {K}")
        dev = torch.device(device)
        self.K, self.N, self.dev = K, N, dev
        self.eng = SDFEngine(K * N, max_samples, dev)
        self.eng._ensure_grads(0, K)                     # pose accumulators f32[K,12], pose gradients f32[K,6]
        self.pstats = torch.zeros((K, STATS_BYTES), dtype=torch.uint8, device=dev)
        self.base = torch.zeros(K, dtype=torch.int32, device=dev)
        self.ctl = torch.zeros((K, _capi.CTL_WORDS), dtype=torch.int32, device=dev)
        self._ctl_init = torch.zeros(_capi.CTL_WORDS, dtype=torch.int32, device=dev)
        self._ctl_init[_capi.CTL_MIN_HIT] = 2 ** 31 - 1
        self.fid = torch.arange(K, dtype=torch.int32, device=dev).repeat_interleave(N).contiguous()
        self.adam_m = torch.zeros((K, 6), device=dev)
        self.adam_v = torch.zeros((K, 6), device=dev)
        self.lr = torch.zeros(K, dtype=torch.float64, device=dev)
        self.last_loss = torch.full((K,), float("nan"), device=dev)
        self._ctl_host = torch.empty((K, _capi.CTL_WORDS), dtype=torch.int32).pin_memory()
        self._loss_host = torch.empty(K, dtype=torch.float32).pin_memory()
        self.batch = _capi.BatchArgs()
        self.read_backs = 0

    def begin(self, lrs):
        """Start of a call: fresh control blocks, Adam state and loss read-out; problem k's rate lrs[k]."""
        self.eng.join_side()
        self.ctl.copy_(self._ctl_init.expand(self.K, -1))
        self.adam_m.zero_()
        self.adam_v.zero_()
        self.last_loss.fill_(float("nan"))
        self.lr.copy_(torch.tensor([float(x) for x in lrs], dtype=torch.float64))

    def render(self, m, cfg, gt=None, cos=None, ray_o=None, ray_d=None, noise=None, noise_rows=0, seeds_dev=None, reference_compat=True):
        """nl_render_samples_batch over the engine's rays (or ray_o / ray_d): the sample list, per-problem statistics in pstats."""
        b = self.batch
        b.n_problems, b.noise_rows = self.K, int(noise_rows)
        b.d_problem_stats, b.d_problem_base = self.pstats.data_ptr(), self.base.data_ptr()
        b.d_problem_seeds = seeds_dev.data_ptr() if seeds_dev is not None else None
        self.eng.render_samples(m, self.K * self.N, cfg, ray_o, ray_d, gt, cos, noise, 0, reference_compat, None, batch=b)

    def step(self, m, bufs, cfg, pose6, dirs, gt, cos, noise=None, noise_rows=0, seeds_dev=None, sel_seeds=None):
        """One iteration of every problem: rays -> batched front end -> per-problem control -> gather -> decoder with per-problem loss
        -> pose accumulators per problem -> per-problem pose gradient, Adam step, loss read-out and seed advances.  No host sync."""
        eng, K = self.eng, self.K
        lib, st = _capi.lib(), _capi.stream_ptr()
        eng.rays_from_poses(pose6, dirs, self.fid)
        self.render(m, cfg, gt, cos, noise=noise, noise_rows=noise_rows, seeds_dev=seeds_dev)
        _capi.check(lib.nl_iter_status_batch(K, C.c_void_p(eng.stats.data_ptr()), _capi.ptr(self.pstats), _capi.ptr(self.ctl), st),
                    "nl_iter_status_batch")
        eng._vs = cfg["voxel_size"]
        eng.gather_forward(m)
        self.decoder(bufs, cfg, gt, cos)
        eng.gradflat.zero_()
        _capi.check(lib.nl_gather_trilinear_bwd(
            eng.max_samples, eng.n_samples_dev, _capi.ptr(eng.s_xyz), _capi.ptr(eng.s_vox), _capi.ptr(m.centres), _capi.ptr(m.vox2row),
            _capi.ptr(m.emb), float(cfg["voxel_size"]), _capi.ptr(eng.dfeats), 1, None, None, _capi.ptr(eng.s_ray), _capi.ptr(eng.s_depth),
            _capi.ptr(dirs), _capi.ptr(self.fid), K, _capi.ptr(eng.pose_acc), st), "nl_gather_trilinear_bwd")
        _capi.check(lib.nl_pose_step_batch(K, _capi.ptr(pose6), _capi.ptr(eng.pose_acc), _capi.ptr(eng.pose_grad), _capi.ptr(self.adam_m),
                                           _capi.ptr(self.adam_v), _capi.ptr(self.lr), 0.9, 0.999, 1e-8, _capi.ptr(self.ctl), _capi.ptr(self.pstats),
                                           float(cfg["fs_weight"]), float(cfg["sdf_weight"]), _capi.ptr(self.last_loss), _capi.ptr(sel_seeds),
                                           SEED_INC_SELECT, _capi.ptr(seeds_dev), SEED_INC_NOISE, st), "nl_pose_step_batch")
        _capi.LAUNCHES += 3

    def decoder(self, bufs, cfg, gt, cos):
        """The frozen decoder over the sample list with every problem's own loss (sdf, dfeats, the problems' squared-error sums)."""
        eng, lib, st = self.eng, _capi.lib(), _capi.stream_ptr()
        pst = _capi.ptr(self.pstats)
        if mlp_impl(bufs.width) == "tc":
            p = bufs.params
            _capi.check(lib.nl_mlp_tc_train_batch(eng.max_samples, eng.n_samples_dev, _capi.ptr(eng.feats), _capi.ptr(bufs.tc_panels), _capi.ptr(p[1]),
                                                  _capi.ptr(p[3]), _capi.ptr(p[4]), _capi.ptr(p[5]), _capi.ptr(eng.s_flag), _capi.ptr(eng.s_depth),
                                                  _capi.ptr(eng.s_ray), _capi.ptr(cos), _capi.ptr(gt), pst, self.N, float(cfg["truncation"]),
                                                  _capi.ptr(eng.sdf), _capi.ptr(eng.dfeats), st), "nl_mlp_tc_train_batch")
        else:
            w = bufs.weights_struct()
            _capi.check(lib.nl_mlp_train_batch(eng.max_samples, eng.n_samples_dev, _capi.ptr(eng.feats), C.byref(w), _capi.ptr(eng.s_flag),
                                               _capi.ptr(eng.s_depth), _capi.ptr(eng.s_ray), _capi.ptr(cos), _capi.ptr(gt), pst, self.N,
                                               float(cfg["truncation"]), _capi.ptr(eng.sdf), _capi.ptr(eng.dfeats), st), "nl_mlp_train_batch")
        _capi.LAUNCHES += 1

    def problem_stats(self):
        """Device -> host copy of the K statistics blocks (synchronises): list of RenderStats."""
        h = self.pstats.cpu().numpy()
        return [RenderStats.from_buffer_copy(h[k].tobytes()) for k in range(self.K)]

    def read_back(self):
        """The end of a call's ONE synchronisation: control blocks (lists of CTL_WORDS ints) and last losses."""
        self._ctl_host.copy_(self.ctl, non_blocking=True)
        self._loss_host.copy_(self.last_loss, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.read_backs += 1
        return self._ctl_host.tolist(), self._loss_host.clone()

    def hit_mask(self, k):
        return (self.eng.hit_rank[k * self.N:(k + 1) * self.N] >= 0).clone()


_TRACKERS = {}


def _tracker(K, N, cap, dev):
    key = (K, N, cap, str(dev))
    t = _TRACKERS.get(key)
    if t is None:
        _TRACKERS.clear()
        t = _TRACKERS[key] = BatchTracker(K, N, cap, dev)
    return t


def _stack_frames(frames, dev, out=None):
    """The scans' device arrays stacked to [K, cap] (cap = the most points of any), point counts int64[K]."""
    arrays = [rh._frame_arrays(f, dev) for f in frames]
    if out is None:
        cap = max(a[0].shape[0] for a in arrays)
        K = len(frames)
        out = (torch.tensor([0.0, 0.0, -1.0], device=dev).repeat(K, cap, 1).contiguous(), torch.ones((K, cap), device=dev),
               torch.ones((K, cap), device=dev), torch.zeros(K, dtype=torch.int64, device=dev))
    dirs, gt, cos, n_dev = out
    for k, (d, c, g) in enumerate(arrays):
        n = d.shape[0]
        dirs[k, :n].copy_(d)
        cos[k, :n].copy_(c)
        gt[k, :n].copy_(g)
        n_dev[k].fill_(n)
    return out


def select_rays_batch(stacked, n_select, seeds, out):
    """nl_select_rays_batch: problem k's n_select rays from scan k with its own seed (seeds int32[K] on the device)."""
    dirs_all, gt_all, cos_all, n_dev = stacked
    K, cap = dirs_all.shape[0], dirs_all.shape[1]
    _capi.check(_capi.lib().nl_select_rays_batch(K, cap, int(n_select), _capi.ptr(n_dev), _capi.ptr(seeds), _capi.ptr(dirs_all), _capi.ptr(gt_all),
                                                 _capi.ptr(cos_all), _capi.ptr(out[0]), _capi.ptr(out[1]), _capi.ptr(out[2]), None,
                                                 _capi.stream_ptr()), "nl_select_rays_batch")
    _capi.LAUNCHES += 1
    return out


def _pack_noise(noise_k, dev):
    """noise_per_iter[it] (one tensor per problem, rows by hit rank within the problem) -> f32[K * rows, stride], rows per problem."""
    rows = max(int(t.shape[0]) for t in noise_k)
    stride = max(int(t.shape[1]) for t in noise_k)
    buf = torch.zeros((len(noise_k), max(rows, 1), stride), dtype=torch.float32, device=dev)
    for k, t in enumerate(noise_k):
        buf[k, :t.shape[0], :t.shape[1]].copy_(t)
    return buf.view(-1, stride), max(rows, 1)


class _TrackBatchGraph:
    """One captured K-problem iteration (_TrackGraph's pattern): per-problem ray selection -> rays -> batched front end -> decoder ->
    per-problem pose steps, every per-call input (scans, poses, rates, seeds) in static device buffers.  Captured once per (map,
    decoder, K, N_rays, sampling mode, capacity); a call is num_iterations replays and one read-back."""

    _cache = {}
    _max_live = 2

    def __init__(self, key, m, sdf_network, cfg, K, N, deterministic, cap, spr):
        dev = m.centres.device
        tr = BatchTracker(K, N, K * N * spr, dev)
        bufs = DecoderBuffers(sdf_network, dev)
        self.key, self.tr, self.bufs, self.m, self.packed, self.K, self.N, self.cap = key, tr, bufs, m, m.packed_children(), K, N, cap
        self.stacked = (torch.tensor([0.0, 0.0, -1.0], device=dev).repeat(K, cap, 1).contiguous(), torch.ones((K, cap), device=dev),
                        torch.ones((K, cap), device=dev), torch.full((K,), cap, dtype=torch.int64, device=dev))
        self.pose6 = torch.zeros((K, 6), device=dev)
        self.seeds_dev = torch.ones(K, dtype=torch.int32, device=dev)
        self.sel_seeds = torch.ones(K, dtype=torch.int32, device=dev)
        self.sel_out = (torch.empty((K * N, 3), device=dev), torch.empty(K * N, device=dev), torch.empty(K * N, device=dev))

        def body():
            dirs, gt, cos = select_rays_batch(self.stacked, N, self.sel_seeds, self.sel_out)
            tr.step(m, bufs, cfg, self.pose6, dirs, gt, cos, seeds_dev=None if deterministic else self.seeds_dev, sel_seeds=self.sel_seeds)

        bufs.refresh_transposes()
        tr.begin([0.0] * K)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            body()
        torch.cuda.current_stream(dev).wait_stream(side)
        l0 = _capi.LAUNCHES
        self.graph = torch.cuda.CUDAGraph()
        with rh._graph_capture(self.graph):
            body()
        self.launches_per_iter = _capi.LAUNCHES - l0 + 1

    @classmethod
    def get(cls, m, sdf_network, cfg, K, N, deterministic, n_points, spr):
        cap = max(1 << 17, 1 << (int(n_points) - 1).bit_length())
        stable = m.stable
        key = (K, N, bool(deterministic), cap, int(spr), m.centres.data_ptr(), m.structure.data_ptr(), m.vox2row.data_ptr(),
               m.packed_children().data_ptr(), m.emb.data_ptr(), -1 if stable else m.n_nodes, -1 if stable else int(m.emb.shape[0]),
               tuple(p.data_ptr() for p in rh._decoder_params(sdf_network)), mlp_impl(sdf_network.pts_linears[0].weight.shape[0]),
               tuple(sorted(cfg.items())))
        g = cls._cache.pop(key, None)
        if g is None:
            if not stable:
                cls._cache.clear()
            while len(cls._cache) >= cls._max_live:
                cls._cache.pop(next(iter(cls._cache)))
            g = cls(key, m, sdf_network, cfg, K, N, deterministic, cap, spr)
        cls._cache[key] = g
        return g

    def run(self, frames, pose6_init, lrs, num_iterations, seeds):
        dev = self.pose6.device
        self.bufs.refresh_transposes()        # the decoder may have been updated in place since the capture
        _stack_frames(frames, dev, self.stacked)
        self.pose6.copy_(pose6_init)
        self.seeds_dev.copy_(torch.tensor([s if s < 2 ** 31 else s - 2 ** 32 for s in seeds], dtype=torch.int32))
        self.sel_seeds.copy_(torch.randint(1, 2 ** 31 - 1, (self.K,), device=dev, dtype=torch.int32))   # follows torch's CUDA generator
        self.tr.begin(lrs)
        for _ in range(num_iterations):
            self.graph.replay()
        _capi.LAUNCHES += self.launches_per_iter * num_iterations
        return self.tr.read_back()


def _run_eager(tr, m, bufs, cfg, frames, pose6, lrs, N, num_iterations, deterministic, noise_per_iter, loss_log, ray_selection, dev):
    K = tr.K
    tr.begin(lrs)
    bufs.refresh_transposes()              # the decoder is frozen while tracking: derive the kernel-side weight images once
    if ray_selection == "device":
        stacked = _stack_frames(frames, dev)
        sel_out = (torch.empty((K * N, 3), device=dev), torch.empty(K * N, device=dev), torch.empty(K * N, device=dev))
    else:
        batch = rh._FrameBatch(frames, dev)
    for it in range(num_iterations):
        sel_seeds = None
        if ray_selection == "device":
            sel_seeds = torch.randint(1, 2 ** 31 - 1, (K,), device=dev, dtype=torch.int32)
            dirs, gt, cos = select_rays_batch(stacked, N, sel_seeds, sel_out)
        else:
            dirs, gt, cos, _ = batch.select(N, dev, track=True, mode="host")
        noise, rows, seeds_dev = None, 0, None
        if noise_per_iter is not None:
            noise, rows = _pack_noise(noise_per_iter[it], dev)
        elif not deterministic:
            seeds_dev = torch.tensor([rh._seed_from_torch() for _ in range(K)], dtype=torch.int32).to(dev)
        tr.step(m, bufs, cfg, pose6, dirs, gt, cos, noise=noise, noise_rows=rows, seeds_dev=seeds_dev, sel_seeds=sel_seeds)
        if loss_log is not None:           # diagnostic path: one read-back per iteration
            ctl = tr.ctl.cpu().tolist()
            for k, s in enumerate(tr.problem_stats()):
                if not ctl[k][_capi.CTL_SKIP_NOW]:
                    loss_log[k].append(s.loss)
    return tr.read_back()


def track_frames(frame_poses, frames, map_states, sdf_network, loss_criteria, voxel_size, N_rays=512, step_size=0.05, num_iterations=10,
                 truncation=0.1, learning_rate=1e-3, max_voxel_hit=10, max_distance=10, *, deterministic=False, noise_per_iter=None,
                 loss_log=None, ray_selection="device", cuda_graph=None):
    """K independent track_frame problems in one launch chain.  Problem k optimises the pose frame_poses[k] of scan frames[k] (the same
    frame object may appear several times: pose hypotheses for one scan) under track_frame's rules -- rate 2 lr if frames[k].index < 2,
    else lr / 3; its own Adam state and step count; the inputs are not modified -- and returns what
    track_frame(frame_poses[k], frames[k], ...) returns alone on the same rays and noise.

    1 <= K <= 31 (one warp per problem in the fused pose step); every scan needs at least N_rays points (the problems are equal ray
    segments).  A problem whose iteration hits nothing stops for the rest of the call, like the reference's `break`: its pose stays
    where it was and its hit mask is None, while the others carry on -- decided on the device, without a host sync per iteration.
    noise_per_iter[it]: a list of K tensors, each in the solo call's layout.  loss_log: a list that receives K lists of per-iteration
    losses.  cuda_graph: as track_frame (default on for maps with stable addresses, device ray selection, no per-iteration host
    inputs / outputs).  Returns a TrackFramesResult: K (OptimizablePose on the GPU, hit_mask bool[N_rays] | None), `.loss` f32[K]."""
    if ray_selection not in ("host", "device"):
        raise ValueError("ray_selection must be 'host' or 'device'")
    frame_poses, frames = list(frame_poses), list(frames)
    K = len(frames)
    if K != len(frame_poses):
        raise ValueError("track_frames: one starting pose per frame")
    if not 1 <= K <= _capi.BATCH_MAX_PROBLEMS:
        raise ValueError(f"track_frames: 1 <= number of problems <= {_capi.BATCH_MAX_PROBLEMS}, got {K}")
    if any(f.points.shape[0] < N_rays for f in frames):
        raise ValueError("track_frames: every scan needs at least N_rays points")
    if noise_per_iter is not None and any(len(n) != K for n in noise_per_iter[:num_iterations]):
        raise ValueError("track_frames: noise_per_iter[it] must hold one tensor per problem")
    if loss_log is not None:
        if len(loss_log) == 0:
            loss_log.extend([] for _ in range(K))
        if len(loss_log) != K:
            raise ValueError("track_frames: loss_log must be empty or hold one list per problem")
    dev = torch.device("cuda")
    graph_ok = ray_selection == "device" and noise_per_iter is None and loss_log is None
    if cuda_graph is None:
        ms = map_states if isinstance(map_states, MapState) else map_states.get("_mapstate")
        cuda_graph = graph_ok and ms is not None and ms.stable and os.environ.get("NL_TRACK_GRAPH", "1") != "0"
    elif cuda_graph and not graph_ok:
        raise ValueError("cuda_graph=True needs ray_selection='device' and no per-iteration host inputs/outputs")
    m = map_states if isinstance(map_states, MapState) else MapState.from_map_states(map_states, dev)
    cfg = rh._cfg(step_size, voxel_size, max_distance, loss_criteria)
    init_poses = []
    for fp in frame_poses:
        p = deepcopy(fp).cuda()
        p.requires_grad_(True)
        init_poses.append(p)
    pose0 = torch.stack([p.data.detach().reshape(6).float() for p in init_poses]).to(dev).contiguous()
    lrs = [learning_rate * 2 if f.index < 2 else learning_rate / 3 for f in frames]   # render_helpers.py:448-450
    N = int(N_rays)
    spr = rh.SAMPLES_PER_RAY_TRACK
    rng = (torch.get_rng_state(), torch.cuda.get_rng_state(dev))
    while True:
        n_log = [len(x) for x in loss_log] if loss_log is not None else None
        if cuda_graph:
            seeds = [0] * K if deterministic else [rh._seed_from_torch() for _ in range(K)]
            g = _TrackBatchGraph.get(m, sdf_network, cfg, K, N, deterministic, max(f.points.shape[0] for f in frames), spr)
            tr = g.tr
            ctl, loss = g.run(frames, pose0, lrs, num_iterations, seeds)
            pose6 = g.pose6
        else:
            tr = _tracker(K, N, K * N * spr, dev)
            pose6 = pose0.clone()
            bufs = DecoderBuffers.of(sdf_network, dev)
            ctl, loss = _run_eager(tr, m, bufs, cfg, frames, pose6, lrs, N, num_iterations, deterministic, noise_per_iter, loss_log,
                                   ray_selection, dev)
        rh._check_ctl(ctl[0], "track_frames")
        if not (ctl[0][_capi.CTL_ERROR] & 2):
            break
        # the shared sample capacity was exceeded somewhere in the call: undo it (the inputs were never touched) and redo it larger
        torch.set_rng_state(rng[0]); torch.cuda.set_rng_state(rng[1], dev)
        if loss_log is not None:
            for x, n in zip(loss_log, n_log):
                del x[n:]
        spr = -(-rh._grown_capacity(K * N * spr, ctl[0], "track_frames") // (K * N))
    out = []
    with torch.no_grad():
        for k, p in enumerate(init_poses):
            p.data.copy_(pose6[k].reshape(p.data.shape))
            stopped = ctl[k][_capi.CTL_SKIPPED] > 0 or num_iterations <= 0
            if stopped and num_iterations > 0:
                print("Encouter a bug while Tracking, currently not be fixed, Restarting!!")  # render_helpers.py:488-491
            out.append((p, None if stopped else tr.hit_mask(k)))
    return TrackFramesResult(out, loss)
