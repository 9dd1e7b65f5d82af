"""A whole sequence: the reference's tracker and mapper (src/tracking.py, src/mapping.py, src/nerfloam.py) as one pipeline, the two
roles concurrent on two host threads and two CUDA streams, writing the trajectory and the meshes.

    slam = NeRFLOAM("configs/kitti/kitti_00.yaml", out_dir)        # the reference's config layout (demo/parser.py)
    summary = slam.run()

`Tracking` and `Mapping` keep the reference's names and rules (each cited below); `run_pipeline` is the scheduler.  The reference
runs the two roles as processes that read whatever the other published last, so two runs differ by timing.  Here the dependency is
fixed (the lag-one schedule, DESIGN.md section 11.3):

  * scan p + 1 is tracked against the map published after scan p - 1's full mapping step (bundle adjustment, create_voxels, publish),
    while the mapper's bundle adjustment of scan p runs on the other stream;
  * the mapper's in-place map update of scan p starts only after the tracker has released its snapshot for scan p + 1;
  * each role draws from its own generator, seeded from `seeding`, so the draws do not depend on how the threads interleave.

Outputs under out_dir, in the reference's layout (loggers.py:17-29, 56-71): mesh/mesh_{index:05d}.ply, mesh/final_mesh_noreplay.ply,
mesh/final_mesh.ply (binary little-endian PLY, float32 xyz and int32 faces, with the -2000 m offset removed as mesh_util.py:139
does) and misc/frame_poses_{index:05d}.txt, misc/frame_poses.txt (one scan per line, the top 3 x 4 of its pose row-major: KITTI's
format, loggers.py:144-159).  NeRFLOAM.save_map(path) writes the finished run's map, decoder, trajectory and settings to one file
(write_map); load_map reads it back onto either octree, and localise.Localiser localises later scans in it.

Deviations from the reference (also in DESIGN.md section 11.3):
  * end_frame is clamped to len - 1: the reference's min(end_frame, len) and range(..., end_frame + 1) index past the last scan
    (tracking.py:43-44, 66-67);
  * the first scan is mapped with `init_calls` 'current' calls; the reference maps it until the tracker's next scan arrives, after a
    20 s sleep (mapping.py:106-107, nerfloam.py:45), which depends on timing;
  * the map is published once per mapping step (and once after the first scan's calls), not after every bundle adjustment;
  * the pose files are written as text only (the reference also writes the .npy it converts them from).
"""
import contextlib
import importlib
import os
import queue
import random
import threading
import time
from collections import namedtuple
from types import SimpleNamespace

import numpy as np
import torch

from . import _capi
from . import render_helpers as rh
from .criterion import Criterion
from .frame import POSE_OFFSET, LidarFrame
from .keyframes import KeyframeGraph
from .lidar import Decoder
from .mapping import MapUpdater
from .mesh import extract_mesh
from .se3pose import OptimizablePose
from .share import SharedMap, _flat_decoder_state, load_flat_decoder_state

SELECTIONS = ("current", "previous", "overlap")


# ----------------------------------------------------------------------------------------------------------------------------
# configuration
# ----------------------------------------------------------------------------------------------------------------------------
def _merge(base, over):
    """demo/parser.py:48-56: `over` into `base`, recursively."""
    for k, v in over.items():
        if k not in base:
            base[k] = dict()
        if isinstance(v, dict):
            _merge(base[k], v)
        else:
            base[k] = v
    return base


def _read_yaml(path):
    """demo/parser.py:23-37: a YAML file with its `base_config` chain merged under it.  A base_config path is taken as given (the
    reference resolves it against the working directory) and, failing that, relative to the including file."""
    import yaml
    with open(path) as f:
        cfg = yaml.safe_load(f) or {}
    base = cfg.get("base_config")
    if base is not None:
        cand = base if os.path.exists(base) else os.path.join(os.path.dirname(os.path.abspath(path)), base)
        if not os.path.exists(cand):
            raise FileNotFoundError(f"{path}: base_config {base!r} not found")
        cfg = _merge(_read_yaml(cand), cfg)
    return cfg


def load_config(config):
    """The reference's configuration as a SimpleNamespace: `config` is a dict, a namespace or a YAML path (base_config merged).
    Optional keys get the reference's defaults (seeding 777, run.py:20-23; final_iter False, mesh_res 8, mapping.py:44-48;
    tracker start/end/read_offset 0/-1/1).  Settings this pipeline does not implement raise ValueError naming the key."""
    if isinstance(config, (str, os.PathLike)):
        cfg = _read_yaml(config)
    elif isinstance(config, dict):
        cfg = _merge({}, config)
    else:
        cfg = _merge({}, vars(config))
    a = SimpleNamespace(**cfg)
    for key in ("data_specs", "criteria", "decoder_specs", "tracker_specs", "mapper_specs"):
        if not isinstance(getattr(a, key, None), dict):
            raise ValueError(f"config: {key} is missing")
    a.debug_args = dict(getattr(a, "debug_args", None) or {})
    a.dataset = getattr(a, "dataset", "kitti")
    if a.dataset == "ncd":
        raise ValueError("config: dataset: ncd is not supported (only kitti and maicity loaders exist)")
    if a.dataset not in ("kitti", "maicity"):
        raise ValueError(f"config: dataset: {a.dataset!r} unknown (kitti or maicity)")
    if a.mapper_specs.get("use_local_coord", False):
        raise ValueError("config: mapper_specs.use_local_coord: True is not supported")
    if (getattr(a, "ckpt_freq", -1) or -1) > 0:
        raise ValueError("config: ckpt_freq > 0 (checkpoints) is not supported")
    if (a.debug_args.get("save_data_freq", 0) or 0) > 0:
        raise ValueError("config: debug_args.save_data_freq > 0 is not supported")
    a.seeding = int(getattr(a, "seeding", 777))
    a.tracker_specs = {"start_frame": 0, "end_frame": -1, "read_offset": 1, **a.tracker_specs}
    a.mapper_specs = {"final_iter": False, "mesh_res": 8, **a.mapper_specs}
    a.debug_args.setdefault("mesh_freq", 0)
    a.data_specs = {"use_gt": False, "max_depth": -1, "min_depth": -1, **a.data_specs}
    return a


# ----------------------------------------------------------------------------------------------------------------------------
# writers
# ----------------------------------------------------------------------------------------------------------------------------
def write_poses(path, poses):
    """One pose per line: the top 3 x 4 of each 4 x 4 pose, row-major, space-separated (loggers.py:144-159, KITTI's format)."""
    with open(path, "w") as f:
        for p in poses:
            f.write(" ".join(f"{float(v):.9g}" for v in np.asarray(p, dtype=np.float64)[:3, :4].reshape(-1)) + "\n")


def write_ply(path, verts, faces):
    """A binary little-endian PLY: float32 x, y, z per vertex and a uchar-counted list of int32 indices per triangle."""
    v = np.ascontiguousarray(np.asarray(verts, dtype="<f4").reshape(-1, 3))
    f = np.asarray(faces, dtype="<i4").reshape(-1, 3)
    rec = np.empty(f.shape[0], dtype=[("n", "u1"), ("v", "<i4", (3,))])
    rec["n"], rec["v"] = 3, f
    head = ("ply\nformat binary_little_endian 1.0\n"
            f"element vertex {v.shape[0]}\nproperty float x\nproperty float y\nproperty float z\n"
            f"element face {f.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as out:
        out.write(head.encode("ascii"))
        out.write(v.tobytes())
        out.write(rec.tobytes())


# ----------------------------------------------------------------------------------------------------------------------------
# host-side rules
# ----------------------------------------------------------------------------------------------------------------------------
def constant_velocity_guess(last_pose, rel_pose):
    """tracking.py:109-114: the last pose with its translation moved by the last relative motion; the rotation is kept.  Returns the
    4 x 4 guess (a copy)."""
    guess = last_pose.detach().clone()
    if rel_pose is not None:
        guess[:3, 3] = (guess @ rel_pose)[:3, 3]
    return guess


def remove_back_points(frame, key_distance):
    """mapping.py:235-255: drop the returns beyond key_distance that lie behind the direction of motion (cosine >= 0.7 between the
    point's xy and minus the relative translation's xy; +x when the frame has no relative pose).  A new LidarFrame sharing the pose."""
    rel_pose = frame.get_rel_pose()
    points = frame.get_points()
    points_norm = torch.norm(points, 2, -1)
    rel_xy = torch.ones((1, 2))
    if rel_pose is None:
        rel_xy[0, 0], rel_xy[0, 1] = 1, 0
    else:
        rel_xy[0, 0], rel_xy[0, 1] = rel_pose[0, 3], rel_pose[1, 3]
    point_cos = torch.sum(-points[:, :2] * rel_xy, dim=-1) / (torch.norm(points[:, :2], 2, -1) * torch.norm(rel_xy, 2, -1))
    keep = ~((point_cos >= 0.7) & (points_norm > key_distance))
    return LidarFrame(frame.index, frame.points[keep], frame.get_pointsCos()[keep], frame.pose, new_keyframe=True)


class KeyframePoses:
    """The mapper's keyframe-relative trajectory (mapping.py:121-125, 341-351): each mapped scan is stored as (index of its
    keyframe in the graph, pose relative to that keyframe); get_updated_poses fixes every stored scan into the trajectory from its
    keyframe's pose at the time of the call and clears the store, so later moves of that keyframe no longer change it."""

    def __init__(self):
        self.frame_poses = []
        self.final_poses = []

    def record(self, keyframe_graph, frame):
        ref = keyframe_graph.current_keyframe.get_pose().detach()
        self.frame_poses.append((len(keyframe_graph.keyframe_graph) - 1, (torch.linalg.inv(ref) @ frame.get_pose().detach()).cpu()))

    @torch.no_grad()
    def get_updated_poses(self, keyframe_graph, offset=-POSE_OFFSET):
        for ref_ind, rel in self.frame_poses:
            pose = keyframe_graph.keyframe_graph[ref_ind].get_pose().detach().cpu() @ rel
            pose[:3, 3] += offset
            self.final_poses.append(pose.numpy())
        self.frame_poses = []
        return self.final_poses


# ----------------------------------------------------------------------------------------------------------------------------
# the two roles
# ----------------------------------------------------------------------------------------------------------------------------
class _Timed:
    def _tick(self, stage, t0):
        self.times.setdefault(stage, []).append((time.perf_counter() - t0) * 1e3)
        self.streams.add(torch.cuda.current_stream().cuda_stream)


class Tracking(_Timed):
    """tracking.py:15-148 against a SharedMap.  track(frame_id, version) tracks one scan against map `version` and returns the
    mapper's copy of it: a new LidarFrame over the same points with its OWN OptimizablePose (the reference's copy crosses a process
    boundary, so the mapper's bundle adjustment never moves the tracker's last_frame)."""

    def __init__(self, args, data_stream, shared, generator=None, place=None):
        self.args, self.data_stream, self.shared, self.generator = args, data_stream, shared, generator
        self.place = place                  # None: the first scan at get_init_pose; else place(frame) sets its pose (NeRFLOAM's base_map)
        ts, ms = args.tracker_specs, args.mapper_specs
        self.loss_criteria = Criterion(args)
        self.voxel_size = ms["voxel_size"]
        self.N_rays, self.num_iterations = ts["N_rays"], ts["num_iterations"]
        self.sdf_truncation = args.criteria["sdf_truncation"]
        self.learning_rate = ts["learning_rate"]
        self.step_size = ts["step_size"] * self.voxel_size
        self.max_voxel_hit = ts["max_voxel_hit"]
        self.max_distance = args.data_specs["max_depth"]
        self.read_offset = ts["read_offset"]
        n = len(data_stream)
        self.end_frame = ts["end_frame"] if ts["end_frame"] > 0 else n - 1
        self.start_frame = min(ts["start_frame"], n)
        self.end_frame = min(self.end_frame, n - 1)      # deviation: the reference clamps to n and then reads scan n (tracking.py:43-44)
        self.last_frame = None
        self.rel_pose = None
        self.times, self.streams = {}, set()

    def first_frame(self):
        """process_first_frame (tracking.py:51-61): the first scan at get_init_pose(start_frame), or where place(frame) puts it."""
        index, points, pointcos, _ = self.data_stream[self.start_frame]
        if self.place is None:
            first = LidarFrame(index, points, pointcos, np.array(self.data_stream.get_init_pose(self.start_frame), dtype=np.float64))
        else:
            first = LidarFrame(index, points, pointcos, OptimizablePose(torch.zeros(6)), new_keyframe=True)
            self.place(first)
        first.pose.requires_grad_(False)
        self.last_frame = first
        self.start_frame += 1
        return self._handoff(first)

    def frame_ids(self):
        """The scans spin() tracks (tracking.py:66-71): start_frame .. end_frame, those divisible by read_offset."""
        return [i for i in range(self.start_frame, self.end_frame + 1) if i % self.read_offset == 0]

    def track(self, frame_id, version):
        t0 = time.perf_counter()
        data_in = self.data_stream[frame_id]
        self._tick("load", t0)
        t0 = time.perf_counter()
        index, points, pointcos, pose = data_in
        if isinstance(pose, np.ndarray):               # tracking.py:78-80: a scan with a pose is passed through untracked
            cur = LidarFrame(index, points, pointcos, pose.copy())
            self.last_frame = cur
        else:
            cur = LidarFrame(index, points, pointcos)
            self._do_tracking(cur, version)
        self._tick("track", t0)
        return self._handoff(cur)

    def _do_tracking(self, cur, version):
        """tracking.py:98-144."""
        guess = constant_velocity_guess(self.last_frame.get_pose(), self.rel_pose)
        input_pose = OptimizablePose(self.last_frame.pose.data.detach().cpu().clone())
        input_pose.requires_grad_(False)
        if self.rel_pose is not None:
            input_pose.data.data[:3] = guess[:3, 3]
        map_state, decoder, slot = self.shared.acquire(version)
        try:
            pose, hit_mask = rh.track_frame(input_pose, cur, map_state, decoder, self.loss_criteria, self.voxel_size, self.N_rays,
                                            self.step_size, self.num_iterations if self.rel_pose is not None else self.num_iterations * 5,
                                            self.sdf_truncation, self.learning_rate, self.max_voxel_hit, self.max_distance,
                                            generator=self.generator)
        finally:
            self.shared.release(slot)
        if hit_mask is None:
            cur.pose = OptimizablePose.from_matrix(guess)
        else:
            cur.pose = OptimizablePose(pose.data.detach().cpu().clone())
        self.rel_pose = torch.linalg.inv(self.last_frame.get_pose().detach()) @ cur.get_pose().detach()
        cur.set_rel_pose(self.rel_pose)
        self.last_frame = cur

    @staticmethod
    def _handoff(frame):
        out = LidarFrame(frame.index, frame.points, frame.pointsCos, OptimizablePose(frame.pose.data.detach().cpu().clone()),
                         new_keyframe=True)
        out.set_rel_pose(None if frame.rel_pose is None else frame.rel_pose.clone())
        return out


class Mapping(_Timed):
    """mapping.py:30-351 on a MapUpdater, a KeyframeGraph and a SharedMap.  init(frame) maps the first scan; optimise(frame) is the
    bundle adjustment of a tracked scan, update(frame) the rest of its mapping step (create_voxels, keyframe, trajectory entry,
    periodic mesh); both of those end with a publication whose version they return.  finish() writes the final outputs.

    map_updater: a MapUpdater to grow (a saved map's) instead of a new one; its rows [0, n_rows) at construction are then held fixed
    (frozen_rows in every bundle_adjust_frames and refine_map call) and the decoder is never stepped."""

    def __init__(self, args, out_dir, shared, decoder, generator=None, selection="current", init_calls=12, reserve_nodes=1 << 20,
                 reserve_rows=1 << 20, map_updater=None):
        if selection not in SELECTIONS:
            raise ValueError(f"selection must be one of {SELECTIONS}, not {selection!r}")
        ms = args.mapper_specs
        self.args, self.shared, self.decoder, self.generator = args, shared, decoder, generator
        self.selection, self.init_calls = selection, int(init_calls)
        self.loss_criteria = Criterion(args)
        self.voxel_size = ms["voxel_size"]
        self.window_size, self.num_iterations, self.n_rays = ms["window_size"], ms["num_iterations"], ms["N_rays_each"]
        self.sdf_truncation = args.criteria["sdf_truncation"]
        self.max_voxel_hit = ms["max_voxel_hit"]
        self.step_size = ms["step_size"] * self.voxel_size
        self.learning_rate = [ms["learning_rate_emb"], ms["learning_rate_decorder"], ms["learning_rate_pose"]]
        self.max_distance = args.data_specs["max_depth"]
        self.freeze_frame, self.keyframe_gap = ms["freeze_frame"], ms["keyframe_gap"]
        self.remove_back, self.key_distance = ms["remove_back"], ms["key_distance"]
        self.final_iter, self.mesh_res = ms["final_iter"], ms["mesh_res"]
        self.mesh_freq = args.debug_args["mesh_freq"]
        if map_updater is None:
            self.map = MapUpdater(self.voxel_size, reserve_nodes=reserve_nodes, reserve_rows=reserve_rows)
            self.frozen_rows, self.train_decoder = 0, True
        else:
            self.map = map_updater                              # new vertices get rows >= n_rows: rows are appended in creation order
            self.frozen_rows, self.train_decoder = int(map_updater.n_rows), False
        self.map.readers = shared
        self.map_state = None
        self.kg = KeyframeGraph(self.window_size, self.keyframe_gap, self.key_distance, self.n_rays, self.voxel_size)
        self.trajectory = KeyframePoses()
        self.keyframe_indices = []
        self.mesh_dir, self.misc_dir = os.path.join(out_dir, "mesh"), os.path.join(out_dir, "misc")
        os.makedirs(self.mesh_dir, exist_ok=True)
        os.makedirs(self.misc_dir, exist_ok=True)
        self.first_frame_id = None
        self.scan_ids = []                  # frame.index of each trajectory entry, in the trajectory's order
        self.times, self.streams = {}, set()

    # -- the steps ---------------------------------------------------------------------------------------------------------
    def init(self, frame):
        """mapping.py:100-108 and 120-147 for the first scan: create_voxels, insert_keyframe, init_calls 'current' mapping calls."""
        t0 = time.perf_counter()
        self.first_frame_id = frame.index
        self._create_voxels(frame)
        self._insert_keyframe(frame)
        for _ in range(self.init_calls):
            self._do_mapping(frame, "current")
        self._tick("init", t0)
        return self._end_step(frame)

    def optimise(self, frame):
        """mapping.py:110-112."""
        t0 = time.perf_counter()
        if self.remove_back:
            frame = remove_back_points(frame, self.key_distance)
        self._do_mapping(frame, self.selection)
        self._tick("map", t0)
        return frame

    def update(self, frame):
        """mapping.py:113-147: create_voxels at the adjusted pose, the keyframe-gap test, the trajectory entry, the periodic mesh."""
        t0 = time.perf_counter()
        self._create_voxels(frame)
        if self.kg.needs_keyframe(frame):
            self._insert_keyframe(frame)
        self._tick("update", t0)
        return self._end_step(frame)

    def finish(self):
        """mapping.py:152-169."""
        self._write_mesh("final_mesh_noreplay.ply")
        if self.final_iter:
            self.refine()
        write_poses(os.path.join(self.misc_dir, "frame_poses.txt"), self.trajectory.get_updated_poses(self.kg))
        self._write_mesh("final_mesh.ply")

    def refine(self):
        """The post-processing passes (mapping.py:128-138, 154-164) as one refine_map call."""
        t0 = time.perf_counter()
        rh.refine_map(self.kg, self.map.embeddings, self.map_state, self.decoder, self.loss_criteria, self.voxel_size, self.step_size,
                      N_rays=2 * self.n_rays, num_iterations=self.num_iterations, truncation=self.sdf_truncation,
                      max_voxel_hit=self.max_voxel_hit, max_distance=self.max_distance, learning_rate=self.learning_rate[0],
                      generator=self.generator, frozen_rows=self.frozen_rows)
        torch.cuda.current_stream().synchronize()
        self._tick("refine", t0)

    # -- helpers -----------------------------------------------------------------------------------------------------------
    def _end_step(self, frame):
        self.trajectory.record(self.kg, frame)
        self.scan_ids.append(frame.index)
        if self.mesh_freq > 0 and frame.index % self.mesh_freq == 0:
            big = self.final_iter and len(self.kg.keyframe_graph) > 20
            if big:
                self.refine()
            self._write_mesh(f"mesh_{frame.index:05d}.ply")
            write_poses(os.path.join(self.misc_dir, f"frame_poses_{frame.index:05d}.txt"), self.trajectory.get_updated_poses(self.kg))
            if big:
                self.kg.keyframe_graph = [self.kg.current_keyframe]      # mapping.py:145-147
        t0 = time.perf_counter()
        version = self.shared.publish(self.map_state, self.decoder)
        self._tick("publish", t0)
        return version

    def _do_mapping(self, frame, selection):
        """mapping.py:172-202 (update_decoder only while index - first < freeze_frame, and never when growing a saved map)."""
        targets = self.kg.select_optimize_targets(frame, selection, generator=self.generator)
        rh.bundle_adjust_frames(targets, self.map.embeddings, self.map_state, self.decoder, self.loss_criteria, self.voxel_size,
                                self.step_size, self.n_rays, self.num_iterations, self.sdf_truncation, self.max_voxel_hit,
                                self.max_distance, learning_rate=self.learning_rate, update_pose=True,
                                update_decoder=self.train_decoder and (frame.index - self.first_frame_id) < self.freeze_frame,
                                generator=self.generator, frozen_rows=self.frozen_rows)

    def _create_voxels(self, frame):
        self.map_state = self.map.create_voxels(frame.points, frame.get_pose().detach())

    def _insert_keyframe(self, frame):
        self.kg.insert_keyframe(frame)
        self.keyframe_indices.append(frame.index)

    def _write_mesh(self, name):
        verts, faces = extract_mesh(self.decoder, self.map_state, self.voxel_size, res=self.mesh_res)
        write_ply(os.path.join(self.mesh_dir, name), verts.double().cpu().numpy() - POSE_OFFSET, faces.cpu().numpy())


# ----------------------------------------------------------------------------------------------------------------------------
# the schedule
# ----------------------------------------------------------------------------------------------------------------------------
class Stopped(Exception):
    """Raised inside a role's thread when the other thread has failed."""


class LagOneSchedule:
    """Host-side state of the lag-one schedule.  Scans are numbered by position p (0: the first scan, mapped by init).  The tracker
    waits in map_version(p) for the version of mapping step max(p - 2, 0) and calls released(p) when it has released that snapshot;
    the mapper waits in wait_released(p + 1) before update(p) and calls published(p, version) after it.  fail(exc) stops both sides:
    every wait then raises Stopped.  `log` records the order of events as (what, position, version) tuples."""

    POLL = 0.05

    def __init__(self):
        self._cv = threading.Condition()
        self.versions = {}
        self.n_released = 0
        self.tracking_done = False
        self.error = None
        self.log = []

    def _wait(self, ready):
        with self._cv:
            while not ready():
                if self.error is not None:
                    raise Stopped()
                self._cv.wait()
            if self.error is not None:
                raise Stopped()

    def map_version(self, p):
        step = max(p - 2, 0)
        self._wait(lambda: step in self.versions)
        with self._cv:
            v = self.versions[step]
            self.log.append(("track", p, v))
        return v

    def released(self, p):
        with self._cv:
            self.n_released = p
            self.log.append(("release", p, None))
            self._cv.notify_all()

    def wait_released(self, p):
        self._wait(lambda: self.n_released >= p or self.tracking_done)
        with self._cv:
            self.log.append(("update", p - 1, None))

    def published(self, p, version):
        with self._cv:
            self.versions[p] = version
            self.log.append(("publish", p, version))
            self._cv.notify_all()

    def finish_tracking(self):
        with self._cv:
            self.tracking_done = True
            self._cv.notify_all()

    def fail(self, exc):
        with self._cv:
            if self.error is None:
                self.error = exc
            self._cv.notify_all()

    def put(self, q, item):
        while True:
            if self.error is not None:
                raise Stopped()
            try:
                return q.put(item, timeout=self.POLL)
            except queue.Full:
                pass

    def get(self, q):
        while True:
            if self.error is not None:
                raise Stopped()
            try:
                return q.get(timeout=self.POLL)
            except queue.Empty:
                pass


_END = object()


def run_pipeline(tracker, mapper, streams=None, schedule=None):
    """Runs `tracker` and `mapper` on two host threads in the lag-one schedule (LagOneSchedule), each under its own CUDA stream when
    `streams` = (tracker_stream, mapper_stream) is given (torch's current stream is per thread).  Tracked scans go from one thread to
    the other through a queue of size 1 (nerfloam.py:29).  The first exception of either thread stops both; both are joined and the
    exception is re-raised here, so no thread outlives the call.  Returns the schedule.

    tracker: first_frame() -> frame, frame_ids() -> ids, track(id, version) -> frame.
    mapper: init(frame) -> version, optimise(frame) -> state, update(state) -> version, finish()."""
    sched = schedule if schedule is not None else LagOneSchedule()
    q = queue.Queue(maxsize=1)

    def on_stream(i):
        return torch.cuda.stream(streams[i]) if streams is not None else contextlib.nullcontext()

    def track_role():
        with on_stream(0):
            sched.put(q, tracker.first_frame())
            for p, fid in enumerate(tracker.frame_ids(), 1):
                frame = tracker.track(fid, sched.map_version(p))
                sched.released(p)
                sched.put(q, frame)
            sched.finish_tracking()
            sched.put(q, _END)

    def map_role():
        with on_stream(1):
            sched.published(0, mapper.init(sched.get(q)))
            p = 0
            while True:
                frame = sched.get(q)
                if frame is _END:
                    break
                p += 1
                state = mapper.optimise(frame)
                # create_voxels rewrites rows of the structural arrays the tracker reads by reference; MapUpdater waits on the
                # stream for the release events that exist when it runs, so the release for scan p + 1 must have been recorded
                sched.wait_released(p + 1)
                sched.published(p, mapper.update(state))
            mapper.finish()

    def guarded(fn):
        def body():
            try:
                fn()
            except Stopped:
                pass
            except BaseException as e:          # noqa: BLE001 -- handed to run_pipeline's caller
                sched.fail(e)
        return body

    threads = [threading.Thread(target=guarded(track_role), name="nerfloam-tracker", daemon=True),
               threading.Thread(target=guarded(map_role), name="nerfloam-mapper", daemon=True)]
    for t in threads:
        t.start()
    try:
        for t in threads:
            t.join()
    except BaseException as e:                  # e.g. KeyboardInterrupt in the caller: stop the roles before leaving
        sched.fail(e)
        for t in threads:
            t.join()
        raise
    if sched.error is not None:
        raise sched.error
    return sched


# ----------------------------------------------------------------------------------------------------------------------------
# map files
# ----------------------------------------------------------------------------------------------------------------------------
MAP_FORMAT = "nerfloam_b200.map/1"
MAP_KEYS = ("format", "map", "decoder", "trajectory", "scan_ids", "config")
CONFIG_KEYS = ("criteria", "tracker_specs", "voxel_size", "data_specs", "dataset")

SavedMap = namedtuple("SavedMap", ["map", "decoder", "decoder_specs", "trajectory", "scan_ids", "config"])
SavedMap.__doc__ = """A run's map: map (mapping.MapUpdater), decoder (lidar.Decoder), decoder_specs (dict), trajectory f64[S,4,4] (the
poses of frame_poses.txt, without POSE_OFFSET), scan_ids i64[S] and config (criteria, tracker_specs, voxel_size, data_specs, dataset
as plain types).  write_map takes one, load_map returns one."""


def _plain(v, where):
    """`v` as built-in types (what torch.load(weights_only=True) reads back); anything else raises ValueError naming `where`."""
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    if isinstance(v, np.integer):
        return int(v)
    if isinstance(v, np.floating):
        return float(v)
    if isinstance(v, (list, tuple)):
        return [_plain(x, f"{where}[{i}]") for i, x in enumerate(v)]
    if isinstance(v, dict):
        return {str(k): _plain(x, f"{where}.{k}") for k, x in v.items()}
    raise ValueError(f"write_map: {where} is a {type(v).__name__}, not a plain type")


def map_config(args):
    """What a map file keeps of a run's configuration (load_config's namespace): criteria, tracker_specs, the mapper's voxel_size,
    data_specs and dataset, as plain types."""
    return _plain({"criteria": args.criteria, "tracker_specs": args.tracker_specs, "voxel_size": args.mapper_specs["voxel_size"],
                   "data_specs": args.data_specs, "dataset": args.dataset}, "config")


def write_map(path, saved):
    """One torch.save file of `saved` (SavedMap) that torch.load(..., weights_only=True) reads: format, map (MapUpdater.state_dict()),
    decoder ({"params": the flat fp32 parameters in state_dict() order, "decoder_specs"}), trajectory f64[S,4,4], scan_ids i64[S]
    and config.  The file is written next to `path` and renamed over it, so a failed write leaves no partial map behind."""
    traj = torch.as_tensor(np.asarray(saved.trajectory, dtype=np.float64)).clone()
    ids = torch.as_tensor(np.asarray(saved.scan_ids, dtype=np.int64)).clone()
    if traj.dim() != 3 or traj.shape[1:] != (4, 4) or traj.shape[0] < 1 or ids.shape != (traj.shape[0],):
        raise ValueError(f"write_map: need trajectory [S,4,4] and scan_ids [S] with S >= 1, got {list(traj.shape)} and {list(ids.shape)}")
    if not bool(torch.isfinite(traj).all()):
        raise ValueError("write_map: the trajectory has non-finite poses")
    config = _plain(dict(saved.config), "config")
    missing = [k for k in CONFIG_KEYS if k not in config]
    if missing:
        raise ValueError(f"write_map: config lacks {', '.join(missing)}")
    if float(config["voxel_size"]) != saved.map.voxel_size:
        raise ValueError(f"write_map: config voxel_size {config['voxel_size']} is not the map's {saved.map.voxel_size}")
    obj = {"format": MAP_FORMAT, "map": saved.map.state_dict(),
           "decoder": {"params": _flat_decoder_state(saved.decoder).to("cpu", copy=True), "decoder_specs": _plain(dict(saved.decoder_specs), "decoder_specs")},
           "trajectory": traj, "scan_ids": ids, "config": config}
    tmp = f"{os.fspath(path)}.part"
    torch.save(obj, tmp)
    os.replace(tmp, path)


def _decoder_size(specs):
    """Number of parameters of Decoder(**specs), built on the meta device (no memory, no draw from torch's generator)."""
    with torch.device("meta"):
        return sum(p.numel() for p in Decoder(**specs).state_dict().values())


def grown_trajectory(saved, poses, scan_ids):
    """The trajectory and scan ids of a saved map grown by a later drive: the saved ones (SavedMap) followed by the drive's poses
    f64[S,4,4] (without POSE_OFFSET) and ids, in that order.  Ids may repeat across drives: the map file only keeps them beside the
    poses.  Returns (f64[S0 + S,4,4], i64[S0 + S])."""
    traj = np.concatenate([np.asarray(saved.trajectory, dtype=np.float64).reshape(-1, 4, 4), np.asarray(poses, dtype=np.float64).reshape(-1, 4, 4)])
    ids = np.concatenate([np.asarray(saved.scan_ids, dtype=np.int64).reshape(-1), np.asarray(scan_ids, dtype=np.int64).reshape(-1)])
    return traj, ids


BASE_KEYS = ("voxel_size", "decoder_specs", "criteria")


def check_base_config(args, saved):
    """A run that grows `saved` (SavedMap) must agree with it on what its decoder was trained for: voxel_size (the run's
    mapper_specs.voxel_size), decoder_specs and criteria (the truncation and loss weights).  ValueError naming the first key that
    differs."""
    ours = {"voxel_size": args.mapper_specs["voxel_size"], "decoder_specs": args.decoder_specs, "criteria": args.criteria}
    theirs = {"voxel_size": saved.config["voxel_size"], "decoder_specs": saved.decoder_specs, "criteria": saved.config["criteria"]}
    for k in BASE_KEYS:
        if _plain(ours[k], k) != _plain(theirs[k], k):
            raise ValueError(f"base_map: the config's {k} {ours[k]!r} differs from the map's {theirs[k]!r}")


def _check_map_file(obj):
    """The checks of a map file above the map itself (from_state_dict checks that); the names of the failed ones."""
    if not isinstance(obj, dict):
        return ["a dict"]
    missing = [k for k in MAP_KEYS if k not in obj]
    if missing:
        return ["keys " + ", ".join(missing)]
    bad = []
    if obj["format"] != MAP_FORMAT:
        bad.append(f"format {obj['format']!r} (this version reads {MAP_FORMAT!r})")
    if not isinstance(obj["map"], dict):
        bad.append("map a dict")
    dec = obj["decoder"]
    if not isinstance(dec, dict) or not isinstance(dec.get("decoder_specs"), dict) or not isinstance(dec.get("params"), torch.Tensor):
        bad.append("decoder a dict of params and decoder_specs")
    elif dec["params"].dtype != torch.float32 or dec["params"].dim() != 1:
        bad.append("decoder params a flat float32 tensor")
    else:
        try:
            n = _decoder_size(dec["decoder_specs"])
        except (TypeError, ValueError, NotImplementedError) as e:
            bad.append(f"decoder_specs a supported decoder ({e})")
        else:
            if dec["params"].numel() != n:
                bad.append(f"decoder params of {n} values for its decoder_specs (got {dec['params'].numel()})")
            elif not bool(torch.isfinite(dec["params"]).all()):
                bad.append("decoder params finite")
    traj, ids = obj["trajectory"], obj["scan_ids"]
    if not isinstance(traj, torch.Tensor) or traj.dtype != torch.float64:
        bad.append("trajectory a float64 tensor")
    elif traj.dim() != 3 or traj.shape[1:] != (4, 4) or traj.shape[0] < 1:
        bad.append(f"trajectory of shape [S,4,4] with S >= 1 (got {list(traj.shape)})")
    elif not bool(torch.isfinite(traj).all()):
        bad.append("trajectory poses finite")
    elif not torch.equal(traj[:, 3], torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=torch.float64).expand(traj.shape[0], 4)):
        bad.append("trajectory poses with last row 0 0 0 1")
    if not isinstance(ids, torch.Tensor) or ids.dtype != torch.int64:
        bad.append("scan_ids an int64 tensor")
    elif isinstance(traj, torch.Tensor) and tuple(ids.shape) != (traj.shape[0],):
        bad.append(f"scan_ids of shape [{traj.shape[0]}] (one per pose, got {list(ids.shape)})")
    cfg = obj["config"]
    if not isinstance(cfg, dict):
        bad.append("config a dict")
    else:
        gone = [k for k in CONFIG_KEYS if k not in cfg]
        if gone:
            bad.append("config keys " + ", ".join(gone))
        else:
            for k in ("criteria", "tracker_specs", "data_specs"):
                if not isinstance(cfg[k], dict):
                    bad.append(f"config {k} a dict")
            if cfg["dataset"] not in ("kitti", "maicity"):
                bad.append(f"config dataset kitti or maicity (got {cfg['dataset']!r})")
            vs = cfg["voxel_size"]
            if isinstance(obj["map"], dict) and (not isinstance(vs, (int, float)) or vs != obj["map"].get("voxel_size")):
                bad.append(f"config voxel_size equal to the map's (got {vs!r} and {obj['map'].get('voxel_size')!r})")
    return bad


def load_map(path, octree="host", device="cuda"):
    """A map file (write_map, NeRFLOAM.save_map) -> SavedMap: the MapUpdater restored onto `octree` ("host" or "device",
    MapUpdater.from_state_dict), a Decoder on `device` carrying the saved parameters, and the other fields.  A malformed file raises
    ValueError naming the failed checks (a missing key, a wrong dtype or shape, a format mismatch, non-finite poses); a malformed map
    inside it raises NerfLoamError (from_state_dict's checks)."""
    try:
        obj = torch.load(path, map_location="cpu", weights_only=True)
    except (OSError, EOFError) as e:
        raise ValueError(f"load_map: cannot read {path}: {e}") from e
    except Exception as e:                  # noqa: BLE001 -- torch.load raises pickle / zip / runtime errors for a foreign file
        raise ValueError(f"load_map: {path} is not a map file: {e}") from e
    bad = _check_map_file(obj)
    if bad:
        raise ValueError(f"load_map: {path} is a malformed map file, failed checks: " + "; ".join(bad))
    mu = MapUpdater.from_state_dict(obj["map"], device=device, octree=octree)
    specs = dict(obj["decoder"]["decoder_specs"])
    with torch.device("meta"):
        decoder = Decoder(**specs)
    decoder = load_flat_decoder_state(decoder.to_empty(device=device), obj["decoder"]["params"].to(device))
    return SavedMap(mu, decoder, specs, obj["trajectory"], obj["scan_ids"], obj["config"])


# ----------------------------------------------------------------------------------------------------------------------------
# the whole system
# ----------------------------------------------------------------------------------------------------------------------------
def load_dataset(args):
    """get_dataset (src/utils/import_util.py): dataset.<name>.DataLoader over data_specs."""
    loader = importlib.import_module(f".dataset.{args.dataset}", __package__).DataLoader
    ds = args.data_specs
    return loader(ds["data_path"], use_gt=ds["use_gt"], max_depth=ds["max_depth"], min_depth=ds["min_depth"])


class NeRFLOAM:
    """nerfloam.py:7-51: the tracker and the mapper of one sequence, run by run() concurrently on two host threads and two CUDA streams.

    config: dict / namespace / YAML path (load_config).  out_dir: where mesh/ and misc/ are written.  data_stream: a loader with
    __len__, __getitem__ -> (index, points, pointsCos, pose or None) and get_init_pose (default: dataset.<dataset>.DataLoader over
    data_specs).  selection: the mapping window, 'current' (the reference's), 'previous' or 'overlap' (KeyframeGraph).  init_calls:
    'current' mapping calls on the first scan.  The constructor seeds torch, numpy and random with `seeding` like run.py:13-23 (the
    decoder's initial weights come from torch's generator); the tracker and the mapper then draw from generators of their own.

    base_map: a map file (write_map) or a SavedMap (on the host octree) to grow with this sequence instead of starting an empty map
    (DESIGN.md section 11.6).  The config must agree with it on BASE_KEYS (check_base_config); its "global_specs" key overrides
    localise.GLOBAL_SPECS.  The first scan is placed as localise.Localiser places it (localise.place_first over the saved trajectory,
    drawing from the tracker's generator), and run() raises NerfLoamError, writing nothing, when no placement hits the map.  The saved
    MapUpdater is grown in place, with reserve_nodes / reserve_rows of room like a new map (MapUpdater.reserve); its decoder is never
    stepped and its rows stay fixed (Mapping's map_updater); frame_poses.txt holds
    this sequence's poses, and save_map writes the saved trajectory followed by them.  None: an empty map, as before."""

    def __init__(self, config, out_dir, data_stream=None, selection="current", init_calls=12, reserve_nodes=1 << 20, reserve_rows=1 << 20,
                 base_map=None):
        args = load_config(config)
        self.args, self.out_dir = args, out_dir
        self.base = None
        if base_map is not None:
            self.base = base_map if isinstance(base_map, SavedMap) else load_map(base_map, octree="host")
            if self.base.map.on_device:
                raise ValueError("base_map: the map must be on the host octree (load_map(..., octree='host'))")
            check_base_config(args, self.base)
            self.base.map.reserve(reserve_nodes, reserve_rows)     # the room a new map would have had
        torch.manual_seed(args.seeding)
        torch.cuda.manual_seed_all(args.seeding)
        np.random.seed(args.seeding)
        random.seed(args.seeding)
        self.data_stream = data_stream if data_stream is not None else load_dataset(args)
        dspec = dict(args.decoder_specs)
        decoder = Decoder(**dspec).cuda() if self.base is None else self.base.decoder
        self.shared = SharedMap(lambda: Decoder(**dspec).cuda())
        self.tracker = Tracking(args, self.data_stream, self.shared, torch.Generator().manual_seed(args.seeding),
                                place=None if self.base is None else self._place_first)
        self.mapper = Mapping(args, out_dir, self.shared, decoder, torch.Generator().manual_seed(args.seeding + 1), selection, init_calls,
                              reserve_nodes, reserve_rows, map_updater=None if self.base is None else self.base.map)
        self.streams = (torch.cuda.Stream(), torch.cuda.Stream())
        self.schedule = None
        self.placement, self.place_ms = None, None

    def _place_first(self, frame):
        """The first scan's pose in the base map, as Localiser places it (localise.place_first over the saved trajectory, with
        localise.GLOBAL_SPECS under the config's global_specs), drawing from the tracker's generator."""
        from .localise import GLOBAL_SPECS, place_first, trajectory_anchors          # localise imports this module
        specs = {**GLOBAL_SPECS, **(getattr(self.args, "global_specs", None) or {})}
        times = {}
        try:
            self.placement = place_first(frame, self.base.map.map_states["_mapstate"], self.base.decoder, self.tracker,
                                         trajectory_anchors(self.base.trajectory), specs, self.tracker.generator, times, "NeRFLOAM")
        finally:
            self.place_ms = {"search": times["place"][0] if "place" in times else None, "track": times.get("polish", [None])[0]}

    def run(self):
        """Runs the sequence and returns a summary: scans, keyframes, the wall time, and per stage the median host milliseconds per
        scan (track, load: the tracker's; map, update, publish: the mapper's) and the refinement times."""
        t0 = time.perf_counter()
        self.schedule = run_pipeline(self.tracker, self.mapper, self.streams)
        torch.cuda.synchronize()
        return self.summary((time.perf_counter() - t0) * 1e3)

    def saved_map(self):
        """The finished run's map as a SavedMap over the live objects (no copy): the mapper's MapUpdater and decoder after the final
        refinement (the map final_mesh.ply was made from), the trajectory frame_poses.txt holds and the scans' ids."""
        m = self.mapper
        if m.map_state is None or m.trajectory.frame_poses or not m.trajectory.final_poses:
            raise RuntimeError("save_map: the run has not finished (call run() first)")
        traj, ids = np.stack(m.trajectory.final_poses).astype(np.float64), np.asarray(m.scan_ids, dtype=np.int64)
        if self.base is not None:
            traj, ids = grown_trajectory(self.base, traj, ids)
        return SavedMap(m.map, m.decoder, dict(self.args.decoder_specs), traj, ids, map_config(self.args))

    def save_map(self, path):
        """Writes the finished run's map to one file (write_map); localise.Localiser and load_map read it."""
        write_map(path, self.saved_map())

    def summary(self, wall_ms):
        times = {**self.tracker.times, **self.mapper.times}
        n = len(self.mapper.trajectory.final_poses)
        out = {"scans": n, "keyframes": len(self.mapper.keyframe_indices), "wall_ms": wall_ms, "ms_per_scan_wall": wall_ms / max(n, 1),
               "ms_per_scan": {k: float(np.median(v)) for k, v in times.items() if k not in ("init", "refine")},
               "init_ms": times.get("init", [0.0])[0], "refine_ms": times.get("refine", []), "out_dir": self.out_dir}
        if self.base is not None:           # the first scan's placement and the saved map's size, rows held fixed
            out["base"] = {"place_ms": self.place_ms, "frozen_rows": self.mapper.frozen_rows, "rows": int(self.mapper.map.n_rows),
                           "nodes": int(self.mapper.map.n_nodes)}
        return out
