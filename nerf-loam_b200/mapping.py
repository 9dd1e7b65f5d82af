"""Map update glue between the octree and the optimisation loop (SURVEY.md section 8 a-14):
Mapping.create_voxels / update_grid_features / get_embeddings of src/mapping.py:283-339.

What changes relative to the reference:
  * no 8 GB `voxel_id2embedding_id` CPU lookup (mapping.py:76): a compact i32[n_nodes] vertex->row table;
  * one embedding row per distinct vertex (the reference allocates a row per *reference* to a new vertex,
    ~70 % orphan rows, SURVEY.md A.1); values are identical because new rows are zero-initialised;
  * the bf16 table grows in place on the device (capacity doubling) instead of CPU cat + full re-upload;
  * the octree export is already in hot-path layout (centres / structure / vertex) -- svo.Octree.export_map.
`map_states` keeps the reference's dict keys so the reference's tracker/mesher can read it, plus
"_mapstate" (engine.MapState) which the fused renderer uses directly.
`octree="device"` keeps the octree itself on the GPU (svo.DeviceOctree): the voxels of a scan never leave the device, and the
update patches the same buffers with the same ids and rows as the host tree.
"""
import ctypes as C

import numpy as np
import torch

from . import _capi
from .engine import MapState
from .svo import DeviceOctree, Octree, grown, malformed_tree, validate_nodes


class _LazyMapStates(dict):
    """The reference-format map_states dict of a device-octree update.  "_mapstate" and "voxel_vertex_emb" are device objects and
    present at once; the CPU tensors (vertex / centres / structure / id table) are copied from the device the first time one of
    them is read, so a loop that never reads them never pays the copy.  The dict belongs to one map version: read it before the
    next update."""
    _LAZY = ("voxel_vertex_idx", "voxel_center_xyz", "voxel_structure", "voxel_id2embedding_id")

    def __init__(self, eager, build):
        super().__init__(eager)
        self._build = build

    def _materialise(self):
        if self._build is not None:
            build, self._build = self._build, None
            super().update(build())

    def __getitem__(self, k):
        if k in self._LAZY:
            self._materialise()
        return super().__getitem__(k)

    def get(self, k, default=None):
        if k in self._LAZY:
            self._materialise()
        return super().get(k, default)

    def __contains__(self, k):
        return k in self._LAZY or super().__contains__(k)

    def __iter__(self):
        self._materialise()
        return super().__iter__()

    def __len__(self):
        self._materialise()
        return super().__len__()

    def keys(self):
        self._materialise()
        return super().keys()

    def values(self):
        self._materialise()
        return super().values()

    def items(self):
        self._materialise()
        return super().items()

    def copy(self):
        self._materialise()
        return dict(super().items())

    def __repr__(self):
        self._materialise()
        return super().__repr__()


class MapUpdater:
    """Device-resident map, updated incrementally (SURVEY.md section 8 f-1).

    All hot-path arrays -- centres, structure, vox2row, the packed traversal image, the bf16 table -- live in capacity-doubling
    DEVICE buffers whose base addresses stay put between doublings.  A map update uploads only the rows the insertion touched
    (svo.Octree.export_dirty: new nodes, nodes that gained a child, leaves that turned SURFACE and their parents), scatters them
    in place, numbers the new vertices and re-packs the touched nodes; the reference re-exports the whole octree with a torch
    dispatcher call per node and re-uploads everything every frame (octree.cpp:293-342, mapping.py:309-337).  Stable addresses are
    also what lets the captured CUDA graphs of the optimisation loops (render_helpers._MapGraph / _TrackGraph) survive map updates.
    `incremental=False` keeps the full-export path (used by the tests as the cross-check).
    `octree="device"` (CUDA, incremental only) inserts into svo.DeviceOctree instead: the scan's voxels stay on the device and the
    update exports, numbers and re-packs the dirty rows there too, reading back only the new-node, dirty-row and embedding-row
    counts (new rows drawn with init_std > 0 still come from the CPU generator, so their values equal the host path's)."""

    def __init__(self, voxel_size, embed_dim=16, grid_dim=256 * 256 * 4, device="cuda", init_std=0.0, seed=0, incremental=True,
                 reserve_nodes=0, reserve_rows=0, octree="host"):
        assert embed_dim == 16
        if octree not in ("host", "device"):
            raise ValueError(f"octree must be 'host' or 'device', not {octree!r}")
        self.voxel_size = float(voxel_size)
        self.device = torch.device(device)
        self.on_device = octree == "device"
        if self.on_device and (self.device.type != "cuda" or not incremental):
            raise ValueError("octree='device' needs a CUDA device and the incremental update")
        self.svo = DeviceOctree(self.device) if self.on_device else Octree()
        self.svo.init(grid_dim, embed_dim, voxel_size)     # mapping.py:81-82
        self.n_rows = 0
        self.n_nodes = 0
        self._emb_buf = torch.zeros((1024, embed_dim), dtype=torch.bfloat16, device=self.device)
        self.init_std = init_std
        self._gen = torch.Generator(device="cpu").manual_seed(seed)
        self.map_states = None
        self.incremental = bool(incremental) and self.device.type == "cuda"
        # capacity-doubling buffers indexed by node id (_grow_nodes): the hot-path arrays on the device; the vertex ids and the
        # vertex -> row table where the tree numbers the rows (host tree: numpy, device tree: device); the host tree also keeps
        # host mirrors of centres and structure for the reference-format dict
        d, i32 = self.device, torch.int32
        self._centres, self._packed = torch.zeros((0, 3), dtype=torch.float32, device=d), torch.zeros(0, dtype=torch.uint8, device=d)
        self._structure, self._vox2row = torch.zeros((0, 9), dtype=i32, device=d), torch.zeros((0, 8), dtype=i32, device=d)
        if self.on_device:
            self._vertex, self._v2r = torch.zeros((0, 8), dtype=i32, device=d), torch.zeros(0, dtype=i32, device=d)
            self._host = ()
        else:
            self._vertex, self._v2r = np.zeros((0, 8), np.int32), np.zeros(0, np.int32)
            self._host = (np.zeros((0, 3), np.float32), np.zeros((0, 9), np.int32))
        self.generation = 0
        self.last_update = {}
        self.readers = None          # optional share.SharedMap: in-place updates wait (on the stream) for its readers
        # reserve_*: initial capacities.  Every capacity doubling moves the buffers (one device copy) and invalidates captured graphs;
        # a run that knows its map size (a KITTI sequence at 0.3 m: ~10^6 nodes = 0.3 GB of the 180 GB) reserves it once
        if self.incremental and reserve_nodes:
            self._grow_nodes(int(reserve_nodes))
        if reserve_rows and reserve_rows > self._emb_buf.shape[0]:
            self._emb_buf = torch.zeros((int(reserve_rows), embed_dim), dtype=torch.bfloat16, device=self.device)

    @property
    def embeddings(self):
        return self._emb_buf[:self.n_rows]

    @property
    def vertex2row(self):
        """i32 vertex (node id) -> embedding row, -1 = none (numpy; copied from the device with octree="device")."""
        return torch.as_tensor(self._v2r[:self.n_nodes]).cpu().numpy()

    # -- checkpoints ------------------------------------------------------------------------------------------------------------
    FORMAT = 1

    def state_dict(self):
        """The map as a plain dict of CPU tensors and Python scalars (loads with torch.load(..., weights_only=True)):
        format, grid_dim, embed_dim, voxel_size, init_std, generation; generator (the CPU generator's state, so rows drawn with
        init_std > 0 continue the same stream); the tree as node arrays child i32[n,8], code i64[n] (u64 bit pattern), type i8[n],
        level u8[n]; vertex2row i32[n] and embeddings bf16[n_rows,16] (the current, trained values).  Host and device trees give
        equal dicts for the same insert history.  Raises NerfLoamError if the tree holds inserts not yet applied to the map
        (svo.insert without update_grid_features): such a map could not continue bit for bit."""
        n = self.n_nodes
        if self.svo.is_dirty() or self.svo.count_nodes() != n:
            raise _capi.NerfLoamError("MapUpdater.state_dict: the octree has inserts that were not applied to the map yet; "
                                      "call update_grid_features() first")
        child, code, type_, level = self.svo.export_nodes()
        gd, _, _ = self.svo._init_args
        return {"format": self.FORMAT, "grid_dim": int(gd), "embed_dim": int(self._emb_buf.shape[1]), "voxel_size": self.voxel_size,
                "init_std": float(self.init_std), "generation": int(self.generation), "generator": self._gen.get_state(),
                "child": child, "code": code, "type": type_, "level": level,
                "vertex2row": torch.from_numpy(np.array(self.vertex2row[:n], dtype=np.int32)),
                "embeddings": self.embeddings.detach().to("cpu", copy=True)}

    _STATE_DTYPES = {"child": torch.int32, "code": torch.int64, "type": torch.int8, "level": torch.uint8, "vertex2row": torch.int32,
                     "embeddings": torch.bfloat16, "generator": torch.uint8}

    @classmethod
    def _check_state(cls, sd):
        """The checks of a checkpoint that need no tree walk; the names of the failed ones."""
        if not isinstance(sd, dict):
            return ["a dict"]
        missing = [k for k in ("format", "grid_dim", "embed_dim", "voxel_size", "init_std", "generation", *cls._STATE_DTYPES) if k not in sd]
        if missing:
            return ["keys " + ", ".join(missing)]
        bad = []
        if sd["format"] != cls.FORMAT:
            bad.append(f"format {sd['format']!r} (this version reads {cls.FORMAT})")
        gd = sd["grid_dim"]
        if not isinstance(gd, int) or gd < 2 or gd > 1 << 20 or gd & (gd - 1):
            bad.append("grid_dim a power of two in [2, 2^20]")
        if sd["embed_dim"] != 16:
            bad.append("embed_dim 16")
        for k, dt in cls._STATE_DTYPES.items():
            if not isinstance(sd[k], torch.Tensor) or sd[k].dtype != dt or sd[k].device.type != "cpu":
                bad.append(f"{k} a CPU {dt} tensor")
        if bad:
            return bad
        n = sd["type"].shape[0]
        shapes = {"child": (n, 8), "code": (n,), "type": (n,), "level": (n,), "vertex2row": (n,)}
        bad += [f"{k} of shape {list(s)}" for k, s in shapes.items() if tuple(sd[k].shape) != s]
        if sd["embeddings"].dim() != 2 or sd["embeddings"].shape[1] != 16:
            bad.append("embeddings of shape [n_rows, 16]")
        return bad

    @classmethod
    def from_state_dict(cls, sd, device="cuda", octree="host", incremental=True, reserve_nodes=0, reserve_rows=0):
        """A new MapUpdater holding the map of `sd` (state_dict()), on either octree whichever tree saved it.  The node arrays and
        the row table are checked (the NL_TREE_* checks of include/nerfloam_b200.h) before anything walks them: a malformed
        checkpoint raises NerfLoamError naming the failed checks.  The buffers, host mirrors, vertex2row, embeddings and map_states
        equal the saved updater's, the tree is clean, and every later create_voxels gives what the saved updater would have given.
        With octree="device" each checkpoint array is copied to the device once and 16 bytes come back."""
        bad = cls._check_state(sd)
        if bad:
            raise _capi.NerfLoamError("MapUpdater.from_state_dict: malformed checkpoint, failed checks: " + "; ".join(bad))
        n, n_rows = sd["type"].shape[0], sd["embeddings"].shape[0]
        nodes = tuple(sd[k].contiguous() for k in ("child", "code", "type", "level"))
        v2r = sd["vertex2row"].contiguous()
        mu = cls(sd["voxel_size"], sd["embed_dim"], sd["grid_dim"], device=device, init_std=sd["init_std"], incremental=incremental,
                 reserve_nodes=max(int(reserve_nodes), n), reserve_rows=max(int(reserve_rows), n_rows), octree=octree)
        mu._gen.set_state(sd["generator"])
        mu._emb_buf[:n_rows].copy_(sd["embeddings"])
        mu.n_rows = n_rows
        mu._v2r = grown(mu._v2r, n, 0, -1)
        torch.as_tensor(mu._v2r)[:n].copy_(v2r)             # numpy (host tree) or device (device tree): one copy either way
        if mu.on_device:
            mu.svo.load_nodes(*nodes, vertex2row=mu._v2r, n_rows=n_rows)
        else:
            bits = validate_nodes(sd["grid_dim"], *nodes, v2r, n_rows)
            if bits:
                raise malformed_tree("MapUpdater.from_state_dict", bits)
            mu.svo.load_nodes(*nodes)
        if mu.incremental:
            ids, m, _ = mu._patch_rows(n, every_row=True)
            mu.n_nodes = n
            mu._pack_rows(ids, m)
            mu._publish()
        else:
            mu._update_full()
        mu.generation = sd["generation"]
        return mu

    def create_voxels(self, points, pose):
        """mapping.py:283-291: sensor-frame points [N,3] + 4x4 pose -> voxel coordinates -> octree -> map_states."""
        pts = torch.as_tensor(points, dtype=torch.float32, device=self.device)
        T = torch.as_tensor(pose, dtype=torch.float32, device=self.device)
        world = pts @ T[:3, :3].transpose(-1, -2) + T[:3, 3]
        voxels = torch.div(world, self.voxel_size, rounding_mode="floor")
        self.svo.insert(voxels.int())
        return self.update_grid_features()

    def insert_voxels(self, voxels_i32):
        self.svo.insert(voxels_i32)
        return self.update_grid_features()

    # ---------------------------------------------------------------------------------------------------------------
    def _grow_rows(self, new_rows):
        self._emb_buf = grown(self._emb_buf, new_rows, self.n_rows, 0)          # grow in place (mapping.py:309-314 re-uploads everything)
        if self.init_std > 0 and new_rows > self.n_rows:                       # reference: zeros (mapping.py:305-307)
            add = torch.randn((new_rows - self.n_rows, 16), generator=self._gen) * self.init_std
            self._emb_buf[self.n_rows:new_rows] = add.to(torch.bfloat16).to(self.device)
        self.n_rows = new_rows

    def reserve(self, nodes=0, rows=0):
        """Room for at least `nodes` nodes and `rows` embedding rows: one move of the buffers now instead of capacity doublings later
        (each of which invalidates the captured graphs).  The map's contents are unchanged; map_states is re-published over the
        moved buffers."""
        moved = False
        if self.incremental and int(nodes) > self._centres.shape[0]:
            self._grow_nodes(int(nodes))
            moved = True
        if int(rows) > self._emb_buf.shape[0]:
            self._emb_buf = grown(self._emb_buf, int(rows), self.n_rows, 0)
            moved = True
        if moved and self.incremental and self.map_states is not None:
            self._publish()

    def _grow_nodes(self, n):
        k = self.n_nodes
        self._centres, self._structure, self._vox2row, self._vertex, self._v2r = (
            grown(b, n, k, fill, 4096) for b, fill in ((self._centres, 0), (self._structure, -1), (self._vox2row, -1), (self._vertex, -1),
                                                       (self._v2r, -1)))
        self._packed = grown(self._packed, 128 * n, 128 * k, 0, 128 * 4096)
        self._host = tuple(grown(b, n, k, None, 4096) for b in self._host)

    def update_grid_features(self):
        """mapping.py:320-339.  Returns the engine.MapState (also stored, with the reference's dict keys, in self.map_states)."""
        if not self.incremental:
            return self._update_full()
        n = self.svo.count_export_nodes()
        if self.readers is not None:
            # a tracker on another stream may still traverse the arrays that are patched below; waiting before the capacity growth
            # also orders this stream after those reads, so a buffer the growth frees cannot be reused under them
            for ev in self.readers.reader_events():
                torch.cuda.current_stream(self.device).wait_event(ev)
        self._grow_nodes(n)
        ids, m, new_rows = self._patch_rows(n)
        self._grow_rows(new_rows)
        self._pack_rows(ids, m)
        self.n_nodes = n
        self.generation += 1
        self.last_update = {"dirty_rows": int(m), "nodes": int(n), "embedding_rows": int(new_rows)}
        return self._publish()

    def _patch_rows(self, n, every_row=False):
        """Writes the rows that changed since the last update (every_row: all n rows of a restored tree) into the node buffers, at
        row = node id, and numbers their new vertices.  Returns (ids, m, rows): ids[:m] are the patched node ids (device), rows
        the new number of embedding rows."""
        if self.on_device:
            if not every_row:
                return self.svo.update_map(self._centres, self._structure, self._vertex, self._v2r, self._vox2row, self.n_rows)
            self.svo.rebuild_map(self._centres, self._structure, self._vertex, self._v2r, self._vox2row, self.n_rows)
            return torch.arange(n, dtype=torch.int32, device=self.device), n, self.n_rows
        if every_row:
            ids, (c, s, v) = np.arange(n, dtype=np.int32), (t.numpy() for t in self.svo.export_map())
        else:
            ids, c, s, v = self.svo.export_dirty()
        m = ids.shape[0]
        rows = np.empty((m, 8), np.int32)
        new_rows = int(_capi.lib().nl_assign_embedding_rows_subset(v.ctypes.data_as(C.c_void_p), m, n, self._v2r.ctypes.data_as(C.c_void_p),
                                                                   self.n_rows, rows.ctypes.data_as(C.c_void_p)))
        if new_rows < 0:
            raise _capi.NerfLoamError(_capi.lib().nl_last_error().decode())
        idx = None
        if m:
            d = self.device
            idx = torch.from_numpy(ids).to(d, non_blocking=True)
            idl = idx.long()
            self._centres.index_copy_(0, idl, torch.from_numpy(c).to(d, non_blocking=True))
            self._structure.index_copy_(0, idl, torch.from_numpy(s).to(d, non_blocking=True))
            self._vox2row.index_copy_(0, idl, torch.from_numpy(rows).to(d, non_blocking=True))
        self._host[0][ids], self._host[1][ids], self._vertex[ids] = c, s, v
        return idx, m, new_rows

    def _pack_rows(self, ids, m):
        """Re-packs the traversal image of the nodes ids[:m]."""
        if m:
            _capi.check(_capi.lib().nl_octree_pack_children_rows(m, _capi.ptr(ids), _capi.ptr(self._centres), _capi.ptr(self._structure),
                                                                 _capi.ptr(self._packed), _capi.stream_ptr()), "nl_octree_pack_children_rows")
            _capi.LAUNCHES += 1

    def _publish(self):
        """The MapState of the current map version over the buffers, and self.map_states."""
        n = self.n_nodes
        # emb_full: the capacity-sized table at a stable address (rows >= n_rows: zero, never referenced); stable: the base addresses
        # survive map updates until a capacity doubling
        ms = MapState.view(self._centres[:n], self._structure[:n], self._vox2row[:n], self.embeddings, emb_full=self._emb_buf,
                           stable=True, packed=self._packed[:n * 128])
        if self.on_device:
            c, s, v, r = self._centres[:n], self._structure[:n], self._vertex[:n], self._v2r[:n]
            build = lambda: {"voxel_vertex_idx": v.cpu(), "voxel_center_xyz": c.cpu(), "voxel_structure": s.cpu(),
                             "voxel_id2embedding_id": r.cpu().view(-1, 1)}
            self.map_states = _LazyMapStates({"voxel_vertex_emb": self.embeddings, "_mapstate": ms}, build)
        else:          # CPU tensors like mapping.py:321-337, over the host mirrors
            c, s = (torch.from_numpy(a[:n]) for a in self._host)
            self.map_states = {"voxel_vertex_idx": torch.from_numpy(self._vertex[:n]), "voxel_center_xyz": c, "voxel_structure": s,
                               "voxel_vertex_emb": self.embeddings, "voxel_id2embedding_id": torch.from_numpy(self._v2r[:n]).view(-1, 1),
                               "_mapstate": ms}
        return ms

    def _update_full(self):
        self.svo.export_dirty()                                                # keep the dirty list from growing without bound
        centres, structure, vertex = self.svo.export_map()                     # mapping.py:321-326
        n = centres.shape[0]
        self._v2r = grown(self._v2r, n, self.n_nodes, -1)
        v = vertex.numpy()
        new_rows = int(_capi.lib().nl_assign_embedding_rows(v.ctypes.data_as(C.c_void_p), n, self._v2r.ctypes.data_as(C.c_void_p), self.n_rows))
        if new_rows < 0:
            raise _capi.NerfLoamError(_capi.lib().nl_last_error().decode())
        self._grow_rows(new_rows)
        self.n_nodes = n
        self.generation += 1
        vox2row = np.where(v >= 0, self._v2r[np.clip(v, 0, None)], -1).astype(np.int32)
        d = self.device
        ms = MapState.view(centres.to(d), structure.to(d), torch.from_numpy(vox2row).to(d), self.embeddings)
        id2 = torch.from_numpy(self._v2r[:n].copy()).view(-1, 1)
        self.map_states = {"voxel_vertex_idx": vertex, "voxel_center_xyz": centres, "voxel_structure": structure,
                           "voxel_vertex_emb": self.embeddings, "voxel_id2embedding_id": id2, "_mapstate": ms}
        return ms
