"""`Octree` with the method set of the reference's torch.classes.svo.Octree
(third_party/sparse_octree/src/bindings.cpp:11-31), backed by the flat-array host octree of
libnerfloam_b200.so (csrc/octree_host.cpp).

Differences from the reference class, all deliberate:
  * node ids are per-tree (the reference's counter is a process global, octree.h:62, so a second
    instance corrupts its exports);
  * `get_centres_and_children()` is a direct array pass (no per-node torch dispatch);
  * `export_map()` returns the arrays already in the layout the hot path consumes (mapping.py:320-326);
  * pickling replays the inserted point tensors like the reference (bindings.cpp:23-31) and is wired; a tree restored from node
    arrays (`load_nodes`), which has no point history, pickles as its node arrays instead.
"""
import ctypes as C

import numpy as np
import torch

from . import _capi


def _np_ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def validate_nodes(grid_dim, child, code, type_, level, vertex2row=None, n_rows=0):
    """nl_octree_validate on CPU node arrays (child i32[n,8], code i64[n], type i8[n], level u8[n], vertex2row i32[n] or None):
    the OR of the failed NL_TREE_* checks' bits, 0 for a well-formed tree (_capi.tree_checks_failed names them)."""
    a = [np.ascontiguousarray(t.numpy() if isinstance(t, torch.Tensor) else t) for t in (child, code, type_, level)]
    v = None if vertex2row is None else np.ascontiguousarray(vertex2row.numpy() if isinstance(vertex2row, torch.Tensor) else vertex2row)
    n = a[2].shape[0]
    bits = int(_capi.lib().nl_octree_validate(int(grid_dim), n, *(_np_ptr(x) for x in a), None if v is None else _np_ptr(v), int(n_rows)))
    if bits < 0:
        raise _capi.NerfLoamError(_capi.lib().nl_last_error().decode())
    return bits


def malformed_tree(what, bits):
    return _capi.NerfLoamError(f"{what}: malformed octree state, failed checks: {', '.join(_capi.tree_checks_failed(bits))}")


def encode(x, y, z):
    """svo.encode (bindings.cpp:6): 63-bit Morton key of integer voxel coordinates (utils.h:106-109)."""
    return int(_capi.lib().nl_morton_encode(int(x), int(y), int(z)))


def grown(buf, n, keep, fill=None, floor=0):
    """`buf` (a torch tensor or a numpy array) if it has room for n rows, else a new buffer like it of max(n, 2 * its rows, floor)
    rows that holds its first `keep` rows, the others set to `fill` (None: uninitialised).  Capacity doubling, so that the
    addresses of a growing buffer change at most log2(size) times."""
    cap = buf.shape[0]
    if n <= cap:
        return buf
    shape = (max(n, 2 * cap, floor), *buf.shape[1:])
    if isinstance(buf, np.ndarray):
        new = np.empty(shape, buf.dtype) if fill is None else np.full(shape, fill, buf.dtype)
    else:
        new = buf.new_empty(shape) if fill is None else buf.new_full(shape, fill)
    new[:keep] = buf[:keep]
    return new


def _int32(vox):
    """Voxel coordinates as the reference's accessor<int,2> takes them: a tensor must be int32, anything else is converted."""
    if not isinstance(vox, torch.Tensor):
        return torch.from_numpy(np.ascontiguousarray(vox, dtype=np.int32))
    if vox.dtype != torch.int32:
        raise RuntimeError("expected an int32 tensor (the reference accessor<int,2> throws here)")
    return vox.detach()


class _ReferenceMethods:
    """The input rules of the reference's methods (octree.cpp, bindings.cpp:11-31), shared by both trees: each method checks its
    input here and hands a well-formed int32 [N,3] batch (a CPU numpy [3] for has_voxel) to the tree's _insert / _try_insert /
    _has_voxel."""

    def _check(self):
        if self._init_args is None:
            raise RuntimeError("Octree not initialized!")  # octree.cpp:56-59 prints this and carries on

    def _check_query(self):
        self._check()

    # -- bindings.cpp:15 insert(Tensor int32[N,3])
    def insert(self, vox):
        self._check()
        v = _int32(vox)
        if v.dim() != 2 or v.shape[1] != 3:
            print(f"Point dimensions mismatch: inputs are {v.shape[-1]} expect 3")  # octree.cpp:62-66
            return
        self._insert(v)

    def try_insert(self, vox):
        """The share of the batch's distinct corner keys that are already in the tree (-1.0 for an empty or malformed batch)."""
        self._check_query()
        v = _int32(vox)
        if v.dim() != 2 or v.shape[1] != 3 or v.shape[0] == 0:
            return -1.0
        return self._try_insert(v)

    def has_voxel(self, xyz):
        self._check()
        v = _int32(xyz).cpu().contiguous().numpy().reshape(-1)
        if v.shape[0] != 3:
            return False
        return self._has_voxel(v)

    def get_features(self, pts):
        """Empty body in the reference (octree.cpp:208-210)."""
        return None


class Octree(_ReferenceMethods):
    def __init__(self):
        self._h = None
        self._all_pts = []              # None: restored from node arrays, no point history
        self._init_args = None

    # -- bindings.cpp:14 init(grid_dim, feat_dim, voxel_size)
    def init(self, grid_dim, feat_dim, voxel_size):
        if self._h is not None:
            _capi.lib().nl_octree_destroy(self._h)
        self._init_args = None
        self._h = _capi.lib().nl_octree_create(int(grid_dim), int(feat_dim), float(voxel_size))
        if not self._h:
            raise _capi.NerfLoamError(_capi.lib().nl_last_error().decode())
        self._init_args = (int(grid_dim), int(feat_dim), float(voxel_size))
        self._all_pts = []

    def _insert(self, v):
        v = v.cpu().contiguous().numpy()
        _capi.check(_capi.lib().nl_octree_insert(self._h, _np_ptr(v), v.shape[0]), "nl_octree_insert")
        if self._all_pts is not None:
            self._all_pts.append(torch.from_numpy(v.copy()))

    def _try_insert(self, v):
        v = v.cpu().contiguous().numpy()
        return float(_capi.lib().nl_octree_try_insert(self._h, _np_ptr(v), v.shape[0]))

    def _has_voxel(self, v):
        return bool(_capi.lib().nl_octree_has_voxel(self._h, _np_ptr(v)))

    def count_nodes(self):
        self._check()
        return int(_capi.lib().nl_octree_count_nodes(self._h))

    def count_leaf_nodes(self):
        self._check()
        return int(_capi.lib().nl_octree_count_leaf_nodes(self._h))

    def get_voxels(self):
        self._check()
        n = self.count_nodes()
        out = np.empty((n, 4), np.float32)
        rows = _capi.lib().nl_octree_get_voxels(self._h, out.ctypes.data_as(C.c_void_p), n)
        return torch.from_numpy(out[:rows])

    def get_leaf_voxels(self):
        self._check()
        n = self.count_leaf_nodes()
        out = np.empty((max(n, 1), 3), np.float32)
        rows = _capi.lib().nl_octree_get_leaf_voxels(self._h, out.ctypes.data_as(C.c_void_p), n)
        return torch.from_numpy(out[:rows])

    # -- bindings.cpp:22 get_centres_and_children() -> (voxels f32[n,4], children f32[n,8], features i32[n,8])
    def get_centres_and_children(self):
        self._check()
        n = int(_capi.lib().nl_octree_count_export_nodes(self._h))
        voxels = np.empty((n, 4), np.float32)
        children = np.empty((n, 8), np.float32)
        features = np.empty((n, 8), np.int32)
        _capi.check(_capi.lib().nl_octree_export(self._h, voxels.ctypes.data_as(C.c_void_p), children.ctypes.data_as(C.c_void_p),
                                                 features.ctypes.data_as(C.c_void_p)), "nl_octree_export")
        return torch.from_numpy(voxels), torch.from_numpy(children), torch.from_numpy(features)

    def export_map(self):
        """(centres f32[n,3], structure i32[n,9], vertex i32[n,8]) == what mapping.py:320-326 derives."""
        self._check()
        n = int(_capi.lib().nl_octree_count_export_nodes(self._h))
        centres = np.empty((n, 3), np.float32)
        structure = np.empty((n, 9), np.int32)
        vertex = np.empty((n, 8), np.int32)
        _capi.check(_capi.lib().nl_octree_export_map(self._h, centres.ctypes.data_as(C.c_void_p),
                                                     structure.ctypes.data_as(C.c_void_p), vertex.ctypes.data_as(C.c_void_p)),
                    "nl_octree_export_map")
        return torch.from_numpy(centres), torch.from_numpy(structure), torch.from_numpy(vertex)

    def export_dirty(self, clear=True):
        """Incremental export: (ids i32[m] ascending, centres f32[m,3], structure i32[m,9], vertex i32[m,8]) of the rows that
        changed since the last clearing call -- scattering them into the previous export gives the full export bit for bit."""
        self._check()
        m = int(_capi.lib().nl_octree_dirty_count(self._h))
        ids = np.empty(m, np.int32)
        centres = np.empty((m, 3), np.float32)
        structure = np.empty((m, 9), np.int32)
        vertex = np.empty((m, 8), np.int32)
        _capi.check(_capi.lib().nl_octree_export_dirty(self._h, ids.ctypes.data_as(C.c_void_p), centres.ctypes.data_as(C.c_void_p),
                                                       structure.ctypes.data_as(C.c_void_p), vertex.ctypes.data_as(C.c_void_p), int(bool(clear))),
                    "nl_octree_export_dirty")
        return ids, centres, structure, vertex

    def count_export_nodes(self):
        self._check()
        return int(_capi.lib().nl_octree_count_export_nodes(self._h))

    def is_dirty(self):
        """True if rows changed since the last clearing export_dirty (inserts a map update has not applied yet)."""
        self._check()
        return int(_capi.lib().nl_octree_dirty_count(self._h)) > 0

    def export_nodes(self):
        """The tree's node arrays as CPU tensors: child i32[n,8], code i64[n] (the u64 bit pattern), type i8[n], level u8[n]
        (side = grid_dim >> level), the layout of DeviceOctree's arrays and of MapUpdater.state_dict()."""
        self._check()
        n = self.count_nodes()
        a = (np.empty((n, 8), np.int32), np.empty(n, np.uint64), np.empty(n, np.int8), np.empty(n, np.uint8))
        _capi.check(_capi.lib().nl_octree_nodes(self._h, *(_np_ptr(x) for x in a)), "nl_octree_nodes")
        return torch.from_numpy(a[0]), torch.from_numpy(a[1].view(np.int64)), torch.from_numpy(a[2]), torch.from_numpy(a[3])

    def load_nodes(self, child, code, type_, level):
        """Replace the tree by node arrays (export_nodes' layout) in O(n), without replaying points.  Malformed arrays raise
        NerfLoamError naming the failed checks and leave the tree as it was.  The restored tree has nothing dirty; having no point
        history, it pickles as its node arrays from now on."""
        self._check()
        a = [np.ascontiguousarray(t.numpy() if isinstance(t, torch.Tensor) else t) for t in (child, code, type_, level)]
        for x, dt in zip(a, (np.int32, np.int64, np.int8, np.uint8)):
            if x.dtype != dt and not (dt == np.int64 and x.dtype == np.uint64):
                raise _capi.NerfLoamError(f"Octree.load_nodes: expected {np.dtype(dt).name} node arrays, got {x.dtype}")
        n = a[2].shape[0]
        if a[0].shape != (n, 8) or a[1].shape != (n,) or a[3].shape != (n,):
            raise _capi.NerfLoamError("Octree.load_nodes: node arrays of mismatched shapes")
        rc = int(_capi.lib().nl_octree_restore(self._h, *(_np_ptr(x) for x in a), n))
        if rc < 0:
            raise _capi.NerfLoamError(_capi.lib().nl_last_error().decode())
        if rc > 0:
            raise malformed_tree("Octree.load_nodes", rc)
        self._all_pts = None

    # -- pickle (bindings.cpp:23-31): state = (size, feat_dim, voxel_size, all inserted tensors), replayed on load.  A tree restored
    # from node arrays has no inserted tensors to replay and pickles as its node arrays.
    def __getstate__(self):
        if self._all_pts is None and self._init_args is not None:
            return {"init": self._init_args, "nodes": tuple(t.numpy() for t in self.export_nodes())}
        return {"init": self._init_args, "all_pts": self._all_pts}

    def __setstate__(self, state):
        self._h = None
        self._all_pts = []
        self._init_args = None
        if state["init"] is not None:
            self.init(*state["init"])
            if "nodes" in state:
                self.load_nodes(*state["nodes"])
            else:
                for p in state["all_pts"]:
                    self.insert(p)

    def __del__(self):
        try:
            if self._h is not None:
                _capi.lib().nl_octree_destroy(self._h)
                self._h = None
        except Exception:
            pass


_NONE_U32 = -1          # 0xffffffff as int32: an empty entry of the pending dirty list
_REST = 2 ** 31 - 1     # resting value of the per-node scratch word


def _at(t, byte_offset):
    return C.c_void_p(t.data_ptr() + byte_offset)


class DeviceOctree(_ReferenceMethods):
    """`Octree` with the tree in device memory (csrc/octree_dev.cu, include/nerfloam_b200.h section 1b): the same node ids,
    exports and counts as the host tree bit for bit, without copying the batch or the tree to the host.

    `insert` accepts CPU or CUDA int32 [N,3] and reads back two counters (the rejection flag and the number of new nodes, to grow
    the capacity-doubling node arrays).  Like the host tree, it rejects a batch with a coordinate outside [0, grid_dim-2] as a
    whole (NerfLoamError) and leaves the tree unchanged.  `export_map` returns CPU tensors like `Octree.export_map`;
    `export_dirty` (numpy, like the host) and `update_map` (straight into a MapUpdater's device buffers) export the rows changed
    since the last dirty export.  `get_centres_and_children`, `get_voxels` and `get_leaf_voxels` return the host tree's CPU
    tensors; `try_insert` takes CPU or CUDA input and reads back 16 bytes.

    Pickling (and so deepcopy and torch.save) stores the init arguments and the node arrays as CPU arrays, 42 bytes per node, not
    the inserted points, and restores onto the current CUDA device.  The arrays are checked on the device before anything walks
    them; a malformed state raises NerfLoamError.  A restored tree is in the state of a restored host tree: every row is dirty, so
    the next `export_dirty` returns all of them, and later inserts and exports equal the host tree's.  It has no embedding-row
    state, so `update_map` refuses it (MapUpdater.from_state_dict restores a tree together with its rows)."""

    def __init__(self, device="cuda"):
        self.device = torch.device(device)
        self._init_args = None
        self._counts = None
        self._restored = False

    def init(self, grid_dim, feat_dim, voxel_size):
        gd = int(grid_dim)
        if gd < 2 or gd > (1 << 20) or gd & (gd - 1):
            raise _capi.NerfLoamError("DeviceOctree.init: grid_dim must be a power of two in [2, 2^20]")
        self._init_args = (gd, int(feat_dim), float(voxel_size))
        self._restored = False
        d = self.device
        self._child = torch.empty((0, 8), dtype=torch.int32, device=d)
        self._code, self._type, self._level, self._scratch = (torch.empty(0, dtype=t, device=d)
                                                              for t in (torch.int64, torch.int8, torch.uint8, torch.int32))
        self._n = 0
        self._grow(4096)
        self._n = 1                     # the root, id 0 (octree.cpp:41-43): its row is the fill values of _grow
        self._base = 0                  # node count at the last dirty export: ids >= base are dirty
        self._pending_points = 0        # points inserted since the last dirty export
        self._list = torch.full((1024,), _NONE_U32, dtype=torch.int32, device=d)
        self._list_used = 0
        self._counts = torch.zeros(8, dtype=torch.int64, device=d)
        self._qcounts = torch.zeros(2, dtype=torch.int64, device=d)   # the queries' read-back block
        self._ws = torch.empty(0, dtype=torch.uint8, device=d)
        self._ids = torch.empty(1024, dtype=torch.int32, device=d)

    @property
    def grid_dim(self):
        return self._init_args[0]

    def _ptrs(self, *names):
        """C pointers of the node arrays `names` ("child", "code", "type", "level", "scratch"); by default the tree's four, in the
        order every entry point takes them."""
        return [_capi.ptr(getattr(self, "_" + k)) for k in names or self._STATE]

    def _grow(self, n):
        k = self._n
        self._child, self._code, self._type, self._level, self._scratch = (
            grown(a, n, k, fill, 4096) for a, fill in zip((self._child, self._code, self._type, self._level, self._scratch), (-1, 0, -1, 0, _REST)))

    def _workspace(self, n_points, query_nodes=None):
        """The workspace of an insert / export of n_points, or with query_nodes given, of a query over that many nodes."""
        L = _capi.lib()
        if query_nodes is None:
            nb = int(L.nl_devoctree_workspace_bytes(int(n_points), self.grid_dim))
        else:
            nb = int(L.nl_devoctree_query_workspace_bytes(int(query_nodes), int(n_points), self.grid_dim))
        if nb < 0:
            raise _capi.NerfLoamError(L.nl_last_error().decode())
        if nb > self._ws.numel():
            self._ws = torch.empty(nb, dtype=torch.uint8, device=self.device)
        return self._ws

    def _check_query(self):
        if self.device.type != "cuda":
            raise NotImplementedError("DeviceOctree's queries run on a CUDA device; use svo.Octree on the CPU")
        self._check()

    def _insert(self, v):
        v = v.to(self.device).contiguous()
        n = v.shape[0]
        if n == 0:
            return
        L = _capi.lib()
        ws = self._workspace(n)
        _capi.check(L.nl_devoctree_insert_count(self.grid_dim, *self._ptrs("child"), _capi.ptr(v), n, _capi.ptr(ws), ws.numel(),
                                                _capi.ptr(self._counts), _capi.stream_ptr()), "nl_devoctree_insert_count")
        bad, n_new = self._counts[:2].tolist()                       # read-back 1: rejection flag, new nodes
        if bad:
            raise _capi.NerfLoamError("DeviceOctree.insert: voxel coordinate outside [0, grid_dim-2]; the batch was rejected "
                                      "and the tree is unchanged")
        n0 = self._n
        self._grow(n0 + n_new)
        need = self._list_used + min(self._base, 10 * n)            # pending-list entries this batch may append
        self._list = grown(self._list, need, self._list_used, _NONE_U32)
        _capi.check(L.nl_devoctree_insert_commit(self.grid_dim, n0, n_new, self._base, *self._ptrs(), *self._ptrs("scratch"),
                                                 _capi.ptr(self._list), n, _capi.ptr(ws), ws.numel(), _capi.ptr(self._counts),
                                                 _capi.stream_ptr()), "nl_devoctree_insert_commit")
        _capi.LAUNCHES += 2
        self._list_used = need
        self._n = n0 + n_new
        self._pending_points += n

    def count_nodes(self):
        self._check()
        return self._n

    def count_export_nodes(self):
        self._check()
        return self._n

    def count_leaf_nodes(self):
        self._check()
        return int((self._type[:self._n] == 0).sum())

    def is_dirty(self):
        """Octree.is_dirty: nodes, pending dirty rows or points since the last dirty export."""
        self._check()
        return self._base != self._n or self._list_used > 0 or self._pending_points > 0

    def _has_voxel(self, v):
        out = torch.empty(1, dtype=torch.int32, device=self.device)
        _capi.check(_capi.lib().nl_devoctree_find(self.grid_dim, *self._ptrs("child"), _capi.ptr(torch.from_numpy(v).to(self.device)), 1,
                                                  _capi.ptr(out), _capi.stream_ptr()), "nl_devoctree_find")
        return bool(int(out[0]) >= 0)

    def _export(self, rows, ids, count_ptr, compact, centres, structure, vertex):
        _capi.check(_capi.lib().nl_devoctree_export(self.grid_dim, self._init_args[2], rows, _capi.ptr(ids), count_ptr, int(compact),
                                                    *self._ptrs(), _capi.ptr(centres), _capi.ptr(structure), _capi.ptr(vertex),
                                                    _capi.stream_ptr()), "nl_devoctree_export")
        _capi.LAUNCHES += 1

    def export_map(self):
        """(centres f32[n,3], structure i32[n,9], vertex i32[n,8]) on the CPU, equal to Octree.export_map()."""
        self._check()
        n, d = self._n, self.device
        c = torch.empty((n, 3), dtype=torch.float32, device=d)
        s = torch.empty((n, 9), dtype=torch.int32, device=d)
        v = torch.empty((n, 8), dtype=torch.int32, device=d)
        self._export(n, None, None, False, c, s, v)
        return c.cpu(), s.cpu(), v.cpu()

    def _dirty_ids(self):
        """Sorted dirty ids into self._ids (device count in counts[2]); returns (their bound, points since the last export)."""
        rows = self._list_used + self._n - self._base
        self._ids = grown(self._ids, rows, 0)
        pts = self._pending_points
        ws = self._workspace(pts)
        _capi.check(_capi.lib().nl_devoctree_dirty_ids(self.grid_dim, self._n, self._base, self._list_used, _capi.ptr(self._list),
                                                       *self._ptrs("scratch"), _capi.ptr(self._ids), pts, _capi.ptr(ws), ws.numel(),
                                                       _capi.ptr(self._counts), _capi.stream_ptr()), "nl_devoctree_dirty_ids")
        _capi.LAUNCHES += 1
        self._base, self._list_used, self._pending_points = self._n, 0, 0
        return rows, pts

    def export_dirty(self, clear=True):
        """Octree.export_dirty(): (ids i32[m] ascending, centres f32[m,3], structure i32[m,9], vertex i32[m,8]) as numpy arrays."""
        self._check()
        if not clear:
            raise NotImplementedError("DeviceOctree.export_dirty always clears the dirty rows")
        rows, _ = self._dirty_ids()
        d = self.device
        c = torch.empty((rows, 3), dtype=torch.float32, device=d)
        s = torch.empty((rows, 9), dtype=torch.int32, device=d)
        v = torch.empty((rows, 8), dtype=torch.int32, device=d)
        self._export(rows, self._ids, _at(self._counts, 16), True, c, s, v)
        m = int(self._counts[2])
        return (self._ids[:m].cpu().numpy(), c[:m].cpu().numpy(), s[:m].cpu().numpy(), v[:m].cpu().numpy())

    def update_map(self, centres, structure, vertex, vertex2row, vox2row, n_emb_rows):
        """The dirty export of a map update, on the device: the changed rows go to their node ids in the (capacity-sized, >= n
        rows) centres / structure / vertex / vox2row buffers, new vertices get embedding rows n_emb_rows.. in vertex2row.
        Reads back the dirty-row count and the new number of embedding rows; returns (ids, m, rows): the first m entries of
        ids (device) are the dirty node ids."""
        self._check()
        if self._restored:
            raise _capi.NerfLoamError("DeviceOctree.update_map: an unpickled tree has no embedding-row state to continue from; "
                                      "a MapUpdater builds its own tree")
        rows, pts = self._dirty_ids()
        self._export(rows, self._ids, _at(self._counts, 16), False, centres, structure, vertex)
        ws = self._workspace(pts)
        _capi.check(_capi.lib().nl_devoctree_assign_rows(self.grid_dim, rows, _capi.ptr(self._ids), self._n, *self._ptrs("type"),
                                                         _capi.ptr(vertex), _capi.ptr(vertex2row), *self._ptrs("scratch"), int(n_emb_rows),
                                                         _capi.ptr(vox2row), pts, _capi.ptr(ws), ws.numel(), _capi.ptr(self._counts),
                                                         _capi.stream_ptr()), "nl_devoctree_assign_rows")
        _capi.LAUNCHES += 1
        m, n_rows = self._counts[2:4].tolist()                      # read-back 2: dirty rows, embedding rows
        return self._ids, m, n_rows

    def rebuild_map(self, centres, structure, vertex, vertex2row, vox2row, n_emb_rows):
        """The full export of a tree loaded together with its embedding rows (MapUpdater.from_state_dict): every row into the
        row = node id buffers of update_map, and vox2row composed from vertex2row.  Every vertex already has its row (the load
        validated it), so no row is numbered and nothing is read back."""
        self._check()
        n = self._n
        self._export(n, None, None, False, centres, structure, vertex)
        ids = torch.arange(n, dtype=torch.int32, device=self.device)
        self._counts[2].fill_(n)                                        # the id list's device-side length
        ws = self._workspace(0, query_nodes=n)
        _capi.check(_capi.lib().nl_devoctree_assign_rows(self.grid_dim, n, _capi.ptr(ids), n, *self._ptrs("type"), _capi.ptr(vertex),
                                                         _capi.ptr(vertex2row), *self._ptrs("scratch"), int(n_emb_rows), _capi.ptr(vox2row),
                                                         0, _capi.ptr(ws), ws.numel(), _capi.ptr(self._counts), _capi.stream_ptr()),
                    "nl_devoctree_assign_rows")
        _capi.LAUNCHES += 1

    def _try_insert(self, v):
        v = v.to(self.device).contiguous()
        n = v.shape[0]
        ws = self._workspace(n, query_nodes=0)
        _capi.check(_capi.lib().nl_devoctree_try_insert(self.grid_dim, *self._ptrs("child"), _capi.ptr(v), n, _capi.ptr(ws), ws.numel(),
                                                        _capi.ptr(self._qcounts), _capi.stream_ptr()), "nl_devoctree_try_insert")
        _capi.LAUNCHES += 1
        hits, keys = self._qcounts.tolist()
        return 1.0 * hits / keys

    def _preorder(self, out, leaves_only):
        ws = self._workspace(0, query_nodes=self._n)
        _capi.check(_capi.lib().nl_devoctree_preorder(self.grid_dim, self._n, *self._ptrs("code", "type", "level"),
                                                      int(leaves_only), _capi.ptr(out), _capi.ptr(self._qcounts),
                                                      _capi.ptr(ws), ws.numel(), _capi.stream_ptr()), "nl_devoctree_preorder")
        _capi.LAUNCHES += 1

    def get_voxels(self):
        """Octree.get_voxels: f32[n,4] (xyz, side) of every node in preorder, on the CPU."""
        self._check_query()
        out = torch.empty((self._n, 4), dtype=torch.float32, device=self.device)
        self._preorder(out, False)
        return out.cpu()

    def get_leaf_voxels(self):
        """Octree.get_leaf_voxels: f32[m,3] of the SURFACE leaves in preorder, on the CPU."""
        self._check_query()
        out = torch.empty((self._n, 3), dtype=torch.float32, device=self.device)
        self._preorder(out, True)
        return out[:int(self._qcounts[0])].cpu()

    def get_centres_and_children(self):
        """Octree.get_centres_and_children: (voxels f32[n,4], children f32[n,8], features i32[n,8]) on the CPU."""
        self._check_query()
        n, d = self._n, self.device
        voxels = torch.empty((n, 4), dtype=torch.float32, device=d)
        children = torch.empty((n, 8), dtype=torch.float32, device=d)
        features = torch.empty((n, 8), dtype=torch.int32, device=d)
        _capi.check(_capi.lib().nl_devoctree_export_nodes(self.grid_dim, self._init_args[2], n, None, None, 0, *self._ptrs(),
                                                          _capi.ptr(voxels), _capi.ptr(children), None, None, _capi.ptr(features),
                                                          _capi.stream_ptr()), "nl_devoctree_export_nodes")
        _capi.LAUNCHES += 1
        return voxels.cpu(), children.cpu(), features.cpu()

    def export_nodes(self):
        """Octree.export_nodes: child i32[n,8], code i64[n], type i8[n], level u8[n] as CPU tensors."""
        self._check()
        n = self._n
        return self._child[:n].cpu(), self._code[:n].cpu(), self._type[:n].cpu(), self._level[:n].cpu()

    def validate(self, vertex2row=None, n_rows=0):
        """nl_devoctree_validate over the tree's n nodes (with vertex2row, a device i32 tensor of >= n entries, the row checks too):
        the OR of the failed NL_TREE_* checks' bits, 0 for a well-formed tree.  Reads back 16 bytes."""
        self._check()
        ws = self._workspace(0, query_nodes=self._n)
        _capi.check(_capi.lib().nl_devoctree_validate(self.grid_dim, self._n, *self._ptrs(), _capi.ptr(vertex2row), int(n_rows), _capi.ptr(ws), ws.numel(),
                                                      _capi.ptr(self._qcounts), _capi.stream_ptr()), "nl_devoctree_validate")
        _capi.LAUNCHES += 1
        structural, rows = self._qcounts.tolist()
        return structural | rows

    def load_nodes(self, child, code, type_, level, vertex2row=None, n_rows=0):
        """Replace the tree by node arrays (CPU tensors in export_nodes' layout, dtypes and shapes checked by the caller): one
        host-to-device copy per array, then `validate` (with vertex2row / n_rows: the caller's device table, already uploaded).
        On success the tree is clean, nothing dirty; malformed arrays raise NerfLoamError naming the failed checks and leave the
        tree uninitialised."""
        self._check()
        n = type_.shape[0]
        self._grow(n)
        for src, dst in zip((child, code, type_, level), (self._child, self._code, self._type, self._level)):
            dst[:n].copy_(src)
        self._n = n
        self._base, self._list_used, self._pending_points = n, 0, 0
        self._restored = False
        bits = self.validate(vertex2row, n_rows)
        if bits:
            self._init_args = None
            raise malformed_tree("DeviceOctree.load_nodes", bits)

    _STATE = ("child", "code", "type", "level")

    def __getstate__(self):
        if self._init_args is None:
            return {"init": None}
        return {"init": self._init_args, **{k: a.numpy() for k, a in zip(self._STATE, self.export_nodes())}}

    def __setstate__(self, state):
        self.device = torch.device("cuda", torch.cuda.current_device())
        self._init_args = None
        self._counts = None
        self._restored = False
        if state["init"] is None:
            return
        self.init(*state["init"])
        self.load_nodes(*(torch.from_numpy(np.ascontiguousarray(state[k])) for k in self._STATE))
        self._base = 0                  # no pending entries, scratch at rest: every row is dirty, as after a host replay
        self._restored = True
