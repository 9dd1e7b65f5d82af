"""Tracker <-> mapper hand-off on the device (SURVEY.md section 8 f-4).

The reference hands the map from the mapper process to the tracker process once per scan through a multiprocessing Manager
(src/share.py:12-121, src/mapping.py:227-232, src/tracking.py:101-106): `deepcopy(decoder)` three times, every map_states tensor moved
to the CPU, the whole dict -- including the 8 GB voxel_id2embedding_id table -- pickled through the Manager's connection, and
the embedding table uploaded again on the other side.

Here the hand-off is a publication of DEVICE state:

  * SharedMap (one process, two CUDA streams): `publish()` takes a consistent snapshot of what the tracker reads -- the embedding
    rows and the decoder parameters, one device-to-device copy each (~1 MB) into a double-buffered slot -- and records an event;
    the structural arrays (centres / structure / vox2row / packed image) are shared by reference, frozen at the published node
    count.  `acquire()` makes the tracker's stream wait for that event, `release()` records the event the mapper's next in-place
    map update waits for.  No host synchronisation, no copy of anything that did not change.
  * ShareData (drop-in for src/share.py's class, for the reference's two-process layout): the same properties and lock discipline,
    but `states` keeps device tensors -- torch's multiprocessing reductions send CUDA tensors through a Manager connection as CUDA IPC
    handles, so nothing is staged through host memory -- the id table is replaced by the compact composed voxel->row table, and
    the decoder travels as one flat device tensor instead of three deep copies of an nn.Module.
"""
from copy import deepcopy
from multiprocessing.managers import NamespaceProxy

import torch
import torch.multiprocessing as mp

from .engine import MapState


def _flat_decoder_state(decoder, out=None):
    """All decoder parameters as one flat fp32 device tensor (order of state_dict())."""
    ps = [p.detach().reshape(-1) for p in decoder.state_dict().values()]
    n = sum(p.numel() for p in ps)
    if out is None or out.numel() != n:
        out = torch.empty(n, dtype=torch.float32, device=ps[0].device)
    o = 0
    for p in ps:
        out[o:o + p.numel()].copy_(p, non_blocking=True)
        o += p.numel()
    return out


def load_flat_decoder_state(decoder, flat):
    """Inverse of _flat_decoder_state: copy the flat snapshot into `decoder`'s parameters (device to device)."""
    o = 0
    with torch.no_grad():
        for p in decoder.state_dict().values():
            p.copy_(flat[o:o + p.numel()].view(p.shape), non_blocking=True)
            o += p.numel()
    return decoder


class _Slot:
    def __init__(self):
        self.emb = None
        self.dec_flat = None
        self.decoder = None
        self.map = None
        self.published = None      # event: snapshot complete
        self.read_done = None      # event: the last reader finished
        self.version = -1


class SharedMap:
    """Publication of the mapper's state to a tracker running on another CUDA stream of the same process."""

    def __init__(self, decoder_factory):
        """decoder_factory(): a fresh decoder module on the device (the tracker's private copy, filled from the snapshots)."""
        self._slots = [_Slot(), _Slot()]
        self._front = -1
        self._factory = decoder_factory
        self.version = 0

    def publish(self, map_state, decoder):
        """Called on the mapper's stream after a map update / optimisation call."""
        s = self._slots[1 - self._front if self._front >= 0 else 0]
        cur = torch.cuda.current_stream()
        if s.read_done is not None:
            cur.wait_event(s.read_done)                      # the previous reader of this slot is done with it
        n_rows = map_state.emb.shape[0]
        if s.emb is None or s.emb.shape[0] < n_rows:
            full = map_state.emb_full                        # a MapUpdater map: mirror its capacity, so the slot's address is as stable as the map's
            want = max(n_rows, 2 * (s.emb.shape[0] if s.emb is not None else 0), full.shape[0] if full is not None else 0)
            s.emb = torch.empty((want, 16), dtype=torch.bfloat16, device=map_state.emb.device)
        s.emb[:n_rows].copy_(map_state.emb, non_blocking=True)
        s.dec_flat = _flat_decoder_state(decoder, s.dec_flat)
        # A MapUpdater map keeps its structural arrays at fixed addresses and each slot's table is a capacity buffer, so a slot is as
        # stable as the map it mirrors: the tracker's captured graph is reused per slot (render_helpers._TrackGraph keeps a few live)
        s.map = map_state.replace(emb=s.emb[:n_rows], emb_full=None)
        s.published = torch.cuda.Event()
        s.published.record(cur)
        self.version += 1
        s.version = self.version
        self._front = self._slots.index(s)
        return s.version

    def acquire(self, version=None):
        """Called on the tracker's stream: (map_state, decoder, slot).  The stream waits for the publication, not the host.
        version: None takes the latest publication; a number takes that publication (publish()'s return value), which must still
        be in one of the two slots -- a reader that lags by at most one publication and releases before the mapper publishes again
        (slam.NeRFLOAM's schedule) always finds it there.  A version that is not (any more, or not yet) held raises RuntimeError."""
        if self._front < 0:
            raise RuntimeError("nothing has been published yet")
        if version is None:
            s = self._slots[self._front]
        else:
            held = [t for t in self._slots if t.version == version]
            if not held:
                raise RuntimeError(f"map version {version} is not held (the slots hold {sorted(t.version for t in self._slots if t.version >= 0)})")
            s = held[0]
        torch.cuda.current_stream().wait_event(s.published)
        if s.decoder is None:
            s.decoder = self._factory()
        load_flat_decoder_state(s.decoder, s.dec_flat)
        return s.map, s.decoder, s

    def release(self, slot):
        slot.read_done = torch.cuda.Event()
        slot.read_done.record(torch.cuda.current_stream())

    def reader_events(self):
        """Events the mapper's next IN-PLACE map update has to wait for (the structural arrays are shared by reference)."""
        return [s.read_done for s in self._slots if s.read_done is not None]


class ShareDataProxy(NamespaceProxy):   # registered by the caller like src/nerfloam.py does (BaseManager.register)
    _exposed_ = ("__getattribute__", "__setattr__")


class ShareData:
    """Same interface as src/share.py:12-121 (decoder / voxels / octree / states / stop_* / tracking_trajectory / push_pose).
    `states` holds device tensors (sent as CUDA IPC handles across processes) and `decoder` is stored as a flat device tensor +
    constructor arguments; `decoder` returns a module rebuilt on the reader's side."""
    _lock = mp.RLock()

    def __init__(self):
        self._stop_mapping = False
        self._stop_tracking = False
        self._decoder_flat = None
        self._decoder_ctor = None
        self._decoder_obj = None
        self._voxels = None
        self._octree = None
        self._states = None
        self._trajectory = []

    @property
    def decoder(self):
        with self._lock:
            if self._decoder_ctor is None:
                return deepcopy(self._decoder_obj)
            cls, kwargs = self._decoder_ctor
            dec = cls(**kwargs).to(self._decoder_flat.device)
            return load_flat_decoder_state(dec, self._decoder_flat)

    @decoder.setter
    def decoder(self, decoder):
        with self._lock:
            kw = getattr(decoder, "ctor_kwargs", None)
            if kw is None or not next(decoder.parameters()).is_cuda:
                self._decoder_ctor, self._decoder_obj = None, deepcopy(decoder)      # unknown module type / host module: the reference's behaviour
                return
            self._decoder_ctor = (type(decoder), dict(kw))
            self._decoder_flat = _flat_decoder_state(decoder).clone()

    @property
    def states(self):
        with self._lock:
            return self._states

    @states.setter
    def states(self, states):
        """Accepts the reference's dict; tensors that are on the device stay there (no `.cpu()` round trip, mapping.py:229-231).
        A dict produced by mapping.MapUpdater is reduced to what the tracker reads."""
        with self._lock:
            ms = states.get("_mapstate") if isinstance(states, dict) else None
            if isinstance(ms, MapState):
                self._states = {"centres": ms.centres, "structure": ms.structure, "vox2row": ms.vox2row, "emb": ms.emb.clone(), "n_nodes": ms.n_nodes}
            else:
                self._states = states

    def map_state(self):
        """The tracker's view: an engine.MapState over the shared device arrays (or over the reference-format dict)."""
        with self._lock:
            st = self._states
            if st is None:
                return None
            if "vox2row" in st:
                return MapState(st["centres"], st["structure"], st["vox2row"], st["emb"], st["emb"].device)
            return MapState.from_map_states(st, "cuda")

    # --- the remaining properties of src/share.py, unchanged in meaning -------------------------------------------------
    @property
    def voxels(self):
        with self._lock:
            return deepcopy(self._voxels)

    @voxels.setter
    def voxels(self, v):
        with self._lock:
            self._voxels = deepcopy(v)

    @property
    def octree(self):
        with self._lock:
            return deepcopy(self._octree)

    @octree.setter
    def octree(self, o):
        with self._lock:
            self._octree = deepcopy(o)

    @property
    def stop_mapping(self):
        with self._lock:
            return self._stop_mapping

    @stop_mapping.setter
    def stop_mapping(self, v):
        with self._lock:
            self._stop_mapping = v

    @property
    def stop_tracking(self):
        with self._lock:
            return self._stop_tracking

    @stop_tracking.setter
    def stop_tracking(self, v):
        with self._lock:
            self._stop_tracking = v

    @property
    def tracking_trajectory(self):
        with self._lock:
            return deepcopy(self._trajectory)

    def push_pose(self, pose):
        with self._lock:
            self._trajectory.append(deepcopy(pose))
