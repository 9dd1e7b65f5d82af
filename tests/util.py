"""Shared helpers for the tests (golden loading, map construction through the product API)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
G = os.path.join(ROOT, "tests", "golden")


PART_BYTES = 900_000


def save_golden(path, **arrays):
    """np.savez_compressed, split into parts <stem>.<i>.npz of at most PART_BYTES of raw array bytes each, so that every stored
    file stays under 1 MB (golden() merges them).  A larger array is stored as row chunks <key>@<j>."""
    stem = path[:-len(".npz")]
    chunks = {}
    for k, v in arrays.items():
        v = np.asarray(v)
        if v.nbytes <= PART_BYTES:
            chunks[k] = v
            continue
        rows = max(1, PART_BYTES // (v.nbytes // v.shape[0]))
        for j in range(0, v.shape[0], rows):
            chunks[f"{k}@{j // rows}"] = v[j:j + rows]
    parts, cur, size = [], {}, 0
    for k, v in chunks.items():
        if cur and size + v.nbytes > PART_BYTES:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    for i, part in enumerate(parts):
        np.savez_compressed(f"{stem}.{i}.npz", **part)


def golden(name):
    """tests/golden/<name>; an archive above 1 MB is stored as parts <stem>.<i>.npz (save_golden), merged here."""
    p = os.path.join(G, name)
    if os.path.exists(p):
        return np.load(p)
    stem = name[:-len(".npz")]
    parts = sorted(f for f in os.listdir(G) if f.startswith(stem + ".") and f[len(stem) + 1:-len(".npz")].isdigit())
    if not parts:
        raise FileNotFoundError(p)
    out, chunks = _Archive(), {}
    for f in parts:
        with np.load(os.path.join(G, f)) as z:
            for k in z.files:
                if "@" in k:
                    name, j = k.rsplit("@", 1)
                    chunks.setdefault(name, {})[int(j)] = z[k]
                else:
                    out[k] = z[k]
    for name, c in chunks.items():
        out[name] = np.concatenate([c[j] for j in range(len(c))])
    return out


class _Archive(dict):
    """The merged parts of a split archive, with np.load's `files`."""

    @property
    def files(self):
        return list(self)


def bf16_from_bits(a):
    return torch.from_numpy(a.copy()).view(torch.bfloat16)


def product_map(vox, voxel_size, id2emb=None, emb_bits=None, device="cuda", grid_dim=256 * 256 * 4):
    """Octree + MapState through the product code (svo.Octree.export_map + engine.MapState)."""
    import nerfloam_b200 as nl
    o = nl.svo.Octree()
    o.init(grid_dim, 16, voxel_size)
    o.insert(torch.from_numpy(np.ascontiguousarray(vox, np.int32)))
    centres, structure, vertex = o.export_map()
    out = {"octree": o, "centres": centres, "structure": structure, "vertex": vertex}
    if id2emb is not None:
        v = vertex.long()
        flat = torch.from_numpy(id2emb.reshape(-1)).long()
        rows = torch.where(v >= 0, flat[v.clamp(min=0)], torch.full_like(v, -1)).int()
        out["vox2row"] = rows
        if emb_bits is not None:
            emb = bf16_from_bits(emb_bits).to(device)
            out["state"] = nl.engine.MapState(centres, structure, rows, emb, device)
    return out


def ref_grid():
    """The compiled, unmodified reference `grid` extension (oracle/_ref/grid), or None when it was not built."""
    p = os.path.join(ROOT, "oracle", "_ref", "grid", "grid_ref.so")
    if not os.path.exists(p):
        return None
    import importlib.util
    spec = importlib.util.spec_from_file_location("grid_ref", p)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_decoder(z, prefix, device="cuda", width=256):
    import nerfloam_b200 as nl
    dec = nl.lidar.Decoder(depth=2, width=width, in_dim=16, skips=[], embedder="none", multires=0)
    sd = {k[len(prefix):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(prefix)}
    dec.load_state_dict(sd)
    return dec.to(device)


class Args:
    def __init__(self, max_depth=40.0, trunc=0.3):
        self.criteria = {"eiko_weight": 0.1, "sdf_weight": 10000.0, "fs_weight": 1, "sdf_truncation": trunc}
        self.data_specs = {"max_depth": max_depth}
