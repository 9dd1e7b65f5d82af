"""Meshing (SURVEY.md section 8 f-3): sparse marching cubes on the GPU over the per-voxel SDF lattices.

Replaces MeshExtractor.create_mesh / marching_cubes of src/utils/mesh_util.py:80-169 up to the Open3D object: the reference
evaluates get_scores, copies every voxel's 8^3 lattice to the host and calls skimage.measure.marching_cubes once per voxel in a
Python loop.  Here the lattice never leaves the device and all voxels are triangulated by two kernel passes (csrc/mc.cu).

    verts, faces = mesh.extract_mesh(decoder, map_states, voxel_size, res=8)         # device tensors f32[V,3], i32[T,3]
    verts, faces = mesh.marching_cubes(centres, sdf_grid, voxel_size)                 # drop-in for MeshExtractor.marching_cubes (numpy out)
"""
import torch

from . import _capi
from .engine import MapState

INT32_MAX = 2 ** 31 - 1


@torch.no_grad()
def marching_cubes_device(sdf, centres, voxel_size, vox_ids=None):
    """sdf f32[n,res,res,res] (CUDA, lattice layout of get_scores), centres f32[N,3] (CUDA), vox_ids i32[n] rows of `centres`
    (None: row v) -> (verts f32[V,3], faces i32[T,3]) on the device.  One 16-byte read-back (the totals) to size the outputs.
    Raises ValueError, before allocating them, when either total is above INT32_MAX (vertex ids and offsets are int32)."""
    if not sdf.is_cuda:
        raise RuntimeError("marching cubes runs on the GPU only (no CPU fallback)")
    sdf = sdf.float().contiguous()
    n, res = sdf.shape[0], sdf.shape[1]
    assert sdf.dim() == 4 and sdf.shape[2] == res and sdf.shape[3] == res
    dev = sdf.device
    centres = centres.detach().to(device=dev, dtype=torch.float32).contiguous()
    if vox_ids is not None:
        vox_ids = vox_ids.to(device=dev, dtype=torch.int32).contiguous()
    counts = torch.empty((4, max(n, 1)), dtype=torch.int32, device=dev)          # nvert, ntri, voff, toff
    totals = torch.zeros(2, dtype=torch.int64, device=dev)
    lib, st = _capi.lib(), _capi.stream_ptr()
    _capi.check(lib.nl_mc_count(n, res, _capi.ptr(sdf), _capi.ptr(counts[0]), _capi.ptr(counts[1]), _capi.ptr(counts[2]), _capi.ptr(counts[3]),
                                _capi.ptr(totals), st), "nl_mc_count")
    nv, nt = (int(x) for x in totals.tolist())
    if max(nv, nt) > INT32_MAX:
        raise ValueError(f"marching cubes: {nv} vertices and {nt} triangles; vertex ids and offsets are int32, so neither may "
                         f"exceed INT32_MAX = {INT32_MAX} (extract fewer voxels per call, or at a lower res)")
    verts = torch.empty((nv, 3), dtype=torch.float32, device=dev)
    faces = torch.empty((nt, 3), dtype=torch.int32, device=dev)
    _capi.check(lib.nl_mc_emit(n, res, float(voxel_size), _capi.ptr(sdf), _capi.ptr(centres), _capi.ptr(vox_ids), _capi.ptr(counts[2]),
                               _capi.ptr(counts[3]), nv, nt, _capi.ptr(verts) if nv else None, _capi.ptr(faces) if nt else None, st), "nl_mc_emit")
    _capi.LAUNCHES += 3
    return verts, faces


def marching_cubes(voxels, sdf, voxel_size):
    """Drop-in for MeshExtractor.marching_cubes(voxels, sdf) (mesh_util.py:145-169): voxels [n,>=3] voxel centres, sdf
    [n,res,res,res,1] -> (verts float32 [V,3], faces int32 [T,3]) as numpy arrays, voxel-major like the reference's loop."""
    dev = torch.device("cuda")
    s = torch.as_tensor(sdf)[..., 0].to(dev)
    c = torch.as_tensor(voxels)[:, :3].detach().to(dev)
    v, f = marching_cubes_device(s, c, voxel_size)
    return v.cpu().numpy(), f.cpu().numpy()


@torch.no_grad()
def extract_mesh(sdf_network, map_states, voxel_size, res=8):
    """create_mesh (mesh_util.py:80-86) without the host round trips: lattice SDF of the SURFACE voxels -> marching cubes,
    everything on the device.  Returns (verts f32[V,3], faces i32[T,3]) CUDA tensors in world coordinates (no -2000 m offset
    applied; the reference adds `offset` when it builds the Open3D mesh, mesh_util.py:139)."""
    from .render_helpers import scores_device
    dev = torch.device("cuda")
    m = map_states if isinstance(map_states, MapState) else MapState.from_map_states(map_states, dev)
    lat, nodes = scores_device(sdf_network, m, voxel_size, res)
    return marching_cubes_device(lat.view(-1, res, res, res), m.centres, voxel_size, vox_ids=nodes)
