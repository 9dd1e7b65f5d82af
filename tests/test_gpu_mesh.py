"""GPU tests of the sparse marching cubes (csrc/mc.cu, nerf-loam_b200/mesh.py; SURVEY.md section 8 f-3) against the numpy / Python
restatement oracle/mc.py and through geometric properties."""
import itertools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nl():
    import nerfloam_b200 as nl
    assert torch.cuda.is_available()
    return nl


def _sphere_block(res=8, nvox=3, vs=0.3, r=0.37, centre=(2000.41, 2000.38, 2000.47)):
    """nvox^3 voxels of side vs around `centre`, each with the res^3 lattice of get_scores sampling the SDF of a sphere."""
    lin = torch.linspace(-0.5, 0.5, res)
    xx, yy, zz = torch.meshgrid(lin, lin, lin, indexing="ij")
    offs = torch.stack([xx, yy, zz], -1).float() * vs                                   # [res,res,res,3]
    idx = torch.tensor(list(itertools.product(range(nvox), repeat=3)), dtype=torch.float32)
    base = torch.tensor(centre) - vs * (nvox - 1) / 2
    centres = (base + idx * vs).float()                                                  # [n,3]
    pts = centres[:, None, None, None, :] + offs[None]
    sdf = (pts.double() - torch.tensor(centre).double()).norm(dim=-1) - r
    return sdf.float(), centres, torch.tensor(centre).double(), r


def _boundary(tris):
    """Directed boundary edges of a set of oriented triangles (interior diagonals of a triangulated polygon cancel): two
    triangulations of the same oriented polygons give the same result."""
    cnt = {}
    for t in tris:
        for i in range(3):
            a, b = t[i], t[(i + 1) % 3]
            if cnt.get((b, a), 0) > 0:
                cnt[(b, a)] -= 1
            else:
                cnt[(a, b)] = cnt.get((a, b), 0) + 1
    return sorted(k for k, v in cnt.items() for _ in range(v))


def test_marching_cubes_vs_python_restatement(nl):
    """Around 2000 m (one fp32 ulp is 1.2e-4 m) and around 0.15 m, where an FMA-contracted vertex formula would differ from the
    separately rounded one in the last bit of a fifth or more of the vertices."""
    import itertools as it
    from oracle import mc as OM
    res = 6
    for centre in ((2000.41, 2000.38, 2000.47), (0.15, 0.11, 0.17)):
        sdf, centres, c, r = _sphere_block(res=res, nvox=2, centre=centre)
        verts, faces = nl.mesh.marching_cubes_device(sdf.cuda(), centres.cuda(), 0.3)
        verts, faces = verts.cpu().numpy(), faces.cpu().numpy()
        vo, to = 0, 0
        for v in range(sdf.shape[0]):
            want_v, _ = OM.marching_cubes_voxel(sdf[v].numpy(), centres[v].numpy(), 0.3)
            nv = len(want_v)
            got_v = verts[vo:vo + nv]
            # vertices bit-exact (same fp32 formula) and in the same order: the kernel's lattice-edge ids, the oracle's edge loop
            want_arr = np.array([np.asarray(p, np.float32) for p in want_v.values()], np.float32).reshape(-1, 3)
            assert np.array_equal(got_v.view(np.uint32), want_arr.view(np.uint32)), \
                (centre, v, int((got_v != want_arr).any(1).sum()), nv)
            pos = {k: tuple(np.asarray(p, np.float32).tolist()) for k, p in want_v.items()}
            neg = sdf[v].numpy() < 0
            # cell by cell (the kernel emits a voxel's triangles in cell order): the same oriented polygons
            for ci, cj, ck in it.product(range(res - 1), repeat=3):
                neg8 = {(x, y, z): bool(neg[ci + x, cj + y, ck + z]) for x, y, z in it.product((0, 1), repeat=3)}
                want = [tuple(pos[(a, ci + x, cj + y, ck + z)] for (a, x, y, z) in t) for t in OM.cell_polygons(neg8)]
                f = faces[to:to + len(want)]
                assert len(want) == 0 or (f.min() >= vo and f.max() < vo + nv)           # a voxel's faces index its own welded vertices
                got = [tuple(tuple(verts[i].tolist()) for i in t) for t in f]
                assert _boundary(got) == _boundary(want), (centre, v, ci, cj, ck)
                to += len(want)
            vo += nv
        assert vo == verts.shape[0] and to == faces.shape[0]


def test_sphere_mesh_properties(nl):
    sdf, centres, c, r = _sphere_block(res=8, nvox=3)
    verts, faces = nl.mesh.marching_cubes_device(sdf.cuda(), centres.cuda(), 0.3)
    assert faces.shape[0] > 500 and int(faces.max()) == verts.shape[0] - 1 and int(faces.min()) == 0
    V = verts.double().cpu()
    h = 0.3 / 7
    assert float(((V - c).norm(dim=-1) - r).abs().max()) < 0.6 * h * h / r + 2e-4      # linear interpolation of a curved SDF: O(h^2 / r)
    T = V[faces.long().cpu()]
    n = torch.cross(T[:, 1] - T[:, 0], T[:, 2] - T[:, 0], dim=-1)
    area = 0.5 * float(n.norm(dim=-1).sum())
    assert abs(area - 4 * np.pi * r * r) < 0.01 * 4 * np.pi * r * r
    # orientation: normals point towards increasing SDF (away from the centre)
    cen = T.mean(1) - c
    assert float(((n * cen).sum(-1) > 0).double().mean()) == 1.0
    # welded inside each voxel, closed across voxels once coincident vertices on shared voxel faces are merged
    # coincident vertices of neighbouring voxels differ in the last fp32 bits (|x| ~ 2000, ulp 1.2e-4 m): merge within 0.5 mm
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    from scipy.spatial import cKDTree
    Vn = V.numpy()
    pairs = cKDTree(Vn).query_pairs(5e-4, output_type="ndarray")
    g = coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(len(Vn), len(Vn)))
    n_uniq, lab = connected_components(g, directed=False)
    inv = torch.from_numpy(lab).long()
    uniq = torch.zeros(n_uniq, 1)
    F = inv[faces.long().cpu()]
    e = torch.cat([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]])
    fwd = {}
    for a, b in e.tolist():
        fwd[(a, b)] = fwd.get((a, b), 0) + 1
    assert all(v == 1 for v in fwd.values()) and all((b, a) in fwd for (a, b) in fwd)  # closed, consistently oriented 2-manifold
    assert uniq.shape[0] - len(fwd) // 2 + F.shape[0] == 2                             # Euler characteristic of a sphere


def test_extract_mesh_and_get_scores_dropin(nl):
    """get_scores on the reference's meshing dict (mapping.py:354-371: SURFACE rows only, no voxel_structure) and the device-side
    extract_mesh on the same map agree; the marching_cubes drop-in reproduces the device result from the CPU lattice."""
    syn = nl.synthetic
    pts, cos, pose = syn.make_scan(n_beams=16, n_az=200, seed=4)
    mu = nl.mapping.MapUpdater(0.3, init_std=0.05, seed=7)
    ms = mu.insert_voxels(torch.from_numpy(syn.voxelize(pts, pose, 0.3)))
    torch.manual_seed(1)
    dec = nl.lidar.Decoder(depth=2, width=256, in_dim=16, skips=[], embedder="none", multires=0).cuda()
    with torch.no_grad():
        dec.sdf_out.bias.zero_()                       # random decoder: centre the values so that the zero level crosses many voxels
    states = mu.map_states
    feats = states["voxel_vertex_idx"]
    keep = ~feats.eq(-1).any(-1)                        # mapping.py:358-361
    enc = {"voxel_vertex_idx": feats[keep], "voxel_center_xyz": states["voxel_center_xyz"][keep], "voxel_vertex_emb": states["voxel_vertex_emb"],
           "voxel_id2embedding_id": states["voxel_id2embedding_id"]}
    grid = nl.render_helpers.get_scores(dec, enc, 0.3, bits=8)
    assert grid.shape == (int(keep.sum()), 8, 8, 8, 1) and not grid.is_cuda
    full = nl.render_helpers.get_scores(dec, states, 0.3, bits=8)          # whole octree: nodes without embeddings hold decoder(0)
    assert full.shape[0] == ms.n_nodes
    np.testing.assert_allclose(full[keep].numpy(), grid.numpy(), atol=1e-6)
    const = full[~keep]
    assert float((const - const.reshape(-1)[0]).abs().max()) == 0.0
    v1, f1 = nl.mesh.extract_mesh(dec, ms, 0.3, res=8)
    v2, f2 = nl.mesh.marching_cubes(enc["voxel_center_xyz"], grid, 0.3)
    assert f1.shape[0] > 100
    assert v1.shape[0] == v2.shape[0] and f1.shape[0] == f2.shape[0]
    np.testing.assert_allclose(v1.cpu().numpy(), v2, atol=2e-4)           # lattice values within 1e-6 of each other move a crossing slightly
    assert np.array_equal(f1.cpu().numpy(), f2)
