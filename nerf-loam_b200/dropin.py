"""Install the native kernels behind the reference's own module names, so that the reference's driver
(demo/run.py -> src/nerfloam.py -> src/mapping.py / src/tracking.py) runs on them unmodified apart from
the one line the reference's README already tells users to edit (mapping.py:19-20, the absolute path of
the svo library).  See INTEGRATION.md.

    import nerfloam_b200.dropin as dropin
    dropin.install(reference_src="/path/to/NeRF-LOAM/src")   # before `import mapping` / `import tracking`
"""
import importlib
import sys


def install(reference_src=None):
    pkg = importlib.import_module(__name__.rsplit(".", 1)[0])
    grid = importlib.import_module(pkg.__name__ + ".grid")
    rh = importlib.import_module(pkg.__name__ + ".render_helpers")
    lidar = importlib.import_module(pkg.__name__ + ".lidar")
    sys.modules["grid"] = grid                                   # `import grid as _ext` (voxel_helpers.py:22)
    if reference_src and reference_src not in sys.path:
        sys.path.insert(0, reference_src)
    try:
        ref_rh = importlib.import_module("variations.render_helpers")
        for name in ("render_rays", "bundle_adjust_frames", "track_frame", "get_scores"):
            setattr(ref_rh, name, getattr(rh, name))
        ref_lidar = importlib.import_module("variations.lidar")
        ref_lidar.Decoder = lidar.Decoder                        # get_decoder: variations.<name>.Decoder (import_util.py:8-10)
    except ModuleNotFoundError:
        pass                                                      # reference sources not on the path: only `grid` is installed
    # the two seams outside the per-iteration path; their reference modules import open3d / skimage / the data loaders, so they are
    # rebound only where those imports succeed (a real NeRF-LOAM environment)
    try:
        mesh_util = importlib.import_module("utils.mesh_util")
        mesh = importlib.import_module(pkg.__name__ + ".mesh")
        mesh_util.get_scores = rh.get_scores                      # mesh_util.py:8 imported the name at module level
        mesh_util.MeshExtractor.marching_cubes = lambda self, voxels, sdf: mesh.marching_cubes(voxels, sdf, self.voxel_size)   # mesh_util.py:145
    except Exception:
        pass
    try:
        ref_share = importlib.import_module("share")
        share = importlib.import_module(pkg.__name__ + ".share")
        ref_share.ShareData, ref_share.ShareDataProxy = share.ShareData, share.ShareDataProxy    # nerfloam.py registers these with its BaseManager
    except Exception:
        pass
    return pkg
