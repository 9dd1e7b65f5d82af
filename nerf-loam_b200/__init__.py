"""nerf-loam_b200 -- H100-native (sm_90a) neural-SDF LiDAR SLAM inner loop behind NeRF-LOAM's own API.

The directory name carries the reference's hyphen; import it as `nerfloam_b200` (the alias module at the
repository root) or with importlib.import_module("nerf-loam_b200").

Public surface (mirrors the reference, see INTEGRATION.md):
    svo.Octree                      <- torch.classes.svo.Octree        (third_party/sparse_octree)
    grid.svo_intersect, grid.inverse_cdf_sampling, ...  <- `grid` extension (third_party/sparse_voxels)
    lidar.Decoder                   <- src/variations/lidar.py
    criterion.Criterion             <- src/criterion.py
    se3pose.OptimizablePose         <- src/se3pose.py
    frame.LidarFrame                <- src/lidarFrame.py
    render_helpers.render_rays / bundle_adjust_frames / track_frame / get_scores  <- src/variations/render_helpers.py
    mapping.MapUpdater              <- Mapping.create_voxels / update_grid_features / get_embeddings (src/mapping.py)
    mesh.extract_mesh / marching_cubes  <- MeshExtractor.create_mesh / marching_cubes (src/utils/mesh_util.py)
Every device computation goes through the C ABI of libnerfloam_b200.so (include/nerfloam_b200.h); there is
no CPU or eager-PyTorch fallback for the kernels.
"""
from . import _capi  # noqa: F401

__all__ = ["svo", "grid", "lidar", "criterion", "se3pose", "frame", "render_helpers", "mapping", "engine", "synthetic", "dist", "dropin", "mesh", "share"]


def __getattr__(name):
    if name in __all__:
        import importlib
        return importlib.import_module("." + name, __name__)
    raise AttributeError(name)
