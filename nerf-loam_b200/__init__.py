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
    track_frames (= render_helpers.track_frames, track_batch)  K independent track_frame problems in one launch chain
    refine_map (= render_helpers.refine_map)  the mapper's key-scan refinement (mapper_specs.final_iter, src/mapping.py:154-164)
    score_poses / relocalise (= render_helpers.*, score)  the loss of up to 65 535 pose hypotheses of one scan; recovering a lost scan
    relocalise_global (globalloc)   a scan placed anywhere within a radius of anchor poses with no guess: millions of placements
                                    scored by occupied-voxel counts on the GPU, the best refined with score_poses and relocalise
    mapping.MapUpdater              <- Mapping.create_voxels / update_grid_features / get_embeddings (src/mapping.py)
    mesh.extract_mesh / marching_cubes  <- MeshExtractor.create_mesh / marching_cubes (src/utils/mesh_util.py)
    evaluate.eval_mesh / sample_surface / voxel_down_sample / nearest_distances  <- the map evaluation of Readme.md ("Evaluation"):
                                    accuracy, completeness, Chamfer distance and F-score of a mesh against a reference cloud, on the GPU
    keyframes.KeyframeGraph / keyframe_overlap / rank_by_overlap  <- Mapping.insert_keyframe / select_optimize_targets (src/mapping.py),
                                    with the 'overlap' window the reference leaves unimplemented (voxel IoU with the scan, on the GPU)
    ground.points_and_cos / segment_ground  <- the Patchwork++ ground segmentation and pointsCos of src/dataset/kitti.py:40-70, on the GPU
    dataset.kitti / dataset.maicity .DataLoader  <- src/dataset/kitti.py, maicity.py (seam: sys.modules["dataset"] = nerfloam_b200.dataset)
    slam.NeRFLOAM / Tracking / Mapping  <- src/nerfloam.py, tracking.py, mapping.py: a whole sequence, tracker and mapper concurrent on
                                    two CUDA streams in a fixed lag-one schedule, writing the trajectory and the meshes;
                                    NeRFLOAM.save_map / slam.load_map: the finished run's map, decoder and trajectory as one file
    localise.Localiser              a sequence localised in a saved map: the first scan placed by relocalise_global with no guess,
                                    the rest tracked by slam.Tracking against the frozen map
    changes.ChangeDetector          what changed since a map was saved: the saved voxels a later drive sees through and the new
                                    ground it hits, counted on the GPU (Localiser's "change_specs")
Every device computation goes through the C ABI of libnerfloam_b200.so (include/nerfloam_b200.h); there is
no CPU or eager-PyTorch fallback for the kernels.
"""
from . import _capi  # noqa: F401

__all__ = ["svo", "grid", "lidar", "criterion", "se3pose", "frame", "render_helpers", "mapping", "engine", "synthetic", "dist", "dropin", "mesh", "share",
           "evaluate", "keyframes", "ground", "dataset", "track_batch", "track_frames", "score", "score_poses", "relocalise", "refine_map", "slam",
           "globalloc", "relocalise_global", "localise", "changes"]


def __getattr__(name):
    import importlib
    if name == "track_frames":
        return importlib.import_module(".track_batch", __name__).track_frames
    if name == "refine_map":
        return importlib.import_module(".render_helpers", __name__).refine_map
    if name in ("score_poses", "relocalise"):
        return getattr(importlib.import_module(".score", __name__), name)
    if name == "relocalise_global":
        return importlib.import_module(".globalloc", __name__).relocalise_global
    if name in __all__:
        return importlib.import_module("." + name, __name__)
    raise AttributeError(name)
