"""ctypes binding of libnerfloam_b200.so (C ABI declared in include/nerfloam_b200.h).

This is the only place the shared library is loaded.  There is no CPU fallback: if the library is
missing it is built with nvcc (nerf-loam_b200/build.py); if that fails, importing raises.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libnerfloam_b200.so")

c_f32p = C.c_void_p
c_i32p = C.c_void_p
vp = C.c_void_p


class RenderStats(C.Structure):
    """nl_render_stats (include/nerfloam_b200.h)."""
    _fields_ = [
        ("n_hit_rays", C.c_int32), ("max_hits", C.c_int32), ("max_samples", C.c_int32), ("n_samples", C.c_int32),
        ("error", C.c_int32), ("max_steps_ceil", C.c_int32), ("_pad", C.c_int32 * 2),
        ("cnt_fs_valid", C.c_int64), ("cnt_sdf_valid", C.c_int64), ("pad_fs_rays", C.c_int64), ("pad_fs_nsamp", C.c_int64),
        ("pad_sdf_rays", C.c_int64), ("pad_sdf_nsamp", C.c_int64), ("pad_sdf_d2", C.c_double), ("pad_sdf_d2_nsamp", C.c_double),
        ("n_fs", C.c_float), ("n_sdf", C.c_float), ("w_fs", C.c_float), ("w_sdf", C.c_float), ("g_fs", C.c_float),
        ("g_sdf", C.c_float), ("pad_fs_sum", C.c_float), ("pad_sdf_sum", C.c_float), ("fs_sum", C.c_double),
        ("sdf_sum", C.c_double), ("loss", C.c_float), ("fs_loss", C.c_float), ("sdf_loss", C.c_float), ("_padf", C.c_float),
    ]


class RenderArgs(C.Structure):
    """nl_render_args."""
    _fields_ = [
        ("n_rays", C.c_int32), ("n_nodes", C.c_int32), ("sample_capacity", C.c_int32), ("reference_compat", C.c_int32),
        ("voxel_size", C.c_float), ("step_size", C.c_float), ("max_distance", C.c_float), ("truncation", C.c_float),
        ("max_depth", C.c_float), ("fs_weight", C.c_float), ("sdf_weight", C.c_float),
        ("d_centres", vp), ("d_structure", vp), ("d_ray_o", vp), ("d_ray_d", vp), ("d_gt_depth", vp), ("d_cos", vp),
        ("d_noise", vp), ("noise_stride", C.c_int32), ("rng_seed", C.c_uint32), ("d_workspace", vp),
        ("workspace_bytes", C.c_int64), ("d_stats", vp), ("d_hit_rank", vp), ("d_s_ray", vp), ("d_s_vox", vp),
        ("d_s_depth", vp), ("d_s_xyz", vp), ("d_s_flag", vp), ("d_ray_nsamp", vp), ("d_ray_offset", vp),
        ("d_packed_children", vp), ("d_rng_seed", vp),
    ]


class BatchArgs(C.Structure):
    """nl_batch_args (K independent problems in one ray batch, nl_render_samples_batch)."""
    _fields_ = [("n_problems", C.c_int32), ("noise_rows", C.c_int32), ("d_problem_stats", vp), ("d_problem_seeds", vp),
                ("d_problem_base", vp)]


class GroundParams(C.Structure):
    """nl_ground_params (include/nerfloam_b200.h section 13)."""
    _fields_ = [("sensor_height", C.c_double), ("min_range", C.c_double), ("max_range", C.c_double),
                ("num_rings_each_zone", C.c_int32 * 4), ("num_sectors_each_zone", C.c_int32 * 4), ("uprightness_thr", C.c_double),
                ("elevation_thr", C.c_double * 4), ("flatness_thr", C.c_double * 4), ("num_iter", C.c_int32), ("num_lpr", C.c_int32),
                ("num_min_pts", C.c_int32), ("_pad", C.c_int32), ("th_seeds", C.c_double), ("th_dist", C.c_double),
                ("adaptive_seed_margin", C.c_double), ("vertical_cell", C.c_double), ("vertical_height", C.c_double)]


GROUND_PATCH_BYTES = 88      # sizeof(nl_ground_patch): mean[3], normal[3], d, lambda_min (f64), n_points, n_ground, ground, ring, n_vertical, pad (i32)


class MlpWeights(C.Structure):
    _fields_ = [("width", C.c_int32), ("W0", vp), ("b0", vp), ("W1", vp), ("b1", vp), ("W2", vp), ("b2", vp),
                ("W0t", vp), ("W1t", vp)]


class MlpGrads(C.Structure):
    _fields_ = [("gW0", vp), ("gb0", vp), ("gW1", vp), ("gb1", vp), ("gW2", vp), ("gb2", vp)]


_SIGNATURES = {
    "nl_last_error": (C.c_char_p, []),
    "nl_version": (C.c_int, []),
    "nl_abi_sizes": (None, [C.POINTER(C.c_int32 * 4)]),
    "nl_octree_create": (vp, [C.c_int64, C.c_int64, C.c_double]),
    "nl_octree_destroy": (None, [vp]),
    "nl_octree_insert": (C.c_int, [vp, vp, C.c_int64]),
    "nl_octree_try_insert": (C.c_double, [vp, vp, C.c_int64]),
    "nl_octree_count_nodes": (C.c_int64, [vp]),
    "nl_octree_count_export_nodes": (C.c_int64, [vp]),
    "nl_octree_count_leaf_nodes": (C.c_int64, [vp]),
    "nl_octree_has_voxel": (C.c_int, [vp, vp]),
    "nl_octree_export": (C.c_int, [vp, vp, vp, vp]),
    "nl_octree_export_map": (C.c_int, [vp, vp, vp, vp]),
    "nl_octree_dirty_count": (C.c_int64, [vp]),
    "nl_octree_export_dirty": (C.c_int, [vp, vp, vp, vp, vp, C.c_int]),
    "nl_assign_embedding_rows_subset": (C.c_int64, [vp, C.c_int64, C.c_int64, vp, C.c_int64, vp]),
    "nl_octree_pack_children_rows": (C.c_int, [C.c_int32, vp, vp, vp, vp, vp]),
    "nl_octree_validate": (C.c_int64, [C.c_int64, C.c_int64, vp, vp, vp, vp, vp, C.c_int64]),
    "nl_octree_nodes": (C.c_int, [vp, vp, vp, vp, vp]),
    "nl_octree_restore": (C.c_int, [vp, vp, vp, vp, vp, C.c_int64]),
    "nl_devoctree_validate": (C.c_int, [C.c_int64, C.c_int64, vp, vp, vp, vp, vp, C.c_int64, vp, C.c_int64, vp, vp]),
    "nl_devoctree_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int64]),
    "nl_devoctree_insert_count": (C.c_int, [C.c_int64, vp, vp, C.c_int64, vp, C.c_int64, vp, vp]),
    "nl_devoctree_insert_commit": (C.c_int, [C.c_int64, C.c_int64, C.c_int64, C.c_int64, vp, vp, vp, vp, vp, vp, C.c_int64, vp, C.c_int64, vp, vp]),
    "nl_devoctree_dirty_ids": (C.c_int, [C.c_int64, C.c_int64, C.c_int64, C.c_int64, vp, vp, vp, C.c_int64, vp, C.c_int64, vp, vp]),
    "nl_devoctree_export": (C.c_int, [C.c_int64, C.c_double, C.c_int64, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]),
    "nl_devoctree_assign_rows": (C.c_int, [C.c_int64, C.c_int64, vp, C.c_int64, vp, vp, vp, vp, C.c_int64, vp, C.c_int64, vp, C.c_int64, vp, vp]),
    "nl_devoctree_find": (C.c_int, [C.c_int64, vp, vp, C.c_int64, vp, vp]),
    "nl_devoctree_query_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int64, C.c_int64]),
    "nl_devoctree_export_nodes": (C.c_int, [C.c_int64, C.c_double, C.c_int64, vp, vp, C.c_int] + [vp] * 10),
    "nl_devoctree_preorder": (C.c_int, [C.c_int64, C.c_int64, vp, vp, vp, C.c_int, vp, vp, vp, C.c_int64, vp]),
    "nl_devoctree_try_insert": (C.c_int, [C.c_int64, vp, vp, C.c_int64, vp, C.c_int64, vp, vp]),
    "nl_octree_get_voxels": (C.c_int64, [vp, vp, C.c_int64]),
    "nl_octree_get_leaf_voxels": (C.c_int64, [vp, vp, C.c_int64]),
    "nl_morton_encode": (C.c_uint64, [C.c_int, C.c_int, C.c_int]),
    "nl_assign_embedding_rows": (C.c_int64, [vp, C.c_int64, vp, C.c_int64]),
    "nl_svo_intersect": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_float, C.c_int] + [vp] * 8),
    "nl_inverse_cdf_sampling": (C.c_int, [C.c_int] * 4 + [C.c_float] + [vp] * 10),
    "nl_render_workspace_bytes": (C.c_int64, [C.c_int32]),
    "nl_render_samples": (C.c_int, [C.POINTER(RenderArgs), vp]),
    "nl_gather_trilinear_fwd": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, C.c_float, vp, vp]),
    "nl_gather_trilinear_bwd": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, C.c_float, vp, C.c_int, vp, vp, vp, vp, vp, vp,
                                          C.c_int, vp, vp]),
    "nl_mlp_prepare": (C.c_int, [C.c_int32, vp, vp, vp, vp, vp]),
    "nl_mlp_forward": (C.c_int, [C.c_int64, vp, vp, C.POINTER(MlpWeights), vp, vp]),
    "nl_mlp_train": (C.c_int, [C.c_int64, vp, vp, C.POINTER(MlpWeights), vp, vp, vp, vp, vp, vp, C.c_float, vp, vp,
                               C.POINTER(MlpGrads), vp, vp, vp, vp]),
    "nl_mlp_tc_panel_bytes": (C.c_int64, []),
    "nl_mlp_tc_prepare": (C.c_int, [vp, vp, vp, vp, vp]),
    "nl_mlp_tc_forward": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "nl_mlp_tc_act_floats": (C.c_int64, [C.c_int64]),
    "nl_mlp_tc_dh1_floats": (C.c_int64, [C.c_int64]),
    "nl_mlp_tc_train": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_float, vp, vp, C.POINTER(MlpGrads),
                                  vp, vp, vp, vp, vp]),
    "nl_octree_packed_bytes": (C.c_int64, [C.c_int32]),
    "nl_octree_pack_children": (C.c_int, [C.c_int32, vp, vp, vp, vp]),
    "nl_loss_prepare": (C.c_int, [vp, C.c_float, C.c_float, vp]),
    "nl_loss_finalize": (C.c_int, [vp, C.c_float, C.c_float, vp]),
    "nl_pose_matrices": (C.c_int, [C.c_int, vp, vp, vp]),
    "nl_rays_from_poses": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp]),
    "nl_pose_grad": (C.c_int, [C.c_int, vp, vp, vp, vp]),
    "nl_rays_from_pose6": (C.c_int, [C.c_int64, C.c_int, vp, vp, vp, vp, vp, vp, vp]),
    "nl_pose_step": (C.c_int, [C.c_int, vp, vp, vp, C.c_uint32, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double, vp, vp, C.c_float, C.c_float,
                               vp, C.c_int32, vp, C.c_int32, vp]),
    "nl_select_rays": (C.c_int, [C.c_int, C.c_int, C.c_int, vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, vp]),
    "nl_adam_f32": (C.c_int, [C.c_int64, vp, vp, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, vp]),
    "nl_adam_bf16": (C.c_int, [C.c_int64, vp, vp, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, vp]),
    "nl_iter_status": (C.c_int, [vp, vp, vp, vp]),
    "nl_adam_f32_ctl": (C.c_int, [C.c_int64, vp, vp, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double, vp, vp]),
    "nl_adam_bf16_ctl": (C.c_int, [C.c_int64, vp, vp, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double, vp, vp]),
    "nl_stats_pack": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, vp]),
    "nl_stats_unpack": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_float, C.c_float, vp]),
    "nl_stats_unpack_peers": (C.c_int, [vp, vp, C.c_int, C.c_float, C.c_float, vp]),
    "nl_peer_reduce_adam_bf16": (C.c_int, [C.c_int64, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double, vp,
                                          C.c_int64, vp, vp, vp, vp]),
    "nl_mc_count": (C.c_int, [C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp, vp]),
    "nl_mc_emit": (C.c_int, [C.c_int32, C.c_int32, C.c_float, vp, vp, vp, vp, vp, C.c_int64, C.c_int64, vp, vp, vp]),
    "nl_mc_case_table": (C.c_int, [vp, vp, vp]),
    # batched tracking (include/nerfloam_b200.h section 3b)
    "nl_abi_sizes_batch": (None, [C.POINTER(C.c_int32 * 2)]),
    "nl_render_samples_batch": (C.c_int, [C.POINTER(RenderArgs), C.POINTER(BatchArgs), vp]),
    "nl_mlp_train_batch": (C.c_int, [C.c_int64, vp, vp, C.POINTER(MlpWeights), vp, vp, vp, vp, vp, vp, C.c_int32, C.c_float, vp, vp, vp]),
    "nl_mlp_tc_train_batch": (C.c_int, [C.c_int64] + [vp] * 13 + [C.c_int32, C.c_float, vp, vp, vp]),
    "nl_iter_status_batch": (C.c_int, [C.c_int, vp, vp, vp, vp]),
    "nl_pose_step_batch": (C.c_int, [C.c_int, vp, vp, vp, vp, vp, vp, C.c_double, C.c_double, C.c_double, vp, vp, C.c_float, C.c_float, vp,
                                     vp, C.c_int32, vp, C.c_int32, vp]),
    "nl_select_rays_batch": (C.c_int, [C.c_int, C.c_int, C.c_int] + [vp] * 10),
    # scoring pose hypotheses (include/nerfloam_b200.h section 3b)
    "nl_abi_sizes_score": (None, [C.POINTER(C.c_int32 * 1)]),
    "nl_mlp_tc_score_batch": (C.c_int, [C.c_int64] + [vp] * 13 + [C.c_int32, C.c_float, vp, vp]),
    "nl_loss_finalize_batch": (C.c_int, [C.c_int, vp, C.c_float, C.c_float, vp, vp]),
    # reconstruction evaluation (include/nerfloam_b200.h section 11)
    "nl_abi_sizes_eval": (None, [C.POINTER(C.c_int32 * 2)]),
    "nl_eval_bounds": (C.c_int, [C.c_int64, vp, vp, vp, vp]),
    "nl_eval_surface_workspace_bytes": (C.c_int64, [C.c_int64]),
    "nl_eval_surface_prepare": (C.c_int, [C.c_int64, vp, C.c_int64, vp, vp, C.c_int64, vp, vp]),
    "nl_eval_sample_surface": (C.c_int, [C.c_int64, vp, C.c_int64, vp, C.c_int64, C.c_uint64, vp, C.c_int64, vp, vp, vp]),
    "nl_eval_voxel_workspace_bytes": (C.c_int64, [C.c_int64]),
    "nl_eval_voxel_down_sample": (C.c_int, [C.c_int64, vp, C.c_double, C.c_double, C.c_double, C.c_double, vp, vp, C.c_int64, vp, vp, vp, vp]),
    "nl_eval_nn_workspace_bytes": (C.c_int64, [C.c_int64]),
    "nl_eval_nearest": (C.c_int, [C.c_int64, vp, C.c_int64, vp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int32, C.c_float, vp,
                                  C.c_int64, vp, vp, vp]),
    "nl_eval_sums_workspace_bytes": (C.c_int64, [C.c_int64]),
    "nl_eval_distance_sums": (C.c_int, [C.c_int64, vp, C.c_float, vp, C.c_int64, vp, vp]),
    # keyframe overlap (include/nerfloam_b200.h section 12)
    "nl_keyframe_overlap_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int64]),
    "nl_keyframe_overlap": (C.c_int, [C.c_int64, vp, C.c_int32, vp, vp, vp, vp, C.c_double, C.c_int64, C.c_int64, vp, C.c_int64, vp, vp]),
    # ground segmentation (include/nerfloam_b200.h section 13)
    "nl_abi_sizes_ground": (None, [C.POINTER(C.c_int32 * 3)]),
    "nl_ground_workspace_bytes": (C.c_int64, [C.c_int64]),
    "nl_ground_segment": (C.c_int, [C.c_int64, vp, C.c_int32, C.POINTER(GroundParams), vp, C.c_int64, vp, vp, vp, vp, vp, vp]),
    "nl_ground_vertical_workspace_bytes": (C.c_int64, [C.c_int64]),
    "nl_ground_segment_vertical": (C.c_int, [C.c_int64, vp, C.c_int32, C.POINTER(GroundParams), vp, C.c_int64, vp, C.c_int64, vp, vp, vp, vp,
                                             vp, vp, vp]),
    "nl_ground_partition": (C.c_int, [C.c_int64, vp, C.c_int32, vp, vp, vp, C.c_int64, vp, vp, vp, vp]),
    # key-scan map refinement (include/nerfloam_b200.h section 14)
    "nl_refine_pass_begin": (C.c_int, [C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int] + [vp] * 15 + [C.c_int64] + [vp] * 5),
    "nl_mark_rows": (C.c_int, [C.c_int64, vp, vp, vp, C.c_int64, vp, vp, vp, vp]),
    "nl_mark_rows_floor": (C.c_int, [C.c_int64, vp, vp, vp, C.c_int64, C.c_int64, vp, vp, vp, vp]),
    "nl_adam_bf16_rows_ctl": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double, vp, vp]),
    "nl_refine_iter_end": (C.c_int, [C.c_int, vp, vp, C.c_int32, vp, C.c_int32, vp]),
    # global localisation, coarse stage (include/nerfloam_b200.h section 15)
    "nl_abi_sizes_globalloc": (None, [C.POINTER(C.c_int32 * 2)]),
    "nl_globalloc_count_leaves": (C.c_int, [C.c_int64, vp, vp, vp]),
    "nl_globalloc_occupied_slots": (C.c_int64, [C.c_int64]),
    "nl_globalloc_occupied": (C.c_int, [C.c_int64, vp, vp, C.c_double, C.c_int64, C.c_int64, vp, vp]),
    "nl_globalloc_cells_workspace_bytes": (C.c_int64, [C.c_int32, vp, C.c_double, C.c_double]),
    "nl_globalloc_cells": (C.c_int, [C.c_int32, vp, vp, C.c_double, C.c_double, vp, C.c_int64, vp, vp]),
    "nl_globalloc_cells_finish": (C.c_int, [C.c_int32, vp, C.c_double, C.c_double, C.c_int64, vp, C.c_int64, vp, vp]),
    "nl_globalloc_matrices": (C.c_int, [C.c_int64, vp, C.c_int64, vp, vp, C.c_int32, C.c_double, vp, vp]),
    "nl_globalloc_score": (C.c_int, [C.c_int64, C.c_int64, C.c_int64, vp, vp, C.c_int32, C.c_double, C.c_int32, vp, vp, C.c_int64, C.c_double,
                                     C.c_int64, vp, vp]),
    "nl_globalloc_select_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int32, C.c_int64]),
    "nl_globalloc_select": (C.c_int, [C.c_int64, vp, C.c_int32, C.c_int64, vp, C.c_int64, vp, vp, vp]),
    "nl_change_votes": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, vp, C.c_int64, C.c_float, C.c_float, vp, vp, vp]),
    "nl_change_rehash": (C.c_int, [C.c_int64, vp, vp, C.c_int64, vp, vp, vp, vp]),
    "nl_change_added": (C.c_int, [C.c_int64, vp, vp, C.c_double, C.c_int64, vp, C.c_int64, C.c_int64, vp, vp, C.c_uint32, vp, vp]),
    "nl_change_finish_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int64]),
    "nl_change_finish": (C.c_int, [C.c_int64, vp, vp, C.c_uint32, C.c_double, C.c_int64, vp, vp, C.c_uint32, C.c_uint32, vp, C.c_int64, vp, vp, vp,
                                   vp, vp]),
}

# words of the device-side iteration control block (include/nerfloam_b200.h section 8)
CTL_ERROR, CTL_SKIPPED, CTL_SKIP_NOW, CTL_ADAM_STEP, CTL_MIN_HIT, CTL_ITERS, CTL_MAX_SAMPLES, CTL_WORDS = 0, 1, 2, 3, 4, 5, 6, 8
CTL_STOPPED = 7              # batched control blocks only (nl_iter_status_batch)
BATCH_MAX_PROBLEMS = 31      # NL_BATCH_MAX_PROBLEMS
SCORE_MAX_PROBLEMS = 65535   # NL_SCORE_MAX_PROBLEMS
EVAL_KEY_BITS = 21           # NL_EVAL_KEY_BITS
EVAL_TILE = 2048             # NL_EVAL_TILE
GROUND_MAX_PATCHES = 1024    # NL_GROUND_MAX_PATCHES
GLOBALLOC_MAX_POINTS = 8192  # NL_GLOBALLOC_MAX_POINTS
# words of the refinement state block (include/nerfloam_b200.h section 14)
REFINE_ITER, REFINE_LISTED, REFINE_PREV, REFINE_STATE_WORDS = 0, 1, 2, 4
STATS_PACK_FIXED = 10
# node-array checks, bit i = 1 << i (NL_TREE_* in include/nerfloam_b200.h section 1)
TREE_CHECKS = ("ROOT", "RANGE", "LINK", "PARENTS", "SHAPE", "ROWS", "VERTICES")


def tree_checks_failed(bits):
    """The names of the NL_TREE_* checks whose bits are set."""
    return [name for i, name in enumerate(TREE_CHECKS) if bits >> i & 1]

EXPORTED_SYMBOLS = tuple(sorted(_SIGNATURES))

_lib = None
LAUNCHES = 0  # number of C-ABI device entry points invoked (each launches >= 1 kernel); see launch_count()


class NerfLoamError(RuntimeError):
    pass


def lib():
    """Load (building first if necessary) the shared library and declare every prototype."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            from . import build as _b
            _b.build()
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        sizes = (C.c_int32 * 4)()
        L.nl_abi_sizes(C.byref(sizes))
        mine = [C.sizeof(RenderStats), RenderStats.n_samples.offset, C.sizeof(RenderArgs), C.sizeof(MlpWeights)]
        if list(sizes) != mine:
            raise ImportError(f"ABI mismatch between _capi.py and libnerfloam_b200.so: {list(sizes)} vs {mine}")
        bsizes = (C.c_int32 * 2)()
        L.nl_abi_sizes_batch(C.byref(bsizes))
        bmine = [C.sizeof(BatchArgs), BATCH_MAX_PROBLEMS]
        if list(bsizes) != bmine:
            raise ImportError(f"ABI mismatch between _capi.py and libnerfloam_b200.so (batch): {list(bsizes)} vs {bmine}")
        ssizes = (C.c_int32 * 1)()
        L.nl_abi_sizes_score(C.byref(ssizes))
        if list(ssizes) != [SCORE_MAX_PROBLEMS]:
            raise ImportError(f"ABI mismatch between _capi.py and libnerfloam_b200.so (score): {list(ssizes)} vs {[SCORE_MAX_PROBLEMS]}")
        esizes = (C.c_int32 * 2)()
        L.nl_abi_sizes_eval(C.byref(esizes))
        if list(esizes) != [EVAL_KEY_BITS, EVAL_TILE]:
            raise ImportError(f"ABI mismatch between _capi.py and libnerfloam_b200.so (eval): {list(esizes)} vs {[EVAL_KEY_BITS, EVAL_TILE]}")
        gsizes = (C.c_int32 * 3)()
        L.nl_abi_sizes_ground(C.byref(gsizes))
        gmine = [C.sizeof(GroundParams), GROUND_MAX_PATCHES, GROUND_PATCH_BYTES]
        if list(gsizes) != gmine:
            raise ImportError(f"ABI mismatch between _capi.py and libnerfloam_b200.so (ground): {list(gsizes)} vs {gmine}")
        lsizes = (C.c_int32 * 2)()
        L.nl_abi_sizes_globalloc(C.byref(lsizes))
        if list(lsizes) != [GLOBALLOC_MAX_POINTS, 3]:
            raise ImportError(f"ABI mismatch between _capi.py and libnerfloam_b200.so (globalloc): {list(lsizes)} vs {[GLOBALLOC_MAX_POINTS, 3]}")
        _lib = L
    return _lib


def check(rc, what=""):
    if rc != 0:
        raise NerfLoamError(f"{what} failed ({rc}): {lib().nl_last_error().decode()}")


def ptr(t):
    """Device/host pointer of a torch tensor (None -> NULL).  The tensor must be contiguous."""
    if t is None:
        return None
    assert t.is_contiguous(), "tensor passed to the C ABI must be contiguous"
    return C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
