/*
 * nerfloam_b200.h -- C ABI of libnerfloam_b200.so: the H100-native (sm_90a) replacement for the
 * per-iteration neural-SDF hot path of NeRF-LOAM (SURVEY.md section 8).
 *
 * Conventions
 *   - plain C: raw pointers, explicit sizes, no torch / C++ types.  `stream` is a cudaStream_t
 *     passed as void* (NULL = legacy default stream).  Every device entry point is asynchronous and
 *     stream-ordered, allocates nothing, never synchronises and NEVER calls exit() (the reference
 *     does: third_party/sparse_voxels/include/cuda_utils.h:37-48).
 *   - all pointers named d_* are device pointers; h_* are host pointers.
 *   - return value: 0 = ok, <0 = error (nl_last_error() returns a thread-local message).
 *   - all reference citations are relative to /root/reference.
 */
#ifndef NERFLOAM_B200_H
#define NERFLOAM_B200_H

#include <stdint.h>

#if defined(__GNUC__)
#define NL_API __attribute__((visibility("default")))
#else
#define NL_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define NL_OK 0
#define NL_ERR_INVALID (-1)
#define NL_ERR_CUDA (-2)
#define NL_ERR_UNSUPPORTED (-3)

#define NL_MAX_HITS 20     /* voxel_helpers.py:533 hard-codes n_max = 20 */
#define NL_EMB_DIM 16      /* configs/*: decoder_specs.in_dim = 16 */
#define NL_SAMPLE_G 200    /* voxel_helpers.py:274: sampler batches */
#define NL_SAMPLE_CHUNK 800 /* voxel_helpers.py:304: 4*G rays per launch and batch */
#define NL_MAX_DEPTH_FILL 80.0f /* voxel_helpers.py:24 MAX_DEPTH */

NL_API const char *nl_last_error(void);
NL_API int nl_version(void);
/* sizeof(nl_render_stats), offsetof(nl_render_stats, n_samples), sizeof(nl_render_args), sizeof(nl_mlp_weights):
 * lets a foreign-language binding verify its struct layout at load time */
NL_API void nl_abi_sizes(int32_t out[4]);

/* ============================================================================================
 * 1. Host octree -- replaces torch.classes.svo.Octree
 *    (third_party/sparse_octree/src/bindings.cpp:11-31, src/octree.cpp, include/octree.h).
 *    Flat-array octree; node ids are creation-order ids, bit-identical to the reference's
 *    Octant::index_ (octree.h:19).  One handle = one independent tree (the reference's node counter
 *    is a process global, octree.h:62; here it is per tree).
 * ============================================================================================ */
typedef struct nl_octree nl_octree;

NL_API nl_octree *nl_octree_create(int64_t grid_dim, int64_t feat_dim, double voxel_size); /* Octree::init   octree.cpp:34-49   */
NL_API void nl_octree_destroy(nl_octree *t);
NL_API int nl_octree_insert(nl_octree *t, const int32_t *h_vox, int64_t n);               /* Octree::insert octree.cpp:51-111  */
NL_API double nl_octree_try_insert(nl_octree *t, const int32_t *h_vox, int64_t n);        /* try_insert     octree.cpp:113-149 */
NL_API int64_t nl_octree_count_nodes(const nl_octree *t);                                  /* count_nodes    octree.cpp:344-364 */
NL_API int64_t nl_octree_count_export_nodes(const nl_octree *t);                           /* rows of get_centres_and_children (octree.cpp:295-297) */
NL_API int64_t nl_octree_count_leaf_nodes(const nl_octree *t);                             /* count_leaf_nodes octree.cpp:366-389 */
NL_API int nl_octree_has_voxel(const nl_octree *t, const int32_t h_xyz[3]);                /* has_voxel      octree.cpp:173-206 */
/* get_centres_and_children (octree.cpp:293-342): voxels f32[n,4], children f32[n,8], features i32[n,8],
 * n = nl_octree_count_export_nodes(). */
NL_API int nl_octree_export(const nl_octree *t, float *h_voxels, float *h_children, int32_t *h_features);
/* The same export already in the layout the hot path consumes (src/mapping.py:320-326):
 * centres f32[n,3] = (xyz + side/2) * voxel_size, structure i32[n,9] = 8 child ids + side, vertex i32[n,8]. */
NL_API int nl_octree_export_map(const nl_octree *t, float *h_centres, int32_t *h_structure, int32_t *h_vertex);
/* Incremental export (SURVEY.md 8 f-1; the reference re-exports the whole tree every frame, octree.cpp:293-342 is O(total nodes)):
 * only the rows that changed since the last call with clear != 0 -- new nodes, nodes that got a child, leaves that became
 * SURFACE and their parents.  ids i32[m] ascending (m = nl_octree_dirty_count), the three arrays hold row ids[o] at row o, in the
 * hot-path layout of nl_octree_export_map.  Rows never move (row = node id), so scattering them into the previous export
 * reproduces a full export bit for bit. */
NL_API int64_t nl_octree_dirty_count(const nl_octree *t);
NL_API int nl_octree_export_dirty(nl_octree *t, int32_t *h_ids, float *h_centres, int32_t *h_structure, int32_t *h_vertex, int clear);
NL_API int64_t nl_octree_get_voxels(const nl_octree *t, float *h_out, int64_t cap_rows);       /* get_voxels      octree.cpp:228-252 : [n,4] preorder */
NL_API int64_t nl_octree_get_leaf_voxels(const nl_octree *t, float *h_out, int64_t cap_rows);  /* get_leaf_voxels octree.cpp:212-226 : [n,3] */
NL_API uint64_t nl_morton_encode(int x, int y, int z);                                         /* svo.encode      utils.h:106-109    */

/* Vertex -> embedding-row table (src/mapping.py:294-317 Mapping.get_embeddings, de-duplicated: one row
 * per distinct vertex id, numbered by first appearance in vertex.reshape(-1)).  vertex2row i32[n_nodes]
 * (-1 = no row yet) is updated in place; returns the new number of rows (>= n_rows_before). */
NL_API int64_t nl_assign_embedding_rows(const int32_t *h_vertex, int64_t n_nodes, int32_t *h_vertex2row, int64_t n_rows_before);
/* The same over a subset of vertex rows (the dirty rows of nl_octree_export_dirty, ascending node id -- which is the order in
 * which a full pass meets the not-yet-numbered vertices, so the numbering is identical); also writes the composed
 * voxel -> embedding-row table for those rows, vox2row_rows i32[n_rows_in, 8]. */
NL_API int64_t nl_assign_embedding_rows_subset(const int32_t *h_vertex_rows, int64_t n_rows_in, int64_t n_nodes, int32_t *h_vertex2row,
                                        int64_t n_rows_before, int32_t *h_vox2row_rows);

/* ============================================================================================
 * 2. Drop-ins for the two live `grid` kernels (third_party/sparse_voxels/src/binding.cpp:12-20)
 * ============================================================================================ */
/* grid.svo_intersect (intersect.cpp:83-112, intersect_gpu.cu:193-272).  ray_start/ray_dir f32[b,m,3],
 * points f32[b,n,3], children i32[b,n,9]; outputs [b,m,n_max] (idx -1 / depths 0 where empty). */
NL_API int nl_svo_intersect(int b, int n, int m, float voxelsize, int n_max, const float *d_ray_start, const float *d_ray_dir,
                     const float *d_points, const int32_t *d_children, int32_t *d_idx, float *d_min_depth,
                     float *d_max_depth, void *stream);
/* grid.inverse_cdf_sampling (sample.cpp:56-95, sample_gpu.cu:133-239), including both index quirks. */
NL_API int nl_inverse_cdf_sampling(int b, int num_rays, int max_hits, int max_steps, float fixed_step_size,
                            const int32_t *d_pts_idx, const float *d_min_depth, const float *d_max_depth,
                            const float *d_noise, const float *d_probs, const float *d_steps, int32_t *d_sampled_idx,
                            float *d_sampled_depth, float *d_sampled_dists, void *stream);

/* ============================================================================================
 * 3. Fused renderer: rays -> compact sample list (no host sync, no padded [R,S] tensors)
 *    replaces ray_intersect + ray_sample (voxel_helpers.py:530-598) and the mask/gather glue of
 *    render_rays (render_helpers.py:207-257).
 * ============================================================================================ */
typedef struct {
    int32_t n_hit_rays;    /* R_hit  = hits.sum()                        render_helpers.py:216   */
    int32_t max_hits;      /* P      = max valid hits per ray            voxel_helpers.py:555    */
    int32_t max_samples;   /* S_max  = max valid samples per ray         voxel_helpers.py:332    */
    int32_t n_samples;     /* M      = sample_mask.sum()                 render_helpers.py:242   */
    int32_t error;         /* bit0: sum(dists) > 10*MAX_DEPTH (ray_sample returns None, voxel_helpers.py:579)
                              bit1: sample capacity exceeded, bit2: DFS stack overflow                  */
    int32_t max_steps_ceil;/* ceil(steps).max(); the reference's noise width is this + P (voxel_helpers.py:294) */
    int32_t _pad[2];
    /* raw loss-mask counters over the padded [R_hit, S_max] matrix (criterion.py:67-88); additive across
     * ray shards (multi-GPU: all-reduce SUM these, MAX max_samples, then call nl_loss_prepare) */
    int64_t cnt_fs_valid, cnt_sdf_valid;     /* front_mask / sdf_mask set among valid samples            */
    int64_t pad_fs_rays, pad_fs_nsamp;       /* rays whose padded cells (z = 80*cos) are front; their sum of nsamp */
    int64_t pad_sdf_rays, pad_sdf_nsamp;     /* same for sdf_mask                                         */
    double pad_sdf_d2, pad_sdf_d2_nsamp;     /* sum depth^2 (and depth^2*nsamp) over those rays           */
    /* derived by nl_loss_prepare */
    float n_fs, n_sdf;     /* count_nonzero(front_mask), count_nonzero(sdf_mask) */
    float w_fs, w_sdf;     /* 1 - n_fs/(n_fs+n_sdf), 1 - n_sdf/(n_fs+n_sdf)      */
    float g_fs, g_sdf;     /* weight * w / (R_hit*S_max): d loss / d(sum of squared errors) */
    float pad_fs_sum, pad_sdf_sum; /* squared-error contribution of the padded (invalid) cells */
    /* accumulated by nl_mlp_train, consumed by nl_loss_finalize */
    double fs_sum, sdf_sum;
    float loss, fs_loss, sdf_loss, _padf;
} nl_render_stats;

typedef struct {
    /* sizes */
    int32_t n_rays;          /* R */
    int32_t n_nodes;         /* octree nodes n */
    int32_t sample_capacity; /* rows available in the d_s_* arrays */
    int32_t reference_compat;/* 1: reproduce the two sampler quirks exactly (SURVEY A.3) */
    float voxel_size, step_size, max_distance;
    float truncation, max_depth;      /* criterion.py: sdf_truncation, data_specs.max_depth */
    float fs_weight, sdf_weight;      /* criterion.py:11-12 */
    /* map (device) */
    const float *d_centres;      /* f32[n,3]  voxel_center_xyz   */
    const int32_t *d_structure;  /* i32[n,9]  voxel_structure    */
    /* rays (device) */
    const float *d_ray_o, *d_ray_d;   /* f32[R,3] */
    const float *d_gt_depth;          /* f32[R] = ||p|| * cos  (criterion.py:30-32), may be NULL for eval */
    const float *d_cos;               /* f32[R]  pointsCos, may be NULL (= 1) */
    /* noise: NULL = constant 0.5 (deterministic=True, voxel_helpers.py:298-299); else f32[R_hit_padded, noise_stride] */
    const float *d_noise;
    int32_t noise_stride;
    uint32_t rng_seed;                /* used when d_noise == NULL and rng_seed != 0: counter-based uniform noise */
    /* workspace (device), sizes from nl_render_workspace_bytes */
    void *d_workspace;
    int64_t workspace_bytes;
    /* outputs (device) */
    nl_render_stats *d_stats;
    int32_t *d_hit_rank;   /* i32[R]: rank among hit rays or -1           (ray_mask)               */
    int32_t *d_s_ray;      /* i32[cap] ray index of each valid sample, row-major (ray, step) order */
    int32_t *d_s_vox;      /* i32[cap] sampled_point_voxel_idx                                      */
    float *d_s_depth;      /* f32[cap] sampled_point_depth                                          */
    float *d_s_xyz;        /* f32[cap,3] ray_o + ray_d * depth (mul then add, unfused) render_helpers.py:9-10 */
    uint8_t *d_s_flag;     /* u8[cap] bit0 front_mask, bit1 sdf_mask (criterion.py:67-82); 0 if d_gt_depth NULL */
    int32_t *d_ray_nsamp;  /* i32[R] valid samples per ray (0 for missed rays); 16-byte aligned (also d_ray_offset, d_hit_rank, d_workspace) */
    int32_t *d_ray_offset; /* i32[R] offset of the ray's first sample in the compact list */
    const void *d_packed_children; /* optional: nl_octree_pack_children() image of (d_centres, d_structure).  With it the
                                    * traversal runs warp-cooperatively (8 lanes per ray, one child each, ballot + shared-memory
                                    * stack); NULL = one thread per ray over the reference's two arrays (same results) */
    const uint32_t *d_rng_seed;    /* optional device-side seed (overrides rng_seed; 0 is mapped to 1): lets a captured CUDA graph draw
                                    * new sampler noise on every replay */
} nl_render_args;

NL_API int64_t nl_render_workspace_bytes(int32_t n_rays);
/* Device-side traversal image of the octree: for node n and child slot u one 16-byte record {child centre xyz, child id
 * (int bits, -1 = none)}, 128 B per node (n_nodes * 128 bytes): the 8 lanes that expand a node read one 128-byte line instead
 * of the node's row of `structure` followed by dependent, scattered reads of `centres`.  Rebuild after every map update.
 * Requires what the reference's octree guarantees: a child's side is half its parent's. */
NL_API int64_t nl_octree_packed_bytes(int32_t n_nodes);
NL_API int nl_octree_pack_children(int32_t n_nodes, const float *d_centres, const int32_t *d_structure, void *d_packed, void *stream);
/* re-pack only the listed nodes (d_ids i32[n_ids]: the dirty rows of an incremental map update) */
NL_API int nl_octree_pack_children_rows(int32_t n_ids, const int32_t *d_ids, const float *d_centres, const int32_t *d_structure, void *d_packed,
                                 void *stream);
NL_API int nl_render_samples(const nl_render_args *args, void *stream);

/* ============================================================================================
 * 4. Embedding gather + trilinear interpolation (render_helpers.py:40-93) and its backward
 * ============================================================================================ */
/* feats[M,16] = sum_k w_k(xyz, centre[vox]) * float(emb[vox2row[vox,k]])   (emb: bf16 [V,16]) */
NL_API int nl_gather_trilinear_fwd(int64_t M, const int32_t *d_M_dev, const float *d_xyz, const int32_t *d_vox,
                            const float *d_centres, const int32_t *d_vox2row, const uint16_t *d_emb_bf16,
                            float voxel_size, float *d_feats, void *stream);
/* Backward: scatters d feats into the fp32 gradient table (atomics; each contribution rounded to bf16 first
 * when round_bf16 != 0, which is where autograd rounds for the reference's bf16 table), and reduces
 * dL/dxyz into per-frame pose accumulators acc[F,12] = (dL/dt[3], dL/dR[3,3]) via rays.
 * Any of d_grad_emb / d_dxyz / d_pose_acc may be NULL. */
NL_API int nl_gather_trilinear_bwd(int64_t M, const int32_t *d_M_dev, const float *d_xyz, const int32_t *d_vox,
                            const float *d_centres, const int32_t *d_vox2row, const uint16_t *d_emb_bf16,
                            float voxel_size, const float *d_dfeats, int round_bf16, float *d_grad_emb, float *d_dxyz,
                            const int32_t *d_s_ray, const float *d_s_depth, const float *d_ray_dir_local,
                            const int32_t *d_ray_frame, int n_frames, float *d_pose_acc, void *stream);

/* ============================================================================================
 * 5. SDF decoder MLP in_dim(16) -> W -> W -> 1 with ReLU (src/variations/lidar.py:109-131) + loss
 *    (src/criterion.py:92-103) + backward.  Weights are nn.Linear layout: W0[W,16], W1[W,W], W2[1,W].
 * ============================================================================================ */
typedef struct {
    int32_t width;                 /* W: 256 (all shipped configs) or any multiple of 32 up to 256 */
    const float *W0, *b0, *W1, *b1, *W2, *b2;   /* device */
    const float *W0t, *W1t;        /* device: transposes [16,W], [W,W] (nl_mlp_prepare writes them) */
} nl_mlp_weights;

typedef struct {
    float *gW0, *gb0, *gW1, *gb1, *gW2, *gb2;   /* device fp32 gradient accumulators (same shapes) */
} nl_mlp_grads;

NL_API int nl_mlp_prepare(int32_t width, const float *d_W0, const float *d_W1, float *d_W0t, float *d_W1t, void *stream);
/* forward only: sdf[M] */
NL_API int nl_mlp_forward(int64_t M, const int32_t *d_M_dev, const float *d_feats, const nl_mlp_weights *w, float *d_sdf,
                   void *stream);
/* forward + loss + backward in one pass.  Per-sample loss terms come from d_s_flag / d_s_depth / rays and the
 * constants in d_stats (nl_loss_prepare).  Writes sdf[M], dfeats[M,16]; accumulates the squared-error sums into
 * d_stats; if grads != NULL also accumulates decoder gradients (d_act_h1 / d_act_dh2: [cap,W] scratch for the
 * dW1 GEMM, required then).  If d_dsdf_ext != NULL the loss is skipped and d loss / d sdf is read from it
 * (f32[M]; this is the backward of a plain Decoder.forward under autograd; d_s_* / d_stats may then be NULL). */
NL_API int nl_mlp_train(int64_t M, const int32_t *d_M_dev, const float *d_feats, const nl_mlp_weights *w,
                 const uint8_t *d_s_flag, const float *d_s_depth, const int32_t *d_s_ray, const float *d_cos,
                 const float *d_gt_depth, nl_render_stats *d_stats, float truncation, float *d_sdf, float *d_dfeats,
                 const nl_mlp_grads *grads, float *d_act_h1, float *d_act_dh2, const float *d_dsdf_ext, void *stream);
/* Tensor-core (wgmma 3xTF32) forward for width 256: weights are pre-split into tf32 hi/lo and pre-swizzled
 * into shared-memory panel images by nl_mlp_tc_prepare (nl_mlp_tc_panel_bytes() bytes of device memory). */
NL_API int64_t nl_mlp_tc_panel_bytes(void);
NL_API int nl_mlp_tc_prepare(const float *d_W0, const float *d_W1, const float *d_w2, void *d_panels, void *stream);
NL_API int nl_mlp_tc_forward(int64_t M, const int32_t *d_M_dev, const float *d_feats, const void *d_panels, const float *d_b0,
                      const float *d_b1, const float *d_w2, const float *d_b2, float *d_sdf, void *stream);
/* Tensor-core forward + loss + backward (same contract as nl_mlp_train, width 256 only).  With grads != NULL d_act is a
 * scratch buffer of nl_mlp_tc_act_floats(M) floats (internal activations for the weight-gradient kernels).
 * The panels must have been prepared from the same W0 / W1 / w2 (the backward panels hold diag(w2) W1).
 * wgrad_stream (may be NULL = stream): the weight-gradient kernels are enqueued there, ordered after the forward/backward
 * kernel by an event, so that they overlap with later work on `stream`; the caller joins the two streams before it reads
 * `grads` or reuses d_act. */
NL_API int64_t nl_mlp_tc_act_floats(int64_t M);
NL_API int nl_mlp_tc_train(int64_t M, const int32_t *d_M_dev, const float *d_feats, const void *d_panels, const float *d_W1,
                    const float *d_b0, const float *d_b1, const float *d_w2, const float *d_b2, const uint8_t *d_s_flag, const float *d_s_depth,
                    const int32_t *d_s_ray, const float *d_cos, const float *d_gt_depth, nl_render_stats *d_stats, float truncation,
                    float *d_sdf, float *d_dfeats, const nl_mlp_grads *grads, float *d_act, const float *d_dsdf_ext, void *wgrad_stream,
                    void *stream);
/* loss constants from the sample statistics (criterion.py:84-88, 97-100); call after nl_render_samples */
NL_API int nl_loss_prepare(nl_render_stats *d_stats, float fs_weight, float sdf_weight, void *stream);
NL_API int nl_loss_finalize(nl_render_stats *d_stats, float fs_weight, float sdf_weight, void *stream);

/* ============================================================================================
 * 6. SE(3) pose (src/se3pose.py): 6-vector [t, w] -> R(w) (11-term Taylor A,B), ray generation and
 *    the pose Jacobian (autograd through rotation()/translation() in the reference).
 * ============================================================================================ */
NL_API int nl_pose_matrices(int n_frames, const float *d_pose6, float *d_Rt12, void *stream);  /* [F,12] = R row-major, t */
NL_API int nl_rays_from_poses(int64_t R, const float *d_dir_local, const int32_t *d_ray_frame, const float *d_Rt12,
                       float *d_ray_o, float *d_ray_d, void *stream);                    /* render_helpers.py:374-376 */
NL_API int nl_pose_grad(int n_frames, const float *d_pose6, const float *d_pose_acc, float *d_grad6, void *stream);
/* nl_pose_matrices + nl_rays_from_poses as one launch (n_frames <= 32; every block evaluates the matrices itself, block 0 also stores
 * them into d_Rt12 if given): a kernel boundary costs as much as either kernel at the reference's 2048-ray iteration size. */
NL_API int nl_rays_from_pose6(int64_t R, int n_frames, const float *d_dir_local, const int32_t *d_ray_frame, const float *d_pose6, float *d_Rt12,
                       float *d_ray_o, float *d_ray_d, void *stream);
/* The tail of an iteration that optimises poses as one launch (n_frames <= 31): nl_pose_grad for every frame; the Adam update
 * (nl_adam_f32_ctl's arithmetic, step count and skip flag from d_ctl) of the rows whose bit is set in row_mask, moments d_m / d_v
 * f32[n_frames,6]; nl_loss_finalize on d_stats (if given); and *d_seed_x += inc_x (wrapping) for up to two device-side RNG seeds
 * that a captured iteration advances (either may be NULL).  Replaces up to n_frames + 4 launches (optim.step() over the pose
 * parameters, render_helpers.py:353-357 / :448-452). */
NL_API int nl_pose_step(int n_frames, float *d_pose6, const float *d_pose_acc, float *d_grad6, uint32_t row_mask, float *d_m, float *d_v,
                 double lr, double beta1, double beta2, double eps, const int32_t *d_ctl, nl_render_stats *d_stats, float fs_weight,
                 float sdf_weight, int32_t *d_seed_a, int32_t inc_a, int32_t *d_seed_b, int32_t inc_b, void *stream);

/* Per-iteration ray selection (LidarFrame.sample_rays, src/lidarFrame.py:55-57 / src/utils/sample_util.py:4-19): for each of
 * n_frames scans, n_select distinct points uniformly at random out of its d_n_points[f] points (int64, device; a scan's arrays have
 * `cap` rows), in ascending point order like the reference's mask, and the gather of their ray data in the same launch:
 * d_dirs f32[n_frames*n_select,3], d_gt, d_cos f32[n_frames*n_select], optional d_idx i32 (the chosen point indices).
 * Seed: *d_seed if given (a captured graph advances it between replays), else `seed`.  The subset is a function of the seed alone
 * (radix select over per-point hashed keys; equal keys go to the lower point index). */
NL_API int nl_select_rays(int n_frames, int cap, int n_select, const int64_t *d_n_points, const uint32_t *d_seed, uint32_t seed,
                   const float *d_dirs_all, const float *d_gt_all, const float *d_cos_all, float *d_dirs, float *d_gt, float *d_cos,
                   int32_t *d_idx, void *stream);

/* ============================================================================================
 * 7. Optimiser (torch.optim.Adam semantics, render_helpers.py:353/448): fp32 tensors and the bf16
 *    embedding table (every intermediate rounded to bf16 where torch's per-op kernels round).
 * ============================================================================================ */
NL_API int nl_adam_f32(int64_t n, float *d_param, const float *d_grad, float *d_m, float *d_v, double lr, double beta1,
                double beta2, double eps, int step, void *stream);
NL_API int nl_adam_bf16(int64_t n, uint16_t *d_param, const float *d_grad_f32, uint16_t *d_m, uint16_t *d_v, double lr,
                 double beta1, double beta2, double eps, int step, void *stream);
/* nl_adam_f32 with the step count in device memory: *d_step is incremented, then used -- so the pair of launches can be
 * captured in a CUDA graph and replayed (the tracking loop, render_helpers.py:452-510, is launch-bound). */
NL_API int nl_adam_f32_devstep(int64_t n, float *d_param, const float *d_grad, float *d_m, float *d_v, double lr, double beta1,
                        double beta2, double eps, int32_t *d_step, void *stream);


/* ============================================================================================
 * 8. Device-side iteration control: lets a whole optimisation call (render_helpers.py:356-423 / :452-510) run without a
 *    host synchronisation per iteration and still behave like the reference's loop.
 *    ctl is int32[NL_CTL_WORDS] in device memory, zeroed by the caller before the first iteration (NL_CTL_MIN_HIT = INT32_MAX).
 * ============================================================================================ */
#define NL_CTL_ERROR 0      /* OR of nl_render_stats.error over all iterations (bit1 capacity, bit2 stack: the call must be redone / fails) */
#define NL_CTL_SKIPPED 1    /* iterations the reference would have skipped (render_rays returned None, render_helpers.py:405-409)        */
#define NL_CTL_SKIP_NOW 2   /* 1 while the current iteration is such an iteration: nl_adam_*_ctl then leave everything untouched           */
#define NL_CTL_ADAM_STEP 3  /* optimiser steps taken so far including the current one (torch.optim.Adam's `step`)                         */
#define NL_CTL_MIN_HIT 4    /* min over iterations of n_hit_rays                                                                           */
#define NL_CTL_ITERS 5      /* iterations seen                                                                                             */
#define NL_CTL_MAX_SAMPLES 6 /* max over iterations of n_samples (what the sample capacity has to hold)                                    */
#define NL_CTL_WORDS 8
/* after an iteration's nl_render_samples (and, multi-GPU, the statistics exchange): d_ctl = fold(d_ctl_prev, d_stats).
 * d_ctl_prev may equal d_ctl (in place); two alternating blocks let work that was deferred to a second stream (the decoder's
 * optimiser step of the previous iteration) keep reading the block of ITS iteration */
NL_API int nl_iter_status(const nl_render_stats *d_stats, const int32_t *d_ctl_prev, int32_t *d_ctl, void *stream);
/* nl_adam_f32 / nl_adam_bf16 with the step count and the skip flag read from the control block */
NL_API int nl_adam_f32_ctl(int64_t n, float *d_param, const float *d_grad, float *d_m, float *d_v, double lr, double beta1, double beta2,
                    double eps, const int32_t *d_ctl, void *stream);
NL_API int nl_adam_bf16_ctl(int64_t n, uint16_t *d_param, const float *d_grad_f32, uint16_t *d_m, uint16_t *d_v, double lr, double beta1,
                     double beta2, double eps, const int32_t *d_ctl, void *stream);

/* ============================================================================================
 * 9. Multi-GPU exchange helpers (SURVEY.md 8 e): the per-iteration statistics that make the loss global are packed into ONE
 *    f64 vector that is all-reduced with SUM (counters and sums as they are; S_max and the error bits in one slot per rank, so
 *    that SUM transports a MAX / OR), and unpacked again.  The collective itself is the caller's (NCCL).
 * ============================================================================================ */
#define NL_STATS_PACK_FIXED 10   /* 6 counters, 2 pad sums, n_hit_rays, reserved */
/* phase 0 (before backward): d_buf = f64[NL_STATS_PACK_FIXED + 2 * world], the sample statistics.
 * phase 1 (after backward):  d_buf = f32[4], the two squared-error sums as (hi, lo) float pairs -- they travel in the header
 *                            of the fp32 gradient buffer, so the gradients and the loss need one collective together. */
NL_API int nl_stats_pack(const nl_render_stats *d_stats, void *d_buf, int rank, int world, int phase, void *stream);
/* phase 0 also re-derives the loss constants (nl_loss_prepare) from the now global statistics */
NL_API int nl_stats_unpack(nl_render_stats *d_stats, const void *d_buf, int world, int phase, float fs_weight, float sdf_weight, void *stream);


/* phase-0 unpack reading every rank's packed vector directly (d_peer_bufs: device array of `world` pointers into symmetric memory):
 * pack -> cross-rank barrier -> this call replaces the all-reduce of the statistics exchange */
NL_API int nl_stats_unpack_peers(nl_render_stats *d_stats, const double *const *d_peer_bufs, int world, float fs_weight, float sdf_weight,
                          void *stream);
/* Fused reduce-scatter -> Adam -> all-gather over NVLink peer memory (csrc/peer.cu): the embedding-gradient reduction and the
 * bf16 Adam step of the embedding table as ONE kernel per rank.  d_grad_peers / d_param_peers: device arrays of `world` pointers
 * to every rank's fp32 gradient table / bf16 parameter table (symmetric memory, n_elems elements each, 16 per row);
 * d_grad_mc / d_param_mc: the NVLS multicast addresses of the same buffers, or both NULL (plain P2P loads / stores then).
 * Rank r reduces and updates rows [r*V/W, (r+1)*V/W) -- d_m / d_v are indexed like the table but only that slice is touched --
 * and writes the new parameters into every rank's table.  Step count and skip flag come from d_ctl (section 8).
 * The caller brackets the call with cross-rank barriers: all scatters complete before, all tables written after. */
NL_API int nl_peer_reduce_adam_bf16(int64_t n_elems, int rank, int world, const float *const *d_grad_peers, const float *d_grad_mc,
                             uint16_t *const *d_param_peers, uint16_t *d_param_mc, uint16_t *d_m, uint16_t *d_v, double lr, double beta1,
                             double beta2, double eps, const int32_t *d_ctl, int64_t hdr_n, const float *const *d_hdr_peers,
                             const float *d_hdr_mc, float *d_hdr_out, void *stream);
/* (hdr_n floats in front of each rank's table -- loss sums, pose accumulators -- are summed over the ranks into the LOCAL
 * d_hdr_out by the same launch; hdr_n % 4 == 0, may be 0) */

/* ============================================================================================
 * 10. Sparse marching cubes over the per-voxel SDF lattices of get_scores -- replaces MeshExtractor.marching_cubes
 *     (src/utils/mesh_util.py:145-169: a Python loop calling skimage.measure.marching_cubes once per voxel on the host).
 *     d_sdf f32[n_vox, res, res, res] (lattice point (i,j,k) of voxel v at ((v*res + i)*res + j)*res + k, the layout of
 *     get_scores, render_helpers.py:97-153); level 0.  Like skimage the mesh of a voxel is welded (one vertex per crossed
 *     lattice edge); voxels are independent (vertices on shared voxel faces are not merged, exactly like the reference's loop,
 *     which offsets each voxel's faces by the running vertex count, mesh_util.py:160-163).
 *     Two calls: nl_mc_count fills per-voxel counts, their exclusive scans and d_totals = {n_vertices, n_triangles} (int64[2]);
 *     the caller allocates the outputs and calls nl_mc_emit.
 *     vertex = ((lattice position) / (res - 1) - 0.5) * voxel_size + centres[vox_ids ? vox_ids[v] : v]   (mesh_util.py:149-161)
 *     Triangles are wound so that the normal points towards increasing SDF.
 * ============================================================================================ */
NL_API int nl_mc_count(int32_t n_vox, int32_t res, const float *d_sdf, int32_t *d_nvert, int32_t *d_ntri, int32_t *d_voff, int32_t *d_toff,
                int64_t *d_totals, void *stream);
NL_API int nl_mc_emit(int32_t n_vox, int32_t res, float voxel_size, const float *d_sdf, const float *d_centres, const int32_t *d_vox_ids,
               const int32_t *d_voff, const int32_t *d_toff, int64_t vert_capacity, int64_t tri_capacity, float *d_verts, int32_t *d_faces,
               void *stream);
/* The 256-case table the kernels use (host call, no GPU needed): tri u8[256][16] = up to 5 edge triples terminated by 255,
 * ntri u8[256], edge_corner u8[12][2].  Corner i sits at (i&1, (i>>1)&1, (i>>2)&1); bit i of the case index is set when the
 * SDF at corner i is negative.  The table is derived (face tracing), not hand-made; see csrc/mc.cu. */
NL_API int nl_mc_case_table(uint8_t *h_tri, uint8_t *h_ntri, uint8_t *h_edge_corner);

#ifdef __cplusplus
}
#endif
#endif /* NERFLOAM_B200_H */
