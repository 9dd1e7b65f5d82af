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

/* Node arrays: the state of a tree, and the layout of a map checkpoint (nerf-loam_b200/mapping.py MapUpdater.state_dict) and of
 * the device tree (section 1b).  child i32[n][8] (every child, FEATURE ones included; -1 = none), code u64[n] (Morton code of the
 * min corner truncated to the node's level), type i8[n] (-1 NONLEAF, 0 SURFACE, 1 FEATURE), level u8[n] (side = grid_dim >> level).
 * Node arrays read from outside the program are checked before any walk of them.  The checks, L = log2(grid_dim), and the bit each
 * one sets when it fails: */
#define NL_TREE_ROOT 1       /* n >= 1; node 0 has level 0, code 0 and is NONLEAF                                                    */
#define NL_TREE_RANGE 2      /* type in {-1, 0, 1}; level <= L; every child id c of node i has i < c < n (parents are created first)  */
#define NL_TREE_LINK 4       /* level[c] = level[i] + 1 and code[c] = code[i] | s << 3 (L - level[c]) for the child c in slot s;
                              * no code bits below a node's level                                                                       */
#define NL_TREE_PARENTS 8    /* every node but the root is the child of exactly one node                                             */
#define NL_TREE_SHAPE 16     /* NONLEAF <=> level < L; every NONLEAF node has a child                                                 */
#define NL_TREE_ROWS 32      /* vertex2row in [-1, n_rows); rows only on level-L nodes; every row in [0, n_rows) used exactly once      */
#define NL_TREE_VERTICES 64  /* the 8 corner leaves of every SURFACE leaf exist; vertex2row[v] >= 0 <=> v is such a corner             */
/* ROWS and VERTICES walk the tree, so they are evaluated only on a tree that passes the first five checks (otherwise they are 0).
 * nl_octree_validate returns the OR of the failed checks' bits (0 = well-formed), or < 0 for bad arguments; vertex2row i32[n] may
 * be NULL (no row checks).  Validation reads every array in O(n) and never follows an id it has not range-checked. */
NL_API int64_t nl_octree_validate(int64_t grid_dim, int64_t n, const int32_t *h_child, const uint64_t *h_code, const int8_t *h_type,
                                  const uint8_t *h_level, const int32_t *h_vertex2row, int64_t n_rows);
/* Copies the tree's node arrays out (n = nl_octree_count_nodes). */
NL_API int nl_octree_nodes(const nl_octree *t, int32_t *h_child, uint64_t *h_code, int8_t *h_type, uint8_t *h_level);
/* Replaces the tree of an initialised handle by node arrays in O(n), without replaying points: runs nl_octree_validate (no rows)
 * first and returns its bits (> 0) without touching the tree if any is set, else NL_OK.  The restored tree has an empty dirty
 * list and an empty set of seen points (a cache: a repeated point only visits existing nodes and changes nothing). */
NL_API int nl_octree_restore(nl_octree *t, const int32_t *h_child, const uint64_t *h_code, const int8_t *h_type, const uint8_t *h_level,
                             int64_t n);

/* ============================================================================================
 * 1b. Device octree -- section 1's insert and the map-update glue around it (Octree::insert octree.cpp:51-111,
 *     Mapping.create_voxels / update_grid_features mapping.py:283-339) on the GPU, bit for bit: the same node ids, types,
 *     dirty rows (ascending id) and embedding-row numbering as nl_octree_insert + nl_octree_export_dirty +
 *     nl_assign_embedding_rows_subset (csrc/octree_dev.cu states the parallel restatement of the creation order).
 *     The tree is capacity-sized device arrays owned by the caller, node id = row:
 *       child i32[cap][8] (every child, FEATURE ones included; -1 = none), code u64[cap] (Morton code of the min corner truncated
 *       to the node's level), type i8[cap] (-1 NONLEAF, 0 SURFACE, 1 FEATURE), level u8[cap] (side = grid_dim >> level),
 *       scratch i32[cap] (resting value INT32_MAX), and a pending dirty list u32[] (resting value 0xffffffff).
 *     The root (id 0: child -1, code 0, NONLEAF, level 0) is written by the caller.
 *     d_counts i64[8]: [0] batch rejected, [1] new nodes, [2] dirty rows, [3] embedding rows after the update, [4] pending entries.
 *     Workspace for n points with L = log2(grid_dim), P = 8n, T = sum_{d=1..L} min(P, 8^d) (bound on the new nodes):
 *       bytes = max(42 P + 8 + 33 T + sort/scan scratch,  4 (P + 2n) + (T + P + 2n) + 68 n + 4 + sort/select/scan scratch), each array
 *       256-byte aligned; the CUB scratch is queried for the current device, so only this call gives the exact figure.
 *     Like nl_octree_insert, a batch with any coordinate outside [0, grid_dim-2] is rejected as a whole: d_counts[0] = 1 and
 *     nothing is written to the tree by insert_count; the caller then does not call insert_commit.
 * ============================================================================================ */
NL_API int64_t nl_devoctree_workspace_bytes(int64_t n_points, int64_t grid_dim);
/* Octree::insert octree.cpp:51-111, step 1 (reads the tree only): validate the batch d_vox i32[n,3] (n <= 2^23), find the nodes
 * it creates.  Writes d_counts[0..1]; the caller reads them back, grows the tree to n_nodes + d_counts[1] and commits. */
NL_API int nl_devoctree_insert_count(int64_t grid_dim, const int32_t *d_child, const int32_t *d_vox, int64_t n, void *d_ws, int64_t ws_bytes,
                              int64_t *d_counts, void *stream);
/* Octree::insert octree.cpp:51-111, step 2 (same batch, same workspace, the tree unchanged since step 1): create the n_new nodes
 * with ids n_nodes.., link them, promote FEATURE leaves visited by corner 0, and append the nodes below `base` (the node count at
 * the last dirty export) whose rows change to the pending list, once each (it needs min(base, 10 n) free entries). */
NL_API int nl_devoctree_insert_commit(int64_t grid_dim, int64_t n_nodes, int64_t n_new, int64_t base, int32_t *d_child, uint64_t *d_code,
                               int8_t *d_type, uint8_t *d_level, int32_t *d_scratch, uint32_t *d_dirty_list, int64_t n, void *d_ws,
                               int64_t ws_bytes, int64_t *d_counts, void *stream);
/* nl_octree_export_dirty's id list (mapping.py:320-326 restricted to the changed rows): d_ids i32[n_list + n_nodes - base] =
 * the pending list sorted, then base .. n_nodes-1; d_counts[2] = their number.  Clears the pending list.  n_points: points
 * inserted since the last call (sizes the workspace). */
NL_API int nl_devoctree_dirty_ids(int64_t grid_dim, int64_t n_nodes, int64_t base, int64_t n_list, uint32_t *d_dirty_list, int32_t *d_scratch,
                           int32_t *d_ids, int64_t n_points, void *d_ws, int64_t ws_bytes, int64_t *d_counts, void *stream);
/* nl_octree_export_map's rows (mapping.py:320-326, octree.cpp:293-342) from the device tree: rows o < n_rows (and o < *d_count if
 * given) of node d_ids[o] (d_ids NULL: node o) into row o (compact != 0) or row = node id of centres f32[.,3], structure i32[.,9],
 * vertex i32[.,8]. */
NL_API int nl_devoctree_export(int64_t grid_dim, double voxel_size, int64_t n_rows, const int32_t *d_ids, const int64_t *d_count, int compact,
                        const int32_t *d_child, const uint64_t *d_code, const int8_t *d_type, const uint8_t *d_level, float *d_centres,
                        int32_t *d_structure, int32_t *d_vertex, void *stream);
/* nl_assign_embedding_rows_subset (mapping.py:294-317) over the dirty rows d_ids[o < d_counts[2]] (n_rows: their bound) of the
 * row = node id arrays written by nl_devoctree_export: numbers the new vertices from n_emb_rows on in d_vertex2row i32[cap],
 * writes d_vox2row rows of those nodes and d_counts[3] = the new number of embedding rows. */
NL_API int nl_devoctree_assign_rows(int64_t grid_dim, int64_t n_rows, const int32_t *d_ids, int64_t n_nodes, const int8_t *d_type,
                             const int32_t *d_vertex, int32_t *d_vertex2row, int32_t *d_scratch, int64_t n_emb_rows, int32_t *d_vox2row,
                             int64_t n_points, void *d_ws, int64_t ws_bytes, int64_t *d_counts, void *stream);
/* find_octant (octree.cpp:151-171) for d_xyz i32[n,3]: leaf id or -1 into d_out i32[n] (has_voxel octree.cpp:173-206). */
NL_API int nl_devoctree_find(int64_t grid_dim, const int32_t *d_child, const int32_t *d_xyz, int64_t n, int32_t *d_out, void *stream);

/* --------------------------------------------------------------------------------------------
 * 1b, queries: the rest of section 1's method set on the device tree, equal to the host tree's results bit for bit.  None of
 * them depends on the order in which atomics land, and none synchronises with the host between its launches.
 *   Query workspace for n_nodes nodes and n points (n = 0 except for try_insert), N = n_nodes, P = 8n:
 *     bytes = max(29 N, 16 P) + CUB sort/select scratch, each array 256-byte aligned; only this call gives the exact figure.
 * -------------------------------------------------------------------------------------------- */
NL_API int64_t nl_devoctree_query_workspace_bytes(int64_t n_nodes, int64_t n_points, int64_t grid_dim);
/* nl_devoctree_export with every output of export_row (octree_host.cpp): get_centres_and_children (octree.cpp:293-342) is
 * voxels4 f32[.,4] (xyz, side; zero for FEATURE nodes), children_f f32[.,8] (visited non-FEATURE children, else -1) and vertex
 * i32[.,8]; centres / structure are nl_devoctree_export's.  Any output but d_vertex may be NULL (not written). */
NL_API int nl_devoctree_export_nodes(int64_t grid_dim, double voxel_size, int64_t n_rows, const int32_t *d_ids, const int64_t *d_count,
                              int compact, const int32_t *d_child, const uint64_t *d_code, const int8_t *d_type, const uint8_t *d_level,
                              float *d_voxels4, float *d_children_f, float *d_centres, int32_t *d_structure, int32_t *d_vertex,
                              void *stream);
/* get_voxels (leaves_only = 0: d_out f32[n_nodes,4] = xyz, side of every node) and get_leaf_voxels (leaves_only = 1: d_out
 * f32[m,3] of the SURFACE leaves, m <= n_nodes written to d_count i64[1]) in preorder (octree.cpp:212-252), without a tree walk:
 * the children are visited in slot order and the slot is the Morton digit of its level, so preorder is the order of (code,
 * level); equal codes are an ancestor chain, created root first, so one stable radix sort of the codes with the node ids as
 * values is the preorder, and the leaves are its SURFACE subset. */
NL_API int nl_devoctree_preorder(int64_t grid_dim, int64_t n_nodes, const uint64_t *d_code, const int8_t *d_type, const uint8_t *d_level,
                          int leaves_only, float *d_out, int64_t *d_count, void *d_ws, int64_t ws_bytes, void *stream);
/* try_insert (octree.cpp:113-149, nl_octree_try_insert) for d_vox i32[n,3], 1 <= n <= 2^23: d_out i64[2] = (number of distinct
 * int32-truncated corner keys of the batch that are keys of the tree, number of distinct corner keys of the batch); the ratio
 * is 1.0 * d_out[0] / d_out[1].  The tree's corner keys are the codes of its level-L nodes, so a key is one iff it decodes to
 * in-grid coordinates whose leaf exists; keys are the host's (21 bits per axis), so negative and out-of-grid points alias alike. */
NL_API int nl_devoctree_try_insert(int64_t grid_dim, const int32_t *d_child, const int32_t *d_vox, int64_t n, void *d_ws, int64_t ws_bytes,
                            int64_t *d_out, void *stream);
/* nl_octree_validate on the device, for node arrays uploaded from outside the program (a checkpoint, a pickle): d_out i64[2] =
 * (bits of the first five checks, bits of ROWS / VERTICES); their OR equals nl_octree_validate's result.  A structural pass (one
 * thread per node and slot; parent counts in the workspace) and a sweep of the parent counts, then, with d_vertex2row i32[n_nodes]
 * given, a row pass that returns at once unless the structural word is 0, so it never walks a malformed tree, and a sweep of its
 * counts.  No result depends on the order in which atomics land; no host synchronisation.  Workspace: three arrays of 4 n_nodes bytes, each 256-byte
 * aligned (nl_devoctree_query_workspace_bytes(n_nodes, 0, grid_dim) covers it). */
NL_API int nl_devoctree_validate(int64_t grid_dim, int64_t n_nodes, const int32_t *d_child, const uint64_t *d_code, const int8_t *d_type,
                                 const uint8_t *d_level, const int32_t *d_vertex2row, int64_t n_rows, void *d_ws, int64_t ws_bytes,
                                 int64_t *d_out, void *stream);

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
    int32_t n_samples;     /* M      = sample_mask.sum()                 render_helpers.py:242
                              summed in 64 bits, stored saturated at INT32_MAX; bit1 of error is set whenever the 64-bit total
                              exceeds sample_capacity, so a call that needs 2^31 samples or more reports INT32_MAX with bit1 set.
                              d_ray_offset saturates the same way and no sample at or past sample_capacity is written.  One ray's
                              stratum count ceil(steps) saturates at INT32_MAX as well. */
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

/* --------------------------------------------------------------------------------------------
 * 3b. Batched front end: K independent problems in one ray batch (render_helpers.track_frames).  Rays [k N, (k+1) N) belong to
 *     problem k, N = n_rays / K.  Every problem is sampled exactly as nl_render_samples over only its N rays would sample it:
 *     its hit ranks, R_hit, P, S_max, max_steps_ceil, error bit 0, the loss-mask counters and the loss constants land in
 *     d_problem_stats[k], and both reference_compat quirks and the 800-ray chunking are keyed by the problem's own (rank, R_hit, P).
 *     args->d_stats receives the call-wide totals that size the rest of the chain: n_hit_rays, n_samples (bit1 of error: the
 *     sample capacity, which all problems share) and bit2 of error.  d_hit_rank holds the rank within the problem, d_s_ray the
 *     global ray index (problem = s_ray / N); the sample list is problem 0's samples in their solo order, then problem 1's, ...
 *     Noise: args->d_noise (if given) is f32[K][noise_rows][noise_stride], rows by hit rank within the problem; otherwise problem
 *     k draws hash noise from d_problem_seeds[k] (0 is mapped to 1, as for args->d_rng_seed) with the ray index WITHIN the problem
 *     as counter, so under one seed it draws what a solo call draws; without d_problem_seeds every problem uses args' seed.
 *     Scoring (render_helpers.score_poses): the front end and the loss alone take up to NL_SCORE_MAX_PROBLEMS problems -- K pose
 *     hypotheses of one scan, which share rays and seed.  Tracking keeps at most NL_BATCH_MAX_PROBLEMS (its pose step and control
 *     blocks).  The gap this fills: a lost scan is never re-localised; the reference falls back to the constant-velocity guess
 *     (src/tracking.py:136-137).
 * -------------------------------------------------------------------------------------------- */
#define NL_BATCH_MAX_PROBLEMS 31     /* the per-problem pose step runs one warp per problem in one block (as nl_pose_step) */
#define NL_SCORE_MAX_PROBLEMS 65535  /* per-problem statistics stay at 160 B x K (about 10 MB) */
typedef struct {
    int32_t n_problems;                 /* K, 1 <= K <= NL_SCORE_MAX_PROBLEMS; args->n_rays must be a multiple of K */
    int32_t noise_rows;                 /* rows per problem of args->d_noise */
    nl_render_stats *d_problem_stats;   /* [K] */
    const uint32_t *d_problem_seeds;    /* [K] or NULL */
    int32_t *d_problem_base;            /* i32[K] written: global hit rank of problem k's first hit ray */
} nl_batch_args;
/* sizeof(nl_batch_args), NL_BATCH_MAX_PROBLEMS: checked by the bindings at load time like nl_abi_sizes */
NL_API void nl_abi_sizes_batch(int32_t out[2]);
/* NL_SCORE_MAX_PROBLEMS: checked by the bindings at load time */
NL_API void nl_abi_sizes_score(int32_t out[1]);
NL_API int nl_render_samples_batch(const nl_render_args *args, const nl_batch_args *batch, void *stream);

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
 * scratch buffer of nl_mlp_tc_act_floats(M) floats: the relu'(h2) bits [cap][8 words] and d loss / d sdf [cap] per sample, which
 * the weight-gradient kernel reads (h1 is recomputed from d_feats; gW0 and gb0 are formed by the forward/backward kernel).
 * d_act_dh1 (may be NULL): if given, nl_mlp_tc_dh1_floats(M) floats that receive dh1 [cap][256] as well; no gradient needs it.
 * The panels must have been prepared from the same W0 / W1 / w2 (the backward panels hold diag(w2) W1).
 * wgrad_stream (may be NULL = stream): the weight-gradient kernel is enqueued there, ordered after the forward/backward
 * kernel by an event, so that it overlaps with later work on `stream`; the caller joins the two streams before it reads
 * `grads`, reuses d_act, changes d_feats or d_panels or changes d_b0 / d_W1 / d_b1 / d_w2 (the weight-gradient kernel reads them). */
NL_API int64_t nl_mlp_tc_act_floats(int64_t M);
NL_API int64_t nl_mlp_tc_dh1_floats(int64_t M);
NL_API int nl_mlp_tc_train(int64_t M, const int32_t *d_M_dev, const float *d_feats, const void *d_panels, const float *d_W1,
                    const float *d_b0, const float *d_b1, const float *d_w2, const float *d_b2, const uint8_t *d_s_flag, const float *d_s_depth,
                    const int32_t *d_s_ray, const float *d_cos, const float *d_gt_depth, nl_render_stats *d_stats, float truncation,
                    float *d_sdf, float *d_dfeats, const nl_mlp_grads *grads, float *d_act, float *d_act_dh1, const float *d_dsdf_ext,
                    void *wgrad_stream, void *stream);
/* Batched loss for a frozen decoder (no weight gradients; the samples of nl_render_samples_batch): sample m belongs to problem
 * d_s_ray[m] / rays_per_problem, reads that problem's loss constants in d_problem_stats and adds its squared errors into that
 * problem's fs_sum / sdf_sum.  sdf and dfeats are per sample the single-problem kernels' values bit for bit. */
NL_API int nl_mlp_train_batch(int64_t M, const int32_t *d_M_dev, const float *d_feats, const nl_mlp_weights *w, const uint8_t *d_s_flag,
                              const float *d_s_depth, const int32_t *d_s_ray, const float *d_cos, const float *d_gt_depth,
                              nl_render_stats *d_problem_stats, int32_t rays_per_problem, float truncation, float *d_sdf, float *d_dfeats,
                              void *stream);
NL_API int nl_mlp_tc_train_batch(int64_t M, const int32_t *d_M_dev, const float *d_feats, const void *d_panels, const float *d_b0,
                                 const float *d_b1, const float *d_w2, const float *d_b2, const uint8_t *d_s_flag, const float *d_s_depth,
                                 const int32_t *d_s_ray, const float *d_cos, const float *d_gt_depth, nl_render_stats *d_problem_stats,
                                 int32_t rays_per_problem, float truncation, float *d_sdf, float *d_dfeats, void *stream);
/* Scoring (section 3b, width 256): nl_mlp_tc_train_batch without the backward -- the forward layers, each problem's squared-error
 * sums, and no d feats.  sdf is nl_mlp_tc_forward's bit for bit; each sample adds what nl_mlp_tc_train_batch adds. */
NL_API int nl_mlp_tc_score_batch(int64_t M, const int32_t *d_M_dev, const float *d_feats, const void *d_panels, const float *d_b0,
                                 const float *d_b1, const float *d_w2, const float *d_b2, const uint8_t *d_s_flag, const float *d_s_depth,
                                 const int32_t *d_s_ray, const float *d_cos, const float *d_gt_depth, nl_render_stats *d_problem_stats,
                                 int32_t rays_per_problem, float truncation, float *d_sdf, void *stream);
/* loss constants from the sample statistics (criterion.py:84-88, 97-100); call after nl_render_samples */
NL_API int nl_loss_prepare(nl_render_stats *d_stats, float fs_weight, float sdf_weight, void *stream);
NL_API int nl_loss_finalize(nl_render_stats *d_stats, float fs_weight, float sdf_weight, void *stream);
/* nl_loss_finalize on each of K <= NL_SCORE_MAX_PROBLEMS problem blocks; d_loss_out f32[K] = its loss, or NaN where render_rays
 * returns None: no hit ray, error bit 0, or no sample */
NL_API int nl_loss_finalize_batch(int n_problems, nl_render_stats *d_problem_stats, float fs_weight, float sdf_weight, float *d_loss_out,
                                  void *stream);

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
/* The same for n_problems independent problems: scan k (row k of the arrays) is selected with its own seed d_seeds[k], exactly as
 * nl_select_rays(1, ...) with that seed selects it, so a batched problem draws the rays of a solo call under the same seed. */
NL_API int nl_select_rays_batch(int n_problems, int cap, int n_select, const int64_t *d_n_points, const uint32_t *d_seeds,
                                const float *d_dirs_all, const float *d_gt_all, const float *d_cos_all, float *d_dirs, float *d_gt,
                                float *d_cos, int32_t *d_idx, void *stream);

/* ============================================================================================
 * 7. Optimiser (torch.optim.Adam semantics, render_helpers.py:353/448): fp32 tensors and the bf16
 *    embedding table (every intermediate rounded to bf16 where torch's per-op kernels round).
 * ============================================================================================ */
NL_API int nl_adam_f32(int64_t n, float *d_param, const float *d_grad, float *d_m, float *d_v, double lr, double beta1,
                double beta2, double eps, int step, void *stream);
NL_API int nl_adam_bf16(int64_t n, uint16_t *d_param, const float *d_grad_f32, uint16_t *d_m, uint16_t *d_v, double lr,
                 double beta1, double beta2, double eps, int step, void *stream);

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
/* Batched tracking (section 3b): one control block per problem, d_ctl int32[K][NL_CTL_WORDS], initialised like a single block.
 * An iteration in which problem k hits nothing (R_hit = 0, error bit 0 or no sample) stops problem k for the rest of the call, like
 * the reference's `break` (render_helpers.py:488-491): NL_CTL_STOPPED is set, and from then on every iteration is a skipped one
 * for it (SKIP_NOW = 1, Adam's step count frozen).  ERROR also receives the call-wide bits 1 and 2 of d_totals, MAX_SAMPLES the
 * call-wide sample count (the capacity all problems share). */
#define NL_CTL_STOPPED 7
NL_API int nl_iter_status_batch(int n_problems, const nl_render_stats *d_totals, const nl_render_stats *d_problem_stats, int32_t *d_ctl,
                                void *stream);
/* nl_pose_step for K independent problems (K <= NL_BATCH_MAX_PROBLEMS), one pose each: warp k forms problem k's pose gradient from
 * its accumulator row, applies Adam with its own rate d_lr[k] (f64), step count and skip flag (d_ctl[k]), finalises its loss
 * (nl_loss_finalize on d_problem_stats[k]; d_last_loss[k] = that loss if the iteration was not skipped) and advances its seeds
 * d_seeds_a[k] += inc_a, d_seeds_b[k] += inc_b (either array may be NULL). */
NL_API int nl_pose_step_batch(int n_problems, float *d_pose6, const float *d_pose_acc, float *d_grad6, float *d_m, float *d_v, const double *d_lr,
                              double beta1, double beta2, double eps, const int32_t *d_ctl, nl_render_stats *d_problem_stats, float fs_weight,
                              float sdf_weight, float *d_last_loss, int32_t *d_seeds_a, int32_t inc_a, int32_t *d_seeds_b, int32_t inc_b,
                              void *stream);

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
 *     the caller allocates the outputs and calls nl_mc_emit.  Offsets and vertex ids are int32: when a total exceeds INT32_MAX
 *     the offsets have wrapped and the mesh cannot be emitted (nl_mc_emit refuses capacities above INT32_MAX).
 *     vertex = ((lattice position) / (res - 1) - 0.5) * voxel_size + centres[vox_ids ? vox_ids[v] : v]   (mesh_util.py:149-161),
 *     each of the four steps rounded separately in fp32 (no FMA contraction).  NaN lattice values count as outside (not < 0).
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

/* ============================================================================================
 * 11. Reconstruction evaluation: a mesh against a reference point cloud -- replaces the evaluation protocol of Readme.md
 *     ("Evaluation": the external SHINE-Mapping script, an Open3D mesh sampled on the host and a CPU KD-tree in both directions).
 *     csrc/eval.cu; nerf-loam_b200/evaluate.py composes the calls.  Every sum is fp64 in a fixed order (tiles of
 *     NL_EVAL_TILE elements, then the tiles in order), so two calls give the same bits on any device and launch shape.
 * ============================================================================================ */
#define NL_EVAL_KEY_BITS 21    /* per axis: voxel and cell keys are 3 x 21 bits; coordinates floor((p - o) / h) in [0, 2^21) */
#define NL_EVAL_TILE 2048      /* elements per fixed-order partial sum */
/* NL_EVAL_KEY_BITS, NL_EVAL_TILE: lets a binding check the constants it relies on */
NL_API void nl_abi_sizes_eval(int32_t out[2]);
/* d_bounds f32[6] = (min x, y, z, max x, y, z) over the finite rows of d_pts f32[n,3] (+inf / -inf when there is none),
 * d_nonfinite i64[1] = number of rows with a NaN or inf coordinate.  n may be 0. */
NL_API int nl_eval_bounds(int64_t n, const float *d_pts, float *d_bounds, int64_t *d_nonfinite, void *stream);
/* Surface sampling, uniform by area.  nl_eval_surface_prepare: fp64 area of every triangle of d_faces i32[n_faces,3] over
 * d_verts f32[n_verts,3] and their fp64 inclusive prefix sum, kept in the workspace; d_info f64[2] = (total area, > 0 when a face
 * index is outside [0, n_verts)).  nl_eval_sample_surface then draws sample i from Philox4x32-10 keyed on `seed` with counter i:
 * the triangle by inverse CDF over the prefix sum (zero-area triangles are never chosen), the point by the square-root barycentric
 * formula, computed in fp64 and rounded to d_out f32[n_samples,3]; d_face i32[n_samples] (may be NULL) gets the triangle. */
NL_API int64_t nl_eval_surface_workspace_bytes(int64_t n_faces);
NL_API int nl_eval_surface_prepare(int64_t n_verts, const float *d_verts, int64_t n_faces, const int32_t *d_faces, void *d_ws, int64_t ws_bytes,
                                   double *d_info, void *stream);
NL_API int nl_eval_sample_surface(int64_t n_verts, const float *d_verts, int64_t n_faces, const int32_t *d_faces, int64_t n_samples, uint64_t seed,
                                  const void *d_ws, int64_t ws_bytes, float *d_out, int32_t *d_face, void *stream);
/* Voxel down-sampling on the grid with origin (ox, oy, oz) and side res: key = floor((p - o) / res) per axis in fp64.  Rows
 * outside the box d_crop f32[6] (min, max as nl_eval_bounds writes it) padded by res are dropped (d_crop may be NULL); rows whose
 * key does not fit NL_EVAL_KEY_BITS are dropped too and counted apart.  Each occupied voxel becomes the centroid of its rows: a
 * stable radix sort by key, then one fp64 sum per voxel in that order.  d_out f32[n,3] (capacity n) gets the centroids in key
 * order, d_keys u64[n] (may be NULL) their keys (x << 42 | y << 21 | z), d_counts i64[3] = (cropped rows, rows outside the key
 * range, voxels). */
NL_API int64_t nl_eval_voxel_workspace_bytes(int64_t n_points);
NL_API int nl_eval_voxel_down_sample(int64_t n, const float *d_pts, double ox, double oy, double oz, double res, const float *d_crop, void *d_ws,
                                     int64_t ws_bytes, float *d_out, uint64_t *d_keys, int64_t *d_counts, void *stream);
/* Truncated nearest distance: d_dist[i] = min(truncation, min_j |q_i - t_j|) in fp32, exact below the truncation.  The target
 * is sorted into cells of side `cell` from origin o (keys as above; d_bad i64[1] counts target rows outside the key range, which
 * are never searched) and every occupied cell's run goes into a hash table.  A query walks Chebyshev rings of cells around its
 * own cell; after ring k every unvisited target is at least k * cell away, so it stops when its best distance is <= k * cell or
 * k * cell >= truncation (max_ring * cell >= truncation is required; max_ring <= 64).  Workspace for n_target rows, about 100
 * bytes per row. */
NL_API int64_t nl_eval_nn_workspace_bytes(int64_t n_target);
NL_API int nl_eval_nearest(int64_t n_query, const float *d_query, int64_t n_target, const float *d_target, double ox, double oy, double oz,
                           double cell, int32_t max_ring, float truncation, void *d_ws, int64_t ws_bytes, float *d_dist, int64_t *d_bad,
                           void *stream);
/* d_out f64[3] = (sum d, sum d^2, number of d < threshold) over d_dist f32[n] */
NL_API int64_t nl_eval_sums_workspace_bytes(int64_t n);
NL_API int nl_eval_distance_sums(int64_t n, const float *d_dist, float threshold, void *d_ws, int64_t ws_bytes, double *d_out, void *stream);

/* ============================================================================================
 * 12. Keyframe overlap: the voxels one scan shares with each of K keyframes -- the counts behind the mapper's 'overlap' window
 *     (Mapping.select_optimize_targets, src/mapping.py:205-225, which declares that method and raises NotImplementedError).
 *     csrc/overlap.cu; nerf-loam_b200/keyframes.py composes the calls.
 * ============================================================================================ */
#define NL_OVERLAP_MAX_CHUNK 1023                   /* keyframes per pass over the table (chunk-local index in the key's top 10 bits) */
#define NL_OVERLAP_MAX_SLOTS ((int64_t)1 << 32)   /* largest table_slots */
/* Voxel of a point p (sensor frame) under the pose row Rt f32[12] (as nl_pose_matrices writes it: R row-major, then t): per axis
 * w_i = ((R_i0 p_x + R_i1 p_y) + R_i2 p_z) + t_i in fp64, v_i = floor(w_i / voxel_size) in fp64.  A point with a v_i outside
 * [0, grid_dim) (grid_dim a power of two <= 2^18), or not finite, is counted as outside and nowhere else.
 * Inputs: the scan d_frame_pts f32[n_frame,3] under row 0 of d_Rt12 f32[n_kf+1,12]; keyframe k has d_kf_n[k] points at d_kf_pts[k]
 * (device arrays of n_kf pointers and counts) under row k + 1, and h_kf_n[k] is the same count on the host: it plans the passes.
 * Output d_out i64[3 n_kf + 1] = (shared[n_kf] = |V_k n V_c|, kf_voxels[n_kf] = |V_k|, outside[n_kf], frame_voxels = |V_c|), with
 * V the set of distinct voxels.  Keyframes go through a table of table_slots slots (a power of two >= 2^10) in passes of up to
 * NL_OVERLAP_MAX_CHUNK keyframes and table_slots / 2 points; a keyframe with more than table_slots / 2 points is an error.  The
 * workspace (256-byte aligned) holds that table and the scan's set.  No host synchronisation; the counts are exact integers, so two
 * calls give identical results. */
NL_API int64_t nl_keyframe_overlap_workspace_bytes(int64_t n_frame, int64_t table_slots);
NL_API int nl_keyframe_overlap(int64_t n_frame, const float *d_frame_pts, int32_t n_kf, const float *const *d_kf_pts, const int64_t *d_kf_n,
                               const int64_t *h_kf_n, const float *d_Rt12, double voxel_size, int64_t grid_dim, int64_t table_slots, void *d_ws,
                               int64_t ws_bytes, int64_t *d_out, void *stream);

/* ============================================================================================
 * 13. Ground segmentation and incidence cosines of one LiDAR scan -- the (points, pointsCos) the data loaders hand to LidarFrame
 *     (src/dataset/kitti.py:40-70, which calls the external Patchwork++ library and a host KD-tree).  This project's own
 *     definition (DESIGN.md section 12; no parity with Patchwork++): a concentric zone model of 4 zones, seeds from the lowest
 *     points of each patch, num_iter principal-component plane fits, an uprightness and elevation verdict, and for a ground point
 *     cos = |n.p| / |p| with n the normal of the ground patch whose mean is nearest.  csrc/ground.cu; nerf-loam_b200/ground.py
 *     composes the calls.  Every sum is fp64 in a fixed order, so two calls give identical bytes.
 *     Opt-in vertical-structure filter (DESIGN.md section 12.1; vertical_cell > 0): a row inside the ranges whose xy column
 *     (floor(x / vertical_cell), floor(y / vertical_cell)) holds returns spread over more than vertical_height in z is vertical:
 *     never a seed candidate nor in a fit, labelled non-ground with cos 1.  The columns' z extents come from a hash table with
 *     integer atomics on order-preserving keys, so they are exact and two calls still give identical bytes.
 * ============================================================================================ */
#define NL_GROUND_MAX_PATCHES 1024   /* sum over the zones of rings x sectors */
#define NL_GROUND_MAX_LPR 1024       /* largest num_lpr */
typedef struct nl_ground_params {     /* Patchwork++'s parameter names; ranges are xy radii in metres */
    double sensor_height, min_range, max_range;
    int32_t num_rings_each_zone[4], num_sectors_each_zone[4];
    double uprightness_thr;
    double elevation_thr[4];          /* first 4 global rings: ground needs mean z + sensor_height below it */
    double flatness_thr[4];           /* carried for completeness; not used by the verdict */
    int32_t num_iter, num_lpr, num_min_pts, _pad;
    double th_seeds, th_dist, adaptive_seed_margin;
    double vertical_cell;             /* column width of the vertical-structure filter in metres; 0 = off */
    double vertical_height;           /* a column whose z extent exceeds it (strictly) is vertical; > 0 when the filter is on */
} nl_ground_params;
typedef struct nl_ground_patch {      /* one patch; the doubles are NaN when the patch has no complete fit */
    double mean[3], normal[3];        /* the last fit: mean, unit normal with normal[2] >= 0 */
    double d, lambda_min;             /* plane n.p + d = 0, smallest covariance eigenvalue */
    int32_t n_points, n_ground, ground, ring;   /* points in the patch (vertical ones included), points labelled ground, verdict, global ring */
    int32_t n_vertical, _pad;         /* vertical points in the patch (0 with the filter off) */
} nl_ground_patch;
/* out = (sizeof(nl_ground_params), NL_GROUND_MAX_PATCHES, sizeof(nl_ground_patch)) */
NL_API void nl_abi_sizes_ground(int32_t out[3]);
NL_API int64_t nl_ground_workspace_bytes(int64_t n);
/* The vertical filter's column table: 16 bytes per slot (8-byte key, u32 z min and max) and a power of two >= 2n slots. */
NL_API int64_t nl_ground_vertical_workspace_bytes(int64_t n);
/* d_points f32 rows of `stride` (3, or 4 with the intensity ignored) floats, n >= 0.  Writes d_label u8[n] (1 = ground),
 * d_cos f32[n] (1 for every non-ground point), d_patch i32[n] (patch id, -1 outside the ranges or not finite; may be NULL),
 * d_patches (one record per patch, zone by zone, ring by ring, sector by sector; may be NULL) and d_counts i64[4] = (ground,
 * non-ground, outside, non-finite); non-ground counts the outside and non-finite rows too.  The workspace (256-byte aligned) has
 * nl_ground_workspace_bytes(n) bytes.  No host synchronisation.  The vertical filter needs nl_ground_segment_vertical. */
NL_API int nl_ground_segment(int64_t n, const float *d_points, int32_t stride, const nl_ground_params *params, void *d_ws, int64_t ws_bytes,
                             uint8_t *d_label, float *d_cos, int32_t *d_patch, nl_ground_patch *d_patches, int64_t *d_counts, void *stream);
/* nl_ground_segment with the vertical filter.  With params->vertical_cell > 0 it needs d_vws (256-byte aligned,
 * nl_ground_vertical_workspace_bytes(n) bytes) and writes d_vertical u8[n] (1 = vertical); with vertical_cell = 0 both may be NULL,
 * no extra kernel runs, the results are nl_ground_segment's, and a non-NULL d_vertical is zeroed. */
NL_API int nl_ground_segment_vertical(int64_t n, const float *d_points, int32_t stride, const nl_ground_params *params, void *d_ws,
                                      int64_t ws_bytes, void *d_vws, int64_t vws_bytes, uint8_t *d_label, float *d_cos, int32_t *d_patch,
                                      nl_ground_patch *d_patches, uint8_t *d_vertical, int64_t *d_counts, void *stream);
/* Stable partition by d_label: the ground rows first, then the rest, each in input order.  d_out_points f32[n,3], d_out_cos f32[n]
 * and d_out_index i32[n] (the input row of each output row). */
NL_API int nl_ground_partition(int64_t n, const float *d_points, int32_t stride, const uint8_t *d_label, const float *d_cos, void *d_ws,
                               int64_t ws_bytes, float *d_out_points, float *d_out_cos, int32_t *d_out_index, void *stream);

/* ============================================================================================
 * 14. Key-scan map refinement (the mapper's final_iter pass, src/mapping.py:154-164): P passes of `iters` iterations, each pass one
 *     bundle_adjust_frames over a random window of keyframes with poses and decoder frozen and a fresh Adam on the embedding table
 *     (render_helpers.py:341-353).  csrc/refine.cu; render_helpers.refine_map captures one iteration and replays it P x iters times.
 *     A fresh Adam makes a row-sparse step exact: a row no sample has reached since the pass began has g = m = v = 0, and the bf16
 *     update leaves it bitwise unchanged, so Adam over the rows touched so far in the pass gives the dense step's table.
 *     State d_state int32[NL_REFINE_STATE_WORDS], zeroed before the first pass: */
#define NL_REFINE_ITER 0         /* iterations completed in the call; pass = ITER / iters                                       */
#define NL_REFINE_LISTED 1       /* rows listed so far in the current pass (length of the row list)                              */
#define NL_REFINE_PREV 2         /* rows the previous pass listed (still in the row list until the next pass's first nl_mark_rows) */
#define NL_REFINE_STATE_WORDS 4
/* Pass boundary, first launch of an iteration.  A no-op unless ITER % iters == 0; then, for pass p = ITER / iters < n_passes:
 * scans d_windows[p][0..n_frames) (keyframe indices) are copied into the selection buffers d_dirs f32[n_frames,cap,3], d_gt, d_cos
 * f32[n_frames,cap] and d_n_points i64[n_frames] from the keyframe table (d_kf_arrays i64[K][3] = device addresses of each keyframe's
 * dirs f32[n,3], cos f32[n], range f32[n]; d_kf_points i64[K] = n <= cap), their poses from d_kf_pose6 f32[K,6] into d_pose6;
 * *d_sel_seed = d_sel_seeds[p], *d_noise_seed = d_noise_seeds[p] (both may be NULL: deterministic sampling); d_ctl[NL_CTL_ADAM_STEP]
 * = 0 (a fresh optimiser); and the moments d_m / d_v (bf16 [n_rows,16]) and the flag bits of the PREV rows of d_rows are zeroed.
 * Replaces the per-call set-up of bundle_adjust_frames (render_helpers.py:341-353: a new optimiser per call) and the upload of its
 * frames and seeds (render_helpers.py:356-391), once per pass. */
NL_API int nl_refine_pass_begin(int n_frames, int64_t cap, int n_keyframes, int iters, int n_passes, const int32_t *d_state,
                                const int32_t *d_windows, const int64_t *d_kf_arrays, const int64_t *d_kf_points, const float *d_kf_pose6,
                                const int32_t *d_sel_seeds, const int32_t *d_noise_seeds, float *d_dirs, float *d_gt, float *d_cos,
                                int64_t *d_n_points, float *d_pose6, int32_t *d_sel_seed, int32_t *d_noise_seed, int32_t *d_ctl,
                                int64_t n_rows, const int32_t *d_rows, uint32_t *d_row_bits, uint16_t *d_m, uint16_t *d_v, void *stream);
/* Flag the embedding rows that nl_gather_trilinear_bwd scatters into (render_helpers.py:60-93, the backward of the trilinear
 * gather): for the first min(*d_M, M) samples, the rows d_vox2row[d_vox[i]][0..8) that are >= 0.  A row whose bit in d_row_bits
 * (u32[ceil(n_rows / 32)]) was clear is set and appended to d_rows at d_state[NL_REFINE_LISTED] (each row once; order unspecified). */
NL_API int nl_mark_rows(int64_t M, const int32_t *d_M, const int32_t *d_vox, const int32_t *d_vox2row, int64_t n_rows, uint32_t *d_row_bits,
                        int32_t *d_rows, int32_t *d_state, void *stream);
/* nl_mark_rows with a floor: only rows >= row_floor are flagged and listed, so nl_adam_bf16_rows_ctl never steps rows [0, row_floor)
 * (the saved rows of a map extended with a later drive, which stay fixed).  0 <= row_floor <= n_rows; row_floor = 0 is nl_mark_rows,
 * with the same bits, list and count. */
NL_API int nl_mark_rows_floor(int64_t M, const int32_t *d_M, const int32_t *d_vox, const int32_t *d_vox2row, int64_t n_rows,
                              int64_t row_floor, uint32_t *d_row_bits, int32_t *d_rows, int32_t *d_state, void *stream);
/* nl_adam_bf16_ctl (optim.step() on the embedding table, render_helpers.py:421-423) over the first min(*d_n_listed, n_rows) rows of d_rows
 * only, 16 elements per row, with the same arithmetic; step count and skip flag from d_ctl.  Every listed row's gradient is cleared
 * after it is read, on a skipped iteration too (its scatter may have run). */
NL_API int nl_adam_bf16_rows_ctl(int64_t n_rows, const int32_t *d_rows, const int32_t *d_n_listed, uint16_t *d_param, float *d_grad_f32,
                                 uint16_t *d_m, uint16_t *d_v, double lr, double beta1, double beta2, double eps, const int32_t *d_ctl,
                                 void *stream);
/* Last launch of an iteration: *d_sel_seed += sel_inc and *d_noise_seed += noise_inc (wrapping; either may be NULL), as the captured
 * mapping iteration advances its seeds (the next iteration's frame.sample_rays and sampler noise, render_helpers.py:365-391);
 * ITER += 1, and at the end of a pass PREV = LISTED, LISTED = 0. */
NL_API int nl_refine_iter_end(int iters, int32_t *d_state, int32_t *d_sel_seed, int32_t sel_inc, int32_t *d_noise_seed, int32_t noise_inc,
                              void *stream);

/* ============================================================================================
 * 15. Global localisation, coarse stage (DESIGN.md section 3.4; csrc/globalloc.cu): for every placement of a scan over a lattice of
 *     positions x headings around anchor poses, how many of M scan points fall in an occupied map voxel, and the n highest counts.
 *     Occupied set: the map's leaf voxels (structure[i][8] == 1, Octree.get_leaf_voxels()), key floor(centre / voxel_size) per axis
 *     packed as vx << 36 | vy << 18 | vz, in an open-addressing set (hash.cuh) of nl_globalloc_occupied_slots(n_leaves) u64 slots.
 *     Anchors: A >= 1 poses, f64[A][12] = the 3x4 matrix row-major (host copy h_anchors for the checks, device copy d_anchors).
 *     Cells: lattice points (i, j) x xy_step within radius (fp64 xy distance) of an anchor, with the nearest anchor (lower index on a
 *     tie of the fp32 distance), numbered in ascending (i, j); d_cells i32[n_cells][3] = (i, j, anchor).
 *     Placement id = cell x yaw_steps + k: rotation Rz(2 pi k / yaw_steps - atan2(R_a10, R_a00)) R_a, translation (i xy_step,
 *     j xy_step, t_a,z), formed in fp64 and rounded to fp32; ids are int32, so n_cells x yaw_steps < 2^31.
 *     Count: the points whose world point ((R0 x + R1 y) + R2 z) + t (fp64 from fp32) has voxel floor(w / voxel_size) inside
 *     [0, grid_dim)^3 and in the set (the arithmetic of section 12).  Every result is an exact integer or a function of integers,
 *     independent of atomics order and launch shape.  Bad arguments return an error code; no entry point aborts.
 * ============================================================================================ */
#define NL_GLOBALLOC_MAX_POINTS 8192   /* M: the scan points are staged in shared memory (12 B each) */
/* out = (NL_GLOBALLOC_MAX_POINTS, ints per cell row) */
NL_API void nl_abi_sizes_globalloc(int32_t out[2]);
/* *d_n_leaves = the rows of d_structure i32[n_nodes][9] with side 1.  n_nodes >= 1. */
NL_API int nl_globalloc_count_leaves(int64_t n_nodes, const int32_t *d_structure, int64_t *d_n_leaves, void *stream);
/* Slots of the occupied set: a power of two >= max(2^10, 2 n_leaves); an error for n_leaves < 1 (an empty map). */
NL_API int64_t nl_globalloc_occupied_slots(int64_t n_leaves);
/* Clears d_set u64[slots] and inserts the key of every leaf row whose voxel lies in [0, grid_dim)^3.  grid_dim a power of two
 * <= 2^18; slots a power of two >= 2 x the leaf count. */
NL_API int nl_globalloc_occupied(int64_t n_nodes, const float *d_centres, const int32_t *d_structure, double voxel_size, int64_t grid_dim,
                                 int64_t slots, uint64_t *d_set, void *stream);
/* Workspace of nl_globalloc_cells / _finish: a hash of (i, j) and a key list sized from the lattice points the anchors' boxes can
 * hold.  Checks A >= 1, finite anchors, radius finite and >= 0, xy_step finite and > 0, and the lattice size. */
NL_API int64_t nl_globalloc_cells_workspace_bytes(int32_t n_anchors, const double *h_anchors, double radius, double xy_step);
/* First half of the cell table: inserts every cell with its nearest anchor and writes *d_n_cells (int64, device).  The caller reads
 * the count back and passes it to nl_globalloc_cells_finish with the same workspace. */
NL_API int nl_globalloc_cells(int32_t n_anchors, const double *h_anchors, const double *d_anchors, double radius, double xy_step, void *d_ws,
                              int64_t ws_bytes, int64_t *d_n_cells, void *stream);
/* Sorts the cells by (i, j) and writes d_cells i32[n_cells][3]. */
NL_API int nl_globalloc_cells_finish(int32_t n_anchors, const double *h_anchors, double radius, double xy_step, int64_t n_cells, void *d_ws,
                                     int64_t ws_bytes, int32_t *d_cells, void *stream);
/* d_Rt12 f32[n][12] (R row-major, then t) of the placements d_ids i64[n]: the device function the scorer uses.  An id outside
 * [0, n_cells x yaw_steps) gets a matrix of NaN. */
NL_API int nl_globalloc_matrices(int64_t n, const int64_t *d_ids, int64_t n_cells, const int32_t *d_cells, const double *d_anchors,
                                 int32_t yaw_steps, double xy_step, float *d_Rt12, void *stream);
/* d_counts[h] for the placements h in [p0, p0 + n): how many of d_points f32[n_points][3] (sensor frame, 1 <= n_points <=
 * NL_GLOBALLOC_MAX_POINTS) land in the occupied set d_set u64[slots]. */
NL_API int nl_globalloc_score(int64_t p0, int64_t n, int64_t n_cells, const int32_t *d_cells, const double *d_anchors, int32_t yaw_steps,
                              double xy_step, int32_t n_points, const float *d_points, const uint64_t *d_set, int64_t slots, double voxel_size,
                              int64_t grid_dim, int32_t *d_counts, void *stream);
NL_API int64_t nl_globalloc_select_workspace_bytes(int64_t n_placements, int32_t n_points, int64_t n_select);
/* The n_select placements of highest d_counts i32[n_placements] ranked by (count desc, id asc): d_ids i32[n_select] and their counts
 * d_sel_counts i32[n_select].  A count outside [0, n_points] is ignored; when fewer than n_select counts are valid, the remaining
 * entries of both outputs are -1.  1 <= n_select <= n_placements; workspace 256-byte aligned. */
NL_API int nl_globalloc_select(int64_t n_placements, const int32_t *d_counts, int32_t n_points, int64_t n_select, void *d_ws, int64_t ws_bytes,
                               int32_t *d_ids, int32_t *d_sel_counts, void *stream);

/* ============================================================================================
 * 16. Change detection against a saved map (DESIGN.md section 11.7; csrc/changes.cu): for every saved voxel, how many rays of a
 *     later drive pass through its surface in space the drive says is empty ("through") and how many end on it ("surface"); and
 *     the voxels where the drive's returns land outside the map's leaves ("added").  Counts are u32 summed with integer atomics,
 *     independent of launch order; the outputs of nl_change_finish are in node order and key order.  No reference counterpart:
 *     the reference treats a map as true once it is built.
 * ============================================================================================ */
/* Votes from the sample list of one nl_render_samples call (rays r in [0, R)) after the decoder forward: d_s_ray, d_s_vox, d_s_depth,
 * d_sdf f32[cap] and d_ray_offset i32[R] as that call and the forward left them, the measured depth d_gt f32[R] of each ray (the
 * point's range).  The sample count is read from d_stats->n_samples, so nothing is read back.  A run is the samples of one ray in one
 * voxel; over the union of a voxel's samples on a ray, with d = gt - depth (fp32): "through" when every d > through_depth
 * (truncation + margin) and the smallest sdf <= 0, adding 1 to d_votes[v][0]; otherwise "surface" when some |d| <= truncation, adding
 * 1 to d_votes[v][1].  d_votes u32[n_nodes][2].  When d_stats->error has bit1 or bit2 set, nothing is added and d_status i32[2] =
 * (error & 6, n_samples); otherwise d_status is not written. */
NL_API int nl_change_votes(int64_t cap, const nl_render_stats *d_stats, const int32_t *d_s_ray, const int32_t *d_s_vox, const float *d_s_depth,
                           const float *d_sdf, const float *d_gt, const int32_t *d_ray_offset, int64_t n_nodes, float truncation,
                           float through_depth, uint32_t *d_votes, int32_t *d_status, void *stream);
/* The added table: d_keys u64[slots] (voxel keys of section 15, NL_HASH_EMPTY = ~0 in free slots) and d_vals u32[slots][3] =
 * (points, distinct scans, last scan id); slots a power of two in [2^10, 2^30].  d_state u32[3] = (keys committed, keys inserted,
 * overflow).  Clears the table and, with old_slots > 0, moves every key of the old table into it with its values (state counts
 * kept); old_slots == 0 zeroes the counts.  The overflow word is cleared either way. */
NL_API int nl_change_rehash(int64_t old_slots, const uint64_t *d_old_keys, const uint32_t *d_old_vals, int64_t slots, uint64_t *d_keys,
                            uint32_t *d_vals, uint32_t *d_state, void *stream);
/* One scan into the added table: each of d_points f32[n_points][3] (sensor frame) posed by d_Rt12 f32[12] (nl_pose_matrices' layout)
 * whose voxel key (section 15's arithmetic) is not in the occupied set d_occ u64[occ_slots] adds 1 to its slot's points, and the
 * scan count rises when the slot's last scan id is not `scan`.  Only when keys committed + n_points <= slots / 2; otherwise the call
 * inserts nothing and sets the overflow word, and the caller rehashes into a larger table and calls again.  scan < 2^32 - 1. */
NL_API int nl_change_added(int64_t n_points, const float *d_points, const float *d_Rt12, double voxel_size, int64_t grid_dim,
                           const uint64_t *d_occ, int64_t occ_slots, int64_t slots, uint64_t *d_keys, uint32_t *d_vals, uint32_t scan,
                           uint32_t *d_state, void *stream);
NL_API int64_t nl_change_finish_workspace_bytes(int64_t n_nodes, int64_t slots);
/* Classification and compaction.  A leaf (d_structure[i][8] == 1) is removed when through >= min_votes and through >= ratio x
 * (through + surface) (fp64), confirmed when it has surface votes and is not removed, unobserved when it has no votes.  d_removed
 * i32[n_nodes]: the removed node ids in ascending order; d_added u64[slots]: the keys with points >= min_points and scans >=
 * min_scans in ascending order, then NL_HASH_EMPTY; d_added_vals u32[slots][2]: their (points, scans); d_totals i64[4] = (confirmed,
 * removed, unobserved, added).  0 < ratio <= 1; the counts >= 1. */
NL_API int nl_change_finish(int64_t n_nodes, const int32_t *d_structure, const uint32_t *d_votes, uint32_t min_votes, double ratio, int64_t slots,
                            const uint64_t *d_keys, const uint32_t *d_vals, uint32_t min_points, uint32_t min_scans, void *d_ws, int64_t ws_bytes,
                            int32_t *d_removed, uint64_t *d_added, uint32_t *d_added_vals, int64_t *d_totals, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NERFLOAM_B200_H */
