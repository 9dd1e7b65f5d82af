// Change detection against a saved map (include/nerfloam_b200.h section 16, DESIGN.md section 11.7): which saved voxels a later
// drive sees through, which it confirms, and where its returns land on ground the map does not hold.
//
//   votes  : one thread per sample of the engine's sample list (nl_render_samples, then the decoder forward).  A run is the samples
//            of one ray in one voxel; the thread at the first sample of a voxel's first run on its ray takes the union of that
//            voxel's samples on the ray (so a ray casts at most one vote per voxel) with d = g_r - depth in fp32:
//              through : every d > truncation + margin and the smallest sdf <= 0 (fminf: a NaN sdf never counts as a crossing);
//              surface : some |d| <= truncation.
//            The two cannot both hold.  u32 counters per node summed with integer atomics, so launch order does not matter.  A call
//            whose sample list overflowed (bit1 / bit2 of the stats' error) adds nothing and records that in d_status.
//   added  : one thread per scan point: the voxel key of voxel.cuh, looked up in the occupied set of globalloc.cu; a miss goes into
//            an open-addressing table (hash.cuh) whose slot carries (points, scans, last scan).  The scan count rises when the
//            slot's last scan changes (atomicExch), so it counts distinct scans while every call inserts one scan.  A call inserts
//            only when the keys committed by earlier calls plus its own points stay within half the slots; otherwise it inserts
//            nothing and raises the overflow word, and the caller rehashes into a larger table and repeats it.  The limit is one
//            value for every thread of the call, so a call inserts everything or nothing.
//   finish : removed node ids in node order (cub::DeviceSelect::Flagged), added keys in key order (a radix sort of the selected
//            keys with the rest set to NL_HASH_EMPTY, which sorts last), and the class totals.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <cmath>
#include <cstdint>

#include "../../include/nerfloam_b200.h"
#include "hash.cuh"
#include "nl_cuda.cuh"
#include "voxel.cuh"

namespace {

constexpr int kThreads = 256;
constexpr uint32_t kNoScan = 0xffffffffu;

int grid_blocks(int64_t n) { return (int)std::min<int64_t>(std::max(1, nl_div_up(n, kThreads)), 16 * nl_num_sms()); }

bool pow2(int64_t v) { return v > 0 && (v & (v - 1)) == 0; }

size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

// ------------------------------------------------------------------------------------------------ votes
__global__ void __launch_bounds__(kThreads) k_votes(int64_t cap, const nl_render_stats *__restrict__ stats, const int32_t *__restrict__ s_ray,
                                                    const int32_t *__restrict__ s_vox, const float *__restrict__ s_depth,
                                                    const float *__restrict__ sdf, const float *__restrict__ gt,
                                                    const int32_t *__restrict__ ray_offset, int64_t n_nodes, float trunc, float through,
                                                    uint32_t *votes, int32_t *status) {
    const int32_t err = stats->error & 6;
    if (err) {
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            status[0] = err;
            status[1] = stats->n_samples;
        }
        return;
    }
    const int64_t M = (int64_t)stats->n_samples < cap ? (int64_t)stats->n_samples : cap;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < M; i += (int64_t)gridDim.x * kThreads) {
        const int32_t r = s_ray[i], v = s_vox[i];
        if (i > 0 && s_ray[i - 1] == r && s_vox[i - 1] == v) continue;           // not the first sample of a run
        if (v < 0 || v >= n_nodes) continue;
        bool first = true;
        for (int64_t j = ray_offset[r]; j < i; ++j) first = first && s_vox[j] != v;
        if (!first) continue;                                                    // an earlier run of this ray took the voxel
        const float g = gt[r];
        bool front = true, surface = false;
        float lo = INFINITY;
        for (int64_t j = i; j < M && s_ray[j] == r; ++j) {
            if (s_vox[j] != v) continue;
            const float d = __fsub_rn(g, s_depth[j]);
            front = front && d > through;
            surface = surface || fabsf(d) <= trunc;
            lo = fminf(lo, sdf[j]);
        }
        if (front && lo <= 0.0f) atomicAdd(&votes[2 * v], 1u);
        else if (surface) atomicAdd(&votes[2 * v + 1], 1u);
    }
}

// ------------------------------------------------------------------------------------------------ added
__global__ void __launch_bounds__(kThreads) k_added(int64_t n, const float *__restrict__ pts, const float *__restrict__ Rt12, double vs, double gd,
                                                    const uint64_t *__restrict__ occ, uint64_t occ_mask, int64_t slots, uint64_t *keys,
                                                    uint32_t *vals, uint32_t scan, uint32_t *state) {
    if ((int64_t)state[0] + n > slots / 2) {            // the same test for every thread: the call inserts everything or nothing
        if (blockIdx.x == 0 && threadIdx.x == 0) state[2] = 1;
        return;
    }
    float Rt[12];
    #pragma unroll
    for (int k = 0; k < 12; ++k) Rt[k] = Rt12[k];
    const uint64_t mask = (uint64_t)slots - 1;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        uint64_t key;
        if (!nl_voxel_key(Rt, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], vs, gd, key)) continue;
        if (nl_hash_contains(occ, occ_mask, key)) continue;
        if (nl_hash_insert(keys, mask, key)) atomicAdd(&state[1], 1u);
        const uint64_t s = nl_hash_slot_of(keys, mask, key);
        atomicAdd(&vals[3 * s], 1u);
        if (atomicExch(&vals[3 * s + 2], scan) != scan) atomicAdd(&vals[3 * s + 1], 1u);
    }
}

__global__ void k_commit(uint32_t *state) { state[0] = state[1]; }

__global__ void __launch_bounds__(kThreads) k_clear(int64_t slots, uint64_t *keys, uint32_t *vals) {
    for (int64_t s = blockIdx.x * (int64_t)kThreads + threadIdx.x; s < slots; s += (int64_t)gridDim.x * kThreads) {
        keys[s] = NL_HASH_EMPTY;
        vals[3 * s] = 0;
        vals[3 * s + 1] = 0;
        vals[3 * s + 2] = kNoScan;
    }
}

__global__ void __launch_bounds__(kThreads) k_rehash(int64_t old_slots, const uint64_t *__restrict__ old_keys, const uint32_t *__restrict__ old_vals,
                                                     int64_t slots, uint64_t *keys, uint32_t *vals) {
    const uint64_t mask = (uint64_t)slots - 1;
    for (int64_t o = blockIdx.x * (int64_t)kThreads + threadIdx.x; o < old_slots; o += (int64_t)gridDim.x * kThreads) {
        const uint64_t k = old_keys[o];
        if (k == NL_HASH_EMPTY) continue;
        nl_hash_insert(keys, mask, k);
        const uint64_t s = nl_hash_slot_of(keys, mask, k);
        vals[3 * s] = old_vals[3 * o];
        vals[3 * s + 1] = old_vals[3 * o + 1];
        vals[3 * s + 2] = old_vals[3 * o + 2];
    }
}

// ------------------------------------------------------------------------------------------------ finish
// totals: confirmed, removed, unobserved, added
__global__ void __launch_bounds__(kThreads) k_classify(int64_t n, const int32_t *__restrict__ structure, const uint32_t *__restrict__ votes,
                                                       uint32_t min_votes, double ratio, uint8_t *flags, unsigned long long *totals) {
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        const bool leaf = structure[9 * i + 8] == 1;
        const uint32_t t = votes[2 * i], s = votes[2 * i + 1];
        const bool removed = leaf && t >= min_votes && (double)t >= ratio * ((double)t + (double)s);
        flags[i] = removed;
        if (removed) atomicAdd(&totals[1], 1ull);
        else if (leaf && s > 0) atomicAdd(&totals[0], 1ull);
        if (leaf && t == 0 && s == 0) atomicAdd(&totals[2], 1ull);
    }
}

__global__ void __launch_bounds__(kThreads) k_select_added(int64_t slots, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                           uint32_t min_points, uint32_t min_scans, uint64_t *out, unsigned long long *totals) {
    for (int64_t s = blockIdx.x * (int64_t)kThreads + threadIdx.x; s < slots; s += (int64_t)gridDim.x * kThreads) {
        const uint64_t k = keys[s];
        const bool sel = k != NL_HASH_EMPTY && vals[3 * s] >= min_points && vals[3 * s + 1] >= min_scans;
        out[s] = sel ? k : NL_HASH_EMPTY;
        if (sel) atomicAdd(&totals[3], 1ull);
    }
}

__global__ void __launch_bounds__(kThreads) k_gather_added(int64_t slots, const uint64_t *__restrict__ sorted, const uint64_t *__restrict__ keys,
                                                           const uint32_t *__restrict__ vals, uint64_t *added, uint32_t *added_vals) {
    const uint64_t mask = (uint64_t)slots - 1;
    for (int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x; r < slots; r += (int64_t)gridDim.x * kThreads) {
        const uint64_t k = sorted[r];
        added[r] = k;
        if (k == NL_HASH_EMPTY) {
            added_vals[2 * r] = added_vals[2 * r + 1] = 0;
            continue;
        }
        const uint64_t s = nl_hash_slot_of(keys, mask, k);
        added_vals[2 * r] = vals[3 * s];
        added_vals[2 * r + 1] = vals[3 * s + 1];
    }
}

struct FinishLayout {                                   // [flags u8[n] | sorted u64[slots] x 2 | selected count | cub temp]
    size_t flags, keys_a, keys_b, count, temp, temp_bytes, bytes;
};

cudaError_t finish_layout(int64_t n_nodes, int64_t slots, FinishLayout *L) {
    size_t sel = 0, sort = 0;
    cudaError_t e;
    if ((e = cub::DeviceSelect::Flagged(nullptr, sel, thrust::counting_iterator<int32_t>(0), (const uint8_t *)nullptr, (int32_t *)nullptr,
                                        (int32_t *)nullptr, (int)n_nodes)) != cudaSuccess)
        return e;
    cub::DoubleBuffer<uint64_t> db(nullptr, nullptr);
    if ((e = cub::DeviceRadixSort::SortKeys(nullptr, sort, db, (int)slots)) != cudaSuccess) return e;
    L->flags = 0;
    L->keys_a = align256((size_t)n_nodes);
    L->keys_b = L->keys_a + align256(8 * (size_t)slots);
    L->count = L->keys_b + align256(8 * (size_t)slots);
    L->temp = L->count + 256;
    L->temp_bytes = std::max(sel, sort);
    L->bytes = L->temp + align256(L->temp_bytes);
    return cudaSuccess;
}

int cuda_fail(const char *what, cudaError_t e) {
    char buf[256];
    std::snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
    return nl_set_error_code(NL_ERR_CUDA, buf);
}

int check_table(const char *what, int64_t slots, const void *keys, const void *vals) {
    if (!pow2(slots) || slots < 1024 || slots > (int64_t(1) << 30)) {
        char buf[160];
        std::snprintf(buf, sizeof(buf), "%s: slots must be a power of two in [2^10, 2^30], got %lld", what, (long long)slots);
        return nl_set_error(buf);
    }
    if (!keys || !vals) {
        char buf[160];
        std::snprintf(buf, sizeof(buf), "%s: null table", what);
        return nl_set_error(buf);
    }
    return NL_OK;
}

}  // namespace

extern "C" {

int nl_change_votes(int64_t cap, const nl_render_stats *d_stats, const int32_t *d_s_ray, const int32_t *d_s_vox, const float *d_s_depth,
                    const float *d_sdf, const float *d_gt, const int32_t *d_ray_offset, int64_t n_nodes, float truncation, float through_depth,
                    uint32_t *d_votes, int32_t *d_status, void *stream) {
    if (cap < 0 || n_nodes < 1) return nl_set_error("nl_change_votes: need cap >= 0 and n_nodes >= 1");
    if (!d_stats || !d_s_ray || !d_s_vox || !d_s_depth || !d_sdf || !d_gt || !d_ray_offset || !d_votes || !d_status)
        return nl_set_error("nl_change_votes: null pointer");
    if (!(truncation >= 0.0f) || !(through_depth >= truncation) || !std::isfinite(through_depth))
        return nl_set_error("nl_change_votes: need 0 <= truncation <= through_depth, both finite");
    if (cap == 0) return NL_OK;
    k_votes<<<grid_blocks(cap), kThreads, 0, (cudaStream_t)stream>>>(cap, d_stats, d_s_ray, d_s_vox, d_s_depth, d_sdf, d_gt, d_ray_offset, n_nodes,
                                                                      truncation, through_depth, d_votes, d_status);
    NL_CHECK_LAUNCH("nl_change_votes");
    return NL_OK;
}

int nl_change_rehash(int64_t old_slots, const uint64_t *d_old_keys, const uint32_t *d_old_vals, int64_t slots, uint64_t *d_keys, uint32_t *d_vals,
                     uint32_t *d_state, void *stream) {
    const char *what = "nl_change_rehash";
    int rc = check_table(what, slots, d_keys, d_vals);
    if (rc != NL_OK) return rc;
    if (old_slots < 0 || (old_slots > 0 && (!d_old_keys || !d_old_vals))) return nl_set_error("nl_change_rehash: bad old table");
    if (old_slots > slots) return nl_set_error("nl_change_rehash: the new table must not be smaller than the old one");
    if (!d_state) return nl_set_error("nl_change_rehash: null state");
    cudaStream_t s = (cudaStream_t)stream;
    k_clear<<<grid_blocks(slots), kThreads, 0, s>>>(slots, d_keys, d_vals);
    NL_CHECK_LAUNCH(what);
    if (old_slots > 0) {
        k_rehash<<<grid_blocks(old_slots), kThreads, 0, s>>>(old_slots, d_old_keys, d_old_vals, slots, d_keys, d_vals);
        NL_CHECK_LAUNCH(what);
    } else {
        cudaError_t e = cudaMemsetAsync(d_state, 0, 2 * sizeof(uint32_t), s);
        if (e != cudaSuccess) return cuda_fail(what, e);
    }
    cudaError_t e = cudaMemsetAsync(d_state + 2, 0, sizeof(uint32_t), s);
    if (e != cudaSuccess) return cuda_fail(what, e);
    return NL_OK;
}

int nl_change_added(int64_t n_points, const float *d_points, const float *d_Rt12, double voxel_size, int64_t grid_dim, const uint64_t *d_occ,
                    int64_t occ_slots, int64_t slots, uint64_t *d_keys, uint32_t *d_vals, uint32_t scan, uint32_t *d_state, void *stream) {
    const char *what = "nl_change_added";
    int rc = check_table(what, slots, d_keys, d_vals);
    if (rc != NL_OK) return rc;
    if (n_points < 0 || n_points > (int64_t(1) << 30)) return nl_set_error("nl_change_added: need 0 <= n_points <= 2^30");
    if ((n_points > 0 && !d_points) || !d_Rt12 || !d_occ || !d_state) return nl_set_error("nl_change_added: null pointer");
    if (!(voxel_size > 0.0) || !std::isfinite(voxel_size)) return nl_set_error("nl_change_added: voxel_size must be finite and > 0");
    if (!pow2(grid_dim) || grid_dim > (int64_t(1) << NL_VOXEL_AXIS_BITS))
        return nl_set_error("nl_change_added: grid_dim must be a power of two <= 2^18");
    if (!pow2(occ_slots)) return nl_set_error("nl_change_added: occ_slots must be a power of two");
    if (scan == kNoScan) return nl_set_error("nl_change_added: scan id 2^32 - 1 is reserved");
    if (n_points == 0) return NL_OK;
    cudaStream_t s = (cudaStream_t)stream;
    k_added<<<grid_blocks(n_points), kThreads, 0, s>>>(n_points, d_points, d_Rt12, voxel_size, (double)grid_dim, d_occ, (uint64_t)occ_slots - 1,
                                                       slots, d_keys, d_vals, scan, d_state);
    NL_CHECK_LAUNCH(what);
    k_commit<<<1, 1, 0, s>>>(d_state);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

int64_t nl_change_finish_workspace_bytes(int64_t n_nodes, int64_t slots) {
    if (n_nodes < 1 || n_nodes > INT32_MAX) return nl_set_error("nl_change_finish_workspace_bytes: need 1 <= n_nodes < 2^31");
    if (!pow2(slots) || slots > (int64_t(1) << 30)) return nl_set_error("nl_change_finish_workspace_bytes: slots must be a power of two <= 2^30");
    FinishLayout L;
    cudaError_t e = finish_layout(n_nodes, slots, &L);
    if (e != cudaSuccess) return cuda_fail("nl_change_finish_workspace_bytes", e);
    return (int64_t)L.bytes;
}

int nl_change_finish(int64_t n_nodes, const int32_t *d_structure, const uint32_t *d_votes, uint32_t min_votes, double ratio, int64_t slots,
                     const uint64_t *d_keys, const uint32_t *d_vals, uint32_t min_points, uint32_t min_scans, void *d_ws, int64_t ws_bytes,
                     int32_t *d_removed, uint64_t *d_added, uint32_t *d_added_vals, int64_t *d_totals, void *stream) {
    const char *what = "nl_change_finish";
    const int64_t need = nl_change_finish_workspace_bytes(n_nodes, slots);
    if (need < 0) return (int)need;
    int rc = check_table(what, slots, d_keys, d_vals);
    if (rc != NL_OK) return rc;
    if (!d_structure || !d_votes || !d_ws || !d_removed || !d_added || !d_added_vals || !d_totals) return nl_set_error("nl_change_finish: null pointer");
    if (ws_bytes < need) return nl_set_error("nl_change_finish: workspace too small");
    if (!(ratio > 0.0 && ratio <= 1.0)) return nl_set_error("nl_change_finish: ratio must lie in (0, 1]");
    if (min_votes < 1 || min_points < 1 || min_scans < 1) return nl_set_error("nl_change_finish: the counts must be >= 1");
    FinishLayout L;
    cudaError_t e = finish_layout(n_nodes, slots, &L);
    if (e != cudaSuccess) return cuda_fail(what, e);
    char *ws = (char *)d_ws;
    uint8_t *flags = (uint8_t *)(ws + L.flags);
    uint64_t *ka = (uint64_t *)(ws + L.keys_a), *kb = (uint64_t *)(ws + L.keys_b);
    int32_t *count = (int32_t *)(ws + L.count);
    void *temp = ws + L.temp;
    size_t temp_bytes = L.temp_bytes;
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long *totals = (unsigned long long *)d_totals;
    if ((e = cudaMemsetAsync(d_totals, 0, 4 * sizeof(int64_t), s)) != cudaSuccess) return cuda_fail(what, e);
    k_classify<<<grid_blocks(n_nodes), kThreads, 0, s>>>(n_nodes, d_structure, d_votes, min_votes, ratio, flags, totals);
    NL_CHECK_LAUNCH(what);
    if ((e = cub::DeviceSelect::Flagged(temp, temp_bytes, thrust::counting_iterator<int32_t>(0), flags, d_removed, count, (int)n_nodes, s)) != cudaSuccess)
        return cuda_fail(what, e);
    k_select_added<<<grid_blocks(slots), kThreads, 0, s>>>(slots, d_keys, d_vals, min_points, min_scans, ka, totals);
    NL_CHECK_LAUNCH(what);
    cub::DoubleBuffer<uint64_t> db(ka, kb);
    temp_bytes = L.temp_bytes;
    if ((e = cub::DeviceRadixSort::SortKeys(temp, temp_bytes, db, (int)slots, 0, 64, s)) != cudaSuccess) return cuda_fail(what, e);
    k_gather_added<<<grid_blocks(slots), kThreads, 0, s>>>(slots, db.Current(), d_keys, d_vals, d_added, d_added_vals);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

}  // extern "C"
