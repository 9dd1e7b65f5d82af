// Voxel overlap of one scan with K keyframes (include/nerfloam_b200.h section 12): the counts behind the mapper's 'overlap'
// keyframe window (src/mapping.py:205-225 declares that method and leaves it unimplemented).
//
//   world point : w_i = ((R_i0 x + R_i1 y) + R_i2 z) + t_i in fp64 from the fp32 matrix and point (voxel.cuh, shared with
//                 globalloc.cu).
//   voxel       : floor(w / voxel_size) in fp64 per axis; a point whose voxel leaves [0, grid_dim)^3 (or is not finite) is not
//                 counted.  Key = vx << 36 | vy << 18 | vz (grid_dim <= 2^18, so 54 bits).
//   frame set   : every point of the scan goes into an open-addressing set (capacity a power of two >= 2N); a first insertion
//                 is one voxel of V_c.
//   keyframes   : split on the host, from the host-side point counts, into chunks of <= 1023 keyframes whose points fill at most
//                 half of the keyframe table.  Per chunk the table is cleared and one launch walks the chunk (grid.y = keyframe)
//                 through the device table of point pointers and counts, so the keyframes are never concatenated.  Every point
//                 inserts (chunk-local keyframe << 54) | key; a first insertion is one voxel of V_k, and one of V_k n V_c when
//                 the key is in the frame set.  The local index stays <= 1022, so no composite key equals NL_HASH_EMPTY (~0).
//   duplicates  : a point whose voxel equals that of the point before it (the lane before it in the warp) skips the table.
//                 Consecutive returns of a scan line mostly share a voxel, so this saves most of the atomics and changes no
//                 count: the earlier point has put the key in the set.
// Every output is an integer count, so it depends neither on the order of the atomics nor on the launch shape.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>

#include "../../include/nerfloam_b200.h"
#include "hash.cuh"
#include "nl_cuda.cuh"
#include "voxel.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kAxisBits = NL_VOXEL_AXIS_BITS;
constexpr int kKfShift = 3 * kAxisBits;                  // composite key: keyframe << 54 | voxel key
constexpr int kMaxChunk = NL_OVERLAP_MAX_CHUNK;          // keyframes per chunk: local index <= 1022 in the top 10 bits
constexpr int64_t kMinSlots = 1024;
constexpr int64_t kMaxPoints = INT32_MAX;

int64_t pow2_at_least(int64_t v) {
    int64_t c = 1;
    while (c < v) c <<= 1;
    return c;
}

int64_t frame_slots(int64_t n) { return std::max(kMinSlots, pow2_at_least(2 * n)); }

bool is_pow2(int64_t v) { return v > 0 && (v & (v - 1)) == 0; }

__device__ __forceinline__ void load_rt(const float *__restrict__ row, float (&Rt)[12]) {
    #pragma unroll
    for (int i = 0; i < 12; ++i) Rt[i] = row[i];
}

__device__ __forceinline__ int64_t warp_sum(int64_t v) {
    #pragma unroll
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

// Is this lane's key the same as the previous lane's (both valid)?  Then the previous point inserts it.
__device__ __forceinline__ bool repeats_previous(bool ok, uint64_t key) {
    const int lane = threadIdx.x & 31;
    const uint64_t prev = __shfl_up_sync(0xffffffffu, key, 1);
    const int prev_ok = __shfl_up_sync(0xffffffffu, (int)ok, 1);
    return lane > 0 && ok && prev_ok && prev == key;
}

// The loops below step a whole warp over 32 consecutive points (the trip count is warp-uniform), so the shuffles see every lane.
__global__ void __launch_bounds__(kThreads) k_frame_set(int64_t n, const float *__restrict__ p, const float *__restrict__ Rt12, double vs,
                                                        double gd, uint64_t *set, uint64_t mask, int64_t *n_voxels) {
    float Rt[12];
    load_rt(Rt12, Rt);
    const int lane = threadIdx.x & 31;
    int64_t added = 0;
    for (int64_t base = blockIdx.x * (int64_t)kThreads + (threadIdx.x & ~31); base < n; base += (int64_t)gridDim.x * kThreads) {
        const int64_t i = base + lane;
        uint64_t key = 0;
        const bool ok = i < n && nl_voxel_key(Rt, p[3 * i], p[3 * i + 1], p[3 * i + 2], vs, gd, key);
        const bool dup = repeats_previous(ok, key);
        if (ok && !dup && nl_hash_insert(set, mask, key)) ++added;
    }
    added = warp_sum(added);
    if (lane == 0 && added) atomicAdd((unsigned long long *)n_voxels, (unsigned long long)added);
}

__global__ void __launch_bounds__(kThreads) k_keyframes(int k0, const float *const *__restrict__ pts, const int64_t *__restrict__ cnt,
                                                        const float *__restrict__ Rt12, double vs, double gd, const uint64_t *__restrict__ fset,
                                                        uint64_t fmask, uint64_t *set, uint64_t mask, int64_t *shared, int64_t *kf_voxels,
                                                        int64_t *outside) {
    const int local = blockIdx.y;
    const int k = k0 + local;
    const int64_t n = cnt[k];
    const float *__restrict__ p = pts[k];
    float Rt[12];
    load_rt(Rt12 + 12 * (1 + k), Rt);
    const int lane = threadIdx.x & 31;
    const uint64_t tag = (uint64_t)local << kKfShift;
    int64_t added = 0, common = 0, out = 0;
    for (int64_t base = blockIdx.x * (int64_t)kThreads + (threadIdx.x & ~31); base < n; base += (int64_t)gridDim.x * kThreads) {
        const int64_t i = base + lane;
        uint64_t key = 0;
        const bool ok = i < n && nl_voxel_key(Rt, p[3 * i], p[3 * i + 1], p[3 * i + 2], vs, gd, key);
        out += (i < n && !ok);
        const bool dup = repeats_previous(ok, key);
        if (ok && !dup && nl_hash_insert(set, mask, tag | key)) {
            ++added;
            common += nl_hash_contains(fset, fmask, key);
        }
    }
    added = warp_sum(added);
    common = warp_sum(common);
    out = warp_sum(out);
    if (lane == 0) {
        if (added) atomicAdd((unsigned long long *)&kf_voxels[k], (unsigned long long)added);
        if (common) atomicAdd((unsigned long long *)&shared[k], (unsigned long long)common);
        if (out) atomicAdd((unsigned long long *)&outside[k], (unsigned long long)out);
    }
}

int cuda_fail(const char *what, cudaError_t e) {
    char buf[256];
    std::snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
    return nl_set_error_code(NL_ERR_CUDA, buf);
}

int grid_blocks(int64_t n) { return (int)std::min<int64_t>(std::max(1, nl_div_up(n, 4 * kThreads)), 8 * nl_num_sms()); }

}  // namespace

extern "C" {

int64_t nl_keyframe_overlap_workspace_bytes(int64_t n_frame, int64_t table_slots) {
    if (n_frame < 0 || n_frame > kMaxPoints) return nl_set_error("nl_keyframe_overlap_workspace_bytes: n_frame must be in [0, 2^31)");
    if (!is_pow2(table_slots) || table_slots < kMinSlots || table_slots > NL_OVERLAP_MAX_SLOTS)
        return nl_set_error("nl_keyframe_overlap_workspace_bytes: table_slots must be a power of two in [2^10, 2^32]");
    return 8 * (frame_slots(n_frame) + table_slots);
}

int nl_keyframe_overlap(int64_t n_frame, const float *d_frame_pts, int32_t n_kf, const float *const *d_kf_pts, const int64_t *d_kf_n,
                        const int64_t *h_kf_n, const float *d_Rt12, double voxel_size, int64_t grid_dim, int64_t table_slots, void *d_ws,
                        int64_t ws_bytes, int64_t *d_out, void *stream) {
    const char *what = "nl_keyframe_overlap";
    if (n_frame < 0 || n_frame > kMaxPoints) return nl_set_error("nl_keyframe_overlap: n_frame must be in [0, 2^31)");
    if (n_kf < 0) return nl_set_error("nl_keyframe_overlap: n_kf must not be negative");
    if (!is_pow2(grid_dim) || grid_dim > (int64_t(1) << kAxisBits))
        return nl_set_error("nl_keyframe_overlap: grid_dim must be a power of two <= 2^18");
    if (!(voxel_size > 0.0) || !std::isfinite(voxel_size)) return nl_set_error("nl_keyframe_overlap: voxel_size must be finite and > 0");
    if (!is_pow2(table_slots) || table_slots < kMinSlots || table_slots > NL_OVERLAP_MAX_SLOTS)
        return nl_set_error("nl_keyframe_overlap: table_slots must be a power of two in [2^10, 2^32]");
    if (!d_Rt12 || !d_ws || !d_out || (n_frame > 0 && !d_frame_pts) || (n_kf > 0 && (!d_kf_pts || !d_kf_n || !h_kf_n)))
        return nl_set_error("nl_keyframe_overlap: null pointer");
    for (int32_t k = 0; k < n_kf; ++k) {
        if (h_kf_n[k] < 0) return nl_set_error("nl_keyframe_overlap: negative keyframe point count");
        if (h_kf_n[k] > table_slots / 2) {
            char buf[192];
            std::snprintf(buf, sizeof(buf), "nl_keyframe_overlap: keyframe %d has %lld points, a table of %lld slots holds at most %lld", (int)k,
                          (long long)h_kf_n[k], (long long)table_slots, (long long)(table_slots / 2));
            return nl_set_error(buf);
        }
    }
    const int64_t fslots = frame_slots(n_frame);
    if (ws_bytes < 8 * (fslots + table_slots)) return nl_set_error("nl_keyframe_overlap: workspace smaller than nl_keyframe_overlap_workspace_bytes");
    if (((uintptr_t)d_ws & 255u) != 0) return nl_set_error("nl_keyframe_overlap: the workspace must be 256-byte aligned");

    cudaStream_t s = (cudaStream_t)stream;
    uint64_t *fset = static_cast<uint64_t *>(d_ws);
    uint64_t *table = fset + fslots;
    int64_t *shared = d_out, *kf_voxels = d_out + n_kf, *outside = d_out + 2 * (int64_t)n_kf, *frame_voxels = d_out + 3 * (int64_t)n_kf;
    const double gd = (double)grid_dim;
    cudaError_t e;
    if ((e = cudaMemsetAsync(d_out, 0, 8 * (3 * (size_t)n_kf + 1), s)) != cudaSuccess) return cuda_fail(what, e);
    if ((e = cudaMemsetAsync(fset, 0xff, 8 * (size_t)fslots, s)) != cudaSuccess) return cuda_fail(what, e);   // NL_HASH_EMPTY
    if (n_frame > 0) {
        k_frame_set<<<grid_blocks(n_frame), kThreads, 0, s>>>(n_frame, d_frame_pts, d_Rt12, voxel_size, gd, fset, (uint64_t)fslots - 1,
                                                              frame_voxels);
        NL_CHECK_LAUNCH(what);
    }
    for (int32_t k0 = 0; k0 < n_kf;) {
        int64_t total = 0, largest = 0;
        int32_t k1 = k0;
        while (k1 < n_kf && k1 - k0 < kMaxChunk && total + h_kf_n[k1] <= table_slots / 2) {
            total += h_kf_n[k1];
            largest = std::max(largest, h_kf_n[k1]);
            ++k1;
        }
        if (total > 0) {
            const int64_t slots = std::min(table_slots, std::max(kMinSlots, pow2_at_least(2 * total)));
            if ((e = cudaMemsetAsync(table, 0xff, 8 * (size_t)slots, s)) != cudaSuccess) return cuda_fail(what, e);
            const dim3 grid(grid_blocks(largest), k1 - k0);
            k_keyframes<<<grid, kThreads, 0, s>>>(k0, d_kf_pts, d_kf_n, d_Rt12, voxel_size, gd, fset, (uint64_t)fslots - 1, table,
                                                  (uint64_t)slots - 1, shared, kf_voxels, outside);
            NL_CHECK_LAUNCH(what);
        }
        k0 = k1;
    }
    return NL_OK;
}

}  // extern "C"
