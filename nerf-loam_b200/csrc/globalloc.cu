// Global localisation, coarse stage (include/nerfloam_b200.h section 15): how many of M scan points land in an occupied map voxel,
// for every placement of a lattice of positions x headings around anchor poses, and the top n of those counts.
//
//   occupied set : the map's finest-level voxels (the rows whose side is 1: Octree.get_leaf_voxels()), keyed as overlap.cu keys
//                  them, in an open-addressing set (hash.cuh) of a power of two >= 2 x the leaf count.  The corner is
//                  floor(centre / voxel_size) in fp64: centre = (corner + 1/2) x voxel_size rounded to fp32 is within 2^-6 voxels of
//                  corner + 1/2 for corners below 2^18, so the floor is exact.
//   cells        : lattice points q = (i, j) x xy_step within `radius` (fp64 distance) of an anchor's xy, each with its nearest
//                  anchor: atomicMin on (fp32 distance bits << 32 | anchor) in a hash keyed by (i, j), so the lower anchor wins a
//                  tie and the winner does not depend on launch order.  The keys are compacted, sorted (bitonic) and numbered in
//                  ascending (i, j) order.
//   placements   : id = cell x Y + k; rotation Rz(2 pi k / Y - psi_a) R_a, translation (q_x, q_y, t_a,z), formed in fp64 and rounded to
//                  fp32 by placement_matrix(), which the scorer and nl_globalloc_matrices share.  Never stored.
//   count        : points whose voxel (voxel.cuh, overlap.cu's arithmetic) is in the occupied set; one warp per placement, the
//                  points in shared memory, the set read from global memory (L2-resident at 10^6 leaves: 32 MB).
//   selection    : the n highest counts by (count desc, id asc): a histogram of counts, the threshold count from its suffix sums,
//                  a stable compaction in id order, and a bitonic sort of the <= n selected (count, id) keys.
// Every output is an integer or a function of integers, so it depends neither on the order of the atomics nor on the launch shape.
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
constexpr int kWarps = kThreads / 32;
constexpr int kTile = 4 * kWarps;                      // placements per scorer CTA
constexpr int kScanTile = 4 * kThreads;                // placements per compaction CTA (4 per thread)
constexpr int64_t kMinSlots = 1024;
constexpr int64_t kLatticeLimit = int64_t(1) << 30;    // |i|, |j| < 2^30: the (i, j) key never equals NL_HASH_EMPTY
constexpr int64_t kMaxBound = int64_t(1) << 30;        // lattice points visited by the cell kernel (anchors x box)
constexpr int64_t kMaxIds = INT32_MAX;                 // placement ids are int32

int64_t pow2_at_least(int64_t v) {
    int64_t c = 1;
    while (c < v) c <<= 1;
    return c;
}

int64_t set_slots(int64_t n) { return std::max(kMinSlots, pow2_at_least(2 * n)); }

int cuda_fail(const char *what, cudaError_t e) {
    char buf[256];
    std::snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
    return nl_set_error_code(NL_ERR_CUDA, buf);
}

int grid_blocks(int64_t n) { return (int)std::min<int64_t>(std::max(1, nl_div_up(n, kThreads)), 16 * nl_num_sms()); }

__device__ __forceinline__ int warp_sum(int v) {
    #pragma unroll
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

// ------------------------------------------------------------------------------------------------ occupied set
__global__ void __launch_bounds__(kThreads) k_count_leaves(int64_t n, const int32_t *__restrict__ structure, unsigned long long *count) {
    int c = 0;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) c += structure[9 * i + 8] == 1;
    c = warp_sum(c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, (unsigned long long)c);
}

__global__ void __launch_bounds__(kThreads) k_occupied(int64_t n, const float *__restrict__ centres, const int32_t *__restrict__ structure,
                                                       double vs, double gd, uint64_t *set, uint64_t mask) {
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        if (structure[9 * i + 8] != 1) continue;
        uint64_t k = 0;
        bool ok = true;
        #pragma unroll
        for (int a = 0; a < 3; ++a) {
            const double v = floor((double)centres[3 * i + a] / vs);
            ok = ok && v >= 0.0 && v < gd;
            k = (k << NL_VOXEL_AXIS_BITS) | (ok ? (uint64_t)v : 0);
        }
        if (ok) nl_hash_insert(set, mask, k);
    }
}

// ------------------------------------------------------------------------------------------------ cells
__host__ __device__ __forceinline__ uint64_t cell_key(int64_t i, int64_t j) {
    return ((uint64_t)(i + kLatticeLimit) << 32) | (uint64_t)(j + kLatticeLimit);
}

// The first lattice index of an anchor's box and the box width: one index of margin beyond [x - r, x + r] on each side, so no
// lattice point within r is missed by rounding.  The same expressions on the host bound the workspace.
__host__ __device__ __forceinline__ int64_t box_first(double x, double r, double step) { return (int64_t)floor((x - r) / step) - 1; }
__host__ __device__ __forceinline__ int64_t box_width(double r, double step) { return (int64_t)ceil(2.0 * r / step) + 4; }

__global__ void __launch_bounds__(kThreads) k_cells(int32_t n_anchors, const double *__restrict__ anchors, double r, double step, int64_t W,
                                                    uint64_t *keys, unsigned long long *vals, uint64_t mask) {
    const int64_t per = W * W, total = per * n_anchors;
    for (int64_t t = blockIdx.x * (int64_t)kThreads + threadIdx.x; t < total; t += (int64_t)gridDim.x * kThreads) {
        const int32_t a = (int32_t)(t / per);
        const int64_t o = t - (int64_t)a * per;
        const double tx = anchors[12 * a + 3], ty = anchors[12 * a + 7];
        const int64_t i = box_first(tx, r, step) + o / W, j = box_first(ty, r, step) + o % W;
        const double dx = __dsub_rn(__dmul_rn((double)i, step), tx), dy = __dsub_rn(__dmul_rn((double)j, step), ty);
        const double d = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
        if (!(d <= r)) continue;
        const uint64_t s = nl_hash_insert_slot(keys, mask, cell_key(i, j));
        atomicMin(&vals[s], ((unsigned long long)__float_as_uint((float)d) << 32) | (unsigned long long)a);
    }
}

__global__ void __launch_bounds__(kThreads) k_compact_keys(int64_t slots, const uint64_t *__restrict__ keys, uint64_t *list,
                                                           unsigned long long *count) {
    for (int64_t s = blockIdx.x * (int64_t)kThreads + threadIdx.x; s < slots; s += (int64_t)gridDim.x * kThreads) {
        const uint64_t k = keys[s];
        if (k != NL_HASH_EMPTY) list[atomicAdd(count, 1ull)] = k;
    }
}

__global__ void __launch_bounds__(kThreads) k_fill(int64_t n, uint64_t *p, uint64_t v) {
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) p[i] = v;
}

// One compare-exchange pass of a bitonic sort of n (a power of two) keys, ascending.
__global__ void __launch_bounds__(kThreads) k_bitonic(int64_t n, uint64_t *v, int64_t j, int64_t k) {
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        const int64_t l = i ^ j;
        if (l <= i) continue;
        const uint64_t a = v[i], b = v[l];
        if (((i & k) == 0) ? (a > b) : (a < b)) {
            v[i] = b;
            v[l] = a;
        }
    }
}

int bitonic_sort(int64_t n, uint64_t *v, cudaStream_t s, const char *what) {
    for (int64_t k = 2; k <= n; k <<= 1)
        for (int64_t j = k >> 1; j > 0; j >>= 1) {
            k_bitonic<<<grid_blocks(n), kThreads, 0, s>>>(n, v, j, k);
            NL_CHECK_LAUNCH(what);
        }
    return NL_OK;
}

__global__ void __launch_bounds__(kThreads) k_cell_table(int64_t n, const uint64_t *__restrict__ list, const uint64_t *__restrict__ keys,
                                                         const unsigned long long *__restrict__ vals, uint64_t mask, int32_t *cells) {
    for (int64_t c = blockIdx.x * (int64_t)kThreads + threadIdx.x; c < n; c += (int64_t)gridDim.x * kThreads) {
        const uint64_t k = list[c];
        cells[3 * c] = (int32_t)((int64_t)(k >> 32) - kLatticeLimit);
        cells[3 * c + 1] = (int32_t)((int64_t)(k & 0xffffffffu) - kLatticeLimit);
        cells[3 * c + 2] = (int32_t)(vals[nl_hash_slot_of(keys, mask, k)] & 0xffffffffu);
    }
}

// ------------------------------------------------------------------------------------------------ placements
// The fp32 matrix of placement `id` (R row-major, then t).
__device__ __forceinline__ void placement_matrix(int64_t id, const int32_t *__restrict__ cells, const double *__restrict__ anchors, int Y,
                                                 double step, float (&Rt)[12]) {
    const int64_t c = id / Y;
    const int k = (int)(id - c * Y);
    const int32_t ci = cells[3 * c], cj = cells[3 * c + 1], a = cells[3 * c + 2];
    const double *A = anchors + 12 * (int64_t)a;
    const double psi = atan2(A[4], A[0]);
    double sn, cs;
    sincos(2.0 * M_PI * (double)k / (double)Y - psi, &sn, &cs);
    #pragma unroll
    for (int col = 0; col < 3; ++col) {
        Rt[col] = (float)(cs * A[col] - sn * A[4 + col]);
        Rt[3 + col] = (float)(sn * A[col] + cs * A[4 + col]);
        Rt[6 + col] = (float)A[8 + col];
    }
    Rt[9] = (float)((double)ci * step);
    Rt[10] = (float)((double)cj * step);
    Rt[11] = (float)A[11];
}

// An id outside [0, n_placements) gets a NaN matrix instead of reading past the cell table.
__global__ void __launch_bounds__(kThreads) k_matrices(int64_t n, const int64_t *__restrict__ ids, int64_t n_placements,
                                                       const int32_t *__restrict__ cells, const double *__restrict__ anchors, int Y, double step,
                                                       float *out) {
    for (int64_t t = blockIdx.x * (int64_t)kThreads + threadIdx.x; t < n; t += (int64_t)gridDim.x * kThreads) {
        float Rt[12];
        const int64_t id = ids[t];
        if (id >= 0 && id < n_placements) {
            placement_matrix(id, cells, anchors, Y, step, Rt);
        } else {
            #pragma unroll
            for (int e = 0; e < 12; ++e) Rt[e] = __int_as_float(0x7fc00000);
        }
        #pragma unroll
        for (int e = 0; e < 12; ++e) out[12 * t + e] = Rt[e];
    }
}

// One warp per placement: the lanes stride over the points in shared memory and the warp sums its hits.
__global__ void __launch_bounds__(kThreads) k_score(int64_t p0, int64_t n, const int32_t *__restrict__ cells, const double *__restrict__ anchors,
                                                    int Y, double step, int M, const float *__restrict__ pts, const uint64_t *__restrict__ set,
                                                    uint64_t mask, double vs, double gd, int32_t *counts) {
    extern __shared__ float sp[];
    for (int e = threadIdx.x; e < 3 * M; e += kThreads) sp[e] = pts[e];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int t = warp; t < kTile; t += kWarps) {
        const int64_t h = p0 + blockIdx.x * (int64_t)kTile + t;
        if (h >= p0 + n) break;
        float Rt[12];
        placement_matrix(h, cells, anchors, Y, step, Rt);
        int hits = 0;
        for (int m = lane; m < M; m += 32) {
            uint64_t key;
            if (nl_voxel_key(Rt, sp[3 * m], sp[3 * m + 1], sp[3 * m + 2], vs, gd, key)) hits += nl_hash_contains(set, mask, key);
        }
        hits = warp_sum(hits);
        if (lane == 0) counts[h] = hits;
    }
}

// ------------------------------------------------------------------------------------------------ selection
// A count outside [0, M] (a caller's M smaller than the scorer's) is never selected and never indexes the histogram.
__device__ __forceinline__ int valid_count(int32_t c, int M) { return (c >= 0 && c <= M) ? c : -1; }

__global__ void __launch_bounds__(kThreads) k_hist(int64_t n, const int32_t *__restrict__ counts, int M, unsigned int *hist) {
    extern __shared__ unsigned int sh[];
    for (int c = threadIdx.x; c <= M; c += kThreads) sh[c] = 0;
    __syncthreads();
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        const int c = valid_count(counts[i], M);
        if (c >= 0) atomicAdd(&sh[c], 1u);
    }
    __syncthreads();
    for (int c = threadIdx.x; c <= M; c += kThreads)
        if (sh[c]) atomicAdd(&hist[c], sh[c]);
}

// thr[0] = T, the count of the n_select-th placement by count; thr[1] = how many placements of count T are selected.
__global__ void k_threshold(const unsigned int *__restrict__ hist, int M, int64_t n_select, int64_t *thr) {
    extern __shared__ unsigned int sh[];
    for (int c = threadIdx.x; c <= M; c += blockDim.x) sh[c] = hist[c];
    __syncthreads();
    if (threadIdx.x != 0) return;
    int64_t above = 0;
    int T = 0;
    for (int c = M; c >= 0; --c) {
        T = c;
        if (above + sh[c] >= n_select) break;
        above += sh[c];
    }
    thr[0] = T;
    thr[1] = n_select - above;
}

__device__ __forceinline__ void tile_flags(const int32_t *__restrict__ counts, int64_t n, int M, int64_t b, const int64_t *__restrict__ thr,
                                           int (&gt)[4], int (&eq)[4], int32_t (&cnt)[4]) {
    const int T = (int)thr[0];
    #pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int64_t h = b * kScanTile + 4 * threadIdx.x + u;
        cnt[u] = h < n ? valid_count(counts[h], M) : -1;
        gt[u] = cnt[u] > T;
        eq[u] = cnt[u] == T;
    }
}

// Exclusive block scan of one int per thread (kThreads threads); returns the block total in *total.
__device__ __forceinline__ int block_scan(int v, int *sh, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
    #pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, s);
        if (lane >= s) x += y;
    }
    if (lane == 31) sh[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = lane < kWarps ? sh[lane] : 0;
        #pragma unroll
        for (int s = 1; s < kWarps; s <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, s);
            if (lane >= s) w += y;
        }
        if (lane < kWarps) sh[kWarps + lane] = w;
    }
    __syncthreads();
    const int before = (warp ? sh[kWarps + warp - 1] : 0) + x - v;
    *total = sh[2 * kWarps - 1];
    __syncthreads();
    return before;
}

__global__ void __launch_bounds__(kThreads) k_tile_counts(int64_t n, const int32_t *__restrict__ counts, int M, const int64_t *__restrict__ thr,
                                                          int64_t *tile_gt, int64_t *tile_eq) {
    __shared__ int sh[2 * kWarps];
    int gt[4], eq[4];
    int32_t cnt[4];
    tile_flags(counts, n, M, blockIdx.x, thr, gt, eq, cnt);
    int tg, te;
    block_scan(gt[0] + gt[1] + gt[2] + gt[3], sh, &tg);
    block_scan(eq[0] + eq[1] + eq[2] + eq[3], sh, &te);
    if (threadIdx.x == 0) {
        tile_gt[blockIdx.x] = tg;
        tile_eq[blockIdx.x] = te;
    }
}

// Exclusive scan of both tile arrays in place, one block, in chunks of kThreads.
__global__ void __launch_bounds__(kThreads) k_tile_scan(int64_t n_tiles, int64_t *tile_gt, int64_t *tile_eq) {
    __shared__ int64_t sh[2 * kThreads];
    int64_t carry_g = 0, carry_e = 0;
    for (int64_t base = 0; base < n_tiles; base += kThreads) {
        const int64_t i = base + threadIdx.x;
        const int64_t g = i < n_tiles ? tile_gt[i] : 0, e = i < n_tiles ? tile_eq[i] : 0;
        sh[threadIdx.x] = g;
        sh[kThreads + threadIdx.x] = e;
        __syncthreads();
        for (int s = 1; s < kThreads; s <<= 1) {      // inclusive Hillis-Steele scan
            const int64_t pg = threadIdx.x >= s ? sh[threadIdx.x - s] : 0, pe = threadIdx.x >= s ? sh[kThreads + threadIdx.x - s] : 0;
            __syncthreads();
            sh[threadIdx.x] += pg;
            sh[kThreads + threadIdx.x] += pe;
            __syncthreads();
        }
        if (i < n_tiles) {
            tile_gt[i] = carry_g + sh[threadIdx.x] - g;
            tile_eq[i] = carry_e + sh[kThreads + threadIdx.x] - e;
        }
        carry_g += sh[kThreads - 1];
        carry_e += sh[2 * kThreads - 1];
        __syncthreads();
    }
}

// Selected placements in id order: every count > T, and the first thr[1] of count T.  Key = (M - count) << 32 | id.
__global__ void __launch_bounds__(kThreads) k_compact_selected(int64_t n, const int32_t *__restrict__ counts, int M, const int64_t *__restrict__ thr,
                                                               const int64_t *__restrict__ off_gt, const int64_t *__restrict__ off_eq, uint64_t *out) {
    __shared__ int sh[2 * kWarps];
    int gt[4], eq[4];
    int32_t cnt[4];
    tile_flags(counts, n, M, blockIdx.x, thr, gt, eq, cnt);
    int tg, te;
    int bg = block_scan(gt[0] + gt[1] + gt[2] + gt[3], sh, &tg);
    int be = block_scan(eq[0] + eq[1] + eq[2] + eq[3], sh, &te);
    const int64_t need = thr[1];
    int64_t g = off_gt[blockIdx.x] + bg, e = off_eq[blockIdx.x] + be;
    #pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int64_t h = blockIdx.x * (int64_t)kScanTile + 4 * threadIdx.x + u;
        if (gt[u] || (eq[u] && e < need)) out[g + (e < need ? e : need)] = ((uint64_t)(M - cnt[u]) << 32) | (uint64_t)h;
        g += gt[u];
        e += eq[u];
    }
}

__global__ void __launch_bounds__(kThreads) k_unpack(int64_t n, const uint64_t *__restrict__ keys, int M, int32_t *ids, int32_t *counts) {
    for (int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x; r < n; r += (int64_t)gridDim.x * kThreads) {
        const uint64_t k = keys[r];
        ids[r] = k == NL_HASH_EMPTY ? -1 : (int32_t)(k & 0xffffffffu);        // fewer than n valid counts: the rest are -1
        counts[r] = k == NL_HASH_EMPTY ? -1 : M - (int32_t)(k >> 32);
    }
}

// ------------------------------------------------------------------------------------------------ host-side checks
int check_lattice(const char *fn, int32_t n_anchors, const double *h_anchors, double radius, double xy_step, int64_t *bound) {
    char buf[224];
    if (n_anchors < 1) { std::snprintf(buf, sizeof(buf), "%s: need at least one anchor", fn); return nl_set_error(buf); }
    if (!h_anchors) { std::snprintf(buf, sizeof(buf), "%s: null anchors", fn); return nl_set_error(buf); }
    if (!std::isfinite(radius) || radius < 0.0) { std::snprintf(buf, sizeof(buf), "%s: radius must be finite and >= 0", fn); return nl_set_error(buf); }
    if (!std::isfinite(xy_step) || !(xy_step > 0.0)) { std::snprintf(buf, sizeof(buf), "%s: xy_step must be finite and > 0", fn); return nl_set_error(buf); }
    for (int64_t e = 0; e < 12 * (int64_t)n_anchors; ++e)
        if (!std::isfinite(h_anchors[e])) {
            std::snprintf(buf, sizeof(buf), "%s: anchor %lld is not finite", fn, (long long)(e / 12));
            return nl_set_error(buf);
        }
    const double w = std::ceil(2.0 * radius / xy_step) + 4.0;
    if (w * w * (double)n_anchors > (double)kMaxBound) {
        std::snprintf(buf, sizeof(buf), "%s: %d anchors x (%.0f lattice points)^2 exceed 2^30 lattice points; raise xy_step or lower radius", fn,
                      (int)n_anchors, w);
        return nl_set_error(buf);
    }
    for (int32_t a = 0; a < n_anchors; ++a)
        for (int c = 0; c < 2; ++c) {
            const double lo = std::floor((h_anchors[12 * a + 3 + 4 * c] - radius) / xy_step) - 1.0;
            if (!(std::fabs(lo) < (double)kLatticeLimit - 2.0 * w)) {
                std::snprintf(buf, sizeof(buf), "%s: anchor %d lies beyond 2^30 lattice steps of the origin", fn, (int)a);
                return nl_set_error(buf);
            }
        }
    *bound = (int64_t)w * (int64_t)w * n_anchors;
    return NL_OK;
}

struct CellsLayout {
    int64_t slots, list;
    int64_t bytes() const { return 8 * (2 * slots + list) + 256; }
};

CellsLayout cells_layout(int64_t bound) { return {set_slots(bound), pow2_at_least(std::max<int64_t>(bound, 1))}; }

struct SelectLayout {
    int64_t hist, tiles, keys;    // hist u32[M+1] (rounded to 8 B), thr i64[2], tile_gt / tile_eq i64[tiles], keys u64[pow2 >= n_select]
    int64_t bytes() const { return 4 * hist + 16 + 16 * tiles + 8 * keys; }
};

SelectLayout select_layout(int64_t n, int M, int64_t n_select) {
    return {(int64_t)(M + 2) & ~int64_t(1), std::max<int64_t>(1, (n + kScanTile - 1) / kScanTile), pow2_at_least(std::max<int64_t>(n_select, 1))};
}

int check_placements(const char *fn, int64_t n_cells, int Y) {
    char buf[192];
    if (Y < 1) { std::snprintf(buf, sizeof(buf), "%s: yaw_steps must be >= 1", fn); return nl_set_error(buf); }
    if (n_cells < 1) { std::snprintf(buf, sizeof(buf), "%s: no cells (no lattice point within radius of an anchor)", fn); return nl_set_error(buf); }
    if (n_cells > kMaxIds / Y) {
        std::snprintf(buf, sizeof(buf), "%s: %lld cells x %d yaws exceed the 2^31 - 1 placement ids", fn, (long long)n_cells, Y);
        return nl_set_error(buf);
    }
    return NL_OK;
}

}  // namespace

extern "C" {

void nl_abi_sizes_globalloc(int32_t out[2]) {
    out[0] = NL_GLOBALLOC_MAX_POINTS;
    out[1] = 3;
}

int nl_globalloc_count_leaves(int64_t n_nodes, const int32_t *d_structure, int64_t *d_n_leaves, void *stream) {
    const char *what = "nl_globalloc_count_leaves";
    if (n_nodes < 1) return nl_set_error("nl_globalloc_count_leaves: the map is empty");
    if (!d_structure || !d_n_leaves) return nl_set_error("nl_globalloc_count_leaves: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e;
    if ((e = cudaMemsetAsync(d_n_leaves, 0, 8, s)) != cudaSuccess) return cuda_fail(what, e);
    k_count_leaves<<<grid_blocks(n_nodes), kThreads, 0, s>>>(n_nodes, d_structure, (unsigned long long *)d_n_leaves);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

int64_t nl_globalloc_occupied_slots(int64_t n_leaves) {
    if (n_leaves < 1) return nl_set_error("nl_globalloc_occupied_slots: the map has no leaf voxels");
    if (n_leaves > (int64_t(1) << 31)) return nl_set_error("nl_globalloc_occupied_slots: more than 2^31 leaf voxels");
    return set_slots(n_leaves);
}

int nl_globalloc_occupied(int64_t n_nodes, const float *d_centres, const int32_t *d_structure, double voxel_size, int64_t grid_dim,
                          int64_t slots, uint64_t *d_set, void *stream) {
    const char *what = "nl_globalloc_occupied";
    if (n_nodes < 1) return nl_set_error("nl_globalloc_occupied: the map is empty");
    if (!d_centres || !d_structure || !d_set) return nl_set_error("nl_globalloc_occupied: null pointer");
    if (!(voxel_size > 0.0) || !std::isfinite(voxel_size)) return nl_set_error("nl_globalloc_occupied: voxel_size must be finite and > 0");
    if (grid_dim < 1 || (grid_dim & (grid_dim - 1)) || grid_dim > (int64_t(1) << NL_VOXEL_AXIS_BITS))
        return nl_set_error("nl_globalloc_occupied: grid_dim must be a power of two <= 2^18");
    if (slots < kMinSlots || (slots & (slots - 1))) return nl_set_error("nl_globalloc_occupied: slots must be a power of two >= 2^10");
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e;
    if ((e = cudaMemsetAsync(d_set, 0xff, 8 * (size_t)slots, s)) != cudaSuccess) return cuda_fail(what, e);   // NL_HASH_EMPTY
    k_occupied<<<grid_blocks(n_nodes), kThreads, 0, s>>>(n_nodes, d_centres, d_structure, voxel_size, (double)grid_dim, d_set, (uint64_t)slots - 1);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

int64_t nl_globalloc_cells_workspace_bytes(int32_t n_anchors, const double *h_anchors, double radius, double xy_step) {
    int64_t bound = 0;
    const int rc = check_lattice("nl_globalloc_cells_workspace_bytes", n_anchors, h_anchors, radius, xy_step, &bound);
    if (rc != NL_OK) return rc;
    return cells_layout(bound).bytes();
}

int nl_globalloc_cells(int32_t n_anchors, const double *h_anchors, const double *d_anchors, double radius, double xy_step, void *d_ws,
                       int64_t ws_bytes, int64_t *d_n_cells, void *stream) {
    const char *what = "nl_globalloc_cells";
    int64_t bound = 0;
    const int rc = check_lattice(what, n_anchors, h_anchors, radius, xy_step, &bound);
    if (rc != NL_OK) return rc;
    if (!d_anchors || !d_ws || !d_n_cells) return nl_set_error("nl_globalloc_cells: null pointer");
    const CellsLayout L = cells_layout(bound);
    if (ws_bytes < L.bytes()) return nl_set_error("nl_globalloc_cells: workspace smaller than nl_globalloc_cells_workspace_bytes");
    if (((uintptr_t)d_ws & 255u) != 0) return nl_set_error("nl_globalloc_cells: the workspace must be 256-byte aligned");
    uint64_t *keys = static_cast<uint64_t *>(d_ws), *vals = keys + L.slots, *list = vals + L.slots;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e;
    if ((e = cudaMemsetAsync(keys, 0xff, 16 * (size_t)L.slots, s)) != cudaSuccess) return cuda_fail(what, e);   // empty keys, +inf values
    if ((e = cudaMemsetAsync(d_n_cells, 0, 8, s)) != cudaSuccess) return cuda_fail(what, e);
    k_cells<<<grid_blocks(bound), kThreads, 0, s>>>(n_anchors, d_anchors, radius, xy_step, box_width(radius, xy_step), keys,
                                                    (unsigned long long *)vals, (uint64_t)L.slots - 1);
    NL_CHECK_LAUNCH(what);
    k_compact_keys<<<grid_blocks(L.slots), kThreads, 0, s>>>(L.slots, keys, list, (unsigned long long *)d_n_cells);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

int nl_globalloc_cells_finish(int32_t n_anchors, const double *h_anchors, double radius, double xy_step, int64_t n_cells, void *d_ws,
                              int64_t ws_bytes, int32_t *d_cells, void *stream) {
    const char *what = "nl_globalloc_cells_finish";
    int64_t bound = 0;
    const int rc = check_lattice(what, n_anchors, h_anchors, radius, xy_step, &bound);
    if (rc != NL_OK) return rc;
    if (n_cells < 1 || n_cells > std::min(bound, kMaxIds))
        return nl_set_error("nl_globalloc_cells_finish: n_cells must be nl_globalloc_cells' count (>= 1 and < 2^31)");
    if (!d_ws || !d_cells) return nl_set_error("nl_globalloc_cells_finish: null pointer");
    const CellsLayout L = cells_layout(bound);
    if (ws_bytes < L.bytes()) return nl_set_error("nl_globalloc_cells_finish: workspace smaller than nl_globalloc_cells_workspace_bytes");
    uint64_t *keys = static_cast<uint64_t *>(d_ws), *vals = keys + L.slots, *list = vals + L.slots;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t P = pow2_at_least(n_cells);
    if (P > n_cells) {
        k_fill<<<grid_blocks(P - n_cells), kThreads, 0, s>>>(P - n_cells, list + n_cells, NL_HASH_EMPTY);
        NL_CHECK_LAUNCH(what);
    }
    if (bitonic_sort(P, list, s, what) != NL_OK) return NL_ERR_CUDA;
    k_cell_table<<<grid_blocks(n_cells), kThreads, 0, s>>>(n_cells, list, keys, (const unsigned long long *)vals, (uint64_t)L.slots - 1, d_cells);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

int nl_globalloc_matrices(int64_t n, const int64_t *d_ids, int64_t n_cells, const int32_t *d_cells, const double *d_anchors, int32_t yaw_steps,
                          double xy_step, float *d_Rt12, void *stream) {
    const char *what = "nl_globalloc_matrices";
    const int rc = check_placements(what, n_cells, yaw_steps);
    if (rc != NL_OK) return rc;
    if (n < 0) return nl_set_error("nl_globalloc_matrices: n must not be negative");
    if (!std::isfinite(xy_step) || !(xy_step > 0.0)) return nl_set_error("nl_globalloc_matrices: xy_step must be finite and > 0");
    if (n == 0) return NL_OK;
    if (!d_ids || !d_cells || !d_anchors || !d_Rt12) return nl_set_error("nl_globalloc_matrices: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    k_matrices<<<grid_blocks(n), kThreads, 0, s>>>(n, d_ids, n_cells * yaw_steps, d_cells, d_anchors, yaw_steps, xy_step, d_Rt12);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

int nl_globalloc_score(int64_t p0, int64_t n, int64_t n_cells, const int32_t *d_cells, const double *d_anchors, int32_t yaw_steps, double xy_step,
                       int32_t n_points, const float *d_points, const uint64_t *d_set, int64_t slots, double voxel_size, int64_t grid_dim,
                       int32_t *d_counts, void *stream) {
    const char *what = "nl_globalloc_score";
    const int rc = check_placements(what, n_cells, yaw_steps);
    if (rc != NL_OK) return rc;
    if (n_points < 1 || n_points > NL_GLOBALLOC_MAX_POINTS) return nl_set_error("nl_globalloc_score: n_points must be in [1, NL_GLOBALLOC_MAX_POINTS]");
    if (p0 < 0 || n < 0 || p0 + n > n_cells * yaw_steps) return nl_set_error("nl_globalloc_score: [p0, p0 + n) must lie within the placements");
    if (!std::isfinite(xy_step) || !(xy_step > 0.0)) return nl_set_error("nl_globalloc_score: xy_step must be finite and > 0");
    if (!(voxel_size > 0.0) || !std::isfinite(voxel_size)) return nl_set_error("nl_globalloc_score: voxel_size must be finite and > 0");
    if (grid_dim < 1 || (grid_dim & (grid_dim - 1)) || grid_dim > (int64_t(1) << NL_VOXEL_AXIS_BITS))
        return nl_set_error("nl_globalloc_score: grid_dim must be a power of two <= 2^18");
    if (slots < kMinSlots || (slots & (slots - 1))) return nl_set_error("nl_globalloc_score: slots must be a power of two >= 2^10");
    if (!d_cells || !d_anchors || !d_points || !d_set || !d_counts) return nl_set_error("nl_globalloc_score: null pointer");
    if (n == 0) return NL_OK;
    static NlPerDevice once;
    const size_t smem = 12 * (size_t)NL_GLOBALLOC_MAX_POINTS;
    cudaError_t e = once.once([&] { return cudaFuncSetAttribute(k_score, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); });
    if (e != cudaSuccess) return cuda_fail(what, e);
    cudaStream_t s = (cudaStream_t)stream;
    for (int64_t q = 0; q < n;) {                           // grid.x <= 2^31 - 1 CTAs per launch
        const int64_t m = std::min<int64_t>(n - q, (int64_t)kTile * 0x7fffffff);
        k_score<<<(unsigned)((m + kTile - 1) / kTile), kThreads, 12 * (size_t)n_points, s>>>(p0 + q, m, d_cells, d_anchors, yaw_steps, xy_step, n_points,
                                                                                           d_points, d_set, (uint64_t)slots - 1, voxel_size,
                                                                                           (double)grid_dim, d_counts);
        NL_CHECK_LAUNCH(what);
        q += m;
    }
    return NL_OK;
}

int64_t nl_globalloc_select_workspace_bytes(int64_t n_placements, int32_t n_points, int64_t n_select) {
    if (n_placements < 1 || n_placements > kMaxIds) return nl_set_error("nl_globalloc_select_workspace_bytes: n_placements must be in [1, 2^31)");
    if (n_points < 1 || n_points > NL_GLOBALLOC_MAX_POINTS)
        return nl_set_error("nl_globalloc_select_workspace_bytes: n_points must be in [1, NL_GLOBALLOC_MAX_POINTS]");
    if (n_select < 1 || n_select > n_placements) return nl_set_error("nl_globalloc_select_workspace_bytes: n_select must be in [1, n_placements]");
    return select_layout(n_placements, n_points, n_select).bytes();
}

int nl_globalloc_select(int64_t n_placements, const int32_t *d_counts, int32_t n_points, int64_t n_select, void *d_ws, int64_t ws_bytes,
                        int32_t *d_ids, int32_t *d_sel_counts, void *stream) {
    const char *what = "nl_globalloc_select";
    const int64_t need_bytes = nl_globalloc_select_workspace_bytes(n_placements, n_points, n_select);
    if (need_bytes < 0) return (int)need_bytes;
    if (!d_counts || !d_ws || !d_ids || !d_sel_counts) return nl_set_error("nl_globalloc_select: null pointer");
    if (ws_bytes < need_bytes) return nl_set_error("nl_globalloc_select: workspace smaller than nl_globalloc_select_workspace_bytes");
    if (((uintptr_t)d_ws & 255u) != 0) return nl_set_error("nl_globalloc_select: the workspace must be 256-byte aligned");
    const SelectLayout L = select_layout(n_placements, n_points, n_select);
    unsigned int *hist = static_cast<unsigned int *>(d_ws);
    int64_t *thr = reinterpret_cast<int64_t *>(hist + L.hist), *tile_gt = thr + 2, *tile_eq = tile_gt + L.tiles;
    uint64_t *keys = reinterpret_cast<uint64_t *>(tile_eq + L.tiles);
    const int M = n_points;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e;
    if ((e = cudaMemsetAsync(hist, 0, 4 * (size_t)L.hist, s)) != cudaSuccess) return cuda_fail(what, e);
    k_hist<<<grid_blocks(n_placements), kThreads, 4 * (size_t)(M + 1), s>>>(n_placements, d_counts, M, hist);
    NL_CHECK_LAUNCH(what);
    k_threshold<<<1, 1024, 4 * (size_t)(M + 1), s>>>(hist, M, n_select, thr);
    NL_CHECK_LAUNCH(what);
    k_tile_counts<<<(unsigned)L.tiles, kThreads, 0, s>>>(n_placements, d_counts, M, thr, tile_gt, tile_eq);
    NL_CHECK_LAUNCH(what);
    k_tile_scan<<<1, kThreads, 0, s>>>(L.tiles, tile_gt, tile_eq);
    NL_CHECK_LAUNCH(what);
    k_fill<<<grid_blocks(L.keys), kThreads, 0, s>>>(L.keys, keys, NL_HASH_EMPTY);     // slots no valid count reaches sort last
    NL_CHECK_LAUNCH(what);
    k_compact_selected<<<(unsigned)L.tiles, kThreads, 0, s>>>(n_placements, d_counts, M, thr, tile_gt, tile_eq, keys);
    NL_CHECK_LAUNCH(what);
    if (bitonic_sort(L.keys, keys, s, what) != NL_OK) return NL_ERR_CUDA;
    k_unpack<<<grid_blocks(n_select), kThreads, 0, s>>>(n_select, keys, M, d_ids, d_sel_counts);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

}  // extern "C"
