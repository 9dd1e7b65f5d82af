// Reconstruction evaluation on the GPU: a mesh against a reference point cloud (include/nerfloam_b200.h section 11).
//
// The reference's README evaluates maps with an external script (a KD-tree over the mesh samples and the ground truth, on the
// host).  Here every step stays on the device:
//
//   surface sampling : fp64 triangle areas -> fixed-tile fp64 inclusive prefix sum (cub::BlockReduce / BlockScan; the tile
//                      size is a constant, so the bits depend on neither the launch shape nor the device) -> one thread per
//                      sample: Philox4x32-10 keyed on the seed, counter = sample index; inverse CDF over the prefix sum picks
//                      the triangle (a zero-area triangle's CDF step is empty, so it is never picked), the square-root
//                      barycentric formula the point.
//   down-sampling    : 3 x 21-bit voxel keys computed in fp64 (points outside an optional crop box get a sentinel key that
//                      sorts last) -> stable radix sort -> run heads -> scan -> one thread per voxel sums its points in fp64
//                      in sorted order and writes the centroid.  Output is in key order.
//   nearest distance : the target is sorted by cell key (cell size chosen by the caller from the data), each occupied cell's
//                      run goes into an open-addressing hash table, and each query walks Chebyshev rings of cells around its
//                      own cell.  After ring k every unvisited target point is at least k*h away, so the walk stops as soon
//                      as the best distance is <= k*h or k*h >= truncation: the search is exact below the truncation.
//   metric sums      : fixed-tile fp64 block reductions, then one block over the tile partials in order.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>

#include "../../include/nerfloam_b200.h"
#include "hash.cuh"
#include "nl_cuda.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kItems = 8;
constexpr int kTile = kThreads * kItems;           // fixed: the fp64 sums' order depends on it and on nothing else
constexpr int kKeyBits = 21;                       // per axis; NL_EVAL_KEY_BITS
constexpr int64_t kKeyDim = int64_t(1) << kKeyBits;
constexpr uint64_t kSentinel = uint64_t(1) << 63;  // cropped point: sorts after every real key (3 x 21 = 63 bits)
constexpr int64_t kMaxN = INT32_MAX;

size_t take(size_t &at, size_t bytes) {
    const size_t o = (at + 255) & ~size_t(255);
    at = o + bytes;
    return o;
}

template <class T>
T *at(void *ws, size_t off) { return reinterpret_cast<T *>(static_cast<char *>(ws) + off); }
template <class T>
const T *at(const void *ws, size_t off) { return reinterpret_cast<const T *>(static_cast<const char *>(ws) + off); }

int cuda_fail(const char *what, cudaError_t e) {
    char buf[256];
    std::snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
    return nl_set_error_code(NL_ERR_CUDA, buf);
}

int short_ws(const char *what, int64_t have, size_t need) {
    char buf[192];
    std::snprintf(buf, sizeof(buf), "%s: workspace of %lld bytes, the matching *_workspace_bytes call asks for %lld", what, (long long)have,
                  (long long)need);
    return nl_set_error(buf);
}

int check_ws(const char *what, const void *ws, int64_t have, size_t need) {
    if (have < (int64_t)need) return short_ws(what, have, need);
    if (((uintptr_t)ws & 255u) != 0) return nl_set_error("nl_eval: the workspace must be 256-byte aligned");
    return NL_OK;
}

// ---- counter-based generator: Philox4x32-10 (Salmon et al., SC'11) --------------------------------------------------------
__device__ __forceinline__ uint4 philox(uint4 c, uint2 k) {
    #pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}

// floor((x - o) / h) in fp64; false when it is outside [0, 2^21)
__device__ __forceinline__ bool axis_key(float x, double o, double h, uint64_t &k) {
    const double v = floor(((double)x - o) / h);
    if (!(v >= 0.0 && v < (double)kKeyDim)) return false;
    k = (uint64_t)v;
    return true;
}

__device__ __forceinline__ uint64_t pack_key(uint64_t kx, uint64_t ky, uint64_t kz) { return (kx << (2 * kKeyBits)) | (ky << kKeyBits) | kz; }

// ---- bounds and finiteness ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ord_of(float f) {        // order-preserving float -> uint32
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_of(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }

__global__ void k_bounds_init(uint32_t *b, int64_t *nonfinite) {
    if (threadIdx.x < 6) b[threadIdx.x] = threadIdx.x < 3 ? 0xffffffffu : 0u;
    if (threadIdx.x == 0) *nonfinite = 0;
}

__global__ void k_bounds(int64_t n, const float *__restrict__ p, uint32_t *b, int64_t *nonfinite) {
    uint32_t lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};
    int bad = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
        if (!(isfinite(x) && isfinite(y) && isfinite(z))) { ++bad; continue; }
        const uint32_t o[3] = {ord_of(x), ord_of(y), ord_of(z)};
        #pragma unroll
        for (int a = 0; a < 3; ++a) { lo[a] = min(lo[a], o[a]); hi[a] = max(hi[a], o[a]); }
    }
    #pragma unroll
    for (int a = 0; a < 3; ++a)
        #pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            lo[a] = min(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], s));
            hi[a] = max(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], s));
        }
    #pragma unroll
    for (int s = 16; s > 0; s >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, s);
    if ((threadIdx.x & 31) == 0) {
        #pragma unroll
        for (int a = 0; a < 3; ++a) { atomicMin(&b[a], lo[a]); atomicMax(&b[3 + a], hi[a]); }
        if (bad) atomicAdd((unsigned long long *)nonfinite, (unsigned long long)bad);
    }
}

__global__ void k_bounds_final(uint32_t *b) {          // in place: encoded -> float (an all-non-finite input leaves +-inf)
    if (threadIdx.x < 6) {
        const uint32_t o = b[threadIdx.x];
        float f;
        if (threadIdx.x < 3 && o == 0xffffffffu) f = INFINITY;
        else if (threadIdx.x >= 3 && o == 0u) f = -INFINITY;
        else f = float_of(o);
        reinterpret_cast<float *>(b)[threadIdx.x] = f;
    }
}

// ---- fixed-order fp64 sums ------------------------------------------------------------------------------------------------
using BlockScanD = cub::BlockScan<double, kThreads>;
using BlockReduceD = cub::BlockReduce<double, kThreads>;

__device__ __forceinline__ double tri_area(const float *__restrict__ v, const int32_t *__restrict__ f, int64_t t, int64_t nv, int &bad) {
    const int32_t a = f[3 * t], b = f[3 * t + 1], c = f[3 * t + 2];
    if (a < 0 || b < 0 || c < 0 || a >= nv || b >= nv || c >= nv) { bad = 1; return 0.0; }
    const double ax = v[3 * a], ay = v[3 * a + 1], az = v[3 * a + 2];
    const double ux = v[3 * b] - ax, uy = v[3 * b + 1] - ay, uz = v[3 * b + 2] - az;
    const double wx = v[3 * c] - ax, wy = v[3 * c + 1] - ay, wz = v[3 * c + 2] - az;
    const double cx = uy * wz - uz * wy, cy = uz * wx - ux * wz, cz = ux * wy - uy * wx;
    const double s = 0.5 * sqrt(cx * cx + cy * cy + cz * cz);
    return isfinite(s) ? s : 0.0;
}

// per tile: the areas (kept for the scan) and their block sum
__global__ void __launch_bounds__(kThreads) k_area_tiles(int64_t nv, const float *__restrict__ v, int64_t nt, const int32_t *__restrict__ f,
                                                        double *area, double *tile_sum, double *info) {
    __shared__ typename BlockReduceD::TempStorage tmp;
    const int64_t base = (int64_t)blockIdx.x * kTile;
    double s[kItems];
    int bad = 0;
    #pragma unroll
    for (int j = 0; j < kItems; ++j) {
        const int64_t t = base + threadIdx.x * kItems + j;            // blocked arrangement: thread-local items are consecutive
        s[j] = t < nt ? tri_area(v, f, t, nv, bad) : 0.0;
        if (t < nt) area[t] = s[j];
    }
    double loc = 0.0;
    #pragma unroll
    for (int j = 0; j < kItems; ++j) loc += s[j];
    const double tot = BlockReduceD(tmp).Sum(loc);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = tot;
    if (bad) atomicAdd(&info[1], 1.0);                                // count of threads that saw a bad index: only "> 0" is used
}

// one block: exclusive prefix of the tile sums in tile order; info[0] = total
__global__ void __launch_bounds__(kThreads) k_tile_prefix(int64_t n_tiles, double *tile_sum, double *info) {
    __shared__ typename BlockScanD::TempStorage tmp;
    double run = 0.0;
    for (int64_t b0 = 0; b0 < n_tiles; b0 += kThreads) {
        const int64_t b = b0 + threadIdx.x;
        const double x = b < n_tiles ? tile_sum[b] : 0.0;
        double ex, agg;
        BlockScanD(tmp).ExclusiveSum(x, ex, agg);
        __syncthreads();
        if (b < n_tiles) tile_sum[b] = run + ex;
        run += agg;
    }
    if (threadIdx.x == 0) info[0] = run;
}

__global__ void __launch_bounds__(kThreads) k_area_scan(int64_t nt, const double *__restrict__ area, const double *__restrict__ tile_off,
                                                       double *cdf) {
    __shared__ typename BlockScanD::TempStorage tmp;
    const int64_t base = (int64_t)blockIdx.x * kTile;
    double s[kItems];
    #pragma unroll
    for (int j = 0; j < kItems; ++j) {
        const int64_t t = base + threadIdx.x * kItems + j;
        s[j] = t < nt ? area[t] : 0.0;
    }
    BlockScanD(tmp).InclusiveSum(s, s);
    const double off = tile_off[blockIdx.x];
    #pragma unroll
    for (int j = 0; j < kItems; ++j) {
        const int64_t t = base + threadIdx.x * kItems + j;
        if (t < nt) cdf[t] = off + s[j];
    }
}

__global__ void k_sample(int64_t nt, const float *__restrict__ v, const int32_t *__restrict__ f, const double *__restrict__ cdf, int64_t ns,
                         uint64_t seed, float *out, int32_t *out_face) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= ns) return;
    const uint4 r = philox(make_uint4((uint32_t)i, (uint32_t)(i >> 32), 0u, 0u), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const double u0 = (double)(((uint64_t)r.x << 21) | (r.y >> 11)) * 0x1.0p-53;    // [0, 1)
    const double u1 = ((double)r.z + 0.5) * 0x1.0p-32, u2 = ((double)r.w + 0.5) * 0x1.0p-32;
    const double total = cdf[nt - 1];
    const double tgt = u0 * total;
    // first t with cdf[t] > tgt: its area is > 0 (cdf[t-1] <= tgt < cdf[t]); u0 * total rounding up to total falls back to the
    // last triangle of positive area
    int64_t lo = 0, hi = nt;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (cdf[mid] > tgt) hi = mid; else lo = mid + 1;
    }
    if (lo == nt) {
        lo = nt - 1;
        while (lo > 0 && cdf[lo - 1] == total) --lo;
    }
    const int32_t a = f[3 * lo], b = f[3 * lo + 1], c = f[3 * lo + 2];
    const double s1 = sqrt(u1);
    const double wa = 1.0 - s1, wb = s1 * (1.0 - u2), wc = s1 * u2;
    #pragma unroll
    for (int k = 0; k < 3; ++k) out[3 * i + k] = (float)(wa * (double)v[3 * a + k] + wb * (double)v[3 * b + k] + wc * (double)v[3 * c + k]);
    if (out_face) out_face[i] = (int32_t)lo;
}

// ---- sort by key, run heads, run starts -----------------------------------------------------------------------------------
struct SortLayout {
    size_t ka = 0, kb = 0, va = 0, vb = 0, flag = 0, rid = 0, start = 0, tmp = 0, tmp_bytes = 0, total = 0;
};

cudaError_t sort_layout(int64_t n, size_t &at_, SortLayout &l) {
    l.ka = take(at_, 8 * (size_t)n); l.kb = take(at_, 8 * (size_t)n);
    l.va = take(at_, 4 * (size_t)n); l.vb = take(at_, 4 * (size_t)n);
    l.flag = take(at_, 4 * (size_t)(n + 1)); l.rid = take(at_, 4 * (size_t)(n + 1)); l.start = take(at_, 4 * (size_t)(n + 1));
    size_t a = 0, b = 0;
    cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    cudaError_t e;
    if ((e = cub::DeviceRadixSort::SortPairs(nullptr, a, k, v, (int)n, 0, 64)) != cudaSuccess) return e;
    if ((e = cub::DeviceScan::ExclusiveSum(nullptr, b, (const int32_t *)nullptr, (int32_t *)nullptr, (int)(n + 1))) != cudaSuccess) return e;
    l.tmp_bytes = std::max(a, b);
    l.tmp = take(at_, l.tmp_bytes);
    return cudaSuccess;
}

__global__ void k_heads(int n, const uint64_t *__restrict__ key, int32_t *flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    flag[i] = (i < n && key[i] != kSentinel && (i == 0 || key[i] != key[i - 1])) ? 1 : 0;
}

// start[rid[i]] = i for every head; start[n_runs] = number of non-sentinel keys (they sort first)
__global__ void k_starts(int n, const uint64_t *__restrict__ key, const int32_t *__restrict__ flag, const int32_t *__restrict__ rid,
                         int32_t *start) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (flag[i]) start[rid[i]] = i;
    const bool last_real = key[i] != kSentinel && (i == n - 1 || key[i + 1] == kSentinel);
    if (last_real) start[rid[n]] = i + 1;
}

// sorts (key, index) pairs held in l.ka / l.va; afterwards the sorted arrays are at *ks / *vs, rid (n + 1) and start (runs + 1)
int sort_runs(const char *what, int n, void *ws, const SortLayout &l, cudaStream_t s, const uint64_t **ks, const uint32_t **vs) {
    cub::DoubleBuffer<uint64_t> dk(at<uint64_t>(ws, l.ka), at<uint64_t>(ws, l.kb));
    cub::DoubleBuffer<uint32_t> dv(at<uint32_t>(ws, l.va), at<uint32_t>(ws, l.vb));
    size_t tb = l.tmp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(at<void>(ws, l.tmp), tb, dk, dv, n, 0, 64, s);     // LSD radix: stable
    if (e != cudaSuccess) return cuda_fail(what, e);
    int32_t *flag = at<int32_t>(ws, l.flag), *rid = at<int32_t>(ws, l.rid), *start = at<int32_t>(ws, l.start);
    k_heads<<<nl_div_up(n + 1, kThreads), kThreads, 0, s>>>(n, dk.Current(), flag);
    NL_CHECK_LAUNCH(what);
    tb = l.tmp_bytes;
    if ((e = cub::DeviceScan::ExclusiveSum(at<void>(ws, l.tmp), tb, flag, rid, n + 1, s)) != cudaSuccess) return cuda_fail(what, e);
    cudaMemsetAsync(start, 0, 4, s);                                  // no real key at all: start[0] = 0
    k_starts<<<nl_div_up(n, kThreads), kThreads, 0, s>>>(n, dk.Current(), flag, rid, start);
    NL_CHECK_LAUNCH(what);
    *ks = dk.Current();
    *vs = dv.Current();
    return NL_OK;
}

// ---- voxel down-sampling --------------------------------------------------------------------------------------------------
// the crop box is padded in fp64, like the origin (min - res), so a kept row never falls below the origin
__device__ __forceinline__ bool in_box(float x, const float *__restrict__ c, int a, double pad) {
    return (double)x >= (double)c[a] - pad && (double)x <= (double)c[3 + a] + pad;
}

__global__ void k_voxel_keys(int n, const float *__restrict__ p, double ox, double oy, double oz, double res, const float *__restrict__ crop,
                             uint64_t *key, uint32_t *val, int64_t *counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
    val[i] = (uint32_t)i;
    if (crop && !(in_box(x, crop, 0, res) && in_box(y, crop, 1, res) && in_box(z, crop, 2, res))) {
        key[i] = kSentinel;
        atomicAdd((unsigned long long *)&counts[0], 1ull);
        return;
    }
    uint64_t kx, ky, kz;
    if (!(axis_key(x, ox, res, kx) & axis_key(y, oy, res, ky) & axis_key(z, oz, res, kz))) {
        key[i] = kSentinel;
        atomicAdd((unsigned long long *)&counts[1], 1ull);
        return;
    }
    key[i] = pack_key(kx, ky, kz);
}

__global__ void k_centroids(int n, const float *__restrict__ p, const uint64_t *__restrict__ key, const uint32_t *__restrict__ idx,
                            const int32_t *__restrict__ rid, const int32_t *__restrict__ start, float *out, uint64_t *out_key,
                            int64_t *counts) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    const int n_runs = rid[n];
    if (r == 0) counts[2] = n_runs;
    if (r >= n_runs) return;
    const int b = start[r], e = start[r + 1];
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (int j = b; j < e; ++j) {                                      // fixed order: the stable sort's
        const uint32_t i = idx[j];
        sx += (double)p[3 * i]; sy += (double)p[3 * i + 1]; sz += (double)p[3 * i + 2];
    }
    const double c = (double)(e - b);
    out[3 * r] = (float)(sx / c); out[3 * r + 1] = (float)(sy / c); out[3 * r + 2] = (float)(sz / c);
    if (out_key) out_key[r] = key[b];
}

// ---- nearest distances ----------------------------------------------------------------------------------------------------
struct NnLayout {
    SortLayout s;
    size_t pts = 0, hkey = 0, hrun = 0, total = 0;
    int64_t cap = 0;
};

cudaError_t nn_layout(int64_t n, NnLayout &l) {
    size_t a = 0;
    l.cap = 1;
    while (l.cap < 2 * n) l.cap <<= 1;                                 // load factor <= 1/2 (cells <= points)
    l.pts = take(a, 16 * (size_t)n);
    l.hkey = take(a, 8 * (size_t)l.cap);
    l.hrun = take(a, 4 * (size_t)l.cap);
    const cudaError_t e = sort_layout(n, a, l.s);
    l.total = a;
    return e;
}

__global__ void k_cell_keys(int n, const float *__restrict__ p, double ox, double oy, double oz, double h, uint64_t *key, uint32_t *val,
                            int64_t *bad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t kx, ky, kz;
    val[i] = (uint32_t)i;
    if (!(axis_key(p[3 * i], ox, h, kx) & axis_key(p[3 * i + 1], oy, h, ky) & axis_key(p[3 * i + 2], oz, h, kz))) {
        key[i] = kSentinel;                                            // cannot happen when h covers the bounds; counted, never searched
        atomicAdd((unsigned long long *)bad, 1ull);
        return;
    }
    key[i] = pack_key(kx, ky, kz);
}

__global__ void k_hash_clear(int64_t cap, uint64_t *hkey) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x) hkey[i] = NL_HASH_EMPTY;
}

__global__ void k_hash_build(int n, const float *__restrict__ p, const uint64_t *__restrict__ key, const uint32_t *__restrict__ idx,
                             const int32_t *__restrict__ flag, const int32_t *__restrict__ rid, float4 *pts, uint64_t *hkey, int32_t *hrun,
                             uint64_t mask) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t j = idx[i];
    pts[i] = make_float4(p[3 * j], p[3 * j + 1], p[3 * j + 2], 0.f);
    if (!flag[i]) return;
    const uint64_t k = key[i];
    for (uint64_t s = nl_hash_mix(k) & mask;; s = (s + 1) & mask) {
        const unsigned long long prev = atomicCAS((unsigned long long *)&hkey[s], (unsigned long long)NL_HASH_EMPTY, (unsigned long long)k);
        if (prev == NL_HASH_EMPTY) { hrun[s] = rid[i]; return; }
    }
}

__device__ __forceinline__ int hash_find(const uint64_t *__restrict__ hkey, const int32_t *__restrict__ hrun, uint64_t mask, uint64_t k) {
    for (uint64_t s = nl_hash_mix(k) & mask;; s = (s + 1) & mask) {
        const uint64_t h = hkey[s];
        if (h == k) return hrun[s];
        if (h == NL_HASH_EMPTY) return -1;
    }
}

__device__ __forceinline__ int64_t query_cell(float x, double o, double h) {
    double v = floor(((double)x - o) / h);
    v = fmin(fmax(v, -1.0e12), 1.0e12);                               // far away: every ring cell is outside the key range
    return (int64_t)v;
}

__global__ void __launch_bounds__(kThreads) k_nn_query(int nq, const float *__restrict__ q, const float4 *__restrict__ pts,
                                                      const int32_t *__restrict__ start, const uint64_t *__restrict__ hkey,
                                                      const int32_t *__restrict__ hrun, uint64_t mask, double ox, double oy, double oz,
                                                      double h, int max_ring, float truncation, float *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const float x = q[3 * i], y = q[3 * i + 1], z = q[3 * i + 2];
    const int64_t cx = query_cell(x, ox, h), cy = query_cell(y, oy, h), cz = query_cell(z, oz, h);
    float best2 = INFINITY;
    for (int k = 0; k <= max_ring; ++k) {
        for (int dx = -k; dx <= k; ++dx) {
            const int64_t gx = cx + dx;
            if (gx < 0 || gx >= kKeyDim) continue;
            for (int dy = -k; dy <= k; ++dy) {
                const int64_t gy = cy + dy;
                if (gy < 0 || gy >= kKeyDim) continue;
                const bool shell = (dx == -k || dx == k || dy == -k || dy == k);
                const int step = shell ? 1 : (k > 0 ? 2 * k : 1);      // inside the shell's x/y faces only the two z caps belong to ring k
                for (int dz = -k; dz <= k; dz += step) {
                    const int64_t gz = cz + dz;
                    if (gz < 0 || gz >= kKeyDim) continue;
                    const int r = hash_find(hkey, hrun, mask, pack_key((uint64_t)gx, (uint64_t)gy, (uint64_t)gz));
                    if (r < 0) continue;
                    const int e = start[r + 1];
                    for (int j = start[r]; j < e; ++j) {
                        const float4 t = pts[j];
                        const float ddx = x - t.x, ddy = y - t.y, ddz = z - t.z;
                        best2 = fminf(best2, ddx * ddx + ddy * ddy + ddz * ddz);
                    }
                }
            }
        }
        // every point outside rings 0..k is at least k*h from the query
        const double reach = (double)k * h;
        if ((double)sqrtf(best2) <= reach || reach >= (double)truncation) break;
    }
    out[i] = fminf(sqrtf(best2), truncation);
}

// ---- distance sums --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) k_sum_tiles(int64_t n, const float *__restrict__ d, float thr, double *part) {
    __shared__ typename BlockReduceD::TempStorage tmp;
    const int64_t base = (int64_t)blockIdx.x * kTile;
    double s1 = 0.0, s2 = 0.0, c = 0.0;
    #pragma unroll
    for (int j = 0; j < kItems; ++j) {
        const int64_t t = base + threadIdx.x * kItems + j;
        if (t < n) {
            const double x = d[t];
            s1 += x; s2 += x * x; c += d[t] < thr ? 1.0 : 0.0;
        }
    }
    s1 = BlockReduceD(tmp).Sum(s1);
    __syncthreads();
    s2 = BlockReduceD(tmp).Sum(s2);
    __syncthreads();
    c = BlockReduceD(tmp).Sum(c);
    if (threadIdx.x == 0) { part[3 * blockIdx.x] = s1; part[3 * blockIdx.x + 1] = s2; part[3 * blockIdx.x + 2] = c; }
}

__global__ void __launch_bounds__(kThreads) k_sum_final(int64_t n_tiles, const double *__restrict__ part, double *out) {
    __shared__ typename BlockReduceD::TempStorage tmp;
    double run[3] = {0.0, 0.0, 0.0};
    for (int64_t b0 = 0; b0 < n_tiles; b0 += kThreads) {
        const int64_t b = b0 + threadIdx.x;
        #pragma unroll
        for (int k = 0; k < 3; ++k) {
            const double x = b < n_tiles ? part[3 * b + k] : 0.0;
            const double t = BlockReduceD(tmp).Sum(x);
            __syncthreads();
            if (threadIdx.x == 0) run[k] += t;
        }
    }
    if (threadIdx.x == 0) { out[0] = run[0]; out[1] = run[1]; out[2] = run[2]; }
}

struct SurfaceLayout {
    size_t area = 0, cdf = 0, tile = 0, total = 0;
};

void surface_layout(int64_t nt, SurfaceLayout &l) {
    size_t a = 0;
    l.area = take(a, 8 * (size_t)nt);
    l.cdf = take(a, 8 * (size_t)nt);
    l.tile = take(a, 8 * (size_t)nl_div_up(nt, kTile));
    l.total = a;
}

bool key_origin_ok(double ox, double oy, double oz, double h) {
    return std::isfinite(ox) && std::isfinite(oy) && std::isfinite(oz) && std::isfinite(h) && h > 0.0;
}

}  // namespace

extern "C" {

void nl_abi_sizes_eval(int32_t out[2]) {
    out[0] = kKeyBits;
    out[1] = kTile;
}

int nl_eval_bounds(int64_t n, const float *d_pts, float *d_bounds, int64_t *d_nonfinite, void *stream) {
    if (n < 0 || n > kMaxN) return nl_set_error("nl_eval_bounds: n must be in [0, 2^31)");
    if (!d_bounds || !d_nonfinite || (n > 0 && !d_pts)) return nl_set_error("nl_eval_bounds: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    uint32_t *b = reinterpret_cast<uint32_t *>(d_bounds);
    k_bounds_init<<<1, 32, 0, s>>>(b, d_nonfinite);
    NL_CHECK_LAUNCH("nl_eval_bounds");
    if (n > 0) {
        k_bounds<<<std::min(nl_div_up(n, kThreads), 4 * nl_num_sms()), kThreads, 0, s>>>(n, d_pts, b, d_nonfinite);
        NL_CHECK_LAUNCH("nl_eval_bounds");
    }
    k_bounds_final<<<1, 32, 0, s>>>(b);
    NL_CHECK_LAUNCH("nl_eval_bounds");
    return NL_OK;
}

int64_t nl_eval_surface_workspace_bytes(int64_t n_faces) {
    if (n_faces < 1 || n_faces > kMaxN) return nl_set_error("nl_eval_surface_workspace_bytes: n_faces must be in [1, 2^31)");
    SurfaceLayout l;
    surface_layout(n_faces, l);
    return (int64_t)l.total;
}

int nl_eval_surface_prepare(int64_t n_verts, const float *d_verts, int64_t n_faces, const int32_t *d_faces, void *d_ws, int64_t ws_bytes,
                            double *d_info, void *stream) {
    const char *what = "nl_eval_surface_prepare";
    if (n_verts < 1 || n_verts > kMaxN || n_faces < 1 || n_faces > kMaxN) return nl_set_error("nl_eval_surface_prepare: bad n_verts or n_faces");
    if (!d_verts || !d_faces || !d_ws || !d_info) return nl_set_error("nl_eval_surface_prepare: null pointer");
    SurfaceLayout l;
    surface_layout(n_faces, l);
    if (int rc = check_ws(what, d_ws, ws_bytes, l.total)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const int tiles = nl_div_up(n_faces, kTile);
    cudaError_t e = cudaMemsetAsync(d_info, 0, 2 * sizeof(double), s);
    if (e != cudaSuccess) return cuda_fail(what, e);
    k_area_tiles<<<tiles, kThreads, 0, s>>>(n_verts, d_verts, n_faces, d_faces, at<double>(d_ws, l.area), at<double>(d_ws, l.tile), d_info);
    NL_CHECK_LAUNCH(what);
    k_tile_prefix<<<1, kThreads, 0, s>>>(tiles, at<double>(d_ws, l.tile), d_info);
    NL_CHECK_LAUNCH(what);
    k_area_scan<<<tiles, kThreads, 0, s>>>(n_faces, at<double>(d_ws, l.area), at<double>(d_ws, l.tile), at<double>(d_ws, l.cdf));
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

int nl_eval_sample_surface(int64_t n_verts, const float *d_verts, int64_t n_faces, const int32_t *d_faces, int64_t n_samples, uint64_t seed,
                           const void *d_ws, int64_t ws_bytes, float *d_out, int32_t *d_face, void *stream) {
    const char *what = "nl_eval_sample_surface";
    if (n_verts < 1 || n_verts > kMaxN || n_faces < 1 || n_faces > kMaxN) return nl_set_error("nl_eval_sample_surface: bad n_verts or n_faces");
    if (n_samples < 0 || n_samples > kMaxN) return nl_set_error("nl_eval_sample_surface: n_samples must be in [0, 2^31)");
    if (!d_verts || !d_faces || !d_ws || (n_samples > 0 && !d_out)) return nl_set_error("nl_eval_sample_surface: null pointer");
    SurfaceLayout l;
    surface_layout(n_faces, l);
    if (int rc = check_ws(what, d_ws, ws_bytes, l.total)) return rc;
    if (n_samples == 0) return NL_OK;
    k_sample<<<nl_div_up(n_samples, kThreads), kThreads, 0, (cudaStream_t)stream>>>(n_faces, d_verts, d_faces, at<double>(d_ws, l.cdf),
                                                                                    n_samples, seed, d_out, d_face);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

int64_t nl_eval_voxel_workspace_bytes(int64_t n_points) {
    if (n_points < 1 || n_points >= kMaxN) return nl_set_error("nl_eval_voxel_workspace_bytes: n_points must be in [1, 2^31 - 1)");
    SortLayout l;
    size_t a = 0;
    const cudaError_t e = sort_layout(n_points, a, l);
    if (e != cudaSuccess) return cuda_fail("nl_eval_voxel_workspace_bytes", e);
    return (int64_t)a;
}

int nl_eval_voxel_down_sample(int64_t n, const float *d_pts, double ox, double oy, double oz, double res, const float *d_crop, void *d_ws,
                              int64_t ws_bytes, float *d_out, uint64_t *d_keys, int64_t *d_counts, void *stream) {
    const char *what = "nl_eval_voxel_down_sample";
    if (n < 1 || n >= kMaxN) return nl_set_error("nl_eval_voxel_down_sample: n must be in [1, 2^31 - 1)");
    if (!key_origin_ok(ox, oy, oz, res)) return nl_set_error("nl_eval_voxel_down_sample: origin must be finite and res finite and > 0");
    if (!d_pts || !d_ws || !d_out || !d_counts) return nl_set_error("nl_eval_voxel_down_sample: null pointer");
    SortLayout l;
    size_t a = 0;
    cudaError_t e = sort_layout(n, a, l);
    if (e != cudaSuccess) return cuda_fail(what, e);
    if (int rc = check_ws(what, d_ws, ws_bytes, a)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    if ((e = cudaMemsetAsync(d_counts, 0, 3 * sizeof(int64_t), s)) != cudaSuccess) return cuda_fail(what, e);
    k_voxel_keys<<<nl_div_up(n, kThreads), kThreads, 0, s>>>((int)n, d_pts, ox, oy, oz, res, d_crop, at<uint64_t>(d_ws, l.ka),
                                                             at<uint32_t>(d_ws, l.va), d_counts);
    NL_CHECK_LAUNCH(what);
    const uint64_t *ks;
    const uint32_t *vs;
    if (int rc = sort_runs(what, (int)n, d_ws, l, s, &ks, &vs)) return rc;
    k_centroids<<<nl_div_up(n, kThreads), kThreads, 0, s>>>((int)n, d_pts, ks, vs, at<int32_t>(d_ws, l.rid), at<int32_t>(d_ws, l.start), d_out,
                                                            d_keys, d_counts);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

int64_t nl_eval_nn_workspace_bytes(int64_t n_target) {
    if (n_target < 1 || n_target >= kMaxN) return nl_set_error("nl_eval_nn_workspace_bytes: n_target must be in [1, 2^31 - 1)");
    NnLayout l;
    const cudaError_t e = nn_layout(n_target, l);
    if (e != cudaSuccess) return cuda_fail("nl_eval_nn_workspace_bytes", e);
    return (int64_t)l.total;
}

int nl_eval_nearest(int64_t n_query, const float *d_query, int64_t n_target, const float *d_target, double ox, double oy, double oz, double cell,
                    int32_t max_ring, float truncation, void *d_ws, int64_t ws_bytes, float *d_dist, int64_t *d_bad, void *stream) {
    const char *what = "nl_eval_nearest";
    if (n_query < 0 || n_query > kMaxN || n_target < 1 || n_target >= kMaxN) return nl_set_error("nl_eval_nearest: bad n_query or n_target");
    if (!key_origin_ok(ox, oy, oz, cell)) return nl_set_error("nl_eval_nearest: origin must be finite and cell finite and > 0");
    if (!(truncation > 0.f) || !std::isfinite(truncation)) return nl_set_error("nl_eval_nearest: truncation must be finite and > 0");
    if (max_ring < 0 || max_ring > 64 || (double)max_ring * cell < (double)truncation)
        return nl_set_error("nl_eval_nearest: max_ring must be in [0, 64] with max_ring * cell >= truncation");
    if (!d_target || !d_ws || !d_bad || (n_query > 0 && (!d_query || !d_dist))) return nl_set_error("nl_eval_nearest: null pointer");
    NnLayout l;
    cudaError_t e = nn_layout(n_target, l);
    if (e != cudaSuccess) return cuda_fail(what, e);
    if (int rc = check_ws(what, d_ws, ws_bytes, l.total)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const int n = (int)n_target;
    if ((e = cudaMemsetAsync(d_bad, 0, sizeof(int64_t), s)) != cudaSuccess) return cuda_fail(what, e);
    k_cell_keys<<<nl_div_up(n, kThreads), kThreads, 0, s>>>(n, d_target, ox, oy, oz, cell, at<uint64_t>(d_ws, l.s.ka), at<uint32_t>(d_ws, l.s.va),
                                                            d_bad);
    NL_CHECK_LAUNCH(what);
    k_hash_clear<<<std::min(nl_div_up(l.cap, kThreads), 8 * nl_num_sms()), kThreads, 0, s>>>(l.cap, at<uint64_t>(d_ws, l.hkey));
    NL_CHECK_LAUNCH(what);
    const uint64_t *ks;
    const uint32_t *vs;
    if (int rc = sort_runs(what, n, d_ws, l.s, s, &ks, &vs)) return rc;
    const uint64_t mask = (uint64_t)l.cap - 1;
    k_hash_build<<<nl_div_up(n, kThreads), kThreads, 0, s>>>(n, d_target, ks, vs, at<int32_t>(d_ws, l.s.flag), at<int32_t>(d_ws, l.s.rid),
                                                             at<float4>(d_ws, l.pts), at<uint64_t>(d_ws, l.hkey), at<int32_t>(d_ws, l.hrun), mask);
    NL_CHECK_LAUNCH(what);
    if (n_query == 0) return NL_OK;
    k_nn_query<<<nl_div_up(n_query, kThreads), kThreads, 0, s>>>((int)n_query, d_query, at<float4>(d_ws, l.pts), at<int32_t>(d_ws, l.s.start),
                                                                 at<uint64_t>(d_ws, l.hkey), at<int32_t>(d_ws, l.hrun), mask, ox, oy, oz, cell,
                                                                 max_ring, truncation, d_dist);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

int64_t nl_eval_sums_workspace_bytes(int64_t n) {
    if (n < 0 || n > kMaxN) return nl_set_error("nl_eval_sums_workspace_bytes: n must be in [0, 2^31)");
    size_t a = 0;
    take(a, 24 * (size_t)std::max(1, nl_div_up(n, kTile)));
    return (int64_t)a;
}

int nl_eval_distance_sums(int64_t n, const float *d_dist, float threshold, void *d_ws, int64_t ws_bytes, double *d_out, void *stream) {
    const char *what = "nl_eval_distance_sums";
    if (n < 0 || n > kMaxN) return nl_set_error("nl_eval_distance_sums: n must be in [0, 2^31)");
    if (!d_ws || !d_out || (n > 0 && !d_dist)) return nl_set_error("nl_eval_distance_sums: null pointer");
    const int tiles = std::max(1, nl_div_up(n, kTile));
    if (int rc = check_ws(what, d_ws, ws_bytes, 24 * (size_t)tiles)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    k_sum_tiles<<<tiles, kThreads, 0, s>>>(n, d_dist, threshold, static_cast<double *>(d_ws));
    NL_CHECK_LAUNCH(what);
    k_sum_final<<<1, kThreads, 0, s>>>(tiles, static_cast<const double *>(d_ws), d_out);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

}  // extern "C"
