// Ground segmentation and incidence cosines of one LiDAR scan (include/nerfloam_b200.h section 13, DESIGN.md section 12).
//
//   binning   : one thread per point: r = sqrt(x^2 + y^2), theta = atan2(y, x) in [0, 2 pi), both fp64 from the fp32 row; zone by
//               the edges b, ring = min(floor((r - b_z) / ring width), rings - 1), sector likewise; patch counts through a block
//               histogram (integer atomics).  Then a stable radix sort of (patch id, input index), an exclusive scan of the
//               counts (patch starts) and a gather of xyz into float4 in patch order.
//   fit       : one CTA per patch, one code path for every size (points stream from global memory, nothing is staged in shared
//               memory).  Seeds: a 4 x 8-bit radix select finds the num_lpr-th smallest candidate z, the smaller ones are ranked
//               in shared memory and summed in ascending order by one thread.  Each of the num_iter fits is two passes (mean,
//               then covariance), reduced in a fixed order (per-thread strided sums, warp butterflies, warps in order), and every
//               thread runs the same cyclic Jacobi eigen-solve on the result.  Then the verdict and the labels.
//   cosine    : one thread per point; every CTA compacts the ground patches (mean, normal) into shared memory in id order.
//   partition : flags -> exclusive scan -> scatter; both halves keep input order (cub::DevicePartition reverses the rejected half).
//   vertical  : only with vertical_cell > 0 (DESIGN.md section 12.1), between binning and the sort.  Column pass: one thread per
//               row inside the ranges inserts its cell key into an open-addressing table (hash.cuh) and folds its z into the slot's
//               min and max with integer atomicMin / atomicMax on order-preserving u32 keys.  Flag pass: one thread per row marks it
//               vertical from its slot's extent.  The gather carries the flag in the float4's .w, and k_fit<true> leaves flagged
//               rows out of the candidates, every S and the labels.  With the filter off none of this runs and k_fit<false> is the
//               unfiltered fit.
// No floating-point atomics anywhere, so two calls give identical bytes.
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
constexpr int kWarps = kThreads / 32;
constexpr int kMaxPatches = NL_GROUND_MAX_PATCHES;
constexpr int kMaxLpr = NL_GROUND_MAX_LPR;
constexpr int kKeyBits = 11;                                  // sort keys 0 .. kMaxPatches (kMaxPatches: outside or not finite)
constexpr int kTablePerThread = kMaxPatches / kThreads;
constexpr int kTableBytes = 48 * kMaxPatches;                 // the cosine kernel's ground-patch table: 6 doubles per patch
constexpr int64_t kMaxN = INT32_MAX;
constexpr double kTwoPi = 6.283185307179586;                  // 2 * pi rounded to fp64, as NumPy's 2 * np.pi
static_assert(kMaxPatches % kThreads == 0, "the cosine kernel's table scan takes kMaxPatches / kThreads entries per thread");
static_assert((1 << kKeyBits) > kMaxPatches, "sort keys must hold kMaxPatches");

struct Geo {
    double edge[5], ring_w[4], sector_w[4];
    int rings[4], sectors[4], patch_off[5], ring_off[4];
};

struct Fit {
    double seed_floor, th_seeds, th_dist, upright, sensor_height, elevation[4];
    int num_iter, num_lpr, num_min_pts;
};

struct Vert {
    double cell = 0.0, height = 0.0;   // cell 0: the filter is off
};

constexpr double kMaxCells = 1073741824.0;                     // max_range / vertical_cell <= 2^30 keeps the cell indices in int32
constexpr int64_t kMinColumnSlots = 256;

int64_t column_slots(int64_t n) {                              // a power of two >= 2n
    int64_t c = kMinColumnSlots;
    while (c < 2 * n) c <<= 1;
    return c;
}

size_t take(size_t &at, size_t bytes) {
    const size_t o = (at + 255) & ~size_t(255);
    at = o + bytes;
    return o;
}

struct Layout {
    size_t key_a = 0, key_b = 0, val_a = 0, val_b = 0, patch = 0, pcount = 0, start = 0, pts = 0, rec = 0, flags = 0, pos = 0, tmp = 0;
    size_t tmp_bytes = 0, total = 0;
};

// with_tmp = false leaves out CUB's temporary storage, whose size query needs the device: the argument checks use that lower bound
cudaError_t layout(int64_t n, Layout &l, bool with_tmp = true) {
    size_t a = 0;
    const size_t m = (size_t)std::max<int64_t>(n, 1);
    l.key_a = take(a, 4 * m); l.key_b = take(a, 4 * m); l.val_a = take(a, 4 * m); l.val_b = take(a, 4 * m);
    l.patch = take(a, 4 * m);
    l.pcount = take(a, 4 * (kMaxPatches + 1)); l.start = take(a, 4 * (kMaxPatches + 1));
    l.pts = take(a, 16 * m);
    l.rec = take(a, sizeof(nl_ground_patch) * kMaxPatches);
    l.flags = take(a, 4 * (m + 1)); l.pos = take(a, 4 * (m + 1));
    l.total = a;
    if (!with_tmp) return cudaSuccess;
    size_t s = 0, c = 0, p = 0;
    cub::DoubleBuffer<uint32_t> k(nullptr, nullptr), v(nullptr, nullptr);
    cudaError_t e;
    if ((e = cub::DeviceRadixSort::SortPairs(nullptr, s, k, v, (int)m, 0, kKeyBits)) != cudaSuccess) return e;
    if ((e = cub::DeviceScan::ExclusiveSum(nullptr, c, (const int32_t *)nullptr, (int32_t *)nullptr, kMaxPatches + 1)) != cudaSuccess) return e;
    if ((e = cub::DeviceScan::ExclusiveSum(nullptr, p, (const int32_t *)nullptr, (int32_t *)nullptr, (int)(m + 1))) != cudaSuccess) return e;
    l.tmp_bytes = std::max(s, std::max(c, p));
    l.tmp = take(a, l.tmp_bytes);
    l.total = a;
    return cudaSuccess;
}

template <class T>
T *at(void *ws, size_t off) { return reinterpret_cast<T *>(static_cast<char *>(ws) + off); }

int cuda_fail(const char *what, cudaError_t e) {
    char buf[256];
    std::snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
    return nl_set_error_code(NL_ERR_CUDA, buf);
}

// ---- binning --------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int patch_of(const Geo &g, float fx, float fy) {
    const double x = fx, y = fy;
    const double r = sqrt(x * x + y * y);                       // x * x is exact in fp64: contraction cannot change r
    if (!(r >= g.edge[0] && r < g.edge[4])) return -1;
    double th = atan2(y, x);
    if (th < 0.0) th += kTwoPi;
    const int z = r < g.edge[1] ? 0 : r < g.edge[2] ? 1 : r < g.edge[3] ? 2 : 3;
    const int ring = (int)fmin(floor((r - g.edge[z]) / g.ring_w[z]), (double)(g.rings[z] - 1));
    const int sec = (int)fmin(floor(th / g.sector_w[z]), (double)(g.sectors[z] - 1));
    return g.patch_off[z] + ring * g.sectors[z] + sec;
}

__global__ void __launch_bounds__(kThreads) k_bin(int n, const float *__restrict__ p, int stride, Geo g, int n_patches, uint32_t *key,
                                                  uint32_t *val, int32_t *patch, int32_t *pcount, uint8_t *label, float *cos,
                                                  int64_t *counts) {
    __shared__ int32_t hist[kMaxPatches];
    for (int b = threadIdx.x; b < n_patches; b += kThreads) hist[b] = 0;
    __syncthreads();
    int outside = 0, bad = 0;
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
        const float x = p[(int64_t)stride * i], y = p[(int64_t)stride * i + 1], z = p[(int64_t)stride * i + 2];
        int id = -1;
        if (!(isfinite(x) && isfinite(y) && isfinite(z))) ++bad;
        else if ((id = patch_of(g, x, y)) < 0) ++outside;
        else atomicAdd(&hist[id], 1);
        key[i] = id < 0 ? (uint32_t)kMaxPatches : (uint32_t)id;
        val[i] = (uint32_t)i;
        patch[i] = id;
        label[i] = 0;
        cos[i] = 1.f;
    }
    __syncthreads();
    for (int b = threadIdx.x; b < n_patches; b += kThreads)
        if (hist[b]) atomicAdd(&pcount[b], hist[b]);
    if (outside) atomicAdd((unsigned long long *)&counts[2], (unsigned long long)outside);
    if (bad) atomicAdd((unsigned long long *)&counts[3], (unsigned long long)bad);
}

// .w = 1 for a vertical row (vert: the flag pass's u8[n], nullptr with the filter off), else 0
__global__ void k_gather(int n, const float *__restrict__ p, int stride, const uint32_t *__restrict__ idx, const int32_t *__restrict__ start,
                         int n_patches, const uint8_t *__restrict__ vert, float4 *pts) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= start[n_patches]) return;                         // the sorted tail is the outside and non-finite rows
    const int64_t i = (int64_t)stride * idx[j];
    pts[j] = make_float4(p[i], p[i + 1], p[i + 2], vert && vert[idx[j]] ? 1.f : 0.f);
}

// ---- fit ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ord_of(float f) {          // order-preserving float -> uint32
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_of(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }

// v[k] <- the block's sum of v[k]: warp butterflies, then the warps in order.  Every thread gets the same bits.
template <int NV>
__device__ __forceinline__ void block_sum(double (&v)[NV], double (*red)[kWarps]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    #pragma unroll
    for (int k = 0; k < NV; ++k) {
        #pragma unroll
        for (int s = 16; s > 0; s >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], s);
        if (lane == 0) red[k][warp] = v[k];
    }
    __syncthreads();
    #pragma unroll
    for (int k = 0; k < NV; ++k) {
        double t = 0.0;
        #pragma unroll
        for (int w = 0; w < kWarps; ++w) t += red[k][w];
        v[k] = t;
    }
    __syncthreads();
}

// Cyclic Jacobi on the symmetric 3x3 a = (a00, a01, a02, a11, a12, a22).  Returns the smallest eigenvalue (ties: the lower index)
// and its unit eigenvector.  tests/ground_ref.py restates it step by step.
__device__ __forceinline__ double eig_min(const double (&c)[6], double (&vec)[3]) {
    double A[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
    double V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
    for (int sweep = 0; sweep < 32; ++sweep) {
        const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
        const double dia = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
        if (!(off > 1e-40 * dia)) break;
        #pragma unroll
        for (int pq = 0; pq < 3; ++pq) {
            const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2, r = 3 - p - q;
            const double apq = A[p][q];
            if (apq == 0.0) continue;
            const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
            const double t = fabs(theta) > 1e150 ? 0.5 / theta : (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
            const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
            A[p][p] -= t * apq;
            A[q][q] += t * apq;
            A[p][q] = A[q][p] = 0.0;
            const double arp = A[r][p], arq = A[r][q];
            A[r][p] = A[p][r] = cs * arp - sn * arq;
            A[r][q] = A[q][r] = sn * arp + cs * arq;
            #pragma unroll
            for (int k = 0; k < 3; ++k) {
                const double vkp = V[k][p], vkq = V[k][q];
                V[k][p] = cs * vkp - sn * vkq;
                V[k][q] = sn * vkp + cs * vkq;
            }
        }
    }
    int m = 0;
    if (A[1][1] < A[m][m]) m = 1;
    if (A[2][2] < A[m][m]) m = 2;
    #pragma unroll
    for (int k = 0; k < 3; ++k) vec[k] = V[k][m];
    return A[m][m];
}

__device__ __forceinline__ double plane_dist(const double (&n)[3], double d, float4 q) {
    return ((n[0] * (double)q.x + n[1] * (double)q.y) + n[2] * (double)q.z) + d;
}

__device__ __forceinline__ int global_ring(const Geo &g, int id) {
    int z = 0;
    while (z < 3 && id >= g.patch_off[z + 1]) ++z;
    return g.ring_off[z] + (id - g.patch_off[z]) / g.sectors[z];
}

// V: the vertical filter is on, and a row with .w != 0 takes no part in the seeds, the fits or the labels
template <bool V>
__global__ void __launch_bounds__(kThreads) k_fit(Geo g, Fit f, const int32_t *__restrict__ start, const float4 *__restrict__ pts,
                                                  const uint32_t *__restrict__ idx, uint8_t *label, nl_ground_patch *rec, int64_t *counts) {
    __shared__ double red[6][kWarps];
    __shared__ uint32_t hist[256];
    __shared__ float low[kMaxLpr], ranked[kMaxLpr];
    __shared__ uint32_t sel_prefix, sel_need, n_low;
    const int id = blockIdx.x;
    const int b = start[id], cnt = start[id + 1] - b;
    const float4 *__restrict__ P = pts + b;
    const bool zone0 = id < g.patch_off[1];
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    double mean[3] = {nan, nan, nan}, nrm[3] = {nan, nan, nan}, d = nan, lam = nan;
    int ground = 0;
    double n_ground = 0.0;
    // candidates: every point, except zone 0's below adaptive_seed_margin * sensor_height (and the vertical ones)
    auto cand = [&](int j, float z) { return !(V && P[j].w != 0.f) && !(zone0 && (double)z < f.seed_floor); };
    auto kept = [](float4 q) { return !(V && q.w != 0.f); };
    int n_vert = 0;
    if (V && cnt > 0) {
        double nv[1] = {0.0};
        for (int j = threadIdx.x; j < cnt; j += kThreads) nv[0] += P[j].w != 0.f ? 1.0 : 0.0;
        block_sum<1>(nv, red);
        n_vert = (int)nv[0];
    }
    const int n_fit = cnt - n_vert;                            // num_min_pts counts the rows a fit may use
    bool fitted = false;
    if (n_fit >= f.num_min_pts && n_fit > 0) {
        double nc[1] = {0.0};
        for (int j = threadIdx.x; j < cnt; j += kThreads) nc[0] += cand(j, P[j].z) ? 1.0 : 0.0;
        block_sum<1>(nc, red);
        const int n_cand = (int)nc[0];
        if (n_cand > 0) {
            const int k = min(f.num_lpr, n_cand);
            // radix select of the k-th smallest candidate z (ordered-key bits, most significant byte first)
            uint32_t prefix = 0, mask = 0, need = (uint32_t)k;
            for (int shift = 24; shift >= 0; shift -= 8) {
                hist[threadIdx.x] = 0;
                __syncthreads();
                for (int j = threadIdx.x; j < cnt; j += kThreads) {
                    const float z = P[j].z;
                    const uint32_t o = ord_of(z);
                    if (cand(j, z) && (o & mask) == prefix) atomicAdd(&hist[(o >> shift) & 255u], 1u);
                }
                __syncthreads();
                if (threadIdx.x == 0) {
                    uint32_t below = 0, digit = 0;
                    while (below + hist[digit] < need) below += hist[digit++];
                    sel_prefix = prefix | (digit << shift);
                    sel_need = need - below;
                }
                __syncthreads();
                prefix = sel_prefix;
                need = sel_need;
                mask |= 255u << shift;
                __syncthreads();
            }
            // the k - need candidates below the k-th smallest value, ranked, then summed in ascending order
            if (threadIdx.x == 0) n_low = 0;
            __syncthreads();
            for (int j = threadIdx.x; j < cnt; j += kThreads) {
                const float z = P[j].z;
                if (cand(j, z) && ord_of(z) < prefix) low[atomicAdd(&n_low, 1u)] = z;
            }
            __syncthreads();
            const int m = (int)n_low;
            for (int i = threadIdx.x; i < m; i += kThreads) {
                const float v = low[i];
                int r = 0;
                for (int j = 0; j < m; ++j) r += (low[j] < v) || (low[j] == v && j < i);
                ranked[r] = v;
            }
            __syncthreads();
            __shared__ double seed_h;
            if (threadIdx.x == 0) {
                double s = 0.0;
                for (int i = 0; i < m; ++i) s += (double)ranked[i];
                const double kth = (double)float_of(prefix);
                for (uint32_t i = 0; i < need; ++i) s += kth;
                seed_h = s / (double)k;
            }
            __syncthreads();
            const double cut = seed_h + f.th_seeds;
            fitted = true;
            for (int t = 0; t < f.num_iter && fitted; ++t) {
                double s[4] = {0.0, 0.0, 0.0, 0.0};
                for (int j = threadIdx.x; j < cnt; j += kThreads) {
                    const float4 q = P[j];
                    const bool in = t == 0 ? (cand(j, q.z) && (double)q.z < cut) : kept(q) && plane_dist(nrm, d, q) < f.th_dist;
                    if (in) { s[0] += 1.0; s[1] += q.x; s[2] += q.y; s[3] += q.z; }
                }
                block_sum<4>(s, red);
                if (s[0] < 3.0) { fitted = false; break; }
                const double mu[3] = {s[1] / s[0], s[2] / s[0], s[3] / s[0]};
                double c[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
                for (int j = threadIdx.x; j < cnt; j += kThreads) {
                    const float4 q = P[j];
                    const bool in = t == 0 ? (cand(j, q.z) && (double)q.z < cut) : kept(q) && plane_dist(nrm, d, q) < f.th_dist;
                    if (in) {
                        const double dx = q.x - mu[0], dy = q.y - mu[1], dz = q.z - mu[2];
                        c[0] += dx * dx; c[1] += dx * dy; c[2] += dx * dz; c[3] += dy * dy; c[4] += dy * dz; c[5] += dz * dz;
                    }
                }
                block_sum<6>(c, red);
                #pragma unroll
                for (int k6 = 0; k6 < 6; ++k6) c[k6] /= s[0];
                lam = eig_min(c, nrm);
                if (nrm[2] < 0.0) { nrm[0] = -nrm[0]; nrm[1] = -nrm[1]; nrm[2] = -nrm[2]; }
                d = -((nrm[0] * mu[0] + nrm[1] * mu[1]) + nrm[2] * mu[2]);
                mean[0] = mu[0]; mean[1] = mu[1]; mean[2] = mu[2];
            }
        }
    }
    const int ring = global_ring(g, id);
    if (fitted) {
        ground = nrm[2] >= f.upright && (ring >= 4 || mean[2] + f.sensor_height < f.elevation[ring]);
        if (ground) {
            double ng[1] = {0.0};
            for (int j = threadIdx.x; j < cnt; j += kThreads)
                if (kept(P[j]) && plane_dist(nrm, d, P[j]) < f.th_dist) { label[idx[b + j]] = 1; ng[0] += 1.0; }
            block_sum<1>(ng, red);
            n_ground = ng[0];
        }
    } else {
        mean[0] = mean[1] = mean[2] = nrm[0] = nrm[1] = nrm[2] = d = lam = nan;
    }
    if (threadIdx.x == 0) {
        nl_ground_patch o;
        for (int k = 0; k < 3; ++k) { o.mean[k] = mean[k]; o.normal[k] = nrm[k]; }
        o.d = d; o.lambda_min = lam;
        o.n_points = cnt; o.n_ground = (int32_t)n_ground; o.ground = ground; o.ring = ring;
        o.n_vertical = n_vert; o._pad = 0;
        rec[id] = o;
        if (o.n_ground) atomicAdd((unsigned long long *)&counts[0], (unsigned long long)o.n_ground);
    }
}

// ---- vertical filter ------------------------------------------------------------------------------------------------------
// The cell (floor(x / cell), floor(y / cell)), fp64 from the fp32 row, packed with each index biased by 2^31.  A row inside the
// ranges has |x|, |y| < max_range <= 2^30 cells, so each biased half lies in [2^30, 3 * 2^30]: never NL_HASH_EMPTY.
__device__ __forceinline__ uint64_t column_key(float fx, float fy, double cell) {
    const int32_t cx = (int32_t)floor((double)fx / cell), cy = (int32_t)floor((double)fy / cell);
    return ((uint64_t)((uint32_t)cx + 0x80000000u) << 32) | (uint64_t)((uint32_t)cy + 0x80000000u);
}

// Column pass: every row inside the ranges (patch >= 0) folds its z into its cell's slot.  zlo starts at ~0, zhi at 0.
__global__ void __launch_bounds__(kThreads) k_columns(int n, const float *__restrict__ p, int stride, const int32_t *__restrict__ patch,
                                                      double cell, uint64_t mask, uint64_t *keys, uint32_t *zlo, uint32_t *zhi) {
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
        if (patch[i] < 0) continue;
        const int64_t r = (int64_t)stride * i;
        const uint64_t s = nl_hash_insert_slot(keys, mask, column_key(p[r], p[r + 1], cell));
        const uint32_t o = ord_of(p[r + 2]);
        atomicMin(&zlo[s], o);
        atomicMax(&zhi[s], o);
    }
}

// Flag pass: vertical = the row's cell spreads over more than `height` in z (the extent of two floats in fp64 is exact).
__global__ void __launch_bounds__(kThreads) k_vertical(int n, const float *__restrict__ p, int stride, const int32_t *__restrict__ patch,
                                                       double cell, double height, uint64_t mask, const uint64_t *__restrict__ keys,
                                                       const uint32_t *__restrict__ zlo, const uint32_t *__restrict__ zhi, uint8_t *vert) {
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
        uint8_t v = 0;
        if (patch[i] >= 0) {
            const int64_t r = (int64_t)stride * i;
            const uint64_t s = nl_hash_slot_of(keys, mask, column_key(p[r], p[r + 1], cell));
            v = (double)float_of(zhi[s]) - (double)float_of(zlo[s]) > height;
        }
        vert[i] = v;
    }
}

// ---- cosine ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) k_cos(int n, const float *__restrict__ p, int stride, const uint8_t *__restrict__ label,
                                                  const nl_ground_patch *__restrict__ rec, int n_patches, float *cos, int64_t *counts) {
    using Scan = cub::BlockScan<int, kThreads>;
    __shared__ typename Scan::TempStorage tmp;
    extern __shared__ double tab_raw[];                        // ground patches in id order: mean xyz, normal xyz
    double (*tab)[6] = reinterpret_cast<double (*)[6]>(tab_raw);
    int flag[kTablePerThread], pos[kTablePerThread], n_tab = 0;
    #pragma unroll
    for (int k = 0; k < kTablePerThread; ++k) {
        const int id = threadIdx.x * kTablePerThread + k;
        flag[k] = id < n_patches && rec[id].ground ? 1 : 0;
    }
    Scan(tmp).ExclusiveSum(flag, pos, n_tab);
    #pragma unroll
    for (int k = 0; k < kTablePerThread; ++k)
        if (flag[k]) {
            const nl_ground_patch &r = rec[threadIdx.x * kTablePerThread + k];
            for (int c = 0; c < 3; ++c) { tab[pos[k]][c] = r.mean[c]; tab[pos[k]][3 + c] = r.normal[c]; }
        }
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x == 0) counts[1] = (int64_t)n - counts[0];
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
        if (!label[i]) continue;
        const double x = p[(int64_t)stride * i], y = p[(int64_t)stride * i + 1], z = p[(int64_t)stride * i + 2];
        double best = INFINITY;
        int arg = 0;
        for (int t = 0; t < n_tab; ++t) {
            const double dx = x - tab[t][0], dy = y - tab[t][1], dz = z - tab[t][2];
            const double d2 = (dx * dx + dy * dy) + dz * dz;
            if (d2 < best) { best = d2; arg = t; }               // strict: ties go to the lower patch id
        }
        const double dot = (tab[arg][3] * x + tab[arg][4] * y) + tab[arg][5] * z;
        cos[i] = (float)(fabs(dot) / sqrt((x * x + y * y) + z * z));
    }
}

// ---- partition ------------------------------------------------------------------------------------------------------------
__global__ void k_flags(int n, const uint8_t *__restrict__ label, int32_t *flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n) flags[i] = i < n && label[i] ? 1 : 0;
}

__global__ void k_scatter(int n, const float *__restrict__ p, int stride, const uint8_t *__restrict__ label, const float *__restrict__ cos,
                          const int32_t *__restrict__ pos, float *out_p, float *out_cos, int32_t *out_idx) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int n_ground = pos[n];
    const int o = label[i] ? pos[i] : n_ground + (i - pos[i]);
    const int64_t s = (int64_t)stride * i;
    out_p[3 * (int64_t)o] = p[s]; out_p[3 * (int64_t)o + 1] = p[s + 1]; out_p[3 * (int64_t)o + 2] = p[s + 2];
    out_cos[o] = cos[i];
    out_idx[o] = i;
}

int check_params(const char *what, const nl_ground_params *q, Geo &g, Fit &f, Vert &v, int &n_patches) {
    char buf[192];
    if (!q) { std::snprintf(buf, sizeof(buf), "%s: null params", what); return nl_set_error(buf); }
    if (!(std::isfinite(q->min_range) && std::isfinite(q->max_range) && q->min_range > 0.0 && q->min_range < q->max_range)) {
        std::snprintf(buf, sizeof(buf), "%s: need 0 < min_range < max_range, both finite", what);
        return nl_set_error(buf);
    }
    int total = 0, rings = 0;
    for (int z = 0; z < 4; ++z) {
        if (q->num_rings_each_zone[z] <= 0 || q->num_sectors_each_zone[z] <= 0) {
            std::snprintf(buf, sizeof(buf), "%s: zone %d: ring and sector counts must be positive", what, z);
            return nl_set_error(buf);
        }
        if (q->num_rings_each_zone[z] > kMaxPatches || q->num_sectors_each_zone[z] > kMaxPatches ||
            (total += q->num_rings_each_zone[z] * q->num_sectors_each_zone[z]) > kMaxPatches) {
            std::snprintf(buf, sizeof(buf), "%s: more patches than NL_GROUND_MAX_PATCHES (%d)", what, kMaxPatches);
            return nl_set_error(buf);
        }
    }
    if (q->num_lpr < 1 || q->num_lpr > kMaxLpr) {
        std::snprintf(buf, sizeof(buf), "%s: num_lpr must be in [1, %d]", what, kMaxLpr);
        return nl_set_error(buf);
    }
    if (q->num_iter < 1) { std::snprintf(buf, sizeof(buf), "%s: num_iter must be >= 1", what); return nl_set_error(buf); }
    const double th[5] = {q->sensor_height, q->uprightness_thr, q->th_seeds, q->th_dist, q->adaptive_seed_margin};
    bool finite = true;
    for (double v : th) finite = finite && std::isfinite(v);
    for (int k = 0; k < 4; ++k) finite = finite && std::isfinite(q->elevation_thr[k]);
    if (!finite) { std::snprintf(buf, sizeof(buf), "%s: thresholds and sensor_height must be finite", what); return nl_set_error(buf); }
    if (!(std::isfinite(q->vertical_cell) && q->vertical_cell >= 0.0)) {
        std::snprintf(buf, sizeof(buf), "%s: vertical_cell must be finite and >= 0 (0 = off)", what);
        return nl_set_error(buf);
    }
    if (q->vertical_cell > 0.0) {
        if (!(std::isfinite(q->vertical_height) && q->vertical_height > 0.0)) {
            std::snprintf(buf, sizeof(buf), "%s: vertical_height must be positive and finite when vertical_cell > 0", what);
            return nl_set_error(buf);
        }
        if (!(q->max_range / q->vertical_cell <= kMaxCells)) {
            std::snprintf(buf, sizeof(buf), "%s: vertical_cell too small: the cell keys need max_range / vertical_cell <= 2^30", what);
            return nl_set_error(buf);
        }
    }
    v.cell = q->vertical_cell;
    v.height = q->vertical_height;
    const double lo = q->min_range, hi = q->max_range;
    const double e[5] = {lo, (7.0 * lo + hi) / 8.0, (3.0 * lo + hi) / 4.0, (lo + hi) / 2.0, hi};
    g.patch_off[0] = 0;
    for (int z = 0; z < 5; ++z) g.edge[z] = e[z];
    for (int z = 0; z < 4; ++z) {
        g.rings[z] = q->num_rings_each_zone[z];
        g.sectors[z] = q->num_sectors_each_zone[z];
        g.ring_w[z] = (e[z + 1] - e[z]) / (double)g.rings[z];
        g.sector_w[z] = kTwoPi / (double)g.sectors[z];
        g.patch_off[z + 1] = g.patch_off[z] + g.rings[z] * g.sectors[z];
        g.ring_off[z] = rings;
        rings += g.rings[z];
    }
    f.seed_floor = q->adaptive_seed_margin * q->sensor_height;
    f.th_seeds = q->th_seeds; f.th_dist = q->th_dist; f.upright = q->uprightness_thr; f.sensor_height = q->sensor_height;
    for (int k = 0; k < 4; ++k) f.elevation[k] = q->elevation_thr[k];
    f.num_iter = q->num_iter; f.num_lpr = q->num_lpr; f.num_min_pts = q->num_min_pts;
    n_patches = total;
    return NL_OK;
}

int check_ws(const char *what, int64_t n, const void *ws, int64_t ws_bytes, Layout &l) {
    char buf[192];
    for (bool with_tmp : {false, true}) {
        const cudaError_t e = layout(n, l, with_tmp);
        if (e != cudaSuccess) return cuda_fail(what, e);
        if (!ws || ws_bytes < (int64_t)l.total) {
            std::snprintf(buf, sizeof(buf), "%s: workspace of %lld bytes, nl_ground_workspace_bytes asks for %lld", what, (long long)ws_bytes,
                          (long long)l.total);
            return nl_set_error(buf);
        }
        if (((uintptr_t)ws & 255u) != 0) { std::snprintf(buf, sizeof(buf), "%s: the workspace must be 256-byte aligned", what); return nl_set_error(buf); }
    }
    return NL_OK;
}

int grid_for(int64_t n) { return (int)std::min<int64_t>(std::max(1, nl_div_up(n, kThreads)), 4 * nl_num_sms()); }

}  // namespace

extern "C" {

void nl_abi_sizes_ground(int32_t out[3]) {
    out[0] = (int32_t)sizeof(nl_ground_params);
    out[1] = kMaxPatches;
    out[2] = (int32_t)sizeof(nl_ground_patch);
}

int64_t nl_ground_workspace_bytes(int64_t n) {
    if (n < 0 || n > kMaxN) return nl_set_error("nl_ground_workspace_bytes: n must be in [0, 2^31)");
    Layout l;
    const cudaError_t e = layout(n, l);
    if (e != cudaSuccess) return cuda_fail("nl_ground_workspace_bytes", e);
    return (int64_t)l.total;
}

int64_t nl_ground_vertical_workspace_bytes(int64_t n) {
    if (n < 0 || n > kMaxN) return nl_set_error("nl_ground_vertical_workspace_bytes: n must be in [0, 2^31)");
    return 16 * column_slots(n);
}

static int ground_segment(const char *what, int64_t n, const float *d_points, int32_t stride, const nl_ground_params *params, void *d_ws,
                          int64_t ws_bytes, void *d_vws, int64_t vws_bytes, uint8_t *d_label, float *d_cos, int32_t *d_patch,
                          nl_ground_patch *d_patches, uint8_t *d_vertical, int64_t *d_counts, void *stream) {
    char buf[192];
    if (n < 0 || n > kMaxN) { std::snprintf(buf, sizeof(buf), "%s: n must be in [0, 2^31)", what); return nl_set_error(buf); }
    if (stride != 3 && stride != 4) { std::snprintf(buf, sizeof(buf), "%s: stride must be 3 or 4", what); return nl_set_error(buf); }
    Geo g;
    Fit f;
    Vert v;
    int n_patches = 0, rc;
    if ((rc = check_params(what, params, g, f, v, n_patches)) != NL_OK) return rc;
    if (!d_counts || (n > 0 && (!d_points || !d_label || !d_cos))) { std::snprintf(buf, sizeof(buf), "%s: null pointer", what); return nl_set_error(buf); }
    const bool vertical = v.cell > 0.0;
    const int64_t slots = column_slots(n);
    if (vertical && n > 0) {
        if (!d_vws || !d_vertical) {
            std::snprintf(buf, sizeof(buf), "%s: null pointer: vertical_cell > 0 needs the vertical workspace and d_vertical "
                          "(nl_ground_segment_vertical)", what);
            return nl_set_error(buf);
        }
        if (vws_bytes < 16 * slots) {
            std::snprintf(buf, sizeof(buf), "%s: vertical workspace of %lld bytes, nl_ground_vertical_workspace_bytes asks for %lld", what,
                          (long long)vws_bytes, (long long)(16 * slots));
            return nl_set_error(buf);
        }
        if (((uintptr_t)d_vws & 255u) != 0) {
            std::snprintf(buf, sizeof(buf), "%s: the vertical workspace must be 256-byte aligned", what);
            return nl_set_error(buf);
        }
    }
    Layout l;
    if ((rc = check_ws(what, n, d_ws, ws_bytes, l)) != NL_OK) return rc;

    cudaStream_t s = (cudaStream_t)stream;
    const int ni = (int)n;
    uint32_t *key_a = at<uint32_t>(d_ws, l.key_a), *key_b = at<uint32_t>(d_ws, l.key_b);
    uint32_t *val_a = at<uint32_t>(d_ws, l.val_a), *val_b = at<uint32_t>(d_ws, l.val_b);
    int32_t *patch = d_patch ? d_patch : at<int32_t>(d_ws, l.patch);
    int32_t *pcount = at<int32_t>(d_ws, l.pcount), *start = at<int32_t>(d_ws, l.start);
    float4 *pts = at<float4>(d_ws, l.pts);
    nl_ground_patch *rec = d_patches ? d_patches : at<nl_ground_patch>(d_ws, l.rec);
    cudaError_t e;
    if ((e = cudaMemsetAsync(d_counts, 0, 4 * sizeof(int64_t), s)) != cudaSuccess) return cuda_fail(what, e);
    if ((e = cudaMemsetAsync(pcount, 0, 4 * (kMaxPatches + 1), s)) != cudaSuccess) return cuda_fail(what, e);
    if (ni > 0) {
        k_bin<<<grid_for(n), kThreads, 0, s>>>(ni, d_points, stride, g, n_patches, key_a, val_a, patch, pcount, d_label, d_cos, d_counts);
        NL_CHECK_LAUNCH(what);
    }
    if (vertical && ni > 0) {                                   // the column table: keys, then z min, then z max, `slots` of each
        uint64_t *keys = at<uint64_t>(d_vws, 0);
        uint32_t *zlo = at<uint32_t>(d_vws, 8 * slots), *zhi = at<uint32_t>(d_vws, 12 * slots);
        if ((e = cudaMemsetAsync(keys, 0xff, 12 * slots, s)) != cudaSuccess) return cuda_fail(what, e);   // NL_HASH_EMPTY keys, zlo = ~0
        if ((e = cudaMemsetAsync(zhi, 0, 4 * slots, s)) != cudaSuccess) return cuda_fail(what, e);
        const uint64_t mask = (uint64_t)slots - 1;
        k_columns<<<grid_for(n), kThreads, 0, s>>>(ni, d_points, stride, patch, v.cell, mask, keys, zlo, zhi);
        NL_CHECK_LAUNCH(what);
        k_vertical<<<grid_for(n), kThreads, 0, s>>>(ni, d_points, stride, patch, v.cell, v.height, mask, keys, zlo, zhi, d_vertical);
        NL_CHECK_LAUNCH(what);
    } else if (d_vertical && ni > 0) {
        if ((e = cudaMemsetAsync(d_vertical, 0, n, s)) != cudaSuccess) return cuda_fail(what, e);
    }
    size_t tb = l.tmp_bytes;
    if ((e = cub::DeviceScan::ExclusiveSum(at<void>(d_ws, l.tmp), tb, pcount, start, n_patches + 1, s)) != cudaSuccess) return cuda_fail(what, e);
    const uint32_t *idx = val_a;
    if (ni > 0) {
        cub::DoubleBuffer<uint32_t> dk(key_a, key_b), dv(val_a, val_b);
        tb = l.tmp_bytes;
        if ((e = cub::DeviceRadixSort::SortPairs(at<void>(d_ws, l.tmp), tb, dk, dv, ni, 0, kKeyBits, s)) != cudaSuccess) return cuda_fail(what, e);
        idx = dv.Current();
        k_gather<<<nl_div_up(n, kThreads), kThreads, 0, s>>>(ni, d_points, stride, idx, start, n_patches, vertical ? d_vertical : nullptr, pts);
        NL_CHECK_LAUNCH(what);
    }
    if (vertical) k_fit<true><<<n_patches, kThreads, 0, s>>>(g, f, start, pts, idx, d_label, rec, d_counts);
    else k_fit<false><<<n_patches, kThreads, 0, s>>>(g, f, start, pts, idx, d_label, rec, d_counts);
    NL_CHECK_LAUNCH(what);
    if (ni > 0) {
        static NlPerDevice opt_in;
        if ((e = opt_in.once([] { return cudaFuncSetAttribute(k_cos, cudaFuncAttributeMaxDynamicSharedMemorySize, kTableBytes); })) != cudaSuccess)
            return cuda_fail(what, e);
        k_cos<<<grid_for(n), kThreads, 48 * n_patches, s>>>(ni, d_points, stride, d_label, rec, n_patches, d_cos, d_counts);
        NL_CHECK_LAUNCH(what);
    }
    return NL_OK;
}

int nl_ground_segment(int64_t n, const float *d_points, int32_t stride, const nl_ground_params *params, void *d_ws, int64_t ws_bytes,
                      uint8_t *d_label, float *d_cos, int32_t *d_patch, nl_ground_patch *d_patches, int64_t *d_counts, void *stream) {
    return ground_segment("nl_ground_segment", n, d_points, stride, params, d_ws, ws_bytes, nullptr, 0, d_label, d_cos, d_patch, d_patches,
                          nullptr, d_counts, stream);
}

int nl_ground_segment_vertical(int64_t n, const float *d_points, int32_t stride, const nl_ground_params *params, void *d_ws, int64_t ws_bytes,
                               void *d_vws, int64_t vws_bytes, uint8_t *d_label, float *d_cos, int32_t *d_patch, nl_ground_patch *d_patches,
                               uint8_t *d_vertical, int64_t *d_counts, void *stream) {
    return ground_segment("nl_ground_segment_vertical", n, d_points, stride, params, d_ws, ws_bytes, d_vws, vws_bytes, d_label, d_cos, d_patch,
                          d_patches, d_vertical, d_counts, stream);
}

int nl_ground_partition(int64_t n, const float *d_points, int32_t stride, const uint8_t *d_label, const float *d_cos, void *d_ws, int64_t ws_bytes,
                        float *d_out_points, float *d_out_cos, int32_t *d_out_index, void *stream) {
    const char *what = "nl_ground_partition";
    if (n < 0 || n > kMaxN) return nl_set_error("nl_ground_partition: n must be in [0, 2^31)");
    if (stride != 3 && stride != 4) return nl_set_error("nl_ground_partition: stride must be 3 or 4");
    if (n > 0 && (!d_points || !d_label || !d_cos || !d_out_points || !d_out_cos || !d_out_index))
        return nl_set_error("nl_ground_partition: null pointer");
    Layout l;
    int rc;
    if ((rc = check_ws(what, n, d_ws, ws_bytes, l)) != NL_OK) return rc;
    if (n == 0) return NL_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const int ni = (int)n;
    int32_t *flags = at<int32_t>(d_ws, l.flags), *pos = at<int32_t>(d_ws, l.pos);
    k_flags<<<nl_div_up(n + 1, kThreads), kThreads, 0, s>>>(ni, d_label, flags);
    NL_CHECK_LAUNCH(what);
    size_t tb = l.tmp_bytes;
    const cudaError_t e = cub::DeviceScan::ExclusiveSum(at<void>(d_ws, l.tmp), tb, flags, pos, ni + 1, s);
    if (e != cudaSuccess) return cuda_fail(what, e);
    k_scatter<<<nl_div_up(n, kThreads), kThreads, 0, s>>>(ni, d_points, stride, d_label, d_cos, pos, d_out_points, d_out_cos, d_out_index);
    NL_CHECK_LAUNCH(what);
    return NL_OK;
}

}  // extern "C"
