// Key-scan map refinement (include/nerfloam_b200.h section 14): the kernels a captured refinement iteration adds around the mapping
// iteration (ray selection -> rays -> samples -> gather -> decoder -> embedding scatter), so that P passes of the mapper's final_iter
// loop (src/mapping.py:154-164) replay one graph without host work between passes, and Adam steps only the rows the pass has reached.
//
//   pass boundary : on the first iteration of a pass, the pass's window and poses go into the selection buffers, its seeds are set,
//                   Adam's step count restarts, and the previous pass's rows get fresh moments and clear flags.
//   row list      : a bit per embedding row; nl_mark_rows sets the bits of the rows the gradient scatter writes and appends each
//                   newly set row to the list (warp-aggregated counter).  nl_mark_rows_floor skips the rows below a floor, so Adam
//                   never steps them (the saved rows of a map being extended).  A plain load filters rows already flagged: bits only go
//                   from 0 to 1 inside the kernel, so a stale 0 costs an atomic and never loses a row.
//   row Adam      : nl_adam_bf16_elem (adam.cuh, shared with nl_adam_bf16_ctl) on the listed rows, two threads per row (8 elements:
//                   one 16-byte load each of p, m, v, two of the gradient); the gradient row is cleared after it is read, which
//                   replaces the dense zero-fill of the fp32 gradient table.
// Exactness: Adam is fresh in every pass, so a row outside the list has g = m = v = 0, and the bf16 update leaves such a row bitwise
// unchanged: the listed-row step equals the dense step over the whole table.
#include <cstdint>

#include "../../include/nerfloam_b200.h"
#include "adam.cuh"
#include "nl_cuda.cuh"

namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads)
    k_refine_pass_begin(int F, long long cap, int iters, int P, const int32_t *__restrict__ state, const int32_t *__restrict__ windows,
                        const long long *__restrict__ kf_arrays, const long long *__restrict__ kf_points, const float *__restrict__ kf_pose6,
                        const int32_t *__restrict__ sel_seeds, const int32_t *__restrict__ noise_seeds, float *__restrict__ dirs,
                        float *__restrict__ gt, float *__restrict__ cosv, long long *__restrict__ n_points, float *__restrict__ pose6,
                        int32_t *__restrict__ sel_seed, int32_t *__restrict__ noise_seed, int32_t *__restrict__ ctl, long long n_rows,
                        const int32_t *__restrict__ rows, uint32_t *__restrict__ row_bits, uint4 *__restrict__ m, uint4 *__restrict__ v) {
    const int it = state[NL_REFINE_ITER];
    if (it % iters != 0 || it / iters >= P) return;
    const int p = it / iters;
    const int32_t *win = windows + (size_t)p * F;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
    if (tid == 0) {
        if (sel_seed) *sel_seed = sel_seeds[p];
        if (noise_seed) *noise_seed = noise_seeds[p];
        ctl[NL_CTL_ADAM_STEP] = 0;
    }
    if (tid < F * 6) pose6[tid] = kf_pose6[(size_t)win[tid / 6] * 6 + tid % 6];
    if (tid < F) n_points[tid] = kf_points[win[tid]];
    // the previous pass's rows: fresh moments (two 16-byte halves per row), flags cleared (all set bits of a word belong to listed rows)
    const long long n_prev = min((long long)state[NL_REFINE_PREV], n_rows);
    for (long long i = tid; i < 2 * n_prev; i += stride) {
        const size_t h = (size_t)rows[i >> 1] * 2 + (i & 1);
        m[h] = make_uint4(0u, 0u, 0u, 0u);
        v[h] = make_uint4(0u, 0u, 0u, 0u);
    }
    for (long long i = tid; i < n_prev; i += stride) row_bits[rows[i] >> 5] = 0u;
    // the window's scans into the selection buffers
    for (int f = 0; f < F; ++f) {
        const int k = win[f];
        const long long n = min(kf_points[k], cap);
        const float *d = reinterpret_cast<const float *>(kf_arrays[k * 3]);
        const float *c = reinterpret_cast<const float *>(kf_arrays[k * 3 + 1]);
        const float *g = reinterpret_cast<const float *>(kf_arrays[k * 3 + 2]);
        float *dd = dirs + (size_t)f * cap * 3, *cc = cosv + (size_t)f * cap, *gg = gt + (size_t)f * cap;
        for (long long i = tid; i < 3 * n; i += stride) dd[i] = d[i];
        for (long long i = tid; i < n; i += stride) {
            cc[i] = c[i];
            gg[i] = g[i];
        }
    }
}

// One thread per (sample, corner): the eight row ids of a sample are contiguous in vox2row, so a warp reads 4 samples' rows at once.
__global__ void __launch_bounds__(kThreads)
    k_mark_rows(long long M_host, const int32_t *__restrict__ M_dev, const int32_t *__restrict__ vox, const int32_t *__restrict__ vox2row,
                int32_t row_floor, uint32_t *row_bits, int32_t *__restrict__ rows, int32_t *__restrict__ n_listed) {
    const long long M = M_dev ? min((long long)*M_dev, M_host) : M_host;
    const long long total = 8 * M;
    const int lane = threadIdx.x & 31;
    for (long long base = (long long)blockIdx.x * blockDim.x; base < total; base += (long long)gridDim.x * blockDim.x) {
        const long long i = base + threadIdx.x;
        bool fresh = false;
        int row = -1;
        if (i < total) {
            row = vox2row[(size_t)vox[i >> 3] * 8 + (i & 7)];
            if (row >= row_floor) {             // row_floor >= 0: also drops the -1 of an unset corner
                const uint32_t bit = 1u << (row & 31);
                if (!(row_bits[row >> 5] & bit)) fresh = !(atomicOr(&row_bits[row >> 5], bit) & bit);
            }
        }
        const unsigned fm = __ballot_sync(0xffffffffu, fresh);
        if (fm == 0u) continue;
        int at = 0;
        if (lane == __ffs(fm) - 1) at = atomicAdd(n_listed, __popc(fm));
        at = __shfl_sync(0xffffffffu, at, __ffs(fm) - 1);
        if (fresh) rows[at + __popc(fm & ((1u << lane) - 1u))] = row;
    }
}

__global__ void __launch_bounds__(kThreads)
    k_adam_bf16_rows_ctl(long long n_rows, const int32_t *__restrict__ rows, const int32_t *__restrict__ n_listed, uint4 *__restrict__ p,
                         float4 *__restrict__ g, uint4 *__restrict__ m, uint4 *__restrict__ v, double lr, double beta1, double beta2,
                         float eps, const int32_t *__restrict__ ctl) {
    const long long n = 2 * min((long long)*n_listed, n_rows);
    const bool skip = ctl[NL_CTL_SKIP_NOW] != 0;
    const NlAdamConst c = nl_adam_const(lr, beta1, beta2, eps, skip ? 1 : ctl[NL_CTL_ADAM_STEP]);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const size_t h = (size_t)rows[i >> 1] * 2 + (i & 1);       // half row: 8 bf16 of p / m / v, 8 floats of the gradient
        const float4 g0 = g[2 * h], g1 = g[2 * h + 1];
        g[2 * h] = make_float4(0.f, 0.f, 0.f, 0.f);
        g[2 * h + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (skip) continue;
        uint4 pw = p[h], mw = m[h], vw = v[h];
        uint16_t *pe = reinterpret_cast<uint16_t *>(&pw), *me = reinterpret_cast<uint16_t *>(&mw), *ve = reinterpret_cast<uint16_t *>(&vw);
        const float ge[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) nl_adam_bf16_elem(c, ge[e], pe[e], me[e], ve[e]);
        p[h] = pw;
        m[h] = mw;
        v[h] = vw;
    }
}

__global__ void k_refine_iter_end(int iters, int32_t *state, int32_t *sel_seed, int32_t sel_inc, int32_t *noise_seed, int32_t noise_inc) {
    if (sel_seed) *sel_seed = (int32_t)((uint32_t)*sel_seed + (uint32_t)sel_inc);
    if (noise_seed) *noise_seed = (int32_t)((uint32_t)*noise_seed + (uint32_t)noise_inc);
    const int it = state[NL_REFINE_ITER] + 1;
    state[NL_REFINE_ITER] = it;
    if (it % iters == 0) {
        state[NL_REFINE_PREV] = state[NL_REFINE_LISTED];
        state[NL_REFINE_LISTED] = 0;
    }
}

int grid_for(long long work, int per_sm) {
    const long long b = (work + kThreads - 1) / kThreads;
    return (int)max(1LL, min(b, (long long)nl_num_sms() * per_sm));
}

}  // namespace

extern "C" int nl_refine_pass_begin(int n_frames, int64_t cap, int n_keyframes, int iters, int n_passes, const int32_t *d_state,
                                    const int32_t *d_windows, const int64_t *d_kf_arrays, const int64_t *d_kf_points, const float *d_kf_pose6,
                                    const int32_t *d_sel_seeds, const int32_t *d_noise_seeds, float *d_dirs, float *d_gt, float *d_cos,
                                    int64_t *d_n_points, float *d_pose6, int32_t *d_sel_seed, int32_t *d_noise_seed, int32_t *d_ctl,
                                    int64_t n_rows, const int32_t *d_rows, uint32_t *d_row_bits, uint16_t *d_m, uint16_t *d_v, void *stream) {
    if (n_frames <= 0 || cap <= 0 || n_keyframes <= 0 || iters <= 0 || n_passes <= 0 || n_rows <= 0 || n_rows > INT32_MAX)
        return nl_set_error("nl_refine_pass_begin: sizes must be positive (n_rows < 2^31)");
    if (!d_state || !d_windows || !d_kf_arrays || !d_kf_points || !d_kf_pose6 || !d_dirs || !d_gt || !d_cos || !d_n_points || !d_pose6 ||
        !d_ctl || !d_rows || !d_row_bits || !d_m || !d_v)
        return nl_set_error("nl_refine_pass_begin: null pointer");
    if (!d_sel_seed != !d_sel_seeds || !d_noise_seed != !d_noise_seeds)
        return nl_set_error("nl_refine_pass_begin: a seed and its per-pass array go together");
    k_refine_pass_begin<<<grid_for(3LL * n_frames * cap, 4), kThreads, 0, (cudaStream_t)stream>>>(
        n_frames, cap, iters, n_passes, d_state, d_windows, reinterpret_cast<const long long *>(d_kf_arrays),
        reinterpret_cast<const long long *>(d_kf_points), d_kf_pose6, d_sel_seeds, d_noise_seeds, d_dirs, d_gt, d_cos,
        reinterpret_cast<long long *>(d_n_points), d_pose6, d_sel_seed, d_noise_seed, d_ctl, n_rows, d_rows, d_row_bits,
        reinterpret_cast<uint4 *>(d_m), reinterpret_cast<uint4 *>(d_v));
    NL_CHECK_LAUNCH("nl_refine_pass_begin");
    return NL_OK;
}

extern "C" int nl_mark_rows_floor(int64_t M, const int32_t *d_M, const int32_t *d_vox, const int32_t *d_vox2row, int64_t n_rows,
                                  int64_t row_floor, uint32_t *d_row_bits, int32_t *d_rows, int32_t *d_state, void *stream) {
    if (M < 0 || n_rows <= 0 || n_rows > INT32_MAX) return nl_set_error("nl_mark_rows: bad sizes (M >= 0, 0 < n_rows < 2^31)");
    if (row_floor < 0 || row_floor > n_rows) return nl_set_error("nl_mark_rows_floor: row_floor must lie in [0, n_rows]");
    if (!d_vox || !d_vox2row || !d_row_bits || !d_rows || !d_state) return nl_set_error("nl_mark_rows: null pointer");
    if (M == 0) return NL_OK;
    k_mark_rows<<<grid_for(8 * M, 8), kThreads, 0, (cudaStream_t)stream>>>(M, d_M, d_vox, d_vox2row, (int32_t)row_floor, d_row_bits,
                                                                             d_rows, d_state + NL_REFINE_LISTED);
    NL_CHECK_LAUNCH("nl_mark_rows");
    return NL_OK;
}

extern "C" int nl_mark_rows(int64_t M, const int32_t *d_M, const int32_t *d_vox, const int32_t *d_vox2row, int64_t n_rows, uint32_t *d_row_bits,
                            int32_t *d_rows, int32_t *d_state, void *stream) {
    return nl_mark_rows_floor(M, d_M, d_vox, d_vox2row, n_rows, 0, d_row_bits, d_rows, d_state, stream);
}

extern "C" int nl_adam_bf16_rows_ctl(int64_t n_rows, const int32_t *d_rows, const int32_t *d_n_listed, uint16_t *d_param, float *d_grad_f32,
                                     uint16_t *d_m, uint16_t *d_v, double lr, double beta1, double beta2, double eps, const int32_t *d_ctl,
                                     void *stream) {
    if (n_rows < 0) return nl_set_error("nl_adam_bf16_rows_ctl: bad arguments");
    if (n_rows == 0) return NL_OK;
    if (!d_rows || !d_n_listed || !d_param || !d_grad_f32 || !d_m || !d_v || !d_ctl) return nl_set_error("nl_adam_bf16_rows_ctl: null pointer");
    k_adam_bf16_rows_ctl<<<grid_for(2 * n_rows, 16), kThreads, 0, (cudaStream_t)stream>>>(
        n_rows, d_rows, d_n_listed, reinterpret_cast<uint4 *>(d_param), reinterpret_cast<float4 *>(d_grad_f32), reinterpret_cast<uint4 *>(d_m),
        reinterpret_cast<uint4 *>(d_v), lr, beta1, beta2, (float)eps, d_ctl);
    NL_CHECK_LAUNCH("nl_adam_bf16_rows_ctl");
    return NL_OK;
}

extern "C" int nl_refine_iter_end(int iters, int32_t *d_state, int32_t *d_sel_seed, int32_t sel_inc, int32_t *d_noise_seed, int32_t noise_inc,
                                  void *stream) {
    if (iters <= 0) return nl_set_error("nl_refine_iter_end: iters must be positive");
    if (!d_state) return nl_set_error("nl_refine_iter_end: null pointer");
    k_refine_iter_end<<<1, 1, 0, (cudaStream_t)stream>>>(iters, d_state, d_sel_seed, sel_inc, d_noise_seed, noise_inc);
    NL_CHECK_LAUNCH("nl_refine_iter_end");
    return NL_OK;
}
