// SDF decoder MLP 16 -> W -> W -> 1 (ReLU) with the SDF / free-space loss and the full backward pass
// fused into one persistent kernel (SURVEY.md section 8 a-8, a-9).
//
// Replaces Decoder.get_values (src/variations/lidar.py:109-123: 3 cuBLAS fp32 GEMMs + bias/ReLU kernels,
// activations [M,256] x2 round-tripping through HBM for autograd), Criterion.forward
// (src/criterion.py:16-115: ~25 elementwise/reduction kernels, 3 .item() syncs) and their autograd graph.
//
// fp32 CUDA-core version (exact fp32 FMA accumulation, SDF parity ~1e-6 against the fp32 reference):
//   * one CTA = 8 warps owns a tile of T = 128 samples; every warp owns 16 samples END TO END (all W
//     output columns of its 16 rows live across its 32 lanes), so the activation tile in shared memory
//     is warp-private by columns: no block barrier is needed between layers, the final 256 -> 1 layer
//     is a lane-local dot + one warp butterfly, and the loss gradient is formed in registers;
//   * activations are kept transposed in shared memory, A^T[k][t] (row stride T+4 floats), so a k-step
//     of the register-tiled GEMM is 4 broadcast LDS.128 (16 rows) + 2 LDS.128 (8 columns) for 128 FMAs;
//   * the WxW weight matrix is streamed from L2 in 16-row chunks (16 KB) with cp.async double buffering;
//   * backward (d/d input features; optional weight gradients) reuses the same tile buffer in place:
//     h1 -> dh2 -> dh1.  ReLU masks are 128 bits per thread in registers.
// Nothing but the input features [M,16], sdf [M], d features [M,16] and -- only when the decoder is being
// trained -- h1 / dh2 [M,W] (for the split-K dW1 GEMM) touches HBM.
#include "loss.cuh"
#include "nl_cuda.cuh"

namespace {

constexpr int T_TILE = 128;       // samples per CTA tile
constexpr int TS = T_TILE + 4;    // row stride of transposed activation tiles (floats)
constexpr int KC = 16;            // weight rows per streamed chunk
constexpr int NTHREADS = 256;

template <int W>
struct Cfg {
    static constexpr int J = W / 32;                 // output columns per lane
    static constexpr int VEC = (J % 4 == 0) ? 4 : 1; // columns are owned in groups of VEC consecutive
    // column owned by (lane, q):  VEC=4: (q/4)*128 + lane*4 + q%4   VEC=1: q*32 + lane
    __device__ static __forceinline__ int col(int lane, int q) {
        return VEC == 4 ? ((q >> 2) * 128 + lane * 4 + (q & 3)) : (q * 32 + lane);
    }
    static constexpr size_t smem_floats(bool wgrad) {
        return (size_t)W * TS          // bufA: h1^T / dh2^T / dh1^T
               + 16 * TS              // x^T
               + 16 * W               // W0^T  [16][W]
               + 2 * KC * W           // streamed weight chunks
               + 3 * W                // b0, b1, w2
               + (wgrad ? (3 * W + 16 * W + 4) : 0);  // gW2, gb1, gb0, gW0, gb2
    }
};

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// acc[16][J] += sum_{k<kc} A[k][t0 + i] * B[k][col(lane,q)]     A: smem row stride TS, B: smem row stride W
template <int W>
__device__ __forceinline__ void mma_rows(float (&acc)[16][Cfg<W>::J], const float *__restrict__ A, const float *__restrict__ B,
                                         int kc, int lane) {
    using C = Cfg<W>;
#pragma unroll 4
    for (int k = 0; k < kc; ++k) {
        float a[16];
        const float4 *ap = reinterpret_cast<const float4 *>(A + k * TS);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const float4 t = ap[v];
            a[4 * v] = t.x; a[4 * v + 1] = t.y; a[4 * v + 2] = t.z; a[4 * v + 3] = t.w;
        }
        float b[C::J];
        if (C::VEC == 4) {
#pragma unroll
            for (int g = 0; g < C::J / 4; ++g) {
                const float4 t = *reinterpret_cast<const float4 *>(B + k * W + g * 128 + lane * 4);
                b[4 * g] = t.x; b[4 * g + 1] = t.y; b[4 * g + 2] = t.z; b[4 * g + 3] = t.w;
            }
        } else {
#pragma unroll
            for (int q = 0; q < C::J; ++q) b[q] = B[k * W + q * 32 + lane];
        }
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
            for (int q = 0; q < C::J; ++q) acc[i][q] = fmaf(a[i], b[q], acc[i][q]);
    }
}

// Stream a [K][W] row-major matrix from global memory through the double-buffered chunk area and accumulate
// acc += A^T(tile) * B.  Block-wide: every thread of the CTA must call it.  Ends with a barrier.
template <int W>
__device__ __forceinline__ void gemm_stream(float (&acc)[16][Cfg<W>::J], const float *__restrict__ A_t0,
                                            const float *__restrict__ Bg, int K, float *chunk, int tid, int lane) {
    constexpr int F4_PER_CHUNK = KC * W / 4;
    const int nch = K / KC;
    for (int f = tid; f < F4_PER_CHUNK; f += NTHREADS) cp_async16(chunk + f * 4, Bg + f * 4);
    cp_async_commit();
    for (int c = 0; c < nch; ++c) {
        float *cur = chunk + (c & 1) * KC * W;
        if (c + 1 < nch) {
            float *nxt = chunk + ((c + 1) & 1) * KC * W;
            const float *src = Bg + (size_t)(c + 1) * KC * W;
            for (int f = tid; f < F4_PER_CHUNK; f += NTHREADS) cp_async16(nxt + f * 4, src + f * 4);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        mma_rows<W>(acc, A_t0 + (size_t)c * KC * TS, cur, KC, lane);
        __syncthreads();
    }
}

template <int W>
__device__ __forceinline__ void zero_acc(float (&acc)[16][Cfg<W>::J]) {
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int q = 0; q < Cfg<W>::J; ++q) acc[i][q] = 0.f;
}

struct MlpParams {
    long long M_host;
    const int32_t *M_dev;
    const float *feats;
    nl_mlp_weights w;
    float *sdf;
    // training
    const uint8_t *s_flag;
    const float *s_depth;
    const int32_t *s_ray;
    const float *cosv, *gt_depth;
    nl_render_stats *stats;
    float truncation;
    float *dfeats;
    nl_mlp_grads g;
    float *act_h1, *act_dh2;
    const float *dsdf_ext;
    int seg_rays;         // SEG: rays per problem; stats = the problems' statistics, problem = s_ray / seg_rays
};

// SEG (training without weight gradients only): nl_mlp_train_batch's loss, per problem (see k_mlp_wg in mlp_tc.cu)
template <int W, bool TRAIN, bool WGRAD, bool SEG = false>
__global__ void __launch_bounds__(NTHREADS, 1) k_mlp(MlpParams p) {
    static_assert(!SEG || (TRAIN && !WGRAD), "the batched loss is for frozen-decoder training only");
    using C = Cfg<W>;
    constexpr int J = C::J;
    constexpr int NMASK = (16 * J + 31) / 32;
    extern __shared__ __align__(16) float smem[];
    float *bufA = smem;
    float *xT = bufA + (size_t)W * TS;
    float *W0t = xT + 16 * TS;
    float *chunk = W0t + 16 * W;
    float *b0s = chunk + 2 * KC * W;
    float *b1s = b0s + W;
    float *w2s = b1s + W;
    float *gW2s = w2s + W;   // only valid when WGRAD
    float *gb1s = gW2s + W;
    float *gb0s = gb1s + W;
    float *gW0s = gb0s + W;  // [W][16]
    float *gb2s = gW0s + 16 * W;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int t0 = warp * 16;
    const long long M = p.M_dev ? min((long long)*p.M_dev, p.M_host) : p.M_host;
    const long long ntiles = (M + T_TILE - 1) / T_TILE;

    for (int i = tid; i < 16 * W; i += NTHREADS) W0t[i] = p.w.W0t[i];
    for (int i = tid; i < W; i += NTHREADS) { b0s[i] = p.w.b0[i]; b1s[i] = p.w.b1[i]; w2s[i] = p.w.W2[i]; }
    if (WGRAD) {
        for (int i = tid; i < 3 * W + 16 * W + 4; i += NTHREADS) gW2s[i] = 0.f;
    }
    const float b2 = p.w.b2[0];
    float g_fs = 0.f, g_sdf = 0.f;
    if (TRAIN && !p.dsdf_ext) { g_fs = p.stats->g_fs; g_sdf = p.stats->g_sdf; }
    double loss_fs = 0.0, loss_sdf = 0.0;
    __syncthreads();

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long m0 = tile * T_TILE;
        // ---- stage the 16 input features of this warp's 16 samples, transposed: xT[e][t] ----
        {
            const int t = tid >> 1, e0 = (tid & 1) * 8;  // t in [t0, t0+16) for this warp
            float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
            if (m0 + t < M) {
                const float4 *src = reinterpret_cast<const float4 *>(p.feats + (size_t)(m0 + t) * 16 + e0);
                v0 = src[0]; v1 = src[1];
            }
            xT[(e0 + 0) * TS + t] = v0.x; xT[(e0 + 1) * TS + t] = v0.y; xT[(e0 + 2) * TS + t] = v0.z; xT[(e0 + 3) * TS + t] = v0.w;
            xT[(e0 + 4) * TS + t] = v1.x; xT[(e0 + 5) * TS + t] = v1.y; xT[(e0 + 6) * TS + t] = v1.z; xT[(e0 + 7) * TS + t] = v1.w;
        }
        __syncwarp();

        float acc[16][J];
        uint32_t mask1[NMASK], mask2[NMASK];
#pragma unroll
        for (int i = 0; i < NMASK; ++i) { mask1[i] = 0u; mask2[i] = 0u; }

        // ---- layer 1: h1 = relu(x W0^T + b0)  (K = 16, B = W0^T resident in smem) ----
        zero_acc<W>(acc);
        mma_rows<W>(acc, xT + t0, W0t, 16, lane);
#pragma unroll
        for (int q = 0; q < J; ++q) {
            const int j = C::col(lane, q);
            const float bias = b0s[j];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                float h = acc[i][q] + bias;
                const bool on = h > 0.f;
                h = on ? h : 0.f;
                acc[i][q] = h;
                if (TRAIN && on) mask1[(i * J + q) >> 5] |= 1u << ((i * J + q) & 31);
            }
            float4 *dst = reinterpret_cast<float4 *>(bufA + (size_t)j * TS + t0);
            dst[0] = make_float4(acc[0][q], acc[1][q], acc[2][q], acc[3][q]);
            dst[1] = make_float4(acc[4][q], acc[5][q], acc[6][q], acc[7][q]);
            dst[2] = make_float4(acc[8][q], acc[9][q], acc[10][q], acc[11][q]);
            dst[3] = make_float4(acc[12][q], acc[13][q], acc[14][q], acc[15][q]);
        }
        if (WGRAD) {  // h1 rows to HBM for the dW1 GEMM (coalesced: a warp writes whole rows)
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                if (m0 + t0 + i < M) {
                    float *row = p.act_h1 + (size_t)(m0 + t0 + i) * W;
                    if (C::VEC == 4) {
#pragma unroll
                        for (int g = 0; g < J / 4; ++g)
                            *reinterpret_cast<float4 *>(row + g * 128 + lane * 4) =
                                make_float4(acc[i][4 * g], acc[i][4 * g + 1], acc[i][4 * g + 2], acc[i][4 * g + 3]);
                    } else {
#pragma unroll
                        for (int q = 0; q < J; ++q) row[q * 32 + lane] = acc[i][q];
                    }
                }
            }
        }
        __syncwarp();

        // ---- layer 2: h2 = relu(h1 W1^T + b1), streamed W1^T ----
        zero_acc<W>(acc);
        gemm_stream<W>(acc, bufA + t0, p.w.W1t, W, chunk, tid, lane);
        float ps[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) ps[i] = 0.f;
#pragma unroll
        for (int q = 0; q < J; ++q) {
            const int j = C::col(lane, q);
            const float bias = b1s[j], w2 = w2s[j];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                float h = acc[i][q] + bias;
                const bool on = h > 0.f;
                h = on ? h : 0.f;
                acc[i][q] = h;
                if (TRAIN && on) mask2[(i * J + q) >> 5] |= 1u << ((i * J + q) & 31);
                ps[i] = fmaf(h, w2, ps[i]);
            }
        }
        // ---- output layer: sdf = h2 . w2 + b2 (butterfly: every lane gets the 16 sums) ----
#pragma unroll
        for (int i = 0; i < 16; ++i) {
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) ps[i] += __shfl_xor_sync(0xffffffffu, ps[i], off);
            ps[i] += b2;
        }
        {
            float mine = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) mine = (lane == i) ? ps[i] : mine;
            if (lane < 16 && m0 + t0 + lane < M) p.sdf[m0 + t0 + lane] = mine;
        }
        if (!TRAIN) continue;

        // ---- loss (criterion.py:92-103) and d loss / d sdf for this warp's 16 samples (lane i <-> sample i) ----
        float my_dsdf = 0.f;
        {
            float mine = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) mine = (lane == i) ? ps[i] : mine;
            const long long m = m0 + t0 + lane;
            int seg_k = -1;                          // SEG: this lane's problem
            double seg_fs = 0.0, seg_sdf = 0.0;
            if (!SEG && lane < 16 && m < M && p.dsdf_ext) {
                my_dsdf = p.dsdf_ext[m];
            } else if (lane < 16 && m < M) {
                const uint32_t fl = p.s_flag[m];
                const int r = p.s_ray[m];
                float gf = g_fs, gs = g_sdf;
                if constexpr (SEG) {
                    seg_k = r / p.seg_rays;
                    gf = p.stats[seg_k].g_fs;
                    gs = p.stats[seg_k].g_sdf;
                }
                const float cosr = p.cosv ? p.cosv[r] : 1.0f;
                const float z = __fmul_rn(p.s_depth[m], cosr);
                const float d = p.gt_depth[r];
                if (fl & 1u) {  // front: (sdf*1*1 - 1)^2
                    const float e = mine - 1.0f;
                    if constexpr (SEG) seg_fs = (double)e * (double)e;
                    else loss_fs += (double)e * (double)e;
                    my_dsdf += 2.0f * gf * e;
                }
                if (fl & 2u) {  // sdf band: ((z + sdf*trunc) - depth)^2
                    const float e = __fsub_rn(__fadd_rn(z, __fmul_rn(mine, p.truncation)), d);
                    if constexpr (SEG) seg_sdf = (double)e * (double)e;
                    else loss_sdf += (double)e * (double)e;
                    my_dsdf += 2.0f * gs * p.truncation * e;
                }
            }
            if constexpr (SEG) nl_seg_loss_add(p.stats, seg_k, seg_fs, seg_sdf);
        }
        float dsdf[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) dsdf[i] = __shfl_sync(0xffffffffu, my_dsdf, i);

        // ---- backward through the output layer: dh2 = dsdf * w2 * relu'(h2); weight grads of W2, b2, b1 ----
        if (WGRAD && lane == 0) {
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) s += dsdf[i];
            atomicAdd(gb2s, s);
        }
#pragma unroll
        for (int q = 0; q < J; ++q) {
            const int j = C::col(lane, q);
            const float w2 = w2s[j];
            float gw2 = 0.f, gb1 = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                if (WGRAD) gw2 = fmaf(acc[i][q], dsdf[i], gw2);
                const bool on = (mask2[(i * J + q) >> 5] >> ((i * J + q) & 31)) & 1u;
                const float d = on ? dsdf[i] * w2 : 0.f;
                acc[i][q] = d;
                gb1 += d;
            }
            if (WGRAD) { atomicAdd(gW2s + j, gw2); atomicAdd(gb1s + j, gb1); }
            float4 *dst = reinterpret_cast<float4 *>(bufA + (size_t)j * TS + t0);
            dst[0] = make_float4(acc[0][q], acc[1][q], acc[2][q], acc[3][q]);
            dst[1] = make_float4(acc[4][q], acc[5][q], acc[6][q], acc[7][q]);
            dst[2] = make_float4(acc[8][q], acc[9][q], acc[10][q], acc[11][q]);
            dst[3] = make_float4(acc[12][q], acc[13][q], acc[14][q], acc[15][q]);
        }
        if (WGRAD) {
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                if (m0 + t0 + i < M) {
                    float *row = p.act_dh2 + (size_t)(m0 + t0 + i) * W;
                    if (C::VEC == 4) {
#pragma unroll
                        for (int g = 0; g < J / 4; ++g)
                            *reinterpret_cast<float4 *>(row + g * 128 + lane * 4) =
                                make_float4(acc[i][4 * g], acc[i][4 * g + 1], acc[i][4 * g + 2], acc[i][4 * g + 3]);
                    } else {
#pragma unroll
                        for (int q = 0; q < J; ++q) row[q * 32 + lane] = acc[i][q];
                    }
                }
            }
        }
        __syncwarp();

        // ---- backward layer 2: dh1 = (dh2 W1) * relu'(h1), streamed W1 (row j = K index) ----
        zero_acc<W>(acc);
        gemm_stream<W>(acc, bufA + t0, p.w.W1, W, chunk, tid, lane);
#pragma unroll
        for (int q = 0; q < J; ++q) {
            const int k = C::col(lane, q);
            float gb0 = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const bool on = (mask1[(i * J + q) >> 5] >> ((i * J + q) & 31)) & 1u;
                const float d = on ? acc[i][q] : 0.f;
                acc[i][q] = d;
                gb0 += d;
            }
            if (WGRAD) atomicAdd(gb0s + k, gb0);
            float4 *dst = reinterpret_cast<float4 *>(bufA + (size_t)k * TS + t0);
            dst[0] = make_float4(acc[0][q], acc[1][q], acc[2][q], acc[3][q]);
            dst[1] = make_float4(acc[4][q], acc[5][q], acc[6][q], acc[7][q]);
            dst[2] = make_float4(acc[8][q], acc[9][q], acc[10][q], acc[11][q]);
            dst[3] = make_float4(acc[12][q], acc[13][q], acc[14][q], acc[15][q]);
        }
        __syncwarp();

        // ---- backward layer 1: dx[t][e] = sum_k dh1[t][k] W0[k][e]; lane = (half th, feature e) ----
        {
            const int e = lane & 15, th = lane >> 4;
            float dx[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) dx[u] = 0.f;
            const float *Ab = bufA + t0 + th * 8;
#pragma unroll 4
            for (int k = 0; k < W; ++k) {
                const float w = __ldg(p.w.W0 + k * 16 + e);
                const float4 a0 = *reinterpret_cast<const float4 *>(Ab + (size_t)k * TS);
                const float4 a1 = *reinterpret_cast<const float4 *>(Ab + (size_t)k * TS + 4);
                dx[0] = fmaf(a0.x, w, dx[0]); dx[1] = fmaf(a0.y, w, dx[1]); dx[2] = fmaf(a0.z, w, dx[2]); dx[3] = fmaf(a0.w, w, dx[3]);
                dx[4] = fmaf(a1.x, w, dx[4]); dx[5] = fmaf(a1.y, w, dx[5]); dx[6] = fmaf(a1.z, w, dx[6]); dx[7] = fmaf(a1.w, w, dx[7]);
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const long long m = m0 + t0 + th * 8 + u;
                if (m < M) p.dfeats[(size_t)m * 16 + e] = dx[u];
            }
            if (WGRAD) {  // gW0[k][e] += sum_{t in warp} dh1[t][k] x[t][e]
                const float4 *xr = reinterpret_cast<const float4 *>(xT + e * TS + t0);
                const float4 x0 = xr[0], x1 = xr[1], x2 = xr[2], x3 = xr[3];
                for (int kk = 0; kk < W / 2; ++kk) {
                    const int k = th * (W / 2) + kk;
                    const float4 *ar = reinterpret_cast<const float4 *>(bufA + (size_t)k * TS + t0);
                    const float4 a0 = ar[0], a1 = ar[1], a2 = ar[2], a3 = ar[3];
                    float s = a0.x * x0.x;
                    s = fmaf(a0.y, x0.y, s); s = fmaf(a0.z, x0.z, s); s = fmaf(a0.w, x0.w, s);
                    s = fmaf(a1.x, x1.x, s); s = fmaf(a1.y, x1.y, s); s = fmaf(a1.z, x1.z, s); s = fmaf(a1.w, x1.w, s);
                    s = fmaf(a2.x, x2.x, s); s = fmaf(a2.y, x2.y, s); s = fmaf(a2.z, x2.z, s); s = fmaf(a2.w, x2.w, s);
                    s = fmaf(a3.x, x3.x, s); s = fmaf(a3.y, x3.y, s); s = fmaf(a3.z, x3.z, s); s = fmaf(a3.w, x3.w, s);
                    atomicAdd(gW0s + k * 16 + e, s);
                }
            }
        }
        __syncwarp();
    }

    if (TRAIN && !SEG && !p.dsdf_ext) {
        for (int off = 16; off > 0; off >>= 1) {
            loss_fs += __shfl_down_sync(0xffffffffu, loss_fs, off);
            loss_sdf += __shfl_down_sync(0xffffffffu, loss_sdf, off);
        }
        if (lane == 0) {
            if (loss_fs != 0.0) atomicAdd(&p.stats->fs_sum, loss_fs);
            if (loss_sdf != 0.0) atomicAdd(&p.stats->sdf_sum, loss_sdf);
        }
    }
    if (WGRAD) {
        __syncthreads();
        for (int i = tid; i < W; i += NTHREADS) {
            atomicAdd(p.g.gW2 + i, gW2s[i]);
            atomicAdd(p.g.gb1 + i, gb1s[i]);
            atomicAdd(p.g.gb0 + i, gb0s[i]);
        }
        for (int i = tid; i < 16 * W; i += NTHREADS) atomicAdd(p.g.gW0 + i, gW0s[i]);
        if (tid == 0) atomicAdd(p.g.gb2, gb2s[0]);
    }
}

// dW1[j][k] += sum_m dh2[m][j] * h1[m][k]   (split-K over samples; 128x128 output tile per CTA)
template <int W>
__global__ void __launch_bounds__(256) k_dw1(long long M_host, const int32_t *__restrict__ M_dev, const float *__restrict__ dh2,
                                              const float *__restrict__ h1, float *__restrict__ gW1, int nsplit) {
    constexpr int TJ = W >= 128 ? 128 : W;
    constexpr int MT = TJ / 16;
    constexpr int VEC = (MT % 4 == 0) ? 4 : 1;
    constexpr int TPD = W / TJ;
    constexpr int MC = 16;
    __shared__ __align__(16) float As[MC][TJ], Bs[MC][TJ];
    const long long M = M_dev ? min((long long)*M_dev, M_host) : M_host;
    const int tile = blockIdx.x % (TPD * TPD), split = blockIdx.x / (TPD * TPD);
    const int j0 = (tile / TPD) * TJ, k0 = (tile % TPD) * TJ;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    auto col = [](int t, int q) { return VEC == 4 ? ((q >> 2) * 64 + t * 4 + (q & 3)) : (q * 16 + t); };
    float acc[MT][MT];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int q = 0; q < MT; ++q) acc[i][q] = 0.f;
    const long long nchunks = (M + MC - 1) / MC;
    for (long long ch = split; ch < nchunks; ch += nsplit) {
        const long long m0 = ch * MC;
        for (int f = tid; f < MC * TJ / 4; f += 256) {
            const int r = f / (TJ / 4), c4 = f % (TJ / 4);
            float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
            if (m0 + r < M) {
                va = *reinterpret_cast<const float4 *>(dh2 + (size_t)(m0 + r) * W + j0 + c4 * 4);
                vb = *reinterpret_cast<const float4 *>(h1 + (size_t)(m0 + r) * W + k0 + c4 * 4);
            }
            *reinterpret_cast<float4 *>(&As[r][c4 * 4]) = va;
            *reinterpret_cast<float4 *>(&Bs[r][c4 * 4]) = vb;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < MC; ++r) {
            float a[MT], b[MT];
#pragma unroll
            for (int i = 0; i < MT; ++i) { a[i] = As[r][col(ty, i)]; b[i] = Bs[r][col(tx, i)]; }
#pragma unroll
            for (int i = 0; i < MT; ++i)
#pragma unroll
                for (int q = 0; q < MT; ++q) acc[i][q] = fmaf(a[i], b[q], acc[i][q]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int q = 0; q < MT; ++q) atomicAdd(gW1 + (size_t)(j0 + col(ty, i)) * W + k0 + col(tx, q), acc[i][q]);
}

__global__ void k_transpose(int rows, int cols, const float *__restrict__ in, float *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < rows * cols) {
        const int r = i / cols, c = i % cols;
        out[(size_t)c * rows + r] = in[i];
    }
}

template <int W, bool TRAIN, bool WGRAD, bool SEG = false>
int launch_mlp(const MlpParams &p, cudaStream_t stream) {
    const size_t smem = Cfg<W>::smem_floats(WGRAD) * sizeof(float);
    static NlPerDevice configured;
    const cudaError_t e = configured.once([&] { return cudaFuncSetAttribute(k_mlp<W, TRAIN, WGRAD, SEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); });
    if (e != cudaSuccess) return nl_set_error_code(NL_ERR_CUDA, cudaGetErrorString(e));
    const long long ntiles = (p.M_host + T_TILE - 1) / T_TILE;
    const int grid = (int)(ntiles < (long long)nl_num_sms() ? ntiles : (long long)nl_num_sms());
    k_mlp<W, TRAIN, WGRAD, SEG><<<grid, NTHREADS, smem, stream>>>(p);
    return NL_OK;
}

template <bool TRAIN, bool WGRAD, bool SEG = false>
int dispatch_width(const MlpParams &p, cudaStream_t stream) {
    switch (p.w.width) {
        case 256: return launch_mlp<256, TRAIN, WGRAD, SEG>(p, stream);
        case 128: return launch_mlp<128, TRAIN, WGRAD, SEG>(p, stream);
        case 64: return launch_mlp<64, TRAIN, WGRAD, SEG>(p, stream);
        case 32: return launch_mlp<32, TRAIN, WGRAD, SEG>(p, stream);
        default: return nl_set_error_code(NL_ERR_UNSUPPORTED, "decoder width must be 32, 64, 128 or 256");
    }
}

bool weights_ok(const nl_mlp_weights *w) {
    return w && w->W0 && w->b0 && w->W1 && w->b1 && w->W2 && w->b2 && w->W0t && w->W1t;
}

}  // namespace

extern "C" int nl_mlp_prepare(int32_t width, const float *W0, const float *W1, float *W0t, float *W1t, void *stream) {
    if (width <= 0 || !W0 || !W1 || !W0t || !W1t) return nl_set_error("nl_mlp_prepare: bad arguments");
    k_transpose<<<nl_div_up((int64_t)width * 16, 256), 256, 0, (cudaStream_t)stream>>>(width, 16, W0, W0t);
    k_transpose<<<nl_div_up((int64_t)width * width, 256), 256, 0, (cudaStream_t)stream>>>(width, width, W1, W1t);
    NL_CHECK_LAUNCH("nl_mlp_prepare");
    return NL_OK;
}

extern "C" int nl_mlp_forward(int64_t M, const int32_t *d_M_dev, const float *feats, const nl_mlp_weights *w, float *sdf,
                              void *stream) {
    if (M < 0) return nl_set_error("nl_mlp_forward: negative M");
    if (M == 0) return NL_OK;
    if (!feats || !sdf || !weights_ok(w)) return nl_set_error("nl_mlp_forward: null pointer");
    MlpParams p = {};
    p.M_host = M; p.M_dev = d_M_dev; p.feats = feats; p.w = *w; p.sdf = sdf;
    int rc = dispatch_width<false, false>(p, (cudaStream_t)stream);
    if (rc != NL_OK) return rc;
    NL_CHECK_LAUNCH("nl_mlp_forward");
    return NL_OK;
}

extern "C" int nl_mlp_train(int64_t M, const int32_t *d_M_dev, const float *feats, const nl_mlp_weights *w,
                            const uint8_t *s_flag, const float *s_depth, const int32_t *s_ray, const float *cosv,
                            const float *gt_depth, nl_render_stats *stats, float truncation, float *sdf, float *dfeats,
                            const nl_mlp_grads *grads, float *act_h1, float *act_dh2, const float *dsdf_ext, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (M < 0) return nl_set_error("nl_mlp_train: negative M");
    if (M == 0) return NL_OK;
    if (!feats || !sdf || !dfeats || !weights_ok(w)) return nl_set_error("nl_mlp_train: null pointer");
    if (!dsdf_ext && (!s_flag || !s_depth || !s_ray || !gt_depth || !stats))
        return nl_set_error("nl_mlp_train: the loss needs s_flag, s_depth, s_ray, gt_depth and stats");
    MlpParams p = {};
    p.M_host = M; p.M_dev = d_M_dev; p.feats = feats; p.w = *w; p.sdf = sdf;
    p.s_flag = s_flag; p.s_depth = s_depth; p.s_ray = s_ray; p.cosv = cosv; p.gt_depth = gt_depth; p.stats = stats;
    p.truncation = truncation; p.dfeats = dfeats; p.dsdf_ext = dsdf_ext;
    int rc;
    if (grads) {
        if (!grads->gW0 || !grads->gb0 || !grads->gW1 || !grads->gb1 || !grads->gW2 || !grads->gb2 || !act_h1 || !act_dh2)
            return nl_set_error("nl_mlp_train: decoder gradients requested but a buffer is null");
        p.g = *grads; p.act_h1 = act_h1; p.act_dh2 = act_dh2;
        rc = dispatch_width<true, true>(p, stream);
        if (rc != NL_OK) return rc;
        const int W = w->width;
        const int tj = W >= 128 ? 128 : W, tiles = (W / tj) * (W / tj);
        int nsplit = nl_num_sms() / tiles;
        if (nsplit < 1) nsplit = 1;
        switch (W) {
            case 256: k_dw1<256><<<tiles * nsplit, 256, 0, stream>>>(M, d_M_dev, act_dh2, act_h1, grads->gW1, nsplit); break;
            case 128: k_dw1<128><<<tiles * nsplit, 256, 0, stream>>>(M, d_M_dev, act_dh2, act_h1, grads->gW1, nsplit); break;
            case 64: k_dw1<64><<<tiles * nsplit, 256, 0, stream>>>(M, d_M_dev, act_dh2, act_h1, grads->gW1, nsplit); break;
            case 32: k_dw1<32><<<tiles * nsplit, 256, 0, stream>>>(M, d_M_dev, act_dh2, act_h1, grads->gW1, nsplit); break;
        }
    } else {
        rc = dispatch_width<true, false>(p, stream);
        if (rc != NL_OK) return rc;
    }
    NL_CHECK_LAUNCH("nl_mlp_train");
    return NL_OK;
}

extern "C" int nl_mlp_train_batch(int64_t M, const int32_t *d_M_dev, const float *feats, const nl_mlp_weights *w, const uint8_t *s_flag,
                                  const float *s_depth, const int32_t *s_ray, const float *cosv, const float *gt_depth,
                                  nl_render_stats *problem_stats, int32_t rays_per_problem, float truncation, float *sdf, float *dfeats,
                                  void *stream) {
    if (M < 0) return nl_set_error("nl_mlp_train_batch: negative M");
    if (rays_per_problem <= 0) return nl_set_error("nl_mlp_train_batch: rays_per_problem must be positive");
    if (M == 0) return NL_OK;
    if (!feats || !sdf || !dfeats || !weights_ok(w) || !s_flag || !s_depth || !s_ray || !gt_depth || !problem_stats)
        return nl_set_error("nl_mlp_train_batch: null pointer");
    MlpParams p = {};
    p.M_host = M; p.M_dev = d_M_dev; p.feats = feats; p.w = *w; p.sdf = sdf;
    p.s_flag = s_flag; p.s_depth = s_depth; p.s_ray = s_ray; p.cosv = cosv; p.gt_depth = gt_depth; p.stats = problem_stats;
    p.truncation = truncation; p.dfeats = dfeats; p.seg_rays = rays_per_problem;
    if (int rc = dispatch_width<true, false, true>(p, (cudaStream_t)stream)) return rc;
    NL_CHECK_LAUNCH("nl_mlp_train_batch");
    return NL_OK;
}
