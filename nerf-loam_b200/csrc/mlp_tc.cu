// Tensor-core version of the SDF decoder MLP (16 -> 256 -> 256 -> 1, ReLU) for sm_90a: Hopper wgmma (m64nNk8, tf32
// inputs, fp32 accumulation in registers) with a 3-term hi/lo split (3xTF32: a*b ~= ah*bh + ah*bl + al*bh), which keeps
// the result within ~1e-6 of an fp32 evaluation -- single-pass TF32 (1e-3) would break the 1e-5 SDF parity bar.
//
// One persistent CTA per SM, two warpgroups; each warpgroup owns 64 samples of a 128-sample tile end to end.
//   * A operands come from registers.  A layer's fp32 accumulator fragment (thread holds columns 8j+2t, 8j+2t+1 of rows g
//     and g+8) is, up to a fixed permutation of K inside every group of 8 (kperm), the tf32 A fragment of the next GEMM
//     (columns t, t+4), so activations never go through shared memory.  The weight panels carry the same permutation.
//   * B operands (weights, pre-split into tf32 hi/lo and pre-swizzled into the 128B-swizzle K-major image wgmma reads,
//     k_tc_prepare) stream from L2 through a 4-slot shared-memory ring: 1-D bulk copies (TMA) completing on mbarriers,
//     issued by thread 0 up to 3 slots ahead; a slot is refilled once the wgmmas of all 8 warps that read it retired.
//   * Every N = 256 GEMM runs as two N = 128 halves, so the previous layer's activations (128 registers per thread) and
//     one accumulator half (64) fit in the register file together.
// Per 128-sample training tile the ring carries 42 items: layer 1 (2 halves), layer 2 (2 halves x 8 K-blocks of 32),
// backward layer 2 (2 x 8) and backward layer 1 (8 K-blocks, N = 16).
//
// Decoder weight gradients (nl_mlp_tc_train with grads): the training kernel stores h1, h2, dh2, dh1 [cap][256] and
// d loss / d sdf; gW1 = dh2^T h1 (K = samples) is a split-K 3xTF32 tensor-core GEMM (k_dw1_tc, mma.sync m16n8k8: both
// operands are sample-major, which wgmma's tf32 forms cannot read), the column sums and gW0 (K = 16) come from one
// streaming pass (k_wg_cols).
#include <mutex>

#include "nl_cuda.cuh"

namespace tc {

constexpr int TM = 128;                  // samples per CTA tile (2 warpgroups x 64)
constexpr int WN = 256;                  // hidden width
constexpr int PANEL_B = WN * 128;        // 32 KB: one weight K-block (256 rows x 32 tf32), hi or lo
constexpr int STAGE_B = 2 * PANEL_B;     // hi + lo, in global memory
constexpr int HALF = 128 * 128;          // 16 KB: 128 rows of a panel (one N = 128 half)
constexpr int SLOT = 2 * HALF;           // ring slot: hi half | lo half
constexpr int NSLOT = 4;
constexpr int STEPS_TRAIN = 25;          // panel stages: layer 1, 8 x layer 2, 8 x backward layer 2, 8 x backward layer 1
constexpr int ITEMS_FWD = 18;
constexpr int ITEMS_TRAIN = 42;
constexpr int NTHREADS = 256;
constexpr int SMEM_TOTAL = NSLOT * SLOT + 3 * WN * 4 + 256 + 1024;   // ring + biases/w2 + barriers + alignment slack

// byte offset of 16-byte chunk c (0..7) of row r inside a K-major SWIZZLE_128B panel
__host__ __device__ __forceinline__ int panel_off(int r, int c) { return (r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4); }
// logical K index stored at panel position k: inside every group of 8, positions 0..3 hold the even, 4..7 the odd columns
__host__ __device__ __forceinline__ int kperm(int k) { const int p = k & 7; return (k & ~7) | (p < 4 ? 2 * p : 2 * (p - 4) + 1); }

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint32_t tf32_rna(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return u;
}

// ---- mbarrier / bulk-copy helpers ------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("{ .reg .b64 st; mbarrier.arrive.shared::cta.b64 st, [%0]; }" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("{ .reg .b64 st; mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1; }" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(bar) : "memory");
}

// ---- wgmma -------------------------------------------------------------------------------------------
// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90): start>>4 [0,14), LBO>>4 [16,30) (unused for swizzled
// K-major, 1), SBO>>4 = 1024>>4 [32,46) (8-row core-matrix groups), layout SWIZZLE_128B = 1 [62,64).  One k-step of 8 tf32
// is 32 bytes further along the row: +2 in the address field.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit_wait() {
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(1));
}
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(1));
}

// A fragment of k-step j of `h` (a 256-column array in accumulator layout, index 4j + x: x = 0,1 row g columns 8j+2t, +1;
// x = 2,3 row g+8) as tf32 hi and lo parts.  Hardware K position t holds column 8j+2t, t+4 holds 8j+2t+1 (see kperm).
__device__ __forceinline__ void frag3(const float (&h)[128], int j, uint32_t (&hi)[4], uint32_t (&lo)[4]) {
    const float v[4] = {h[4 * j], h[4 * j + 2], h[4 * j + 1], h[4 * j + 3]};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        hi[i] = tf32_rna(v[i]);
        lo[i] = tf32_rna(v[i] - __uint_as_float(hi[i]));
    }
}
// D[64 x N] += A x B with 3 terms: ah*bh + ah*bl + al*bh
template <int NACC>
__device__ __forceinline__ void mma3(float (&d)[NACC], const uint32_t (&a)[4], const uint32_t (&l)[4], uint64_t bh, uint64_t bl) {
    if constexpr (NACC == 64) {
        wgmma_n128(d, a[0], a[1], a[2], a[3], bh);
        wgmma_n128(d, a[0], a[1], a[2], a[3], bl);
        wgmma_n128(d, l[0], l[1], l[2], l[3], bh);
    } else {
        wgmma_n16(d, a[0], a[1], a[2], a[3], bh);
        wgmma_n16(d, a[0], a[1], a[2], a[3], bl);
        wgmma_n16(d, l[0], l[1], l[2], l[3], bh);
    }
}
template <int NACC>
__device__ __forceinline__ float (&sub64(float (&a)[NACC], int off))[64] { return *reinterpret_cast<float(*)[64]>(a + off); }

// ------------------------------------------------------------------------------------------------
// Weight panels: the exact shared-memory image (K-major, 128B swizzle, K permuted by kperm, tf32 hi then lo) of every
// weight K-block, laid out contiguously in global memory so that bulk copies fill a ring slot.
//   stage 0       : W0  [256 x 16]  (row j, k = e; only the first 64 B of each 128 B row are meaningful)
//   stage 1 + kb  : W1[:, 32kb : 32kb+32]              forward layer 2
//   stage 9 + jb  : (diag(w2) W1)^T[:, 32jb : 32jb+32] backward layer 2 (d h1 = dsdf * (relu'(h2) . diag(w2) W1) * relu'(h1))
//   stage 17 + kb : W0^T[:, 32kb : 32kb+32] (16 rows)  backward layer 1 (d x  = d h1 . W0)
// ------------------------------------------------------------------------------------------------
__global__ void k_tc_prepare(const float *__restrict__ W0, const float *__restrict__ W1, const float *__restrict__ w2,
                             uint8_t *__restrict__ panels) {
    const int stage = blockIdx.y;                         // 0..24
    const int t = blockIdx.x * blockDim.x + threadIdx.x;  // (row, chunk)
    if (t >= WN * 8) return;
    const int r = t >> 3, c = t & 7;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (stage >= 17 && r >= 16) return;
    for (int i = 0; i < 4; ++i) {
        const int k = kperm(c * 4 + i);                   // logical K index inside the 32-wide block
        if (stage == 0) {                                 // layer 1:   B[j][e] = W0[j][e]
            if (c < 4) v[i] = W0[r * 16 + k];
        } else if (stage <= 8) {                          // layer 2:   B[j][k] = W1[j][k]
            v[i] = W1[(size_t)r * WN + (stage - 1) * 32 + k];
        } else if (stage <= 16) {                         // bwd layer 2: B[k][j] = w2[j] W1[j][k]
            const int j = (stage - 9) * 32 + k;
            v[i] = __fmul_rn(w2[j], W1[(size_t)j * WN + r]);
        } else {                                          // bwd layer 1: B[e][k] = W0[k][e]
            v[i] = W0[(size_t)((stage - 17) * 32 + k) * 16 + r];
        }
    }
    float hi[4], lo[4];
    for (int i = 0; i < 4; ++i) { hi[i] = __uint_as_float(tf32_rna(v[i])); lo[i] = __uint_as_float(tf32_rna(v[i] - hi[i])); }
    uint8_t *base = panels + (size_t)stage * STAGE_B;
    *reinterpret_cast<float4 *>(base + panel_off(r, c)) = make_float4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<float4 *>(base + PANEL_B + panel_off(r, c)) = make_float4(lo[0], lo[1], lo[2], lo[3]);
}

struct Params {
    long long M_host;
    const int32_t *M_dev;
    const float *feats;        // [M,16]
    const uint8_t *panels;     // 25 stages x 64 KB
    const float *b0, *b1, *w2, *b2;
    float *sdf, *dfeats;
    const uint8_t *s_flag;
    const float *s_depth;
    const int32_t *s_ray;
    const float *cosv, *gt_depth;
    nl_render_stats *stats;
    float truncation;
    const float *dsdf_ext;
    float *act_h1, *act_h2, *act_dh2, *act_dh1, *act_d;   // WGRAD: [cap][256] x 4, [cap]
};

// ring item i of a tile -> panel stage and N half
__device__ __forceinline__ void item_of(int i, int &stage, int &half) {
    if (i < 2) { stage = 0; half = i; }
    else if (i < 18) { half = (i - 2) >> 3; stage = 1 + ((i - 2) & 7); }
    else if (i < 34) { half = (i - 18) >> 3; stage = 9 + ((i - 18) & 7); }
    else { half = 0; stage = 17 + (i - 34); }
}

template <bool TRAIN, bool WGRAD>
__global__ void __launch_bounds__(NTHREADS, 1) k_mlp_wg(Params p) {
    constexpr int IPT = TRAIN ? ITEMS_TRAIN : ITEMS_FWD;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;    // SWIZZLE_128B panels need 1024-byte alignment
    uint8_t *sm = smem_raw + (base - raw);
    const uint32_t ring = base;
    float *b0s = reinterpret_cast<float *>(sm + NSLOT * SLOT);
    float *b1s = b0s + WN;
    float *w2s = b1s + WN;
    const uint32_t bar0 = smem_u32(w2s + WN);       // FULL[s] at 8s, EMPTY[s] at 8 (NSLOT + s)
    auto FULL = [&](uint32_t s) { return bar0 + 8u * s; };
    auto EMPTY = [&](uint32_t s) { return bar0 + 8u * (NSLOT + s); };

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const long long M = p.M_dev ? min((long long)*p.M_dev, p.M_host) : p.M_host;
    const long long ntiles = (M + TM - 1) / TM;
    const long long my_tiles = (long long)blockIdx.x < ntiles ? (ntiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const uint32_t total = (uint32_t)(my_tiles * IPT);

    for (int i = tid; i < WN; i += NTHREADS) { b0s[i] = p.b0[i]; b1s[i] = p.b1[i]; w2s[i] = p.w2[i]; }
    if (tid == 0) {
        for (int s = 0; s < NSLOT; ++s) { mbar_init(FULL(s), 1); mbar_init(EMPTY(s), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // thread 0 feeds the ring: item n is always issued before anyone waits for it; items up to n + NSLOT - 1 are issued
    // when their slot is already free (non-blocking test), so the copies run ahead of the MMAs
    uint32_t issued = 0;
    auto issue = [&](uint32_t n) {
        const uint32_t s = n % NSLOT;
        mbar_wait(EMPTY(s), ((n / NSLOT) & 1) ^ 1);
        int stage, half;
        item_of((int)(n % IPT), stage, half);
        const uint32_t bytes = stage >= 17 ? 16 * 128 : HALF;
        mbar_expect_tx(FULL(s), 2 * bytes);
        const uint8_t *src = p.panels + (size_t)stage * STAGE_B + half * HALF;
        bulk_g2s(ring + s * SLOT, src, bytes, FULL(s));
        bulk_g2s(ring + s * SLOT + HALF, src + PANEL_B, bytes, FULL(s));
    };
    uint32_t n = 0;   // ring items consumed by this thread
    // wait for item n; returns the descriptors of its hi and lo halves.  The caller computes its A fragments first and then
    // issues wgmma.fence (registers written after the fence may not feed the wgmmas behind it)
    auto acquire = [&](uint64_t &bh, uint64_t &bl) {
        if (tid == 0) {
            while (issued < total && issued < n + NSLOT) {
                if (issued > n && !mbar_test(EMPTY(issued % NSLOT), ((issued / NSLOT) & 1) ^ 1)) break;
                issue(issued++);
            }
        }
        __syncwarp();
        const uint32_t s = n % NSLOT;
        mbar_wait(FULL(s), (n / NSLOT) & 1);
        bh = make_desc(ring + s * SLOT);
        bl = make_desc(ring + s * SLOT + HALF);
    };
    auto release = [&]() {
        wg_commit_wait();
        __syncwarp();
        if (lane == 0) mbar_arrive(EMPTY(n % NSLOT));
        ++n;
    };

    const float b2 = p.b2[0];
    float g_fs = 0.f, g_sdf = 0.f;
    if (TRAIN && !p.dsdf_ext) { g_fs = p.stats->g_fs; g_sdf = p.stats->g_sdf; }
    double loss_fs = 0.0, loss_sdf = 0.0;

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long m0 = tile * TM + warp * 16 + g, m1 = m0 + 8;   // this thread's two rows
        const bool live0 = m0 < M, live1 = m1 < M;

        // ---- layer 1: D1 = x . W0^T (K = 16: two k-steps; A fragment of k-step ks = columns 8ks+2t, 8ks+2t+1) ----
        float h[128];
        {
            float xa[8];
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                const float2 r0 = live0 ? *reinterpret_cast<const float2 *>(p.feats + (size_t)m0 * 16 + 8 * ks + 2 * t) : make_float2(0.f, 0.f);
                const float2 r1 = live1 ? *reinterpret_cast<const float2 *>(p.feats + (size_t)m1 * 16 + 8 * ks + 2 * t) : make_float2(0.f, 0.f);
                xa[4 * ks] = r0.x; xa[4 * ks + 1] = r0.y; xa[4 * ks + 2] = r1.x; xa[4 * ks + 3] = r1.y;
            }
            float xh[128];   // only the first 8 entries are used: frag3 reads a k-step's fragment from a 128-entry array
#pragma unroll
            for (int i = 0; i < 8; ++i) xh[i] = xa[i];
#pragma unroll
            for (int i = 0; i < 128; ++i) h[i] = 0.f;
            uint32_t ah[2][4], al[2][4];
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) frag3(xh, ks, ah[ks], al[ks]);
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                uint64_t bh, bl;
                acquire(bh, bl);
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < 2; ++ks) mma3<64>(sub64(h, 64 * half), ah[ks], al[ks], bh + 2 * ks, bl + 2 * ks);
                release();
            }
        }
        // h1 = relu(D1 + b0), relu'(h1) bits: bit (4j + x) of the 128-bit mask
        uint32_t mask1[4] = {0u, 0u, 0u, 0u}, mask2[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int j = 0; j < 32; ++j)
#pragma unroll
            for (int x = 0; x < 4; ++x) {
                const float v = h[4 * j + x] + b0s[8 * j + 2 * t + (x & 1)];
                const bool on = v > 0.f;
                h[4 * j + x] = on ? v : 0.f;
                if (on) mask1[j >> 3] |= 1u << ((j & 7) * 4 + x);
            }
        if (WGRAD) {
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                if (live0) *reinterpret_cast<float2 *>(p.act_h1 + (size_t)m0 * WN + 8 * j + 2 * t) = make_float2(h[4 * j], h[4 * j + 1]);
                if (live1) *reinterpret_cast<float2 *>(p.act_h1 + (size_t)m1 * WN + 8 * j + 2 * t) = make_float2(h[4 * j + 2], h[4 * j + 3]);
            }
        }

        // ---- layer 2 (two N halves) + output layer partial sums ----
        float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            float d[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) d[i] = 0.f;
#pragma unroll
            for (int kb = 0; kb < 8; ++kb) {
                uint32_t ah[4][4], al[4][4];
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) frag3(h, 4 * kb + ks, ah[ks], al[ks]);
                uint64_t bh, bl;
                acquire(bh, bl);
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) mma3<64>(d, ah[ks], al[ks], bh + 2 * ks, bl + 2 * ks);
                release();
            }
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
#pragma unroll
                for (int x = 0; x < 4; ++x) {
                    const int col = 128 * half + 8 * jj + 2 * t + (x & 1), j = 16 * half + jj;
                    const float v = d[4 * jj + x] + b1s[col];
                    const bool on = v > 0.f;
                    const float hv = on ? v : 0.f;
                    d[4 * jj + x] = hv;
                    if (on) mask2[j >> 3] |= 1u << ((j & 7) * 4 + x);
                    if (x < 2) ps0 = fmaf(hv, w2s[col], ps0); else ps1 = fmaf(hv, w2s[col], ps1);
                }
            if (WGRAD) {
#pragma unroll
                for (int jj = 0; jj < 16; ++jj) {
                    const int col = 128 * half + 8 * jj + 2 * t;
                    if (live0) *reinterpret_cast<float2 *>(p.act_h2 + (size_t)m0 * WN + col) = make_float2(d[4 * jj], d[4 * jj + 1]);
                    if (live1) *reinterpret_cast<float2 *>(p.act_h2 + (size_t)m1 * WN + col) = make_float2(d[4 * jj + 2], d[4 * jj + 3]);
                }
            }
        }
        // the 4 threads of a quad hold the 4 column classes of the same two rows
        ps0 += __shfl_xor_sync(0xffffffffu, ps0, 1); ps0 += __shfl_xor_sync(0xffffffffu, ps0, 2);
        ps1 += __shfl_xor_sync(0xffffffffu, ps1, 1); ps1 += __shfl_xor_sync(0xffffffffu, ps1, 2);
        const float sdf0 = ps0 + b2, sdf1 = ps1 + b2;
        if (t == 0) {
            if (live0) p.sdf[m0] = sdf0;
            if (live1) p.sdf[m1] = sdf1;
        }
        if constexpr (TRAIN) {
            // ---- loss (criterion.py:92-103) and d loss / d sdf for both rows ----
            float dsdf[2] = {0.f, 0.f};
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const long long m = r ? m1 : m0;
                const float s = r ? sdf1 : sdf0;
                if (!(r ? live1 : live0)) continue;
                if (p.dsdf_ext) { dsdf[r] = p.dsdf_ext[m]; continue; }
                const uint32_t fl = p.s_flag[m];
                const int ray = p.s_ray[m];
                const float z = __fmul_rn(p.s_depth[m], p.cosv ? p.cosv[ray] : 1.0f);
                const float dgt = p.gt_depth[ray];
                if (fl & 1u) {
                    const float e = s - 1.0f;
                    if (t == 0) loss_fs += (double)e * (double)e;
                    dsdf[r] += 2.0f * g_fs * e;
                }
                if (fl & 2u) {
                    const float e = __fsub_rn(__fadd_rn(z, __fmul_rn(s, p.truncation)), dgt);
                    if (t == 0) loss_sdf += (double)e * (double)e;
                    dsdf[r] += 2.0f * g_sdf * p.truncation * e;
                }
            }
            if (WGRAD) {
                if (t == 0) {
                    if (live0) p.act_d[m0] = dsdf[0];
                    if (live1) p.act_d[m1] = dsdf[1];
                }
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const int col = 8 * j + 2 * t;
                    float v[4];
#pragma unroll
                    for (int x = 0; x < 4; ++x)
                        v[x] = ((mask2[j >> 3] >> ((j & 7) * 4 + x)) & 1u) ? dsdf[x >> 1] * w2s[col + (x & 1)] : 0.f;
                    if (live0) *reinterpret_cast<float2 *>(p.act_dh2 + (size_t)m0 * WN + col) = make_float2(v[0], v[1]);
                    if (live1) *reinterpret_cast<float2 *>(p.act_dh2 + (size_t)m1 * WN + col) = make_float2(v[2], v[3]);
                }
            }
            // ---- backward layer 2: D3 = relu'(h2) . (diag(w2) W1).  The A operand is the 0/1 mask (exact in tf32: 2 terms) ----
#pragma unroll
            for (int i = 0; i < 128; ++i) h[i] = 0.f;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
#pragma unroll
                for (int kb = 0; kb < 8; ++kb) {
                    uint32_t a[4][4];
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) {
                        const int j = 4 * kb + ks;
                        const uint32_t w = mask2[j >> 3] >> ((j & 7) * 4);
                        a[ks][0] = (w & 1u) ? 0x3f800000u : 0u; a[ks][1] = (w & 4u) ? 0x3f800000u : 0u;
                        a[ks][2] = (w & 2u) ? 0x3f800000u : 0u; a[ks][3] = (w & 8u) ? 0x3f800000u : 0u;
                    }
                    uint64_t bh, bl;
                    acquire(bh, bl);
                    wg_fence();
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) {
                        wgmma_n128(sub64(h, 64 * half), a[ks][0], a[ks][1], a[ks][2], a[ks][3], bh + 2 * ks);
                        wgmma_n128(sub64(h, 64 * half), a[ks][0], a[ks][1], a[ks][2], a[ks][3], bl + 2 * ks);
                    }
                    release();
                }
            }
            // dh1 = dsdf * D3 * relu'(h1)
#pragma unroll
            for (int j = 0; j < 32; ++j)
#pragma unroll
                for (int x = 0; x < 4; ++x)
                    h[4 * j + x] = ((mask1[j >> 3] >> ((j & 7) * 4 + x)) & 1u) ? dsdf[x >> 1] * h[4 * j + x] : 0.f;
            if (WGRAD) {
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    if (live0) *reinterpret_cast<float2 *>(p.act_dh1 + (size_t)m0 * WN + 8 * j + 2 * t) = make_float2(h[4 * j], h[4 * j + 1]);
                    if (live1) *reinterpret_cast<float2 *>(p.act_dh1 + (size_t)m1 * WN + 8 * j + 2 * t) = make_float2(h[4 * j + 2], h[4 * j + 3]);
                }
            }
            // ---- backward layer 1: d x = dh1 . W0 (N = 16) ----
            float dx[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) dx[i] = 0.f;
#pragma unroll
            for (int kb = 0; kb < 8; ++kb) {
                uint32_t ah[4][4], al[4][4];
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) frag3(h, 4 * kb + ks, ah[ks], al[ks]);
                uint64_t bh, bl;
                acquire(bh, bl);
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) mma3<8>(dx, ah[ks], al[ks], bh + 2 * ks, bl + 2 * ks);
                release();
            }
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
                if (live0) *reinterpret_cast<float2 *>(p.dfeats + (size_t)m0 * 16 + 8 * jj + 2 * t) = make_float2(dx[4 * jj], dx[4 * jj + 1]);
                if (live1) *reinterpret_cast<float2 *>(p.dfeats + (size_t)m1 * 16 + 8 * jj + 2 * t) = make_float2(dx[4 * jj + 2], dx[4 * jj + 3]);
            }
        }
    }
    if (TRAIN && !p.dsdf_ext) {
        for (int off = 16; off > 0; off >>= 1) {
            loss_fs += __shfl_down_sync(0xffffffffu, loss_fs, off);
            loss_sdf += __shfl_down_sync(0xffffffffu, loss_sdf, off);
        }
        if (lane == 0) {
            if (loss_fs != 0.0) atomicAdd(&p.stats->fs_sum, loss_fs);
            if (loss_sdf != 0.0) atomicAdd(&p.stats->sdf_sum, loss_sdf);
        }
    }
}

// gW1[j][k] += sum_s dh2[s][j] h1[s][k]: CTA = 128 x 128 output tile, split-K over samples (grid = 4 tiles x nsplit, one CTA
// per SM: 148 registers per thread).
// Chunks of 32 samples of both operands are double-buffered in shared memory by cp.async (rows padded to 136 floats: the
// fragment loads (sample t / t+4, column g) hit 32 distinct banks); warp w owns rows 64 (w & 1) .. +63 and columns
// 32 (w >> 1) .. +31 of the tile, 4 x 4 m16n8 accumulators.  hi/lo split of both operands at fragment load.
constexpr int DW_KC = 32, DW_LD = 136;
constexpr int DW_SMEM = 2 * 2 * DW_KC * DW_LD * 4;   // 68 KB: 2 operands x 2 buffers
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__global__ void __launch_bounds__(256) k_dw1_tc(long long M_host, const int32_t *__restrict__ M_dev, const float *__restrict__ dh2,
                                                const float *__restrict__ h1, float *__restrict__ gW1, int nsplit) {
    extern __shared__ float4 dw_smem[];
    auto As = reinterpret_cast<float(*)[DW_KC][DW_LD]>(dw_smem);
    auto Bs = reinterpret_cast<float(*)[DW_KC][DW_LD]>(reinterpret_cast<float *>(dw_smem) + 2 * DW_KC * DW_LD);
    const long long M = M_dev ? min((long long)*M_dev, M_host) : M_host;
    const int tile = blockIdx.x & 3, split = blockIdx.x >> 2;
    const int j0 = (tile >> 1) * 128, k0 = (tile & 1) * 128;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int wj = (warp & 1) * 64, wk = (warp >> 1) * 32;
    float acc[4][4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
    const long long nch = (M + DW_KC - 1) / DW_KC;
    auto load = [&](long long ch, int buf) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int f = tid + i * 256, r = f >> 5, c4 = (f & 31) * 4;   // 32 rows x 32 float4
            const long long s = ch * DW_KC + r;
            const bool v = s < M;
            const size_t o = (size_t)(v ? s : 0) * WN;
            cp_async16(smem_u32(&As[buf][r][c4]), dh2 + o + j0 + c4, v);
            cp_async16(smem_u32(&Bs[buf][r][c4]), h1 + o + k0 + c4, v);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    int buf = 0;
    if (split < nch) load(split, 0);
    for (long long ch = split; ch < nch; ch += nsplit, buf ^= 1) {
        if (ch + nsplit < nch) {
            load(ch + nsplit, buf ^ 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
#pragma unroll
        for (int ks = 0; ks < DW_KC / 8; ++ks) {
            const int s0 = ks * 8 + t;
            uint32_t ah[4][4], al[4][4], bh[4][2], bl[4][2];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi) {
                const int j = wj + mi * 16 + g;
                const float v[4] = {As[buf][s0][j], As[buf][s0][j + 8], As[buf][s0 + 4][j], As[buf][s0 + 4][j + 8]};
#pragma unroll
                for (int i = 0; i < 4; ++i) { ah[mi][i] = tf32_rna(v[i]); al[mi][i] = tf32_rna(v[i] - __uint_as_float(ah[mi][i])); }
            }
#pragma unroll
            for (int ni = 0; ni < 4; ++ni) {
                const int n = wk + ni * 8 + g;
                const float v[2] = {Bs[buf][s0][n], Bs[buf][s0 + 4][n]};
#pragma unroll
                for (int i = 0; i < 2; ++i) { bh[ni][i] = tf32_rna(v[i]); bl[ni][i] = tf32_rna(v[i] - __uint_as_float(bh[ni][i])); }
            }
#pragma unroll
            for (int mi = 0; mi < 4; ++mi)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    mma_tf32(acc[mi][ni], ah[mi], bh[ni][0], bh[ni][1]);
                    mma_tf32(acc[mi][ni], ah[mi], bl[ni][0], bl[ni][1]);
                    mma_tf32(acc[mi][ni], al[mi], bh[ni][0], bh[ni][1]);
                }
        }
        __syncthreads();
    }
    if (split >= nch) return;
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
            const int j = j0 + wj + mi * 16 + g, k = k0 + wk + ni * 8 + 2 * t;
            atomicAdd(gW1 + (size_t)j * WN + k, acc[mi][ni][0]);
            atomicAdd(gW1 + (size_t)j * WN + k + 1, acc[mi][ni][1]);
            atomicAdd(gW1 + (size_t)(j + 8) * WN + k, acc[mi][ni][2]);
            atomicAdd(gW1 + (size_t)(j + 8) * WN + k + 1, acc[mi][ni][3]);
        }
}

// Column sums of the stored activations, thread = column k, one contiguous range of samples per CTA:
//   gW0[k][e] += sum_s dh1[s][k] x[s][e]   gb0[k] += sum_s dh1[s][k]   gW2[k] += sum_s d[s] h2[s][k]
//   gb1[k]    += sum_s dh2[s][k]           gb2    += sum_s d[s]
constexpr int COLS_CHUNK = 64;
__global__ void __launch_bounds__(WN) k_wg_cols(long long M_host, const int32_t *__restrict__ M_dev, const float *__restrict__ feats,
                                                const float *__restrict__ dh1, const float *__restrict__ h2, const float *__restrict__ dh2,
                                                const float *__restrict__ d, nl_mlp_grads g) {
    __shared__ float xs[COLS_CHUNK][16];
    __shared__ float ds[COLS_CHUNK];
    const long long M = M_dev ? min((long long)*M_dev, M_host) : M_host;
    const long long per = ((M + gridDim.x - 1) / gridDim.x + COLS_CHUNK - 1) / COLS_CHUNK * COLS_CHUNK;
    const long long s0 = (long long)blockIdx.x * per, s1 = min(M, s0 + per);
    const int k = threadIdx.x;
    float gw0[16], gb0 = 0.f, gw2 = 0.f, gb1 = 0.f, gb2 = 0.f;
#pragma unroll
    for (int e = 0; e < 16; ++e) gw0[e] = 0.f;
    for (long long c0 = s0; c0 < s1; c0 += COLS_CHUNK) {
        const int n = (int)min((long long)COLS_CHUNK, s1 - c0);
        __syncthreads();
        for (int i = k; i < n * 16; i += WN) xs[i >> 4][i & 15] = feats[(size_t)c0 * 16 + i];
        if (k < n) ds[k] = d[c0 + k];
        __syncthreads();
        for (int i = 0; i < n; ++i) {
            const size_t o = (size_t)(c0 + i) * WN + k;
            const float a = dh1[o];
#pragma unroll
            for (int e = 0; e < 16; ++e) gw0[e] = fmaf(a, xs[i][e], gw0[e]);
            gb0 += a;
            gw2 = fmaf(ds[i], h2[o], gw2);
            gb1 += dh2[o];
            if (k == 0) gb2 += ds[i];
        }
    }
    if (s0 >= s1) return;
#pragma unroll
    for (int e = 0; e < 16; ++e) atomicAdd(g.gW0 + k * 16 + e, gw0[e]);
    atomicAdd(g.gb0 + k, gb0);
    atomicAdd(g.gW2 + k, gw2);
    atomicAdd(g.gb1 + k, gb1);
    if (k == 0) atomicAdd(g.gb2, gb2);
}

template <bool TRAIN, bool WGRAD>
int launch(const Params &p, cudaStream_t stream) {
    static NlPerDevice configured;
    const cudaError_t e = configured.once([] { return cudaFuncSetAttribute(k_mlp_wg<TRAIN, WGRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL); });
    if (e != cudaSuccess) return nl_set_error_code(NL_ERR_CUDA, cudaGetErrorString(e));
    const long long ntiles = (p.M_host + TM - 1) / TM;
    const int grid = (int)(ntiles < (long long)nl_num_sms() ? ntiles : (long long)nl_num_sms());
    k_mlp_wg<TRAIN, WGRAD><<<grid, NTHREADS, SMEM_TOTAL, stream>>>(p);
    return NL_OK;
}

}  // namespace tc

extern "C" int64_t nl_mlp_tc_panel_bytes(void) { return (int64_t)tc::STEPS_TRAIN * tc::STAGE_B; }

extern "C" int nl_mlp_tc_prepare(const float *W0, const float *W1, const float *w2, void *panels, void *stream) {
    if (!W0 || !W1 || !w2 || !panels) return nl_set_error("nl_mlp_tc_prepare: null pointer");
    dim3 grid(nl_div_up(tc::WN * 8, 256), tc::STEPS_TRAIN);
    tc::k_tc_prepare<<<grid, 256, 0, (cudaStream_t)stream>>>(W0, W1, w2, (uint8_t *)panels);
    NL_CHECK_LAUNCH("nl_mlp_tc_prepare");
    return NL_OK;
}

extern "C" int nl_mlp_tc_forward(int64_t M, const int32_t *d_M_dev, const float *feats, const void *panels, const float *b0,
                                 const float *b1, const float *w2, const float *b2, float *sdf, void *stream) {
    if (M < 0) return nl_set_error("nl_mlp_tc_forward: negative M");
    if (M == 0) return NL_OK;
    if (!feats || !panels || !b0 || !b1 || !w2 || !b2 || !sdf) return nl_set_error("nl_mlp_tc_forward: null pointer");
    tc::Params p = {};
    p.M_host = M; p.M_dev = d_M_dev; p.feats = feats; p.panels = (const uint8_t *)panels;
    p.b0 = b0; p.b1 = b1; p.w2 = w2; p.b2 = b2; p.sdf = sdf;
    if (int rc = tc::launch<false, false>(p, (cudaStream_t)stream)) return rc;
    NL_CHECK_LAUNCH("nl_mlp_tc_forward");
    return NL_OK;
}

// h1, h2, dh2, dh1 [cap][256] and d loss / d sdf [cap], cap = M rounded up to whole tiles
extern "C" int64_t nl_mlp_tc_act_floats(int64_t M) { return ((M + tc::TM - 1) / tc::TM) * tc::TM * (4 * tc::WN + 1); }

extern "C" int nl_mlp_tc_train(int64_t M, const int32_t *d_M_dev, const float *feats, const void *panels, const float *W1, const float *b0,
                               const float *b1, const float *w2, const float *b2, const uint8_t *s_flag, const float *s_depth,
                               const int32_t *s_ray, const float *cosv, const float *gt_depth, nl_render_stats *stats,
                               float truncation, float *sdf, float *dfeats, const nl_mlp_grads *grads, float *act,
                               const float *dsdf_ext, void *wgrad_stream_, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (M < 0) return nl_set_error("nl_mlp_tc_train: negative M");
    if (M == 0) return NL_OK;
    if (!feats || !panels || !W1 || !b0 || !b1 || !w2 || !b2 || !sdf || !dfeats) return nl_set_error("nl_mlp_tc_train: null pointer");
    if (!dsdf_ext && (!s_flag || !s_depth || !s_ray || !gt_depth || !stats))
        return nl_set_error("nl_mlp_tc_train: the loss needs s_flag, s_depth, s_ray, gt_depth and stats");
    if (grads && (!grads->gW0 || !grads->gb0 || !grads->gW1 || !grads->gb1 || !grads->gW2 || !grads->gb2 || !act))
        return nl_set_error("nl_mlp_tc_train: decoder gradients requested but a buffer is null");
    tc::Params p = {};
    p.M_host = M; p.M_dev = d_M_dev; p.feats = feats; p.panels = (const uint8_t *)panels;
    p.b0 = b0; p.b1 = b1; p.w2 = w2; p.b2 = b2; p.sdf = sdf; p.dfeats = dfeats;
    p.s_flag = s_flag; p.s_depth = s_depth; p.s_ray = s_ray; p.cosv = cosv; p.gt_depth = gt_depth; p.stats = stats;
    p.truncation = truncation; p.dsdf_ext = dsdf_ext;
    if (!grads) {
        if (int rc = tc::launch<true, false>(p, stream)) return rc;
        NL_CHECK_LAUNCH("nl_mlp_tc_train");
        return NL_OK;
    }
    const size_t cap = (size_t)((M + tc::TM - 1) / tc::TM) * tc::TM, plane = cap * tc::WN;
    p.act_h1 = act; p.act_h2 = act + plane; p.act_dh2 = act + 2 * plane; p.act_dh1 = act + 3 * plane; p.act_d = act + 4 * plane;
    if (int rc = tc::launch<true, true>(p, stream)) return rc;
    // The weight-gradient kernels only need what the kernel above wrote; on a second stream they overlap with whatever the
    // caller enqueues next on `stream` (the embedding scatter).
    cudaStream_t ws = wgrad_stream_ ? (cudaStream_t)wgrad_stream_ : stream;
    if (ws != stream) {
        constexpr int NL_MAX_DEV = 64;
        static std::mutex mu;
        static cudaEvent_t ev_dev[NL_MAX_DEV] = {};
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= NL_MAX_DEV) return nl_set_error_code(NL_ERR_CUDA, "nl_mlp_tc_train: cudaGetDevice");
        std::lock_guard<std::mutex> lock(mu);
        cudaEvent_t &ev = ev_dev[dev];
        if (!ev && cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) return nl_set_error_code(NL_ERR_CUDA, "cudaEventCreate");
        if (cudaEventRecord(ev, stream) != cudaSuccess || cudaStreamWaitEvent(ws, ev, 0) != cudaSuccess)
            return nl_set_error_code(NL_ERR_CUDA, "nl_mlp_tc_train: could not order the weight-gradient stream behind the decoder kernel");
    }
    static NlPerDevice dw_configured;
    const cudaError_t e = dw_configured.once([] { return cudaFuncSetAttribute(tc::k_dw1_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::DW_SMEM); });
    if (e != cudaSuccess) return nl_set_error_code(NL_ERR_CUDA, cudaGetErrorString(e));
    const int nsplit = nl_num_sms() / 4 > 0 ? nl_num_sms() / 4 : 1;
    tc::k_dw1_tc<<<4 * nsplit, 256, tc::DW_SMEM, ws>>>(M, d_M_dev, p.act_dh2, p.act_h1, grads->gW1, nsplit);
    tc::k_wg_cols<<<nl_num_sms() * 4, tc::WN, 0, ws>>>(M, d_M_dev, feats, p.act_dh1, p.act_h2, p.act_dh2, p.act_d, *grads);
    NL_CHECK_LAUNCH("nl_mlp_tc_train");
    return NL_OK;
}
