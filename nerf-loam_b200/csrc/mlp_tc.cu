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
//   * The K = 256 GEMMs are software-pipelined in commit groups of 2 k-steps (wgmma.wait_group 1): a warpgroup builds its next
//     A fragments and waits for the ring while its previous group runs (gemm in k_mlp_wg).
//   * Every N = 256 GEMM runs as two N = 128 halves, so the previous layer's activations (128 registers per thread) and
//     one accumulator half (64) fit in the register file together.
// Per 128-sample training tile the ring carries 42 items: layer 1 (2 halves), layer 2 (2 halves x 8 K-blocks of 32),
// backward layer 2 (2 x 8) and backward layer 1 (8 K-blocks, N = 16).
//
// Decoder weight gradients (nl_mlp_tc_train with grads): the training kernel forms gW0 = dh1^T x and gb0 = sum dh1 itself, from
// dh1 staged in shared memory during backward layer 1, and stores the relu'(h2) bits (32 B per sample) and d loss / d sdf (and,
// only when asked to, dh1 [cap][256]).  The output layer has one unit, so dh2 = dsdf * w2 * m2 (m2 = relu'(h2)) and everything
// that would read h2 or dh2 follows from G = m2^T (dsdf * h1) and c = m2^T dsdf:
//   gW1 = diag(w2) G   gW2[j] = sum_k W1[j,k] G[j,k] + b1[j] c[j]   gb1 = w2 * c
// h1 = relu(x W0^T + b0) is not stored: its input x (K = 16, 64 B per sample) is, and recomputing h1 costs a tenth of G.  One
// split-K kernel (k_wgrad_tc) recomputes h1 and forms G on wgmma, both transposed so that the sample is wgmma's K: h1^T = W0 x^T
// with A = W0 from registers and B = x (K-major as stored), then G^T = (dsdf h1)^T m2 on fp16 wgmma with A = the h1^T accumulator
// from registers (each row scaled by a power of two into fp16's range and split into hi + lo) and B = the exact 0/1 mask expanded
// into a K-major tile.  The column sums c and gb2 run beside it.
#include <mutex>
#include <type_traits>

#include "loss.cuh"
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
// k_mlp_wg's shared memory, from the 1024-aligned base: the ring, b0 / b1 / w2, the ring's mbarriers; training adds every thread's
// relu'(h1) and relu'(h2) bits and loss sums (kept out of the register file so that ptxas need not serialise the wgmmas); weight
// gradients add one staging area per warpgroup for dh1 and the activations that leave through bulk copies, and the CTA's gW0 / gb0
// sums.
constexpr int SM_BIAS = NSLOT * SLOT;
constexpr int SM_BAR = SM_BIAS + 3 * WN * 4;
constexpr int SM_MASK = SM_BAR + 256;                     // mask1 [4][NTHREADS], mask2 [4][NTHREADS] words
constexpr int SM_LOSS = SM_MASK + 2 * 4 * NTHREADS * 4;   // fs, sdf squared-error sums [2][NTHREADS] doubles
constexpr int SM_STG = SM_LOSS + 2 * NTHREADS * 8;
// Staging area of a warpgroup: one N = 64 quarter of dh1 for its 64 rows, pitch STG_LD floats (STG_LD = 8 mod 32: a half-warp's
// 8-byte stores of an accumulator fragment and a warp's mma.sync B-fragment loads -- sample t / t + 4, column g -- hit 32 distinct
// banks; rows stay 16-byte aligned for the bulk copies), then its relu'(h2) words and dsdf.
constexpr int STG_LD = 72;
constexpr int STG_M2 = 64 * STG_LD * 4, STG_D = STG_M2 + 64 * 8 * 4, STG_WG = STG_D + 64 * 4;
// gW0 [2][256][16] then gb0 [2][256] floats, summed over the CTA's tiles: one copy per warpgroup, every entry of a copy owned by
// one thread, so they need no atomics.  Then each warpgroup's x tile: its 64 rows' features, [64][16] floats, row s holding feature
// e at column e ^ xt_swz(s), so that the gW0 A-fragment loads (sample t / t + 4, feature g / g + 8) hit 32 distinct banks.
constexpr int SM_GW0 = SM_STG + 2 * STG_WG, SM_GB0 = SM_GW0 + 2 * WN * 16 * 4, SM_XT = SM_GB0 + 2 * WN * 4;
constexpr int SMEM_FWD = SM_MASK + 1024;                  // + alignment slack
constexpr int SMEM_TRAIN = SM_STG + 1024;
constexpr int SMEM_WGRAD = SM_XT + 2 * 64 * 16 * 4 + 1024;
static_assert(SMEM_WGRAD <= 227 * 1024, "k_mlp_wg<train, wgrad> exceeds the 227 KB of shared memory a CTA may use");
static_assert(SM_LOSS % 8 == 0 && SM_STG % 16 == 0 && STG_LD * 4 % 16 == 0 && STG_D % 16 == 0 && STG_WG % 16 == 0 && SM_GW0 % 16 == 0 && SM_XT % 16 == 0,
              "alignment");
static_assert(STG_LD % 32 == 8, "bank-conflict-free staging stores and B-fragment loads");
__host__ __device__ __forceinline__ int xt_swz(int s) { return (s & 2) << 2; }

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
// shared -> global bulk copy, tracked in the issuing thread's bulk groups
__device__ __forceinline__ void bulk_s2g(void *dst, uint32_t src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every bulk copy this thread committed has finished reading shared memory (the source may be overwritten)
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... and has completed its writes
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// generic-proxy shared-memory writes made visible to the async proxy (the bulk copies that read them)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// v += x for a float in shared memory owned by this thread
__device__ __forceinline__ void add_shared(uint32_t addr, float x) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v + x) : "memory");
}
__device__ __forceinline__ float ld_shared(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
    return v;
}
// named barrier 1 + wg over the 128 threads of warpgroup wg (barrier 0 is __syncthreads')
__device__ __forceinline__ void wg_bar_sync(int wg) {
    if (wg == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
    else asm volatile("bar.sync 2, 128;" ::: "memory");
}

// ---- wgmma -------------------------------------------------------------------------------------------
// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90): start>>4 [0,14), LBO>>4 [16,30) (unused for swizzled
// K-major, 1), SBO>>4 = 1024>>4 [32,46) (8-row core-matrix groups), layout SWIZZLE_128B = 1 [62,64).  One k-step of 8 tf32
// is 32 bytes further along the row: +2 in the address field.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// every commit group of this warpgroup but the N committed last has completed
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void wg_commit_wait() {
    wg_commit();
    wg_wait<0>();
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
// D = A x B (scale-d = 0: the accumulator's previous contents are not read) and D += A x B, as used by k_wgrad_tc
__device__ __forceinline__ void wgmma_n64_z(float (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]), "=f"(d[17]), "=f"(d[18]), "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]), "=f"(d[24]), "=f"(d[25]), "=f"(d[26]), "=f"(d[27]), "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(0));
}
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(1));
}

// D (=, +=) A x B in fp16 (m64n128k16, fp32 accumulation), as used by k_wgrad_tc for G: A register i holds two adjacent K
// columns (lower K in the lower half) of row g + 8 (i & 1), columns 2t + 8 (i >> 1); B K-major (imm-trans-b = 0)
__device__ __forceinline__ void wgmma_f16_n128_z(float (&d)[64], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]), "=f"(d[17]), "=f"(d[18]), "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]), "=f"(d[24]), "=f"(d[25]), "=f"(d[26]), "=f"(d[27]), "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31]), "=f"(d[32]), "=f"(d[33]), "=f"(d[34]), "=f"(d[35]), "=f"(d[36]), "=f"(d[37]), "=f"(d[38]), "=f"(d[39]), "=f"(d[40]), "=f"(d[41]), "=f"(d[42]), "=f"(d[43]), "=f"(d[44]), "=f"(d[45]), "=f"(d[46]), "=f"(d[47]), "=f"(d[48]), "=f"(d[49]), "=f"(d[50]), "=f"(d[51]), "=f"(d[52]), "=f"(d[53]), "=f"(d[54]), "=f"(d[55]), "=f"(d[56]), "=f"(d[57]), "=f"(d[58]), "=f"(d[59]), "=f"(d[60]), "=f"(d[61]), "=f"(d[62]), "=f"(d[63])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(0));
}
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
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
// gW0^T = x^T dh1 (both kernels' weight gradients): one m16n8k8 tf32 term, A[e][s] = x[s][e], B[s][n] = dh1[s][n]
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void split4(const float (&v)[4], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) { hi[i] = tf32_rna(v[i]); lo[i] = tf32_rna(v[i] - __uint_as_float(hi[i])); }
}
// tf32_rna for finite x in two integer operations (cvt.rna.tf32.f32 adds an inf / NaN test to the same round-half-away-from-zero)
__device__ __forceinline__ uint32_t tf32_rna_finite(float x) { return (__float_as_uint(x) + 0x1000u) & 0xffffe000u; }
__device__ __forceinline__ void split_finite(float v, uint32_t &hi, uint32_t &lo) {
    hi = tf32_rna_finite(v);
    lo = tf32_rna_finite(v - __uint_as_float(hi));
}
// v0, v1 as fp16 pairs hi + lo (v0 in the lower halves): hi = rn(v), lo = rn(v - hi); v - hi is exact in fp32
__device__ __forceinline__ void split_f16x2(float v0, float v1, uint32_t &hi, uint32_t &lo) {
    float h0, h1;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(v1), "f"(v0));
    asm("{\n\t.reg .f16 a, b;\n\tmov.b32 {a, b}, %2;\n\tcvt.f32.f16 %0, a;\n\tcvt.f32.f16 %1, b;\n\t}" : "=f"(h0), "=f"(h1) : "r"(hi));
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(v1 - h1), "f"(v0 - h0));
}
// s with mx 2^s in [2^14, 2^15) for mx >= 0 (s = 0 for mx = 0), at most 126 so that 2^s and 2^-s are normal floats
__device__ __forceinline__ int f16_shift(float mx) { return mx == 0.f ? 0 : min(141 - (int)(__float_as_uint(mx) >> 23), 126); }
__device__ __forceinline__ float exp2_int(int s) { return __uint_as_float((uint32_t)(127 + s) << 23); }

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
    float *act_dh1, *act_d;            // WGRAD: [cap][256] (may be null: dh1 is not copied out), [cap]
    uint32_t *act_m2;                  // WGRAD: relu'(h2) rows, [cap][8] (see m2_word)
    float *gW0, *gb0;                  // WGRAD: [256][16], [256], accumulated
    int seg_rays;                      // SEG: rays per problem; stats = the problems' statistics, problem = s_ray / seg_rays
};

// relu'(h2) of one sample as 8 words (32 B): quad thread t of the training kernel holds columns 8j + 2t + e (j = 0..31,
// e = 0, 1) and stores them as 64 bits at word 2t, bit 2j + e.  Column c is therefore bit m2_bit(c) of word m2_word(c).
__host__ __device__ __forceinline__ int m2_word(int c) { return 2 * ((c >> 1) & 3) + (c >> 7); }
__host__ __device__ __forceinline__ int m2_bit(int c) { return (2 * (c >> 3) + (c & 1)) & 31; }
// bits 0 and 1 of nibble i of `m` -> bits 2i and 2i + 1 of the result (16 bits)
__device__ __forceinline__ uint32_t m2_pack(uint32_t m) {
    m &= 0x33333333u;
    m = (m | (m >> 2)) & 0x0F0F0F0Fu;
    m = (m | (m >> 4)) & 0x00FF00FFu;
    return (m | (m >> 8)) & 0x0000FFFFu;
}

// Phase breakdown of k_mlp_wg (scripts/time_decoder_phases.py builds a copy of the library with -DNL_TC_STAMPS; without it the
// stamps compile to nothing).  Thread 0 of each warpgroup adds the clock64() cycles since its previous stamp to the counter of the
// phase the stamp closes, in shared memory beside the ring's mbarriers, and adds its counters into tc_stamps at kernel end.
enum StampPhase { PH_RING, PH_ABUILD, PH_WAIT, PH_EPI1, PH_EPI2, PH_LOSS, PH_WGRAD, PH_REST, NPH };
#ifdef NL_TC_STAMPS
__device__ unsigned long long tc_stamps[2][NPH];
#endif

// ring item i of a tile -> panel stage and N half
__device__ __forceinline__ void item_of(int i, int &stage, int &half) {
    if (i < 2) { stage = 0; half = i; }
    else if (i < 18) { half = (i - 2) >> 3; stage = 1 + ((i - 2) & 7); }
    else if (i < 34) { half = (i - 18) >> 3; stage = 9 + ((i - 18) & 7); }
    else { half = 0; stage = 17 + (i - 34); }
}

// SEG (without weight gradients only): the loss of nl_mlp_tc_train_batch -- every sample reads the loss constants of its problem and
// adds its squared errors into that problem's sums; the per-sample arithmetic is the single-problem kernel's.  SEG without TRAIN is
// nl_mlp_tc_score_batch: the forward ring items, the same sums, no backward layers and no d feats.
template <bool TRAIN, bool WGRAD, bool SEG = false>
__global__ void __launch_bounds__(NTHREADS, 1) k_mlp_wg(Params p) {
    static_assert(!SEG || !WGRAD, "the batched loss is for a frozen decoder only");
    constexpr int IPT = TRAIN ? ITEMS_TRAIN : ITEMS_FWD;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;    // SWIZZLE_128B panels need 1024-byte alignment
    uint8_t *sm = smem_raw + (base - raw);
    const uint32_t ring = base;
    float *b0s = reinterpret_cast<float *>(sm + SM_BIAS);
    float *b1s = b0s + WN;
    float *w2s = b1s + WN;
    const uint32_t bar0 = base + SM_BAR;            // FULL[s] at 8s, EMPTY[s] at 8 (NSLOT + s)
    auto FULL = [&](uint32_t s) { return bar0 + 8u * s; };
    auto EMPTY = [&](uint32_t s) { return bar0 + 8u * (NSLOT + s); };

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    // TRAIN: relu'(h1) / relu'(h2) bit words i of this thread at [i * NTHREADS + tid]; squared-error sums at [tid], [NTHREADS + tid]
    uint32_t *mask1s = reinterpret_cast<uint32_t *>(sm + SM_MASK), *mask2s = mask1s + 4 * NTHREADS;
    double *lsum = reinterpret_cast<double *>(sm + SM_LOSS);
    const long long M = p.M_dev ? min((long long)*p.M_dev, p.M_host) : p.M_host;
    const long long ntiles = (M + TM - 1) / TM;
    const long long my_tiles = (long long)blockIdx.x < ntiles ? (ntiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const uint32_t total = (uint32_t)(my_tiles * IPT);

    for (int i = tid; i < WN; i += NTHREADS) { b0s[i] = p.b0[i]; b1s[i] = p.b1[i]; w2s[i] = p.w2[i]; }
    if constexpr (WGRAD) {
        float *acc = reinterpret_cast<float *>(sm + SM_GW0);   // WGRAD: gW0 copy w: [w][n][e]; gb0 copy c: [c][n]
        for (int i = tid; i < 2 * WN * 16 + 2 * WN; i += NTHREADS) acc[i] = 0.f;
    }
    if (tid == 0) {
        for (int s = 0; s < NSLOT; ++s) { mbar_init(FULL(s), 1); mbar_init(EMPTY(s), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
#ifdef NL_TC_STAMPS
    static_assert(16 * NSLOT + 2 * NPH * 8 <= 256, "the phase counters share the mbarriers' 256 bytes");
    unsigned long long *st_acc = reinterpret_cast<unsigned long long *>(sm + SM_BAR + 16 * NSLOT) + NPH * (tid >> 7);
    if ((tid & 127) == 0)
        for (int i = 0; i < NPH; ++i) st_acc[i] = 0ull;
#endif
    __syncthreads();
#ifdef NL_TC_STAMPS
    long long st_last = clock64();
    auto stamp = [&](int ph) {
        if ((tid & 127) == 0) { const long long now = clock64(); st_acc[ph] += (unsigned long long)(now - st_last); st_last = now; }
    };
#else
    auto stamp = [](int) {};
#endif

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
    uint32_t n = 0, nrel = 0;   // ring items acquired / released by this thread
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
        ++n;
    };
    // the oldest acquired item's slot is free again: the caller has waited for every wgmma that read it
    auto release = [&]() {
        __syncwarp();
        if (lane == 0) mbar_arrive(EMPTY(nrel % NSLOT));
        ++nrel;
    };
    // A GEMM of NG / 2 ring items (K-blocks of 4 k-steps), software-pipelined in NG commit groups of 2 k-steps: group q runs k-steps
    // 2 (q & 1), + 1 of item q / 2 with the A fragments in set q & 1.  build(q) forms group q's fragments and mma(q, bh, bl) issues
    // its wgmmas, in the order an unpipelined K-block would.  Once group q - 1 is committed, wgmma.wait_group 1 retires group q - 2,
    // and group q is built into the registers q - 2 read while q - 1 runs, so a warpgroup keeps a group on the tensor pipe while it
    // splits its next activations or waits for the ring.  An item is released when its second group has retired, one group after
    // the next item was acquired.  That cannot deadlock the ring: when thread 0 acquires item n, its own warpgroup still holds only
    // item n - 1 (its second group in flight) and has released n - 2 and everything before, while the one blocking wait in the feed
    // is for item n's slot, last held by item n - NSLOT.  The other warpgroup needs nothing from thread 0 to release n - NSLOT: every
    // item up to n - 1 was issued before thread 0 came here.  The last group is waited for (wait_group 0) before gemm returns, so
    // the accumulators may be read after it.
    auto gemm = [&](auto ng, auto &&build, auto &&mma) {
        constexpr int NG = decltype(ng)::value;
        static_assert(NG % 2 == 0, "two commit groups per ring item");
        uint64_t bh = 0, bl = 0;
#pragma unroll
        for (int q = 0; q < NG; ++q) {
            if (q >= 2) {
                wg_wait<1>();
                if (q & 1) release();
                stamp(PH_WAIT);
            }
            build(q);
            stamp(PH_ABUILD);
            if (!(q & 1)) { acquire(bh, bl); stamp(PH_RING); }
            wg_fence();
            mma(q, bh, bl);
            wg_commit();
            stamp(PH_REST);
        }
        wg_wait<0>();
        release();
        stamp(PH_WAIT);
    };

    const float b2 = p.b2[0];
    if constexpr (TRAIN) { lsum[tid] = 0.0; lsum[NTHREADS + tid] = 0.0; }

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
            stamp(PH_REST);
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) frag3(xh, ks, ah[ks], al[ks]);
            stamp(PH_ABUILD);
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                uint64_t bh, bl;
                acquire(bh, bl);
                stamp(PH_RING);
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < 2; ++ks) mma3<64>(sub64(h, 64 * half), ah[ks], al[ks], bh + 2 * ks, bl + 2 * ks);
                stamp(PH_REST);
                wg_commit_wait();
                release();
                stamp(PH_WAIT);
            }
        }
        // h1 = relu(D1 + b0), relu'(h1) bits: bit (4j + x) of the 128-bit mask, parked in shared memory until dh1
        {
            uint32_t mask1[4] = {0u, 0u, 0u, 0u};
#pragma unroll
            for (int j = 0; j < 32; ++j)
#pragma unroll
                for (int x = 0; x < 4; ++x) {
                    const float v = h[4 * j + x] + b0s[8 * j + 2 * t + (x & 1)];
                    const bool on = v > 0.f;
                    h[4 * j + x] = on ? v : 0.f;
                    if (on) mask1[j >> 3] |= 1u << ((j & 7) * 4 + x);
                }
            if constexpr (TRAIN) {
#pragma unroll
                for (int i = 0; i < 4; ++i) mask1s[i * NTHREADS + tid] = mask1[i];
            }
        }
        stamp(PH_EPI1);

        // ---- layer 2 (two N halves) + output layer partial sums ----
        float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            float d[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) d[i] = 0.f;
            uint32_t ah[2][2][4], al[2][2][4];   // [set][k-step of the group]: 8 K-blocks of 4 k-steps, 16 groups
            stamp(PH_REST);
            gemm(
                std::integral_constant<int, 16>{},
                [&](int q) {
#pragma unroll
                    for (int ks = 0; ks < 2; ++ks) frag3(h, 2 * q + ks, ah[q & 1][ks], al[q & 1][ks]);
                },
                [&](int q, uint64_t bh, uint64_t bl) {
#pragma unroll
                    for (int ks = 0; ks < 2; ++ks) {
                        const int k = 2 * (q & 1) + ks;   // k-step inside the K-block
                        mma3<64>(d, ah[q & 1][ks], al[q & 1][ks], bh + 2 * k, bl + 2 * k);
                    }
                });
            // relu'(h2) bits: bit (4j + x) of the 128-bit mask (j = 16 half + jj), words 2 half and 2 half + 1 of it
            uint32_t mask2[2] = {0u, 0u};
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
#pragma unroll
                for (int x = 0; x < 4; ++x) {
                    const int col = 128 * half + 8 * jj + 2 * t + (x & 1);
                    const float v = d[4 * jj + x] + b1s[col];
                    const bool on = v > 0.f;
                    const float hv = on ? v : 0.f;
                    d[4 * jj + x] = hv;
                    if (on) mask2[jj >> 3] |= 1u << ((jj & 7) * 4 + x);
                    if (x < 2) ps0 = fmaf(hv, w2s[col], ps0); else ps1 = fmaf(hv, w2s[col], ps1);
                }
            if constexpr (TRAIN) {
                mask2s[(2 * half) * NTHREADS + tid] = mask2[0];
                mask2s[(2 * half + 1) * NTHREADS + tid] = mask2[1];
            }
            stamp(PH_EPI2);
        }
        // the 4 threads of a quad hold the 4 column classes of the same two rows
        ps0 += __shfl_xor_sync(0xffffffffu, ps0, 1); ps0 += __shfl_xor_sync(0xffffffffu, ps0, 2);
        ps1 += __shfl_xor_sync(0xffffffffu, ps1, 1); ps1 += __shfl_xor_sync(0xffffffffu, ps1, 2);
        const float sdf0 = ps0 + b2, sdf1 = ps1 + b2;
        if (t == 0) {
            if (live0) p.sdf[m0] = sdf0;
            if (live1) p.sdf[m1] = sdf1;
        }
        if constexpr (TRAIN || SEG) {
            // ---- loss (criterion.py:92-103) and d loss / d sdf for both rows ----
            float dsdf[2] = {0.f, 0.f};
            int seg_k[2] = {-1, -1};                 // SEG: problem of each row (-1: no row)
            double seg_fs[2] = {0.0, 0.0}, seg_sdf[2] = {0.0, 0.0};
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const long long m = r ? m1 : m0;
                const float s = r ? sdf1 : sdf0;
                if (!(r ? live1 : live0)) continue;
                if (!SEG && p.dsdf_ext) { dsdf[r] = p.dsdf_ext[m]; continue; }
                const uint32_t fl = p.s_flag[m];
                const int ray = p.s_ray[m];
                int k = 0;
                if constexpr (SEG) k = seg_k[r] = ray / p.seg_rays;
                const float gf = p.stats[k].g_fs, gs = p.stats[k].g_sdf;
                const float z = __fmul_rn(p.s_depth[m], p.cosv ? p.cosv[ray] : 1.0f);
                const float dgt = p.gt_depth[ray];
                if (fl & 1u) {
                    const float e = s - 1.0f;
                    if (t == 0) {
                        if constexpr (SEG) seg_fs[r] = (double)e * (double)e;
                        else lsum[tid] += (double)e * (double)e;
                    }
                    dsdf[r] += 2.0f * gf * e;
                }
                if (fl & 2u) {
                    const float e = __fsub_rn(__fadd_rn(z, __fmul_rn(s, p.truncation)), dgt);
                    if (t == 0) {
                        if constexpr (SEG) seg_sdf[r] = (double)e * (double)e;
                        else lsum[NTHREADS + tid] += (double)e * (double)e;
                    }
                    dsdf[r] += 2.0f * gs * p.truncation * e;
                }
            }
            if constexpr (SEG) {                     // one quad thread per row carries its squared errors
#pragma unroll
                for (int r = 0; r < 2; ++r) nl_seg_loss_add(p.stats, t == 0 ? seg_k[r] : -1, seg_fs[r], seg_sdf[r]);
            }
            stamp(PH_LOSS);
            if constexpr (!TRAIN) continue;          // scoring: the tile ends with its loss
            // WGRAD: the activation buffer rows of this warpgroup leave through bulk copies from its staging area (dh1 quarter |
            // relu'(h2) words | dsdf).  The first warp's lanes issue them (two dh1 rows each, when dh1 is copied out at all); a staged
            // quarter is overwritten only after those lanes saw their copies finish reading it and the warpgroup passed a barrier
            // behind them, which also orders it after the gW0 / gb0 reads of the previous quarter.  Everything here is derived from
            // tid and tile where it is used.
            auto staging = [&]() { return reinterpret_cast<float *>(sm + SM_STG + (warp >> 2) * STG_WG); };
            if (WGRAD) {
                const int lr = (warp & 3) * 16 + g;   // this thread's rows inside the warpgroup's 64: lr, lr + 8
                // mask2 bit 4j + x: row x >> 1, column 8j + 2t + (x & 1).  The previous tile's copies of these words finished reading
                // them before its second dh1 half was staged.
                uint32_t w[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) w[i] = mask2s[i * NTHREADS + tid];
                uint32_t *stg_m2 = reinterpret_cast<uint32_t *>(staging() + STG_M2 / 4);
                *reinterpret_cast<uint2 *>(stg_m2 + lr * 8 + 2 * t) =
                    make_uint2(m2_pack(w[0]) | m2_pack(w[1]) << 16, m2_pack(w[2]) | m2_pack(w[3]) << 16);
                *reinterpret_cast<uint2 *>(stg_m2 + (lr + 8) * 8 + 2 * t) =
                    make_uint2(m2_pack(w[0] >> 2) | m2_pack(w[1] >> 2) << 16, m2_pack(w[2] >> 2) | m2_pack(w[3] >> 2) << 16);
                if (t == 0) {   // dsdf leaves in whole 16-byte pieces of 4 rows; the rows of a partly live piece are stored directly
                    float *stg_d = staging() + STG_D / 4;
                    stg_d[lr] = dsdf[0];
                    stg_d[lr + 8] = dsdf[1];
                    if (live0 && (m0 | 3) >= M) p.act_d[m0] = dsdf[0];
                    if (live1 && (m1 | 3) >= M) p.act_d[m1] = dsdf[1];
                }
                stamp(PH_WGRAD);
            }
            // stage dh1 columns 64 qq .. 64 qq + 63 (and with qq = 0 the relu'(h2) words, dsdf and the x tile) and start their copies
            auto stage_quarter = [&](int qq) {
                const int wg = warp >> 2, lr = (warp & 3) * 16 + g;
                float *stg = staging();
                if ((warp & 3) == 0) bulk_wait_read();
                wg_bar_sync(wg);
                if (qq == 0) {   // thread (row r, quarter t): features 4t .. 4t + 3 of rows r and r + 8 of the warpgroup's 64, exactly 0
                                 // past M, where the feature array may hold anything (indices read afresh, as in gw0_quarter)
                    uint32_t th;
                    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(th));
                    const int r = ((th >> 5) & 3) * 16 + ((th >> 2) & 7), c = 4 * (th & 3);
                    const long long s = tile * TM + 64 * (th >> 7) + r;
                    float *xt = reinterpret_cast<float *>(sm + SM_XT) + (th >> 7) * 64 * 16;
                    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                    const float4 v0 = s < M ? __ldg(reinterpret_cast<const float4 *>(p.feats + (size_t)s * 16 + c)) : z;
                    const float4 v1 = s + 8 < M ? __ldg(reinterpret_cast<const float4 *>(p.feats + (size_t)(s + 8) * 16 + c)) : z;
                    *reinterpret_cast<float4 *>(xt + r * 16 + (c ^ xt_swz(r))) = v0;
                    *reinterpret_cast<float4 *>(xt + (r + 8) * 16 + (c ^ xt_swz(r + 8))) = v1;
                }
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    const int j = 8 * qq + jj;
                    *reinterpret_cast<float2 *>(stg + lr * STG_LD + 8 * jj + 2 * t) = make_float2(h[4 * j], h[4 * j + 1]);
                    *reinterpret_cast<float2 *>(stg + (lr + 8) * STG_LD + 8 * jj + 2 * t) = make_float2(h[4 * j + 2], h[4 * j + 3]);
                }
                fence_proxy_async();
                wg_bar_sync(wg);
                if ((warp & 3) == 0) {
                    const long long r0 = tile * TM + 64 * wg;               // rows r0 .. r0 + nrows - 1
                    const int nrows = (int)min(max(M - r0, 0LL), 64LL);
                    if (p.act_dh1)
                        for (int r = lane; r < nrows; r += 32)
                            bulk_s2g(p.act_dh1 + (size_t)(r0 + r) * WN + 64 * qq, smem_u32(stg + r * STG_LD), 64 * 4);
                    if (qq == 0 && lane == 0 && nrows > 0) {
                        bulk_s2g(p.act_m2 + (size_t)r0 * 8, smem_u32(stg + STG_M2 / 4), nrows * 8 * 4);
                        if (nrows >= 4) bulk_s2g(p.act_d + r0, smem_u32(stg + STG_D / 4), (nrows & ~3) * 4);
                    }
                    bulk_commit();
                }
            };
            // gW0^T += x^T dh1 and gb0 += sum dh1 over the warpgroup's 64 rows, for the staged quarter qq.  Warp w of the warpgroup owns
            // columns 64 qq + 16 w .. + 15 (two n8 tiles) and uses k_wgrad_tc's former 3xTF32 terms, each accumulator restarted every 32
            // samples (see the truncation note at k_wgrad_tc).  x comes from the warpgroup's x tile, exactly 0 on rows at or past M; dh1 is
            // 0 there already.  Both are finite, so they are split with tf32_rna_finite.  The B fragments a warp loads cover all 64
            // rows of its 16 columns (lanes t = 0..3 of a column together), so gb0 is their sum over the k-steps and the 4 lanes.
            auto gw0_quarter = [&](int qq) {
                uint32_t th;   // read afresh: nothing here is computed early and held through the forward layers
                asm volatile("mov.u32 %0, %%tid.x;" : "=r"(th));
                const int wg = th >> 7, wq = (th >> 5) & 3, g = (th >> 2) & 7, t = th & 3, sw = xt_swz(t);
                const float *stg = reinterpret_cast<const float *>(sm + SM_STG + wg * STG_WG);
                const float *xt = reinterpret_cast<const float *>(sm + SM_XT) + wg * 64 * 16;
                float cs[2] = {0.f, 0.f};   // gb0 partial of column 16 wq + 8 nt + g
#pragma unroll 1
                for (int hk = 0; hk < 2; ++hk) {
                    float pw[2][3][4];
#pragma unroll
                    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
                        for (int m = 0; m < 3; ++m)
#pragma unroll
                            for (int i = 0; i < 4; ++i) pw[nt][m][i] = 0.f;
#pragma unroll
                    for (int k4 = 0; k4 < 4; ++k4) {
                        const int ks = 4 * hk + k4;
                        const float *xa = xt + (8 * ks + t) * 16, *xb = xa + 4 * 16;   // rows 8 ks + t and + 4: same swizzle
                        const float av[4] = {xa[g ^ sw], xa[(g + 8) ^ sw], xb[g ^ sw], xb[(g + 8) ^ sw]};
                        uint32_t xh[4], xl[4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) split_finite(av[i], xh[i], xl[i]);
#pragma unroll
                        for (int nt = 0; nt < 2; ++nt) {
                            const float *qr = stg + (8 * ks + t) * STG_LD + 16 * wq + 8 * nt + g;
                            const float bv[2] = {qr[0], qr[4 * STG_LD]};
                            uint32_t bh[2], bl[2];
#pragma unroll
                            for (int i = 0; i < 2; ++i) split_finite(bv[i], bh[i], bl[i]);
                            cs[nt] += bv[0] + bv[1];
                            mma_tf32(pw[nt][0], xh, bh[0], bh[1]);
                            mma_tf32(pw[nt][1], xh, bl[0], bl[1]);
                            mma_tf32(pw[nt][2], xl, bh[0], bh[1]);
                        }
                    }
                    // fragment entry i: row (e) g + 8 (i >> 1), column (n) 2t + (i & 1) of n8 tile nt
#pragma unroll
                    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            add_shared(base + SM_GW0 + 4 * ((wg * WN + 64 * qq + 16 * wq + 8 * nt + 2 * t + (i & 1)) * 16 + g + 8 * (i >> 1)),
                                       pw[nt][0][i] + pw[nt][1][i] + pw[nt][2][i]);
                }
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) {
                    float c = cs[nt];
                    c += __shfl_xor_sync(0xffffffffu, c, 1);
                    c += __shfl_xor_sync(0xffffffffu, c, 2);
                    if (t == 0) add_shared(base + SM_GB0 + 4 * (wg * WN + 64 * qq + 16 * wq + 8 * nt + g), c);
                }
            };
            // ---- backward layer 2: D3 = relu'(h2) . (diag(w2) W1).  The A operand is the 0/1 mask (exact in tf32: 2 terms) ----
#pragma unroll
            for (int i = 0; i < 128; ++i) h[i] = 0.f;
            // one pipeline over both N halves (groups 0..15: columns 0..127, 16..31: 128..255); K-block kb of a half holds k-steps
            // 4 kb .. 4 kb + 3, whose mask bits are in word kb / 2
            {
                uint32_t a[2][2][4];   // [set][k-step of the group]
                stamp(PH_REST);
                gemm(
                    std::integral_constant<int, 32>{},
                    [&](int q) {
                        const int kb = (q & 15) >> 1;
                        const uint32_t wk = mask2s[(kb >> 1) * NTHREADS + tid];
#pragma unroll
                        for (int ks = 0; ks < 2; ++ks) {
                            const int j = 4 * kb + 2 * (q & 1) + ks;
                            const uint32_t w = wk >> ((j & 7) * 4);
                            uint32_t(&f)[4] = a[q & 1][ks];
                            f[0] = (w & 1u) ? 0x3f800000u : 0u; f[1] = (w & 4u) ? 0x3f800000u : 0u;
                            f[2] = (w & 2u) ? 0x3f800000u : 0u; f[3] = (w & 8u) ? 0x3f800000u : 0u;
                        }
                    },
                    [&](int q, uint64_t bh, uint64_t bl) {
#pragma unroll
                        for (int ks = 0; ks < 2; ++ks) {
                            const int k = 2 * (q & 1) + ks;
                            const uint32_t(&f)[4] = a[q & 1][ks];
                            wgmma_n128(sub64(h, 64 * (q >> 4)), f[0], f[1], f[2], f[3], bh + 2 * k);
                            wgmma_n128(sub64(h, 64 * (q >> 4)), f[0], f[1], f[2], f[3], bl + 2 * k);
                        }
                    });
            }
            // dh1 = dsdf * D3 * relu'(h1)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t m1w = mask1s[i * NTHREADS + tid];
#pragma unroll
                for (int j = 8 * i; j < 8 * i + 8; ++j)
#pragma unroll
                    for (int x = 0; x < 4; ++x)
                        h[4 * j + x] = ((m1w >> ((j & 7) * 4 + x)) & 1u) ? dsdf[x >> 1] * h[4 * j + x] : 0.f;
            }
            // ---- backward layer 1: d x = dh1 . W0 (N = 16); each dh1 quarter is staged (and copied out) before its two K-blocks,
            // and its gW0 / gb0 terms run while the first commit group of the first of them is in flight ----
            float dx[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) dx[i] = 0.f;
            {
                uint32_t ah[2][2][4], al[2][2][4];   // [set][k-step of the group]: 8 K-blocks of 4 k-steps, 16 groups
                stamp(PH_REST);
                gemm(
                    std::integral_constant<int, 16>{},
                    [&](int q) {
                        if (WGRAD && q % 4 == 0) { stage_quarter(q / 4); stamp(PH_WGRAD); }
#pragma unroll
                        for (int ks = 0; ks < 2; ++ks) frag3(h, 2 * q + ks, ah[q & 1][ks], al[q & 1][ks]);
                    },
                    [&](int q, uint64_t bh, uint64_t bl) {
#pragma unroll
                        for (int ks = 0; ks < 2; ++ks) {
                            const int k = 2 * (q & 1) + ks;
                            mma3<8>(dx, ah[q & 1][ks], al[q & 1][ks], bh + 2 * k, bl + 2 * k);
                        }
                        if (WGRAD && q % 4 == 0) { stamp(PH_REST); gw0_quarter(q / 4); stamp(PH_WGRAD); }
                    });
            }
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
                if (live0) *reinterpret_cast<float2 *>(p.dfeats + (size_t)m0 * 16 + 8 * jj + 2 * t) = make_float2(dx[4 * jj], dx[4 * jj + 1]);
                if (live1) *reinterpret_cast<float2 *>(p.dfeats + (size_t)m1 * 16 + 8 * jj + 2 * t) = make_float2(dx[4 * jj + 2], dx[4 * jj + 3]);
            }
        }
    }
    if (WGRAD && (warp & 3) == 0) bulk_wait();   // the staging areas stay valid until the copies out of them have completed
    if constexpr (WGRAD) {                        // the CTA's gW0 / gb0 (if it had a tile): one fp32 atomic per entry
        __syncthreads();
        if (n > 0) {
            uint32_t th;
            asm volatile("mov.u32 %0, %%tid.x;" : "=r"(th));
            const uint32_t acc = (smem_u32(smem_raw) + 1023u & ~1023u) + SM_GW0, acb = acc + (SM_GB0 - SM_GW0);
            for (uint32_t i = th; i < WN * 16; i += NTHREADS) atomicAdd(p.gW0 + i, ld_shared(acc + 4 * i) + ld_shared(acc + 4 * (WN * 16 + i)));
            atomicAdd(p.gb0 + th, ld_shared(acb + 4 * th) + ld_shared(acb + 4 * (WN + th)));
        }
    }
    if (TRAIN && !SEG && !p.dsdf_ext) {
        // every thread's sums in the order it added them, then over the warp: the same fp64 partials as register accumulators
        double loss_fs = lsum[tid], loss_sdf = lsum[NTHREADS + tid];
        for (int off = 16; off > 0; off >>= 1) {
            loss_fs += __shfl_down_sync(0xffffffffu, loss_fs, off);
            loss_sdf += __shfl_down_sync(0xffffffffu, loss_sdf, off);
        }
        if (lane == 0) {
            if (loss_fs != 0.0) atomicAdd(&p.stats->fs_sum, loss_fs);
            if (loss_sdf != 0.0) atomicAdd(&p.stats->sdf_sum, loss_sdf);
        }
    }
#ifdef NL_TC_STAMPS
    stamp(PH_REST);
    if ((tid & 127) == 0)
        for (int i = 0; i < NPH; ++i) atomicAdd(&tc_stamps[tid >> 7][i], st_acc[i]);
#endif
}

// The decoder weight gradients past layer 1 from x = feats, the relu'(h2) bits and dsdf; h1 is recomputed from x instead of stored.
// With G = m2^T (dsdf * h1) and c = m2^T dsdf (section at the top of the file):
//   gW1 = diag(w2) G   gW2[j] = sum_k W1[j,k] G[j,k] + b1[j] c[j]   gb1 = w2 * c   gb2 = sum_s dsdf
// (gW0 = dh1^T x and gb0 = sum_s dh1 are formed by the training kernel, where dh1 is.)
// Grid = 4 tiles x nsplit (one CTA per SM), split-K over samples.  CTA (tile, split) owns the 128 x 128 tile (k0, j0) of G^T.
// The reduction index is the sample, and wgmma takes A from registers or K-major shared memory and B from shared memory, so G is
// formed transposed with K = samples, G^T[k, j] = sum_s (dsdf * h1)^T[k, s] m2[s, j]: A comes from registers and B, the mask, is
// rebuilt per chunk as a K-major tile.
// Warpgroup w owns rows k0 + 64 w .. +63 (wgmma M = 64) and all 128 columns j.  Per chunk of WG_KC = 64 samples it
//   1. recomputes h1^T[k, s] = W0[k, :] x[s, :]^T (N = 64 samples, K = 16) with 3xTF32 wgmma, terms in the training kernel's
//      order: A = the tf32 hi / lo parts of W0 that the training kernel multiplies (the layer-1 panel), held in 16 registers for
//      the whole kernel; B = the chunk's x split into hi / lo tiles (x's own [s][e] rows are K-major).  This is the training
//      kernel's z1, so both kernels agree on every relu'(h1);
//   2. forms v = dsdf * relu(h1^T + b0) in the accumulator registers (b0 per row, dsdf per column), scales each row by the power
//      of two 2^s that puts the row's largest |v| over the chunk in [2^14, 2^15), and splits it into fp16 hi = rn(v 2^s) and
//      lo = rn(v 2^s - hi).  fp16 has tf32's 11 significant bits, so hi + lo is v 2^s to 2^-22 relative while lo is normal and to
//      2^-25 absolute (2^-39 of the row's maximum) below; the scaling is exact, and it is what keeps the row inside fp16's range.
//      Columns 16 kk .. 16 kk + 15 of the n64 accumulator fragment are, as they stand, the fp16 A fragment of k-step kk;
//   3. accumulates G^T with 2 fp16 terms (hi m2 + lo m2; the mask is exact in fp16, and fp16 products are exact in the fp32
//      accumulator): A from the registers of step 2, B = the mask expanded from its bits into a [128 j][64 s] tile of 0 / 1.0
//      halves (K-major, 128-byte swizzle: one 128-byte row per j), shared by both warpgroups.  The chunk's rows are scaled back by
//      2^-s as they are added into the running sums.
// While the G wgmmas run, the warps form the column sums c (the k0 = 0 tiles) and gb2 (tile 0), and build the next chunk's x and
// mask tiles into the other of two tile buffers.  x, the mask rows and dsdf stream through a WG_NS-slot shared-memory ring filled
// by cp.async WG_NS - 1 chunks ahead; one __syncthreads per chunk publishes the next chunk's data and tiles.
// The tensor core truncates the sums it accumulates, a bias that grows with the number of MMAs into one accumulator; so every
// chunk's first wgmma starts from zero (scale-d = 0) and the chunk sums are added up in fp32 (G) or fp64 (the rest) over the ~2e4
// samples of a split.
// Samples at or past the device-side count are zero-filled in every streamed array (the feature array behind them holds stale
// values, possibly non-finite): x = dsdf = 0 and an empty mask, so they add exact zeros everywhere.
// The partial G is folded into the gradients it determines before the atomics:
//   gW1[j][k] += w2[j] G[j][k]      gW2[j] += sum_k W1[j][k] G[j][k] (+ b1[j] c[j] from the k0 = 0 tiles)
constexpr int WG_KC = 64, WG_NS = 4;
constexpr int WG_LDX = 20;     // x rows in the ring: fragment loads (row g, column t) hit 32 distinct banks
constexpr int WG_OM = WG_KC * WG_LDX, WG_OD = WG_OM + WG_KC * 8;   // slot: x | mask rows | dsdf
constexpr int WG_SLOT = WG_OD + WG_KC;                             // floats
constexpr int WG_MT = 128 * 128;             // mask tile: 128 rows (j) x 64 fp16 samples
constexpr int WG_XT = WG_KC * 128;           // x tile (hi or lo): a 128-byte row per sample, the 16 features in its first 64 B
constexpr int WG_SMEM = 2 * (WG_MT + 2 * WG_XT) + WG_NS * WG_SLOT * 4 + 1024;   // 94 KB: 2 tile buffers, ring, alignment slack
static_assert(WG_OM % 4 == 0 && WG_OD % 4 == 0 && WG_SLOT % 4 == 0, "cp.async 16-byte destinations");
static_assert(WG_KC == 64, "the loaders and the x-tile build assign one 16-byte piece of x per thread, a mask row is 128 bytes");
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void *src, bool valid) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(valid ? 4 : 0) : "memory");
}
// keeps the compiler from moving reads of wgmma accumulators above the wgmma.wait_group that completes them
template <int N>
__device__ __forceinline__ void wg_fence_acc(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__global__ void __launch_bounds__(256, 1) k_wgrad_tc(long long M_host, const int32_t *__restrict__ M_dev, const float *__restrict__ x,
                                                     const uint32_t *__restrict__ m2, const float *__restrict__ dsdf,
                                                     const uint8_t *__restrict__ panels, const float *__restrict__ b0, const float *__restrict__ W1,
                                                     const float *__restrict__ b1, const float *__restrict__ w2, nl_mlp_grads grads, int nsplit) {
    extern __shared__ uint8_t wg_smem[];
    const uint32_t raw = smem_u32(wg_smem);
    const uint32_t base = (raw + 1023u) & ~1023u;    // SWIZZLE_128B tiles need 1024-byte alignment
    // tile buffer b: mask tile at b * WG_MT, x hi / lo at 2 WG_MT + (2b, 2b + 1) WG_XT; then the ring
    uint8_t *tiles = wg_smem + (base - raw);
    float *ring = reinterpret_cast<float *>(tiles + 2 * (WG_MT + 2 * WG_XT));
    __shared__ float red[8][128];     // gW2 partials of the 8 warps
    __shared__ double cred[2][128];   // c partials of the two sample halves
    const long long M = M_dev ? min((long long)*M_dev, M_host) : M_host;
    const int tile = blockIdx.x & 3, split = blockIdx.x >> 2;
    const int j0 = (tile >> 1) * 128, k0 = (tile & 1) * 128;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int kr = k0 + 64 * (warp >> 2) + 16 * (warp & 3) + g;   // this thread's rows of h1^T and G^T: kr and kr + 8

    // W0 as A fragments of k-steps 0, 1 (K position q of k-step ks = feature 8 ks + q).  The layer-1 panel holds W0 row k at panel
    // row k and feature kperm(p) at position p.
    uint32_t w0h[2][4], w0l[2][4];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
        for (int i = 0; i < 4; ++i) {   // i: row kr + 8 (i & 1), feature 8 ks + t + 4 (i >> 1)
            const int e = 8 * ks + t + 4 * (i >> 1), pos = (e & ~7) | ((e & 1) << 2) | ((e & 7) >> 1);
            const int off = panel_off(kr + 8 * (i & 1), pos >> 2) + (pos & 3) * 4;
            w0h[ks][i] = *reinterpret_cast<const uint32_t *>(panels + off);
            w0l[ks][i] = *reinterpret_cast<const uint32_t *>(panels + PANEL_B + off);
        }
    const float b0a = b0[kr], b0b = b0[kr + 8];

    float tot[64];   // G^T: tot[4 jn + x] is row kr + 8 (x >> 1), column j0 + 8 jn + 2t + (x & 1)
#pragma unroll
    for (int i = 0; i < 64; ++i) tot[i] = 0.f;
    double c_acc = 0.0, gb2 = 0.0;
    const long long nch = (M + WG_KC - 1) / WG_KC;
    // Every thread commits one cp.async group per chunk, empty past the last chunk, so that wait_group n always means "all but the
    // n chunks issued last have landed".
    auto load = [&](long long ch, int buf) {
        if (ch >= nch) { asm volatile("cp.async.commit_group;" ::: "memory"); return; }
        float *sl = ring + buf * WG_SLOT;
        const long long s0 = ch * WG_KC;
        {                                                              // x: 64 rows x 4 float4
            const int r = tid >> 2, c4 = (tid & 3) * 4;
            const bool v = s0 + r < M;
            cp_async16(smem_u32(sl + r * WG_LDX + c4), x + (size_t)(v ? s0 + r : 0) * 16 + c4, v);
        }
        if (tid < 2 * WG_KC) {                                           // mask: 64 rows x 2 x 16 B
            const int r = tid >> 1, h = tid & 1;
            const bool v = s0 + r < M;
            cp_async16(smem_u32(sl + WG_OM + r * 8 + 4 * h), m2 + (size_t)(v ? s0 + r : 0) * 8 + 4 * h, v);
        } else if (tid < 3 * WG_KC) {                                    // dsdf
            const int r = tid - 2 * WG_KC;
            const bool v = s0 + r < M;
            cp_async4(smem_u32(sl + WG_OD + r), dsdf + (v ? s0 + r : 0), v);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    // x hi / lo and mask tiles of the chunk in ring slot `sl` into tile buffer b.  Thread tid writes mask tile row bj for samples
    // 32 bh .. 32 bh + 31, in sample order (16-byte pieces 4 bh .. 4 bh + 3 of the row).  The k0 = 0 tiles also add those samples'
    // dsdf into c[j0 + bj] here.
    const int bj = tid & 127, bh = tid >> 7, bw = m2_word(bj) + (j0 >> 7), bb = m2_bit(bj);
    auto build = [&](const float *sl, int b) {
        {
            const int r = tid >> 2, c = tid & 3;
            const float4 v = *reinterpret_cast<const float4 *>(sl + r * WG_LDX + 4 * c);
            const float a[4] = {v.x, v.y, v.z, v.w};
            uint32_t hi[4], lo[4];
            split4(a, hi, lo);
            uint8_t *xt = tiles + 2 * WG_MT + 2 * b * WG_XT;
            *reinterpret_cast<uint4 *>(xt + panel_off(r, c)) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            *reinterpret_cast<uint4 *>(xt + WG_XT + panel_off(r, c)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
        const uint32_t *Ms = reinterpret_cast<const uint32_t *>(sl + WG_OM);
        const float *Ds = sl + WG_OD;
        uint8_t *mt = tiles + b * WG_MT;
        float sc = 0.f;
#pragma unroll
        for (int q = 4 * bh; q < 4 * bh + 4; ++q) {
            uint32_t f[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int s = 8 * q + 2 * i;
                const bool on0 = (Ms[s * 8 + bw] >> bb) & 1u, on1 = (Ms[(s + 1) * 8 + bw] >> bb) & 1u;
                f[i] = (on0 ? 0x3C00u : 0u) | (on1 ? 0x3C000000u : 0u);
                if (k0 == 0) { sc += on0 ? Ds[s] : 0.f; sc += on1 ? Ds[s + 1] : 0.f; }
            }
            *reinterpret_cast<uint4 *>(mt + panel_off(bj, q)) = make_uint4(f[0], f[1], f[2], f[3]);
        }
        c_acc += sc;
    };

#pragma unroll
    for (int i = 0; i < WG_NS - 1; ++i) load(split + (long long)i * nsplit, i);
    asm volatile("cp.async.wait_group %0;" ::"n"(WG_NS - 2) : "memory");
    __syncthreads();
    if (split < nch) build(ring, 0);
    for (long long ch = split, it = 0; ch < nch; ch += nsplit, ++it) {
        asm volatile("cp.async.wait_group %0;" ::"n"(WG_NS - 3) : "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the tiles were written by ordinary stores, wgmma reads them
        // chunk `it`'s tiles and chunk it + 1's data are visible; every thread is done with ring slot (it + WG_NS - 1) % WG_NS and
        // its wgmmas on tile buffer (it + 1) & 1 have completed
        __syncthreads();
        load(ch + (long long)(WG_NS - 1) * nsplit, (int)((it + WG_NS - 1) % WG_NS));
        const float *sl = ring + (it % WG_NS) * WG_SLOT;
        const int b = (int)(it & 1);
        const uint64_t xd = make_desc(base + 2 * WG_MT + 2 * b * WG_XT), md = make_desc(base + b * WG_MT);

        // ---- 1. h1^T = W0 x^T ----
        float d1[32];
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const uint64_t xh = xd + 2 * ks, xl = xh + (WG_XT >> 4);
            if (ks == 0) wgmma_n64_z(d1, w0h[0][0], w0h[0][1], w0h[0][2], w0h[0][3], xh);
            else wgmma_n64(d1, w0h[ks][0], w0h[ks][1], w0h[ks][2], w0h[ks][3], xh);
            wgmma_n64(d1, w0l[ks][0], w0l[ks][1], w0l[ks][2], w0l[ks][3], xh);
            wgmma_n64(d1, w0h[ks][0], w0h[ks][1], w0h[ks][2], w0h[ks][3], xl);
        }
        wg_commit_wait();
        wg_fence_acc(d1);

        // ---- 2. fp16 A fragments of k-step kk (samples 16 kk .. +15) of 2^s dsdf * relu(h1^T + b0), s per row ----
        uint32_t ah[WG_KC / 16][4], al[WG_KC / 16][4];
        float inv_a, inv_b;   // 2^-s of rows kr, kr + 8
        {
            const float *Ds = sl + WG_OD;
            float ma = 0.f, mb = 0.f;
#pragma unroll
            for (int j = 0; j < WG_KC / 8; ++j) {   // d1[4 j + x]: row kr + 8 (x >> 1), sample 8 j + 2t + (x & 1)
                const float2 ds = *reinterpret_cast<const float2 *>(Ds + 8 * j + 2 * t);
                const float v0 = d1[4 * j] + b0a, v1 = d1[4 * j + 1] + b0a, v2 = d1[4 * j + 2] + b0b, v3 = d1[4 * j + 3] + b0b;
                d1[4 * j] = ds.x * (v0 > 0.f ? v0 : 0.f);
                d1[4 * j + 1] = ds.y * (v1 > 0.f ? v1 : 0.f);
                d1[4 * j + 2] = ds.x * (v2 > 0.f ? v2 : 0.f);
                d1[4 * j + 3] = ds.y * (v3 > 0.f ? v3 : 0.f);
                ma = fmaxf(ma, fmaxf(fabsf(d1[4 * j]), fabsf(d1[4 * j + 1])));
                mb = fmaxf(mb, fmaxf(fabsf(d1[4 * j + 2]), fabsf(d1[4 * j + 3])));
            }
            ma = fmaxf(ma, __shfl_xor_sync(0xffffffffu, ma, 1)); ma = fmaxf(ma, __shfl_xor_sync(0xffffffffu, ma, 2));
            mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 1)); mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 2));
            const int sa = f16_shift(ma), sb = f16_shift(mb);
            const float ua = exp2_int(sa), ub = exp2_int(sb);
            inv_a = exp2_int(-sa); inv_b = exp2_int(-sb);
#pragma unroll
            for (int kk = 0; kk < WG_KC / 16; ++kk) {
                const float *v = d1 + 8 * kk;
                split_f16x2(v[0] * ua, v[1] * ua, ah[kk][0], al[kk][0]);   // row kr, samples 16 kk + 2t, + 1
                split_f16x2(v[2] * ub, v[3] * ub, ah[kk][1], al[kk][1]);   // row kr + 8
                split_f16x2(v[4] * ua, v[5] * ua, ah[kk][2], al[kk][2]);   // row kr, samples 16 kk + 8 + 2t, + 1
                split_f16x2(v[6] * ub, v[7] * ub, ah[kk][3], al[kk][3]);   // row kr + 8
            }
        }

        // ---- 3. this chunk's 2^s G^T = (2^s dsdf h1)^T m2, left running while the warps do the rest ----
        float part[64];
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < WG_KC / 16; ++kk) {
            const uint64_t bd = md + 2 * kk;
            if (kk == 0) wgmma_f16_n128_z(part, ah[0][0], ah[0][1], ah[0][2], ah[0][3], bd);
            else wgmma_f16_n128(part, ah[kk][0], ah[kk][1], ah[kk][2], ah[kk][3], bd);
            wgmma_f16_n128(part, al[kk][0], al[kk][1], al[kk][2], al[kk][3], bd);
        }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");

        // ---- column sum gb2 (tile 0); c is summed in build() ----
        if (tile == 0 && tid < WG_KC) gb2 += sl[WG_OD + tid];

        // ---- the next chunk's tiles, into the buffer that the previous chunk's wgmmas read ----
        if (ch + nsplit < nch) build(ring + ((it + 1) % WG_NS) * WG_SLOT, b ^ 1);
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        wg_fence_acc(part);
#pragma unroll
        for (int i = 0; i < 64; ++i) tot[i] = fmaf(part[i], (i & 2) ? inv_b : inv_a, tot[i]);   // the product is exact
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    if (split >= nch) return;
#pragma unroll
    for (int jn = 0; jn < 16; ++jn)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int j = j0 + 8 * jn + 2 * t + e;
            const float s = w2[j], ga = tot[4 * jn + e], gb = tot[4 * jn + 2 + e];
            atomicAdd(grads.gW1 + (size_t)j * WN + kr, s * ga);
            atomicAdd(grads.gW1 + (size_t)j * WN + kr + 8, s * gb);
            float r = fmaf(W1[(size_t)j * WN + kr], ga, W1[(size_t)j * WN + kr + 8] * gb);
            r += __shfl_xor_sync(0xffffffffu, r, 4);
            r += __shfl_xor_sync(0xffffffffu, r, 8);
            r += __shfl_xor_sync(0xffffffffu, r, 16);
            if (g == 0) red[warp][8 * jn + 2 * t + e] = r;
        }
    if (k0 == 0) cred[tid >> 7][tid & 127] = c_acc;
    if (tile == 0 && warp < WG_KC / 32) {
        for (int off = 16; off > 0; off >>= 1) gb2 += __shfl_xor_sync(0xffffffffu, gb2, off);
        if (lane == 0) atomicAdd(grads.gb2, (float)gb2);
    }
    __syncthreads();
    if (tid < 128) {
        const int j = j0 + tid;
        float r = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) r += red[w][tid];
        if (k0 == 0) {
            const float c = (float)(cred[0][tid] + cred[1][tid]);
            atomicAdd(grads.gb1 + j, w2[j] * c);
            r += b1[j] * c;
        }
        atomicAdd(grads.gW2 + j, r);
    }
}

template <bool TRAIN, bool WGRAD, bool SEG = false>
int launch(const Params &p, cudaStream_t stream) {
    constexpr int smem = WGRAD ? SMEM_WGRAD : TRAIN ? SMEM_TRAIN : SMEM_FWD;
    static NlPerDevice configured;
    const cudaError_t e = configured.once([] { return cudaFuncSetAttribute(k_mlp_wg<TRAIN, WGRAD, SEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); });
    if (e != cudaSuccess) return nl_set_error_code(NL_ERR_CUDA, cudaGetErrorString(e));
    const long long ntiles = (p.M_host + TM - 1) / TM;
    const int grid = (int)(ntiles < (long long)nl_num_sms() ? ntiles : (long long)nl_num_sms());
    k_mlp_wg<TRAIN, WGRAD, SEG><<<grid, NTHREADS, smem, stream>>>(p);
    return NL_OK;
}

}  // namespace tc

#ifdef NL_TC_STAMPS
// k_mlp_wg's phase counters (cycles summed over CTAs and launches), [2 warpgroups][tc::NPH] in StampPhase order, then zeroed
extern "C" NL_API int nl_mlp_tc_stamps(unsigned long long *out) {
    const unsigned long long zero[2 * tc::NPH] = {};
    if (cudaMemcpyFromSymbol(out, tc::tc_stamps, sizeof(zero)) != cudaSuccess || cudaMemcpyToSymbol(tc::tc_stamps, zero, sizeof(zero)) != cudaSuccess)
        return nl_set_error_code(NL_ERR_CUDA, "nl_mlp_tc_stamps");
    return NL_OK;
}
#endif

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

// relu'(h2) bits [cap][8 words] and d loss / d sdf [cap]; the optional dh1 plane is [cap][256].  cap = M rounded up to whole tiles
extern "C" int64_t nl_mlp_tc_act_floats(int64_t M) { return ((M + tc::TM - 1) / tc::TM) * tc::TM * (8 + 1); }
extern "C" int64_t nl_mlp_tc_dh1_floats(int64_t M) { return ((M + tc::TM - 1) / tc::TM) * tc::TM * tc::WN; }

extern "C" int nl_mlp_tc_train(int64_t M, const int32_t *d_M_dev, const float *feats, const void *panels, const float *W1, const float *b0,
                               const float *b1, const float *w2, const float *b2, const uint8_t *s_flag, const float *s_depth,
                               const int32_t *s_ray, const float *cosv, const float *gt_depth, nl_render_stats *stats,
                               float truncation, float *sdf, float *dfeats, const nl_mlp_grads *grads, float *act, float *act_dh1,
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
    const size_t cap = (size_t)((M + tc::TM - 1) / tc::TM) * tc::TM;
    p.act_dh1 = act_dh1; p.act_m2 = reinterpret_cast<uint32_t *>(act); p.act_d = act + cap * 8;
    p.gW0 = grads->gW0; p.gb0 = grads->gb0;
    if (int rc = tc::launch<true, true>(p, stream)) return rc;
    static NlPerDevice configured;
    const cudaError_t e = configured.once([] { return cudaFuncSetAttribute(tc::k_wgrad_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::WG_SMEM); });
    if (e != cudaSuccess) return nl_set_error_code(NL_ERR_CUDA, cudaGetErrorString(e));
    // The weight-gradient kernel only needs what the kernel above wrote, the features, the layer-1 panel and b0 / W1 / b1 / w2; on a
    // second stream it overlaps with whatever the caller enqueues next on `stream` (the embedding scatter).
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
    const int nsplit = nl_num_sms() / 4 > 0 ? nl_num_sms() / 4 : 1;
    tc::k_wgrad_tc<<<4 * nsplit, 256, tc::WG_SMEM, ws>>>(M, d_M_dev, feats, p.act_m2, p.act_d, p.panels, b0, W1, b1, w2, *grads, nsplit);
    NL_CHECK_LAUNCH("nl_mlp_tc_train");
    return NL_OK;
}

extern "C" int nl_mlp_tc_train_batch(int64_t M, const int32_t *d_M_dev, const float *feats, const void *panels, const float *b0, const float *b1,
                                     const float *w2, const float *b2, const uint8_t *s_flag, const float *s_depth, const int32_t *s_ray,
                                     const float *cosv, const float *gt_depth, nl_render_stats *problem_stats, int32_t rays_per_problem,
                                     float truncation, float *sdf, float *dfeats, void *stream) {
    if (M < 0) return nl_set_error("nl_mlp_tc_train_batch: negative M");
    if (rays_per_problem <= 0) return nl_set_error("nl_mlp_tc_train_batch: rays_per_problem must be positive");
    if (M == 0) return NL_OK;
    if (!feats || !panels || !b0 || !b1 || !w2 || !b2 || !sdf || !dfeats || !s_flag || !s_depth || !s_ray || !gt_depth || !problem_stats)
        return nl_set_error("nl_mlp_tc_train_batch: null pointer");
    tc::Params p = {};
    p.M_host = M; p.M_dev = d_M_dev; p.feats = feats; p.panels = (const uint8_t *)panels;
    p.b0 = b0; p.b1 = b1; p.w2 = w2; p.b2 = b2; p.sdf = sdf; p.dfeats = dfeats;
    p.s_flag = s_flag; p.s_depth = s_depth; p.s_ray = s_ray; p.cosv = cosv; p.gt_depth = gt_depth; p.stats = problem_stats;
    p.truncation = truncation; p.seg_rays = rays_per_problem;
    if (int rc = tc::launch<true, false, true>(p, (cudaStream_t)stream)) return rc;
    NL_CHECK_LAUNCH("nl_mlp_tc_train_batch");
    return NL_OK;
}

extern "C" int nl_mlp_tc_score_batch(int64_t M, const int32_t *d_M_dev, const float *feats, const void *panels, const float *b0, const float *b1,
                                     const float *w2, const float *b2, const uint8_t *s_flag, const float *s_depth, const int32_t *s_ray,
                                     const float *cosv, const float *gt_depth, nl_render_stats *problem_stats, int32_t rays_per_problem,
                                     float truncation, float *sdf, void *stream) {
    if (M < 0) return nl_set_error("nl_mlp_tc_score_batch: negative M");
    if (rays_per_problem <= 0) return nl_set_error("nl_mlp_tc_score_batch: rays_per_problem must be positive");
    if (M == 0) return NL_OK;
    if (!feats || !panels || !b0 || !b1 || !w2 || !b2 || !sdf || !s_flag || !s_depth || !s_ray || !gt_depth || !problem_stats)
        return nl_set_error("nl_mlp_tc_score_batch: null pointer");
    tc::Params p = {};
    p.M_host = M; p.M_dev = d_M_dev; p.feats = feats; p.panels = (const uint8_t *)panels;
    p.b0 = b0; p.b1 = b1; p.w2 = w2; p.b2 = b2; p.sdf = sdf;
    p.s_flag = s_flag; p.s_depth = s_depth; p.s_ray = s_ray; p.cosv = cosv; p.gt_depth = gt_depth; p.stats = problem_stats;
    p.truncation = truncation; p.seg_rays = rays_per_problem;
    if (int rc = tc::launch<false, false, true>(p, (cudaStream_t)stream)) return rc;
    NL_CHECK_LAUNCH("nl_mlp_tc_score_batch");
    return NL_OK;
}
