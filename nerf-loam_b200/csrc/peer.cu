// Multi-GPU gradient reduction FUSED with the optimiser step over NVLink peer memory (SURVEY.md section 8 e, "fused with the
// collective"): reduce-scatter -> Adam -> all-gather as ONE kernel per rank instead of ncclAllReduce + a separate Adam launch.
//
// Every rank has scattered its embedding gradients into its own fp32 table G_r (L2 atomics, gather.cu).  The tables and the
// bf16 parameter tables live in symmetric memory: every rank can address every peer's copy (NVLink P2P), and on an NVSwitch
// system there is additionally ONE multicast address per buffer (NVLS).  Rank r owns the rows [r*V/W, (r+1)*V/W):
//
//     g      = sum over ranks of G_q[row]        multimem.ld_reduce.add.v4.f32 -- the reduction happens INSIDE the switch and the
//                                                 16 B that come back are already the sum (W P2P loads + adds without NVLS)
//     p,m,v  = Adam(p, g, m, v)                   exactly nl_adam_bf16_ctl (optim.cu); m and v exist only for the owned rows
//     P_q[row] = p  for every rank q              multimem.st.v4 -- one store, the switch replicates it (W P2P stores without NVLS)
//
// so that afterwards every rank holds the identical updated table.  Compared with all-reduce + Adam the gradient crosses
// NVLink once as a reduce-scatter (4 B/element in, from W sources, summed in the switch) and the result once as bf16
// (2 B/element out) instead of a full fp32 all-reduce, the optimiser state is sharded W ways (ZeRO-1), every element's Adam
// arithmetic is done once instead of W times, and one kernel launch replaces two.  The caller orders it between two
// symmetric-memory barriers (all scatters finished / all tables written); see dist.PeerReduceAdam.
#include "nl_cuda.cuh"
#include "adam.cuh"

namespace {

__device__ __forceinline__ float4 mc_ld_reduce_f32x4(const float *mc) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
    return v;
}
__device__ __forceinline__ void mc_st_b32x4(void *mc, uint4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)),
                 "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w)) : "memory");
}

// One thread per 8 consecutive elements (half an embedding row): 2 x 16 B of reduced gradient in, 16 B of parameters out.
template <bool MC>
__global__ void __launch_bounds__(256) k_reduce_adam_bf16(long long e0, long long e1, int rank, int world, const float *const *grad_peers,
                                                           const float *grad_mc, uint16_t *const *param_peers, uint16_t *param_mc,
                                                           uint16_t *__restrict__ m, uint16_t *__restrict__ v, double lr, double beta1, double beta2,
                                                           float eps, const int32_t *__restrict__ ctl, int hdr_n4, const float *const *hdr_peers,
                                                           const float *hdr_mc, float *__restrict__ hdr_out) {
    // the small vector in front of the table (loss sums, pose accumulators): every rank reduces all of it into a LOCAL buffer
    if (blockIdx.x == gridDim.x - 1) {
        for (int i = threadIdx.x; i < hdr_n4; i += blockDim.x) {
            float4 s4;
            if (MC) {
                s4 = mc_ld_reduce_f32x4(hdr_mc + 4 * i);
            } else {
                s4 = make_float4(0.f, 0.f, 0.f, 0.f);
                for (int q = 0; q < world; ++q) {
                    const float4 a = *reinterpret_cast<const float4 *>(hdr_peers[q] + 4 * i);
                    s4.x += a.x; s4.y += a.y; s4.z += a.z; s4.w += a.w;
                }
            }
            *reinterpret_cast<float4 *>(hdr_out + 4 * i) = s4;
        }
        return;
    }
    const long long e = e0 + ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8;
    if (e >= e1 || ctl[NL_CTL_SKIP_NOW]) return;        // a skipped iteration leaves parameters and moments untouched on every rank
    float g[8];
    if (MC) {
        const float4 a = mc_ld_reduce_f32x4(grad_mc + e), b = mc_ld_reduce_f32x4(grad_mc + e + 4);
        g[0] = a.x; g[1] = a.y; g[2] = a.z; g[3] = a.w; g[4] = b.x; g[5] = b.y; g[6] = b.z; g[7] = b.w;
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) g[i] = 0.f;
        for (int q = 0; q < world; ++q) {               // fixed order 0..W-1 on every rank: the sum does not depend on who computes it
            const float4 a = *reinterpret_cast<const float4 *>(grad_peers[q] + e), b = *reinterpret_cast<const float4 *>(grad_peers[q] + e + 4);
            g[0] += a.x; g[1] += a.y; g[2] += a.z; g[3] += a.w; g[4] += b.x; g[5] += b.y; g[6] += b.z; g[7] += b.w;
        }
    }
    const NlAdamConst c = nl_adam_const(lr, beta1, beta2, eps, ctl[NL_CTL_ADAM_STEP]);
    uint4 pw = *reinterpret_cast<const uint4 *>(param_peers[rank] + e);
    uint4 mw = *reinterpret_cast<const uint4 *>(m + e), vw = *reinterpret_cast<const uint4 *>(v + e);
    uint16_t *p16 = reinterpret_cast<uint16_t *>(&pw), *m16 = reinterpret_cast<uint16_t *>(&mw), *v16 = reinterpret_cast<uint16_t *>(&vw);
#pragma unroll
    for (int i = 0; i < 8; ++i) nl_adam_bf16_elem(c, g[i], p16[i], m16[i], v16[i]);
    *reinterpret_cast<uint4 *>(m + e) = mw;
    *reinterpret_cast<uint4 *>(v + e) = vw;
    if (MC) {
        mc_st_b32x4(param_mc + e, pw);
    } else {
        for (int q = 0; q < world; ++q) *reinterpret_cast<uint4 *>(param_peers[q] + e) = pw;
    }
}

}  // namespace

extern "C" int nl_peer_reduce_adam_bf16(int64_t n_elems, int rank, int world, const float *const *d_grad_peers, const float *d_grad_mc,
                                        uint16_t *const *d_param_peers, uint16_t *d_param_mc, uint16_t *d_m, uint16_t *d_v, double lr,
                                        double beta1, double beta2, double eps, const int32_t *d_ctl, int64_t hdr_n, const float *const *d_hdr_peers,
                                        const float *d_hdr_mc, float *d_hdr_out, void *stream) {
    if (hdr_n < 0 || (hdr_n & 3) || (hdr_n > 0 && (!d_hdr_peers || !d_hdr_out))) return nl_set_error("nl_peer_reduce_adam_bf16: bad header arguments");
    if (n_elems < 0 || (n_elems & 15) || world < 1 || rank < 0 || rank >= world) return nl_set_error("nl_peer_reduce_adam_bf16: bad sizes");
    if (!d_grad_peers || !d_param_peers || !d_m || !d_v || !d_ctl) return nl_set_error("nl_peer_reduce_adam_bf16: null pointer");
    if ((d_grad_mc == nullptr) != (d_param_mc == nullptr)) return nl_set_error("nl_peer_reduce_adam_bf16: both or neither multicast address");
    // row-aligned contiguous slice of this rank
    const long long rows = n_elems / 16;
    const long long e0 = rows * rank / world * 16, e1 = rows * (rank + 1) / world * 16;
    const int blocks = nl_div_up((e1 - e0) / 8, 256) + 1;          // + one block for the header
    if (d_grad_mc)
        k_reduce_adam_bf16<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(e0, e1, rank, world, d_grad_peers, d_grad_mc, d_param_peers, d_param_mc,
                                                                           d_m, d_v, lr, beta1, beta2, (float)eps, d_ctl, (int)(hdr_n / 4), d_hdr_peers,
                                                                           d_hdr_mc, d_hdr_out);
    else
        k_reduce_adam_bf16<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(e0, e1, rank, world, d_grad_peers, nullptr, d_param_peers, nullptr,
                                                                            d_m, d_v, lr, beta1, beta2, (float)eps, d_ctl, (int)(hdr_n / 4), d_hdr_peers,
                                                                            nullptr, d_hdr_out);
    NL_CHECK_LAUNCH("nl_peer_reduce_adam_bf16");
    return NL_OK;
}
