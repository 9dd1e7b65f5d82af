// One element of torch.optim.Adam on an fp32 tensor, shared by the per-tensor kernels (optim.cu) and the fused pose step (pose.cu):
//     m = lerp(m, g, 1-b1);  v = v*b2;  v = v + (1-b2)*g*g;  denom = sqrt(v) / sqrt(1-b2^t) + eps;  p = p + (-(lr/(1-b1^t))) * (m/denom)
// with every operation rounded where torch's per-op kernels round.
#pragma once
#include "nl_cuda.cuh"

struct NlAdamConst {
    float w1, b2, w2, eps, step_size, bc2_sqrt;
};
// bias corrections for step t, evaluated in double like torch's host code
__device__ __forceinline__ NlAdamConst nl_adam_const(double lr, double beta1, double beta2, float eps, int t) {
    const double bc1 = 1.0 - pow(beta1, (double)t), bc2 = 1.0 - pow(beta2, (double)t);
    return {(float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), eps, (float)(lr / bc1), (float)sqrt(bc2)};
}
__device__ __forceinline__ void nl_adam_f32_elem(const NlAdamConst &c, float gi, float &p, float &m, float &v) {
    const float mi = __fadd_rn(m, __fmul_rn(c.w1, __fsub_rn(gi, m)));                         // lerp (weight < 0.5)
    float vi = __fmul_rn(v, c.b2);
    vi = __fadd_rn(vi, __fmul_rn(__fmul_rn(c.w2, gi), gi));                                   // addcmul
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vi), c.bc2_sqrt), c.eps);
    p = __fadd_rn(p, __fmul_rn(-c.step_size, __fdiv_rn(mi, denom)));                          // addcdiv
    m = mi;
    v = vi;
}
// The same on the bf16 embedding table (optim.cu's nl_adam_bf16_ctl, refine.cu's row-list step): parameter and moments are bf16,
// every operation rounds its result to bf16, and the fp32 gradient sum is rounded first.  With g = m = v = 0 it leaves p bitwise
// unchanged (m = v = +0, and p + (-step_size) * (+0 / d) = p, also for p = -0).
__device__ __forceinline__ void nl_adam_bf16_elem(const NlAdamConst &c, float g32, uint16_t &p, uint16_t &m, uint16_t &v) {
    const float gi = nl_round_bf16(g32);
    float mi = nl_bf16_to_f32(m), vi = nl_bf16_to_f32(v), pi = nl_bf16_to_f32(p);
    mi = nl_round_bf16(__fadd_rn(mi, __fmul_rn(c.w1, __fsub_rn(gi, mi))));
    vi = nl_round_bf16(__fmul_rn(vi, c.b2));
    vi = nl_round_bf16(__fadd_rn(vi, __fmul_rn(__fmul_rn(c.w2, gi), gi)));
    float d = nl_round_bf16(__fsqrt_rn(vi));
    d = nl_round_bf16(__fdiv_rn(d, c.bc2_sqrt));
    d = nl_round_bf16(__fadd_rn(d, c.eps));
    pi = nl_round_bf16(__fadd_rn(pi, __fmul_rn(-c.step_size, __fdiv_rn(mi, d))));
    p = nl_f32_to_bf16(pi);
    m = nl_f32_to_bf16(mi);
    v = nl_f32_to_bf16(vi);
}
