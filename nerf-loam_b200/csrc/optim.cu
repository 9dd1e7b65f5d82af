// Adam with torch.optim.Adam semantics (render_helpers.py:353, :448; defaults betas (0.9, 0.999),
// eps 1e-8, no weight decay, no amsgrad), one fused kernel per parameter tensor instead of torch's
// sequence of per-op (foreach) kernels:
//     m = lerp(m, g, 1-b1);  v = v*b2;  v = v + (1-b2)*g*g;
//     denom = sqrt(v) / sqrt(1-b2^t) + eps;  p = p + (-(lr/(1-b1^t))) * (m/denom)
// nl_adam_bf16 is for the reference's bf16 embedding table (mapping.py:305-306): parameter, gradient
// and both moments are bf16 tensors there, so every op above rounds its result to bf16; the fused
// kernel rounds at the same points (the gradient arrives as the fp32 scatter sum and is rounded first,
// which is what autograd's bf16 embedding backward produces).
#include "nl_cuda.cuh"
#include "adam.cuh"

namespace {

__global__ void k_adam_f32(long long n, float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m,
                           float *__restrict__ v, float w1, float beta2, float w2, float eps, float step_size, float bc2_sqrt) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float gi = g[i];
    const float mi = __fadd_rn(m[i], __fmul_rn(w1, __fsub_rn(gi, m[i])));                      // lerp (weight < 0.5)
    float vi = __fmul_rn(v[i], beta2);
    vi = __fadd_rn(vi, __fmul_rn(__fmul_rn(w2, gi), gi));                                      // addcmul
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vi), bc2_sqrt), eps);
    p[i] = __fadd_rn(p[i], __fmul_rn(-step_size, __fdiv_rn(mi, denom)));                       // addcdiv
    m[i] = mi;
    v[i] = vi;
}

__global__ void k_adam_bf16(long long n, uint16_t *__restrict__ p, const float *__restrict__ g32, uint16_t *__restrict__ m,
                            uint16_t *__restrict__ v, float w1, float beta2, float w2, float eps, float step_size, float bc2_sqrt) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float gi = nl_round_bf16(g32[i]);
    float mi = nl_bf16_to_f32(m[i]), vi = nl_bf16_to_f32(v[i]), pi = nl_bf16_to_f32(p[i]);
    mi = nl_round_bf16(__fadd_rn(mi, __fmul_rn(w1, __fsub_rn(gi, mi))));
    vi = nl_round_bf16(__fmul_rn(vi, beta2));
    vi = nl_round_bf16(__fadd_rn(vi, __fmul_rn(__fmul_rn(w2, gi), gi)));
    float d = nl_round_bf16(__fsqrt_rn(vi));
    d = nl_round_bf16(__fdiv_rn(d, bc2_sqrt));
    d = nl_round_bf16(__fadd_rn(d, eps));
    pi = nl_round_bf16(__fadd_rn(pi, __fmul_rn(-step_size, __fdiv_rn(mi, d))));
    p[i] = nl_f32_to_bf16(pi);
    m[i] = nl_f32_to_bf16(mi);
    v[i] = nl_f32_to_bf16(vi);
}

// Adam driven by the device-side iteration control block (nl_iter_status): the step count is ctl[NL_CTL_ADAM_STEP] and the whole
// update is skipped when ctl[NL_CTL_SKIP_NOW] is set -- the reference `continue`s past optim.step() when an iteration hits nothing
// (render_helpers.py:405-409), and a skipped step advances neither the moments nor Adam's step count.
template <bool BF16>
__global__ void k_adam_ctl(long long n, void *__restrict__ p_, const float *__restrict__ g, void *__restrict__ m_, void *__restrict__ v_,
                           double lr, double beta1, double beta2, float eps, const int32_t *__restrict__ ctl) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || ctl[NL_CTL_SKIP_NOW]) return;
    const int t = ctl[NL_CTL_ADAM_STEP];
    const double bc1 = 1.0 - pow(beta1, (double)t), bc2 = 1.0 - pow(beta2, (double)t);
    const float w1 = (float)(1.0 - beta1), b2 = (float)beta2, w2 = (float)(1.0 - beta2), step_size = (float)(lr / bc1), bc2_sqrt = (float)sqrt(bc2);
    if (BF16) {
        uint16_t *p = (uint16_t *)p_, *m = (uint16_t *)m_, *v = (uint16_t *)v_;
        nl_adam_bf16_elem(NlAdamConst{w1, b2, w2, eps, step_size, bc2_sqrt}, g[i], p[i], m[i], v[i]);
    } else {
        float *p = (float *)p_, *m = (float *)m_, *v = (float *)v_;
        nl_adam_f32_elem(NlAdamConst{w1, b2, w2, eps, step_size, bc2_sqrt}, g[i], p[i], m[i], v[i]);
    }
}

}  // namespace

#include <cmath>

extern "C" int nl_adam_f32(int64_t n, float *p, const float *g, float *m, float *v, double lr, double beta1, double beta2,
                           double eps, int step, void *stream) {
    if (n < 0 || step < 1) return nl_set_error("nl_adam_f32: bad arguments");
    if (n == 0) return NL_OK;
    if (!p || !g || !m || !v) return nl_set_error("nl_adam_f32: null pointer");
    const double bc1 = 1.0 - std::pow(beta1, step), bc2 = 1.0 - std::pow(beta2, step);
    k_adam_f32<<<nl_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(n, p, g, m, v, (float)(1.0 - beta1), (float)beta2,
                                                                    (float)(1.0 - beta2), (float)eps, (float)(lr / bc1),
                                                                    (float)std::sqrt(bc2));
    NL_CHECK_LAUNCH("nl_adam_f32");
    return NL_OK;
}

extern "C" int nl_adam_bf16(int64_t n, uint16_t *p, const float *g, uint16_t *m, uint16_t *v, double lr, double beta1,
                            double beta2, double eps, int step, void *stream) {
    if (n < 0 || step < 1) return nl_set_error("nl_adam_bf16: bad arguments");
    if (n == 0) return NL_OK;
    if (!p || !g || !m || !v) return nl_set_error("nl_adam_bf16: null pointer");
    const double bc1 = 1.0 - std::pow(beta1, step), bc2 = 1.0 - std::pow(beta2, step);
    k_adam_bf16<<<nl_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(n, p, g, m, v, (float)(1.0 - beta1), (float)beta2,
                                                                     (float)(1.0 - beta2), (float)eps, (float)(lr / bc1),
                                                                     (float)std::sqrt(bc2));
    NL_CHECK_LAUNCH("nl_adam_bf16");
    return NL_OK;
}

extern "C" int nl_adam_f32_ctl(int64_t n, float *p, const float *g, float *m, float *v, double lr, double beta1, double beta2, double eps,
                               const int32_t *d_ctl, void *stream) {
    if (n < 0) return nl_set_error("nl_adam_f32_ctl: bad arguments");
    if (n == 0) return NL_OK;
    if (!p || !g || !m || !v || !d_ctl) return nl_set_error("nl_adam_f32_ctl: null pointer");
    k_adam_ctl<false><<<nl_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(n, p, g, m, v, lr, beta1, beta2, (float)eps, d_ctl);
    NL_CHECK_LAUNCH("nl_adam_f32_ctl");
    return NL_OK;
}

extern "C" int nl_adam_bf16_ctl(int64_t n, uint16_t *p, const float *g, uint16_t *m, uint16_t *v, double lr, double beta1, double beta2,
                                double eps, const int32_t *d_ctl, void *stream) {
    if (n < 0) return nl_set_error("nl_adam_bf16_ctl: bad arguments");
    if (n == 0) return NL_OK;
    if (!p || !g || !m || !v || !d_ctl) return nl_set_error("nl_adam_bf16_ctl: null pointer");
    k_adam_ctl<true><<<nl_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(n, p, g, m, v, lr, beta1, beta2, (float)eps, d_ctl);
    NL_CHECK_LAUNCH("nl_adam_bf16_ctl");
    return NL_OK;
}
