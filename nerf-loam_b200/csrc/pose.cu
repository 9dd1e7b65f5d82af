// SE(3) pose parameterisation of src/se3pose.py (OptimizablePose): data = [t(3), w(3)],
// R = I + A(theta) [w]x + B(theta) [w]x^2 with the 11-term Taylor polynomials of se3pose.py:63-82,
// ray generation (render_helpers.py:372-376 / 467-471) and the pose Jacobian that the reference gets
// from autograd through rotation() / translation().
#include "nl_cuda.cuh"
#include "adam.cuh"
#include "loss.cuh"

namespace {

// se3pose.py:63-72: sum_{i<=10} (-1)^i x^(2i) / (2i+1)!   (denominators accumulated like the Python loop)
// One warp per pose: lane i evaluates term i (the powf / pow calls are what the evaluation costs, and they are independent), then
// every lane adds the 11 terms up in the loop's order -- the same operations in the same order as the serial loop, a tenth of its
// latency (these two kernels sit on the critical path of every tracking iteration: 13 + 6 us serial).
__device__ __forceinline__ void taylor_AB(float x, float &A, float &B, float &dA, float &dB) {
    // values in fp32 term by term (the reference evaluates in fp32 tensors), derivatives in double
    const int i = threadIdx.x & 31;
    double denA = 1.0, denB = 1.0;
    for (int k = 0; k <= min(i, 10); ++k) {
        if (k > 0) denA *= (double)((2 * k) * (2 * k + 1));
        denB *= (double)((2 * k + 1) * (2 * k + 2));
    }
    float ta = 0.f, tb = 0.f;
    double tda = 0.0, tdb = 0.0;
    if (i <= 10) {
        const float sgn = (i & 1) ? -1.f : 1.f;
        const float xp = powf(x, (float)(2 * i));  // x ** (2*i); pow(0,0) = 1
        ta = sgn * xp / (float)denA;
        tb = sgn * xp / (float)denB;
        if (i > 0) {
            const double dxp = (double)(2 * i) * pow((double)x, (double)(2 * i - 1));
            tda = (double)sgn * dxp / denA;
            tdb = (double)sgn * dxp / denB;
        }
    }
    float a = 0.f, b = 0.f;
    double da = 0.0, db = 0.0;
#pragma unroll
    for (int k = 0; k <= 10; ++k) {
        a = a + __shfl_sync(0xffffffffu, ta, k);
        b = b + __shfl_sync(0xffffffffu, tb, k);
        if (k > 0) {
            da += __shfl_sync(0xffffffffu, tda, k);
            db += __shfl_sync(0xffffffffu, tdb, k);
        }
    }
    A = a; B = b; dA = (float)da; dB = (float)db;
}

__device__ __forceinline__ void rotation_from_w(const float w[3], float R[9]) {
    const float theta = sqrtf(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    float A, B, dA, dB;
    taylor_AB(theta, A, B, dA, dB);
    const float W[9] = {0.f, -w[2], w[1], w[2], 0.f, -w[0], -w[1], w[0], 0.f};  // se3pose.py:53-61
    float W2[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) W2[r * 3 + c] = W[r * 3] * W[c] + W[r * 3 + 1] * W[3 + c] + W[r * 3 + 2] * W[6 + c];
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = ((i % 4 == 0) ? 1.f : 0.f) + A * W[i] + B * W2[i];
}

constexpr int POSE_WARPS = 4;      // poses per block (one warp each)

__global__ void __launch_bounds__(POSE_WARPS * 32) k_pose_matrices(int F, const float *__restrict__ pose6, float *__restrict__ Rt12) {
    const int f = blockIdx.x * POSE_WARPS + (threadIdx.x >> 5);
    if (f >= F) return;                                  // warp-uniform
    float R[9];
    rotation_from_w(pose6 + f * 6 + 3, R);
    if ((threadIdx.x & 31) != 0) return;
#pragma unroll
    for (int i = 0; i < 9; ++i) Rt12[f * 12 + i] = R[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) Rt12[f * 12 + 9 + i] = pose6[f * 6 + i];
}

// rays_d = dirs @ R^T, rays_o = t (render_helpers.py:374-376)
__global__ void k_rays_from_poses(long long n, const float *__restrict__ dir_local, const int32_t *__restrict__ ray_frame,
                                  const float *__restrict__ Rt12, float *__restrict__ ray_o, float *__restrict__ ray_d) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const float *P = Rt12 + (size_t)(ray_frame ? ray_frame[r] : 0) * 12;
    const float x = dir_local[r * 3], y = dir_local[r * 3 + 1], z = dir_local[r * 3 + 2];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        ray_d[r * 3 + a] = fmaf(z, P[a * 3 + 2], fmaf(y, P[a * 3 + 1], x * P[a * 3]));
        ray_o[r * 3 + a] = P[9 + a];
    }
}

// grad6 = [dL/dt, dL/dw] from acc = (dL/dt[3], dL/dR[3][3]).
// dR/dw_i = A' (w_i/theta) W + A E_i + B' (w_i/theta) W^2 + B (E_i W + W E_i), theta' = w_i/theta (0 at theta = 0,
// matching torch's norm backward).
// one warp: d loss / d (t, w) of frame f
__device__ __forceinline__ void pose_grad_warp(int f, const float *__restrict__ pose6, const float *__restrict__ acc, float *__restrict__ grad6) {
    const float *w = pose6 + f * 6 + 3;
    const float *G = acc + f * 12 + 3;
    const float theta = sqrtf(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    float A, B, dA, dB;
    taylor_AB(theta, A, B, dA, dB);
    const int i = threadIdx.x & 31;                      // lane i < 3: the derivative with respect to w_i
    if (i >= 3) return;
    const float W[9] = {0.f, -w[2], w[1], w[2], 0.f, -w[0], -w[1], w[0], 0.f};
    float W2[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) W2[r * 3 + c] = W[r * 3] * W[c] + W[r * 3 + 1] * W[3 + c] + W[r * 3 + 2] * W[6 + c];
    float E[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (i == 0) { E[5] = -1.f; E[7] = 1.f; }
    if (i == 1) { E[2] = 1.f; E[6] = -1.f; }
    if (i == 2) { E[1] = -1.f; E[3] = 1.f; }
    const float dth = theta > 0.f ? w[i] / theta : 0.f;
    float g = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float EW = E[r * 3] * W[c] + E[r * 3 + 1] * W[3 + c] + E[r * 3 + 2] * W[6 + c];
            const float WE = W[r * 3] * E[c] + W[r * 3 + 1] * E[3 + c] + W[r * 3 + 2] * E[6 + c];
            const float dR = dA * dth * W[r * 3 + c] + A * E[r * 3 + c] + dB * dth * W2[r * 3 + c] + B * (EW + WE);
            g += G[r * 3 + c] * dR;
        }
    grad6[f * 6 + 3 + i] = g;
    grad6[f * 6 + i] = acc[f * 12 + i];
}

__global__ void __launch_bounds__(POSE_WARPS * 32) k_pose_grad(int F, const float *__restrict__ pose6, const float *__restrict__ acc, float *__restrict__ grad6) {
    const int f = blockIdx.x * POSE_WARPS + (threadIdx.x >> 5);
    if (f >= F) return;                                  // warp-uniform
    pose_grad_warp(f, pose6, acc, grad6);
}

// rays straight from the 6-vectors: every block first evaluates the (few) pose matrices into shared memory -- a warp per pose, the same
// code as k_pose_matrices -- then transforms its rays; block 0 also stores the matrices.  One launch instead of two on the critical
// path of every iteration (at 2048 rays a kernel boundary costs as much as either kernel).
constexpr int RAYS_MAX_FRAMES = 32;
__global__ void __launch_bounds__(256) k_rays_from_pose6(long long n, int F, const float *__restrict__ dir_local, const int32_t *__restrict__ ray_frame,
                                                          const float *__restrict__ pose6, float *__restrict__ Rt12, float *__restrict__ ray_o,
                                                          float *__restrict__ ray_d) {
    __shared__ float sRt[RAYS_MAX_FRAMES][12];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int f = w; f < F; f += 8) {                     // warp-uniform
        float R[9];
        rotation_from_w(pose6 + f * 6 + 3, R);
        if (lane < 9) sRt[f][lane] = R[lane];
        else if (lane < 12) sRt[f][lane] = pose6[f * 6 + lane - 9];
    }
    __syncthreads();
    if (blockIdx.x == 0 && Rt12)
        for (int i = threadIdx.x; i < F * 12; i += blockDim.x) Rt12[i] = sRt[i / 12][i % 12];
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const float *P = sRt[ray_frame ? ray_frame[r] : 0];
    const float x = dir_local[r * 3], y = dir_local[r * 3 + 1], z = dir_local[r * 3 + 2];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        ray_d[r * 3 + a] = fmaf(z, P[a * 3 + 2], fmaf(y, P[a * 3 + 1], x * P[a * 3]));
        ray_o[r * 3 + a] = P[9 + a];
    }
}

// The tail of an iteration that optimises poses, as ONE launch instead of up to F + 4: warp f < F = k_pose_grad for frame f followed,
// if bit f of row_mask is set, by the Adam update of its six parameters (nl_adam_f32_ctl's arithmetic: adam.cuh); warp F = the loss
// read-out of nl_loss_finalize and the advance of the device-side RNG seeds a captured iteration carries.
__global__ void __launch_bounds__(1024) k_pose_step(int F, float *__restrict__ pose6, const float *__restrict__ acc, float *__restrict__ grad6,
                                                     uint32_t row_mask, float *__restrict__ m, float *__restrict__ v, double lr, double beta1,
                                                     double beta2, float eps, const int32_t *__restrict__ ctl, nl_render_stats *stats,
                                                     float fs_weight, float sdf_weight, int32_t *seed_a, int32_t inc_a, int32_t *seed_b, int32_t inc_b) {
    const int f = threadIdx.x >> 5, i = threadIdx.x & 31;
    if (f == F) {
        if (i == 0 && stats) nl_loss_finalize_dev(stats, fs_weight, sdf_weight);
        if (i == 1 && seed_a) *seed_a = (int32_t)((uint32_t)*seed_a + (uint32_t)inc_a);
        if (i == 2 && seed_b) *seed_b = (int32_t)((uint32_t)*seed_b + (uint32_t)inc_b);
        return;
    }
    if (f > F) return;
    pose_grad_warp(f, pose6, acc, grad6);
    if (!((row_mask >> f) & 1u) || ctl[NL_CTL_SKIP_NOW]) return;
    __syncwarp();                                        // lanes 0..2 wrote grad6[f][0..5]
    if (i < 6) {
        const NlAdamConst c = nl_adam_const(lr, beta1, beta2, eps, ctl[NL_CTL_ADAM_STEP]);
        nl_adam_f32_elem(c, grad6[f * 6 + i], pose6[f * 6 + i], m[f * 6 + i], v[f * 6 + i]);
    }
}

// k_pose_step for K independent problems: warp k = problem k's pose gradient, its Adam step under its own rate, step count and skip
// flag (control block k), its loss read-out and the advance of its two seeds.
__global__ void __launch_bounds__(1024) k_pose_step_batch(int K, float *__restrict__ pose6, const float *__restrict__ acc, float *__restrict__ grad6,
                                                           float *__restrict__ m, float *__restrict__ v, const double *__restrict__ lr, double beta1,
                                                           double beta2, float eps, const int32_t *__restrict__ ctl, nl_render_stats *stats,
                                                           float fs_weight, float sdf_weight, float *__restrict__ last_loss, int32_t *seeds_a,
                                                           int32_t inc_a, int32_t *seeds_b, int32_t inc_b) {
    const int k = threadIdx.x >> 5, i = threadIdx.x & 31;
    if (k >= K) return;                                  // warp-uniform
    const int32_t *c = ctl + k * NL_CTL_WORDS;
    const bool skip = c[NL_CTL_SKIP_NOW] != 0;
    pose_grad_warp(k, pose6, acc, grad6);
    __syncwarp();                                        // lanes 0..2 wrote grad6[k][0..5]; every lane has read pose6[k]
    if (!skip && i < 6) {
        const NlAdamConst a = nl_adam_const(lr[k], beta1, beta2, eps, c[NL_CTL_ADAM_STEP]);
        nl_adam_f32_elem(a, grad6[k * 6 + i], pose6[k * 6 + i], m[k * 6 + i], v[k * 6 + i]);
    }
    if (i == 6 && stats) {
        nl_loss_finalize_dev(stats + k, fs_weight, sdf_weight);
        if (last_loss && !skip) last_loss[k] = stats[k].loss;
    }
    if (i == 7 && seeds_a) seeds_a[k] = (int32_t)((uint32_t)seeds_a[k] + (uint32_t)inc_a);
    if (i == 8 && seeds_b) seeds_b[k] = (int32_t)((uint32_t)seeds_b[k] + (uint32_t)inc_b);
}

}  // namespace

extern "C" int nl_pose_step_batch(int K, float *pose6, const float *acc, float *grad6, float *m, float *v, const double *d_lr, double beta1,
                                  double beta2, double eps, const int32_t *d_ctl, nl_render_stats *d_problem_stats, float fs_weight,
                                  float sdf_weight, float *d_last_loss, int32_t *d_seeds_a, int32_t inc_a, int32_t *d_seeds_b, int32_t inc_b,
                                  void *stream) {
    if (K < 1 || K > NL_BATCH_MAX_PROBLEMS) return nl_set_error("nl_pose_step_batch: need 1 <= n_problems <= 31");
    if (!pose6 || !acc || !grad6 || !m || !v || !d_lr || !d_ctl) return nl_set_error("nl_pose_step_batch: null pointer");
    k_pose_step_batch<<<1, K * 32, 0, (cudaStream_t)stream>>>(K, pose6, acc, grad6, m, v, d_lr, beta1, beta2, (float)eps, d_ctl, d_problem_stats,
                                                              fs_weight, sdf_weight, d_last_loss, d_seeds_a, inc_a, d_seeds_b, inc_b);
    NL_CHECK_LAUNCH("nl_pose_step_batch");
    return NL_OK;
}

extern "C" int nl_pose_matrices(int F, const float *pose6, float *Rt12, void *stream) {
    if (F <= 0 || !pose6 || !Rt12) return nl_set_error("nl_pose_matrices: bad arguments");
    k_pose_matrices<<<nl_div_up(F, POSE_WARPS), POSE_WARPS * 32, 0, (cudaStream_t)stream>>>(F, pose6, Rt12);
    NL_CHECK_LAUNCH("nl_pose_matrices");
    return NL_OK;
}

extern "C" int nl_rays_from_poses(int64_t R, const float *dir_local, const int32_t *ray_frame, const float *Rt12,
                                  float *ray_o, float *ray_d, void *stream) {
    if (R < 0 || !dir_local || !Rt12 || !ray_o || !ray_d) return nl_set_error("nl_rays_from_poses: bad arguments");
    if (R == 0) return NL_OK;
    k_rays_from_poses<<<nl_div_up(R, 256), 256, 0, (cudaStream_t)stream>>>(R, dir_local, ray_frame, Rt12, ray_o, ray_d);
    NL_CHECK_LAUNCH("nl_rays_from_poses");
    return NL_OK;
}

extern "C" int nl_pose_grad(int F, const float *pose6, const float *acc, float *grad6, void *stream) {
    if (F <= 0 || !pose6 || !acc || !grad6) return nl_set_error("nl_pose_grad: bad arguments");
    k_pose_grad<<<nl_div_up(F, POSE_WARPS), POSE_WARPS * 32, 0, (cudaStream_t)stream>>>(F, pose6, acc, grad6);
    NL_CHECK_LAUNCH("nl_pose_grad");
    return NL_OK;
}

extern "C" int nl_rays_from_pose6(int64_t R, int F, const float *dir_local, const int32_t *ray_frame, const float *pose6, float *Rt12,
                                  float *ray_o, float *ray_d, void *stream) {
    if (R < 0 || F <= 0 || F > RAYS_MAX_FRAMES) return nl_set_error("nl_rays_from_pose6: need R >= 0 and 1 <= n_frames <= 32");
    if (!dir_local || !pose6 || !ray_o || !ray_d) return nl_set_error("nl_rays_from_pose6: null pointer");
    if (R == 0) return NL_OK;
    k_rays_from_pose6<<<nl_div_up(R, 256), 256, 0, (cudaStream_t)stream>>>(R, F, dir_local, ray_frame, pose6, Rt12, ray_o, ray_d);
    NL_CHECK_LAUNCH("nl_rays_from_pose6");
    return NL_OK;
}

extern "C" int nl_pose_step(int F, float *pose6, const float *acc, float *grad6, uint32_t row_mask, float *m, float *v, double lr, double beta1,
                            double beta2, double eps, const int32_t *d_ctl, nl_render_stats *d_stats, float fs_weight, float sdf_weight,
                            int32_t *d_seed_a, int32_t inc_a, int32_t *d_seed_b, int32_t inc_b, void *stream) {
    if (F <= 0 || F > 31) return nl_set_error("nl_pose_step: need 1 <= n_frames <= 31");
    if (!pose6 || !acc || !grad6 || !d_ctl || (row_mask && (!m || !v))) return nl_set_error("nl_pose_step: null pointer");
    k_pose_step<<<1, (F + 1) * 32, 0, (cudaStream_t)stream>>>(F, pose6, acc, grad6, row_mask, m, v, lr, beta1, beta2, (float)eps, d_ctl, d_stats,
                                                               fs_weight, sdf_weight, d_seed_a, inc_a, d_seed_b, inc_b);
    NL_CHECK_LAUNCH("nl_pose_step");
    return NL_OK;
}
