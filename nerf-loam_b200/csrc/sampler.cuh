// The stratified inverse-CDF walk along one ray, shared by the fused sampler (render.cu, k_sample) and the `grid.inverse_cdf_sampling`
// drop-in (grid_dropin.cu).  Behaviour to reproduce: third_party/sparse_voxels/src/sample_gpu.cu:165-238 (including its two index
// quirks, which the callers express through the two tail predicates); every floating-point operation is spelled with explicit
// rounding so that both users give the reference kernel's bits.
//
// A ray's hits are "bins" [lo, hi) with probability mass prob = length / total length.  The unit interval is cut into
// ceil(steps) strata; stratum i contributes the abscissa t = (i + noise_i) / steps.  Whenever t lies beyond the current bin, the
// bin is closed with one sample reaching to its far end; otherwise t is mapped linearly into the bin and a sample spans from the
// previous cut to the new one.  After the last stratum the open remainder of the current bin -- and, while `tail_allowed`, of
// the bins after it -- is flushed.  A sample is reported as emit(voxel id, z_from, z_to); callers derive mid-point / length.
#pragma once
#include <cstdint>

#include "nl_cuda.cuh"

// ceil(steps) as a stratum count.  The float -> int conversion is undefined at 2^31 and above, so the count saturates at INT32_MAX
// there (and is 0 for NaN); below that it is (int)ceilf(steps) exactly.
__device__ __forceinline__ int nl_strata_count(float steps) {
    const float c = ceilf(steps);
    return c >= 2147483648.0f ? INT32_MAX : (c > 0.0f ? (int)c : 0);
}

template <class Bins, class Noise, class Emit, class TailAllowed, class TailNextIdx>
__device__ __forceinline__ void nl_inverse_cdf_walk(int n_bins, const Bins &bins, float steps, float fixed_step, Noise noise, Emit emit,
                                                    TailAllowed tail_allowed, TailNextIdx tail_next_idx) {
    int b = 0;
    float lo = bins.lo(0), hi = bins.hi(0);
    float mass_before = 0.f, mass_upto = bins.prob(0);                  // cumulative probability at the two ends of bin b
    const float dt = fixed_step > 0.0f ? fixed_step : __frcp_rn(steps);  // (float)(1.0 / (double)steps) is the correctly rounded reciprocal
    float cut = lo;                                                      // where the previous sample ended
    const int n_strata = nl_strata_count(steps);
    bool exhausted = false;                                              // ran past the ray's last valid bin
    for (int i = 0; i < n_strata; ++i) {
        const float t = __fmul_rn(__fadd_rn((float)i, noise(i)), dt);
        while (t > mass_upto) {
            emit(bins.idx(b), cut, hi);
            ++b;
            if (b >= n_bins || bins.idx(b) == -1) { exhausted = true; break; }
            lo = bins.lo(b); hi = bins.hi(b);
            mass_before = mass_upto;
            mass_upto = __fadd_rn(mass_upto, bins.prob(b));
            cut = lo;
        }
        if (exhausted) break;
        const float frac = __fdiv_rn(__fsub_rn(t, mass_before), __fsub_rn(mass_upto, mass_before));
        const float z = __fmaf_rn(frac, __fsub_rn(hi, lo), lo);          // one FMA in the reference binary (nvcc -fmad default)
        emit(bins.idx(b), cut, z);
        cut = z;
    }
    while (cut < hi && !exhausted && tail_allowed(b)) {
        emit(bins.idx(b), cut, hi);
        ++b;
        if (b >= n_bins || tail_next_idx(b) == -1) break;
        lo = bins.lo(b); hi = bins.hi(b);
        cut = lo;
    }
}
