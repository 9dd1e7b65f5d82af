// The loss read-out of one iteration (criterion.py:84-100 after the masked sums): shared by nl_loss_finalize (render.cu) and the fused
// pose step (pose.cu).
#pragma once
#include "nl_cuda.cuh"

__device__ __forceinline__ void nl_loss_finalize_dev(nl_render_stats *s, float fs_weight, float sdf_weight) {
    const double N = (double)((long long)s->n_hit_rays * (long long)s->max_samples);
    s->fs_loss = (float)((s->fs_sum + (double)s->pad_fs_sum) / N) * s->w_fs;
    s->sdf_loss = (float)((s->sdf_sum + (double)s->pad_sdf_sum) / N) * s->w_sdf;
    s->loss = fs_weight * s->fs_loss + sdf_weight * s->sdf_loss;
}

// Batched loss (nl_render_samples_batch): adds this lane's squared-error sums into stats[k].fs_sum / sdf_sum, k = its problem or -1
// (nothing to add).  Called by all 32 lanes together.  Samples are ordered by problem, so a warp almost always holds one problem:
// then one reduction and one atomic per sum; a warp that straddles a problem boundary adds lane by lane.
__device__ __forceinline__ void nl_seg_loss_add(nl_render_stats *stats, int k, double fs, double sdf) {
    const int kmax = __reduce_max_sync(0xffffffffu, k);
    if (__all_sync(0xffffffffu, k < 0 || k == kmax)) {
        for (int off = 16; off > 0; off >>= 1) {
            fs += __shfl_down_sync(0xffffffffu, fs, off);
            sdf += __shfl_down_sync(0xffffffffu, sdf, off);
        }
        if ((threadIdx.x & 31) == 0 && kmax >= 0) {
            if (fs != 0.0) atomicAdd(&stats[kmax].fs_sum, fs);
            if (sdf != 0.0) atomicAdd(&stats[kmax].sdf_sum, sdf);
        }
    } else if (k >= 0) {
        if (fs != 0.0) atomicAdd(&stats[k].fs_sum, fs);
        if (sdf != 0.0) atomicAdd(&stats[k].sdf_sum, sdf);
    }
}
