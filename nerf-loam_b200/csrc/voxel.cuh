// Voxel key of a posed scan point, shared by overlap.cu (keyframe overlap) and globalloc.cu (global localisation), so both
// count a point in the same voxel:
//   world point : w_i = ((R_i0 x + R_i1 y) + R_i2 z) + t_i in fp64 from the fp32 matrix and point.  The products are exact in
//                 fp64, so FMA contraction cannot change the result; the parentheses fix the order of the additions.
//   voxel       : floor(w / voxel_size) in fp64 per axis; a point whose voxel leaves [0, grid_dim)^3 (or is not finite) has no key.
//   key         : vx << 36 | vy << 18 | vz (grid_dim <= 2^18, so 54 bits).
// Rt is the 3x4 matrix as 12 floats: R row-major, then t (nl_pose_matrices' layout).
#pragma once
#include <cstdint>

constexpr int NL_VOXEL_AXIS_BITS = 18;   // log2 of the largest grid_dim (MapUpdater's default, 256 * 256 * 4)

__device__ __forceinline__ bool nl_voxel_key(const float (&Rt)[12], float x, float y, float z, double vs, double gd, uint64_t &key) {
    uint64_t k = 0;
    #pragma unroll
    for (int i = 0; i < 3; ++i) {
        const double w = (((double)Rt[3 * i] * (double)x + (double)Rt[3 * i + 1] * (double)y) + (double)Rt[3 * i + 2] * (double)z) +
                         (double)Rt[9 + i];
        const double v = floor(w / vs);
        if (!(v >= 0.0 && v < gd)) return false;
        k = (k << NL_VOXEL_AXIS_BITS) | (uint64_t)v;
    }
    key = k;
    return true;
}
