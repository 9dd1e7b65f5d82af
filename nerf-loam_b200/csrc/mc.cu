// Sparse marching cubes on the GPU over the per-voxel SDF lattices of get_scores (SURVEY.md section 8 f-3).
//
// Replaces MeshExtractor.marching_cubes (src/utils/mesh_util.py:145-169): a Python loop over every voxel that copies its
// res^3 lattice to the host and runs skimage.measure.marching_cubes on it (~0.3 ms per voxel, seconds per mesh).  Here all
// voxels are processed by two kernel passes with no host round trip:
//
//   k_mc_count : one block per voxel.  Counts the lattice edges the zero level crosses (= vertices: like skimage, a
//                voxel's mesh is welded -- one vertex per crossed edge, shared by the triangles around it) and the
//                triangles of its (res-1)^3 cells.
//   (scan)       exclusive scans of both counts over the voxels -> output offsets, totals.
//   k_mc_emit  : one block per voxel.  Ranks the crossed edges in a fixed order (block-wide scan in shared memory), writes
//                vertex (rank) at the linearly interpolated zero crossing in world coordinates,
//                   v = ((lattice position) / (res-1) - 0.5) * voxel_size + centre          (mesh_util.py:152-161)
//                and the triangles as vertex ids, in voxel-major, cell-major order.
//
// The case table is not the classic hand-made 256 x 16 list: it is DERIVED at first use by tracing, for each of the 256 sign
// configurations, the zero-level segments across the six faces of the cube (marching squares per face) and joining them into
// closed loops, which are fan-triangulated.  The two-segment (ambiguous) face case is resolved by a rule that depends on the
// face's own four corner signs only (the negative corners are cut off separately), so the two cells sharing a face always
// agree on it: the surface is watertight across cells, which the classic table does not guarantee.  Triangles are oriented
// with their normal towards increasing SDF (outside).
#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "nl_cuda.cuh"

namespace {

constexpr int MC_MAX_TRI = 5;              // checked when the table is built
constexpr int MC_ROW = 3 * MC_MAX_TRI + 1; // edge triples, terminated by 255

// corner i sits at (i & 1, (i >> 1) & 1, (i >> 2) & 1); edge e = 4 * axis + k joins the two corners that differ along `axis`,
// k enumerating the 4 positions of the other two coordinates (lower axis = low bit)
struct McTables {
    uint8_t tri[256][MC_ROW];
    uint8_t ntri[256];
    uint8_t edge_corner[12][2];
};

inline int corner_of(int x, int y, int z) { return x | (y << 1) | (z << 2); }

void edge_corners(int e, int &c0, int &c1) {
    const int axis = e >> 2, k = e & 3;
    int xyz[3];
    const int o0 = (axis + 1) % 3, o1 = (axis + 2) % 3;
    const int lo = std::min(o0, o1), hi = std::max(o0, o1);
    xyz[lo] = k & 1; xyz[hi] = k >> 1;
    xyz[axis] = 0; c0 = corner_of(xyz[0], xyz[1], xyz[2]);
    xyz[axis] = 1; c1 = corner_of(xyz[0], xyz[1], xyz[2]);
}

int edge_between(int ca, int cb) {
    for (int e = 0; e < 12; ++e) {
        int c0, c1;
        edge_corners(e, c0, c1);
        if ((c0 == ca && c1 == cb) || (c0 == cb && c1 == ca)) return e;
    }
    return -1;
}

bool build_tables(McTables &T) {
    for (int e = 0; e < 12; ++e) {
        int c0, c1;
        edge_corners(e, c0, c1);
        T.edge_corner[e][0] = (uint8_t)c0; T.edge_corner[e][1] = (uint8_t)c1;
    }
    // the six faces as corner cycles (consecutive corners share a cube edge)
    int faces[6][4];
    for (int axis = 0; axis < 3; ++axis)
        for (int side = 0; side < 2; ++side) {
            const int a = (axis + 1) % 3, b = (axis + 2) % 3;
            const int uv[4][2] = {{0, 0}, {1, 0}, {1, 1}, {0, 1}};
            for (int i = 0; i < 4; ++i) {
                int xyz[3];
                xyz[axis] = side; xyz[a] = uv[i][0]; xyz[b] = uv[i][1];
                faces[axis * 2 + side][i] = corner_of(xyz[0], xyz[1], xyz[2]);
            }
        }
    int max_tri = 0;
    for (int cfg = 0; cfg < 256; ++cfg) {
        auto inside = [&](int c) { return (cfg >> c) & 1; };     // bit set: sdf < 0 at that corner
        int nbr[12][2], deg[12];
        for (int e = 0; e < 12; ++e) { deg[e] = 0; nbr[e][0] = nbr[e][1] = -1; }
        auto link = [&](int ea, int eb) { nbr[ea][deg[ea]++] = eb; nbr[eb][deg[eb]++] = ea; };
        for (int f = 0; f < 6; ++f) {
            int ce[4], nc = 0;                                   // crossed edges of this face, in cycle order: edge i joins corner i and i+1
            for (int i = 0; i < 4; ++i) {
                const int ca = faces[f][i], cb = faces[f][(i + 1) & 3];
                if (inside(ca) != inside(cb)) ce[nc++] = i;
            }
            auto E = [&](int i) { return edge_between(faces[f][i], faces[f][(i + 1) & 3]); };
            if (nc == 2) {
                link(E(ce[0]), E(ce[1]));
            } else if (nc == 4) {
                // two inside corners on a diagonal: cut each of them off on its own (edges i-1 and i around inside corner i)
                for (int i = 0; i < 4; ++i)
                    if (inside(faces[f][i])) link(E((i + 3) & 3), E(i));
            }
        }
        int nt = 0;
        bool seen[12] = {};
        for (int e0 = 0; e0 < 12; ++e0) {
            if (deg[e0] == 0 || seen[e0]) continue;
            if (deg[e0] != 2) return false;
            std::vector<int> loop;
            int prev = -1, cur = e0;
            while (cur != -1 && !seen[cur]) {
                seen[cur] = true;
                loop.push_back(cur);
                const int nx = (nbr[cur][0] != prev) ? nbr[cur][0] : nbr[cur][1];
                prev = cur; cur = nx;
                if (cur == e0) break;
            }
            if (loop.size() < 3) return false;
            // orientation: polygon normal (edge mid-points) must point from the inside corners towards the outside ones
            double P[12][3], n[3] = {0, 0, 0}, dir[3] = {0, 0, 0};
            for (size_t i = 0; i < loop.size(); ++i) {
                const int c0 = T.edge_corner[loop[i]][0], c1 = T.edge_corner[loop[i]][1];
                for (int a = 0; a < 3; ++a) {
                    const double x0 = (c0 >> a) & 1, x1 = (c1 >> a) & 1;
                    P[i][a] = 0.5 * (x0 + x1);
                    dir[a] += inside(c0) ? (x1 - x0) : (x0 - x1);
                }
            }
            for (size_t i = 0; i < loop.size(); ++i) {           // Newell's method
                const double *a = P[i], *b = P[(i + 1) % loop.size()];
                n[0] += (a[1] - b[1]) * (a[2] + b[2]);
                n[1] += (a[2] - b[2]) * (a[0] + b[0]);
                n[2] += (a[0] - b[0]) * (a[1] + b[1]);
            }
            if (n[0] * dir[0] + n[1] * dir[1] + n[2] * dir[2] < 0) std::reverse(loop.begin(), loop.end());
            for (size_t i = 1; i + 1 < loop.size(); ++i) {
                if (nt >= MC_MAX_TRI) return false;
                T.tri[cfg][3 * nt] = (uint8_t)loop[0]; T.tri[cfg][3 * nt + 1] = (uint8_t)loop[i]; T.tri[cfg][3 * nt + 2] = (uint8_t)loop[i + 1];
                ++nt;
            }
        }
        for (int i = 3 * nt; i < MC_ROW; ++i) T.tri[cfg][i] = 255;
        T.ntri[cfg] = (uint8_t)nt;
        max_tri = std::max(max_tri, nt);
    }
    return max_tri <= MC_MAX_TRI;
}

const McTables *host_tables() {
    static McTables T;
    static int state = 0;   // 0 not built, 1 ok, -1 failed
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    if (state == 0) state = build_tables(T) ? 1 : -1;
    return state == 1 ? &T : nullptr;
}

__constant__ McTables c_mc;

// lattice edge id inside one voxel: axis a in {0:x, 1:y, 2:z}, base point (i,j,k) with the coordinate along a < res-1.
// lattice point (i,j,k) <-> sdf[(i*res + j)*res + k]   (get_scores: meshgrid(x,y,z) 'ij', render_helpers.py:113-117)
__device__ __forceinline__ int lat(int i, int j, int k, int res) { return (i * res + j) * res + k; }

struct McShape {
    int res, ncell, nedge_axis;   // (res-1)^3 cells, res*res*(res-1) edges per axis
};

__device__ __forceinline__ void edge_decode(int id, const McShape &s, int &axis, int &i, int &j, int &k) {
    axis = id / s.nedge_axis;
    int r = id - axis * s.nedge_axis;
    const int m = s.res - 1;
    // the coordinate along `axis` runs over res-1 values, the other two over res
    if (axis == 0) { i = r / (s.res * s.res); r -= i * s.res * s.res; j = r / s.res; k = r - j * s.res; }
    else if (axis == 1) { i = r / (m * s.res); r -= i * m * s.res; j = r / s.res; k = r - j * s.res; }
    else { i = r / (s.res * m); r -= i * s.res * m; j = r / m; k = r - j * m; }
}
__device__ __forceinline__ int edge_encode(int axis, int i, int j, int k, const McShape &s) {
    const int m = s.res - 1;
    if (axis == 0) return (i * s.res + j) * s.res + k;
    if (axis == 1) return s.nedge_axis + (i * m + j) * s.res + k;
    return 2 * s.nedge_axis + (i * s.res + j) * m + k;
}

__device__ __forceinline__ bool neg(float v) { return v < 0.0f; }

constexpr int MC_THREADS = 256;
constexpr int MC_MAX_RES = 16;             // lattice staged in shared memory: 16^3 floats = 16 KB

__device__ __forceinline__ int cell_config(const float *s_sdf, int ci, int cj, int ck, int res) {
    int cfg = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c)
        cfg |= neg(s_sdf[lat(ci + (c & 1), cj + ((c >> 1) & 1), ck + ((c >> 2) & 1), res)]) ? (1 << c) : 0;
    return cfg;
}

__global__ void __launch_bounds__(MC_THREADS) k_mc_count(int n_vox, int res, const float *__restrict__ sdf, int32_t *__restrict__ nvert,
                                                          int32_t *__restrict__ ntri) {
    __shared__ float s_sdf[MC_MAX_RES * MC_MAX_RES * MC_MAX_RES];
    __shared__ int s_cnt[2];
    const int v = blockIdx.x;
    if (v >= n_vox) return;
    const McShape sh = {res, (res - 1) * (res - 1) * (res - 1), res * res * (res - 1)};
    const int npt = res * res * res;
    for (int i = threadIdx.x; i < npt; i += MC_THREADS) s_sdf[i] = sdf[(size_t)v * npt + i];
    if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    int nv = 0, nt = 0;
    for (int id = threadIdx.x; id < 3 * sh.nedge_axis; id += MC_THREADS) {
        int a, i, j, k;
        edge_decode(id, sh, a, i, j, k);
        const float s0 = s_sdf[lat(i, j, k, res)], s1 = s_sdf[lat(i + (a == 0), j + (a == 1), k + (a == 2), res)];
        nv += neg(s0) != neg(s1);
    }
    const int m = res - 1;
    for (int c = threadIdx.x; c < sh.ncell; c += MC_THREADS) {
        const int ci = c / (m * m), cj = (c / m) % m, ck = c % m;
        nt += c_mc.ntri[cell_config(s_sdf, ci, cj, ck, res)];
    }
    for (int off = 16; off > 0; off >>= 1) { nv += __shfl_down_sync(0xffffffffu, nv, off); nt += __shfl_down_sync(0xffffffffu, nt, off); }
    if ((threadIdx.x & 31) == 0) { atomicAdd(&s_cnt[0], nv); atomicAdd(&s_cnt[1], nt); }
    __syncthreads();
    if (threadIdx.x == 0) { nvert[v] = s_cnt[0]; ntri[v] = s_cnt[1]; }
}

// exclusive scan of two int arrays of n entries (n = voxels: 1e4..1e6), one block; totals -> totals[0..1]
__global__ void __launch_bounds__(1024) k_mc_scan(int n, const int32_t *__restrict__ a, const int32_t *__restrict__ b, int32_t *__restrict__ oa,
                                                   int32_t *__restrict__ ob, int64_t *__restrict__ totals) {
    __shared__ long long wsum[2][32];
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    long long ca = 0, cb = 0;
    for (int base = 0; base < n; base += 1024) {
        const int i = base + t;
        const long long xa = i < n ? a[i] : 0, xb = i < n ? b[i] : 0;
        long long ia = xa, ib = xb;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const long long ya = __shfl_up_sync(0xffffffffu, ia, off), yb = __shfl_up_sync(0xffffffffu, ib, off);
            if (lane >= off) { ia += ya; ib += yb; }
        }
        if (lane == 31) { wsum[0][w] = ia; wsum[1][w] = ib; }
        __syncthreads();
        long long pa = 0, pb = 0, ta = 0, tb = 0;
        for (int k = 0; k < 32; ++k) {
            if (k < w) { pa += wsum[0][k]; pb += wsum[1][k]; }
            ta += wsum[0][k]; tb += wsum[1][k];
        }
        if (i < n) { oa[i] = (int32_t)(ca + pa + ia - xa); ob[i] = (int32_t)(cb + pb + ib - xb); }
        ca += ta; cb += tb;
        __syncthreads();
    }
    if (t == 0) { totals[0] = ca; totals[1] = cb; }
}

__global__ void __launch_bounds__(MC_THREADS) k_mc_emit(int n_vox, int res, float voxel_size, const float *__restrict__ sdf,
                                                         const float *__restrict__ centres, const int32_t *__restrict__ vox_ids,
                                                         const int32_t *__restrict__ voff, const int32_t *__restrict__ toff,
                                                         int64_t vcap, int64_t tcap, float *__restrict__ verts, int32_t *__restrict__ faces) {
    __shared__ float s_sdf[MC_MAX_RES * MC_MAX_RES * MC_MAX_RES];
    __shared__ int16_t s_rank[3 * MC_MAX_RES * MC_MAX_RES * (MC_MAX_RES - 1)];   // rank of a crossed edge among the voxel's vertices, -1 otherwise
    __shared__ int s_warp[MC_THREADS / 32];
    __shared__ int s_carry;
    const int v = blockIdx.x;
    if (v >= n_vox) return;
    const McShape sh = {res, (res - 1) * (res - 1) * (res - 1), res * res * (res - 1)};
    const int npt = res * res * res, nedge = 3 * sh.nedge_axis;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    for (int i = t; i < npt; i += MC_THREADS) s_sdf[i] = sdf[(size_t)v * npt + i];
    if (t == 0) s_carry = 0;
    __syncthreads();
    const int node = vox_ids ? vox_ids[v] : v;
    const float cx = centres[(size_t)node * 3], cy = centres[(size_t)node * 3 + 1], cz = centres[(size_t)node * 3 + 2];
    const float inv = 1.0f / (float)(res - 1);
    const int vbase = voff[v];
    // ---- vertices: rank the crossed edges in id order (tiles of MC_THREADS ids, block scan per tile) ----
    for (int base = 0; base < nedge; base += MC_THREADS) {
        const int id = base + t;
        int a = 0, i = 0, j = 0, k = 0;
        float s0 = 1.f, s1 = 1.f;
        bool cross = false;
        if (id < nedge) {
            edge_decode(id, sh, a, i, j, k);
            s0 = s_sdf[lat(i, j, k, res)];
            s1 = s_sdf[lat(i + (a == 0), j + (a == 1), k + (a == 2), res)];
            cross = neg(s0) != neg(s1);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, cross);
        if (lane == 0) s_warp[w] = __popc(bal);
        __syncthreads();
        int pre = s_carry;
        for (int q = 0; q < w; ++q) pre += s_warp[q];
        const int rank = pre + __popc(bal & ((1u << lane) - 1u));
        if (id < nedge) s_rank[id] = cross ? (int16_t)rank : (int16_t)-1;
        if (cross && (int64_t)vbase + rank < vcap) {
            const float tt = s0 / (s0 - s1);                                  // zero crossing between the two lattice points
            float p[3] = {(float)i, (float)j, (float)k};
            p[a] += tt;
            float *o = verts + (size_t)(vbase + rank) * 3;
            // mesh_util.py:149-161: spacing 1/(res-1), -0.5, * voxel_size, + centre -- four separately rounded steps, written
            // with explicit roundings so that nvcc does not contract them into two FMAs (tests/mesh_ref.py restates them)
            o[0] = __fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(p[0], inv), 0.5f), voxel_size), cx);
            o[1] = __fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(p[1], inv), 0.5f), voxel_size), cy);
            o[2] = __fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(p[2], inv), 0.5f), voxel_size), cz);
        }
        __syncthreads();
        if (t == 0) { int tot = 0; for (int q = 0; q < MC_THREADS / 32; ++q) tot += s_warp[q]; s_carry += tot; }
        __syncthreads();
    }
    // ---- triangles: cells in order, block scan of the per-cell counts per tile ----
    if (t == 0) s_carry = 0;
    __syncthreads();
    const int m = res - 1;
    const int tbase = toff[v];
    for (int base = 0; base < sh.ncell; base += MC_THREADS) {
        const int c = base + t;
        int cfg = 0, nt = 0, ci = 0, cj = 0, ck = 0;
        if (c < sh.ncell) {
            ci = c / (m * m); cj = (c / m) % m; ck = c % m;
            cfg = cell_config(s_sdf, ci, cj, ck, res);
            nt = c_mc.ntri[cfg];
        }
        int incl = nt;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= off) incl += y;
        }
        if (lane == 31) s_warp[w] = incl;
        __syncthreads();
        int pre = s_carry;
        for (int q = 0; q < w; ++q) pre += s_warp[q];
        int64_t out = (int64_t)tbase + pre + incl - nt;
        for (int q = 0; q < nt; ++q, ++out) {
            if (out >= tcap) break;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const int e = c_mc.tri[cfg][3 * q + r];
                const int c0 = c_mc.edge_corner[e][0];
                const int axis = e >> 2;
                const int id = edge_encode(axis, ci + (c0 & 1), cj + ((c0 >> 1) & 1), ck + ((c0 >> 2) & 1), sh);
                faces[(size_t)out * 3 + r] = vbase + (int)s_rank[id];
            }
        }
        __syncthreads();
        if (t == 0) { int tot = 0; for (int q = 0; q < MC_THREADS / 32; ++q) tot += s_warp[q]; s_carry += tot; }
        __syncthreads();
    }
}

NlPerDevice g_tables_uploaded;

int upload_tables() {
    const McTables *T = host_tables();
    if (!T) return nl_set_error("marching cubes: case table construction failed");
    const cudaError_t e = g_tables_uploaded.once([&] { return cudaMemcpyToSymbol(c_mc, T, sizeof(McTables)); });
    if (e != cudaSuccess) return nl_set_error_code(NL_ERR_CUDA, cudaGetErrorString(e));
    return NL_OK;
}

}  // namespace

extern "C" int nl_mc_case_table(uint8_t *h_tri, uint8_t *h_ntri, uint8_t *h_edge_corner) {
    const McTables *T = host_tables();
    if (!T) return nl_set_error("nl_mc_case_table: construction failed");
    if (h_tri) std::memcpy(h_tri, T->tri, sizeof(T->tri));
    if (h_ntri) std::memcpy(h_ntri, T->ntri, sizeof(T->ntri));
    if (h_edge_corner) std::memcpy(h_edge_corner, T->edge_corner, sizeof(T->edge_corner));
    return NL_OK;
}

extern "C" int nl_mc_count(int32_t n_vox, int32_t res, const float *d_sdf, int32_t *d_nvert, int32_t *d_ntri, int32_t *d_voff, int32_t *d_toff,
                           int64_t *d_totals, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (n_vox < 0 || res < 2 || res > MC_MAX_RES) return nl_set_error("nl_mc_count: need n_vox >= 0 and 2 <= res <= 16");
    // no voxels (an empty map): nothing is read or written but the totals, so the per-voxel pointers may be null
    if ((n_vox > 0 && (!d_sdf || !d_nvert || !d_ntri || !d_voff || !d_toff)) || !d_totals) return nl_set_error("nl_mc_count: null pointer");
    if (int rc = upload_tables()) return rc;
    if (n_vox > 0) k_mc_count<<<n_vox, MC_THREADS, 0, stream>>>(n_vox, res, d_sdf, d_nvert, d_ntri);
    k_mc_scan<<<1, 1024, 0, stream>>>(n_vox, d_nvert, d_ntri, d_voff, d_toff, d_totals);
    NL_CHECK_LAUNCH("nl_mc_count");
    return NL_OK;
}

extern "C" int nl_mc_emit(int32_t n_vox, int32_t res, float voxel_size, const float *d_sdf, const float *d_centres, const int32_t *d_vox_ids,
                          const int32_t *d_voff, const int32_t *d_toff, int64_t vert_capacity, int64_t tri_capacity, float *d_verts,
                          int32_t *d_faces, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (n_vox < 0 || res < 2 || res > MC_MAX_RES) return nl_set_error("nl_mc_emit: need n_vox >= 0 and 2 <= res <= 16");
    if ((n_vox > 0 && (!d_sdf || !d_centres || !d_voff || !d_toff)) || (vert_capacity > 0 && !d_verts) || (tri_capacity > 0 && !d_faces))
        return nl_set_error("nl_mc_emit: null pointer");
    // offsets and face entries are int32 vertex / triangle ids: a mesh with more than INT32_MAX of either cannot be written
    if (vert_capacity > INT32_MAX || tri_capacity > INT32_MAX) return nl_set_error("nl_mc_emit: capacities above INT32_MAX");
    if (int rc = upload_tables()) return rc;
    if (n_vox > 0)
        k_mc_emit<<<n_vox, MC_THREADS, 0, stream>>>(n_vox, res, voxel_size, d_sdf, d_centres, d_vox_ids, d_voff, d_toff, vert_capacity, tri_capacity,
                                                   d_verts, d_faces);
    NL_CHECK_LAUNCH("nl_mc_emit");
    return NL_OK;
}
