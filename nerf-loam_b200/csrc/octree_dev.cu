// Device-side octree insertion (include/nerfloam_b200.h section 1b): the host octree's insert (octree_host.cpp, the reference's
// octree.cpp:51-111) and the map-update glue around it (mapping.py:283-339) as kernels, producing the same node ids, types,
// dirty rows and embedding-row numbering bit for bit.
//
// The host loops over points i, corners j = 0..7 and levels d = 1..L and creates every missing node it visits, so a new node's
// id is its rank among the new nodes ordered by their first visiting triple (i, j, d).  A node's first visit is the smallest
// p = 8i + j whose corner lies inside it, at the node's own level; ancestors have a superset of corners, so ordering the new nodes
// by pmin * L + (d - 1) reproduces the creation order.  One insert:
//   count  k_corners   validate the batch, descend the existing tree per (point, corner) to the first missing level dm
//          sort        the 8n corner Morton keys (stable: equal keys keep ascending p); corners whose leaf exists sort last
//          k_count     a level-d node is a run of keys sharing their top 3d bits; position k starts new nodes at the levels
//                      max(dm, first level at which key[k] differs from key[k-1]) .. L  -> exclusive scan = slot offsets
//   commit k_slots     one slot per new node, with the slot (or existing id) of its parent
//          k_pmin      leaf runs carry their first p up the parent chain with atomicMin (a walk stops where a smaller value already
//                      is: the thread that stored it carries it further); j == 0 corners flag their leaf SURFACE
//          sort        slots by pmin * L + (d - 1) -> ids n_before + rank
//          k_build, k_link, k_promote   node arrays, child slots (exactly one writer each), FEATURE -> SURFACE promotion,
//                      existing dirty rows appended once (CAS on a per-node scratch word) to a pending list
//   export k_dirty_tail  sorted pending list + the new id range = dirty rows in ascending id order; k_export writes them in
//                      nl_octree_export_map's layout; k_first / k_rflag / scan / k_assign number the new embedding rows in
//                      nl_assign_embedding_rows_subset's order, k_vox2row composes the rows of the dirty nodes.
// No step depends on the order in which atomics land, so every run gives the same arrays.
//
// The queries (get_centres_and_children, get_voxels, get_leaf_voxels, try_insert) follow the insert path: k_export with the
// host export_row's optional outputs, preorder as one stable sort of the node codes, try_insert as two sorts of the batch's
// corner keys (see the comment above k_pre_init).
#include <cub/cub.cuh>

#include <climits>
#include <cstdint>
#include <cstdio>

#include "../../include/nerfloam_b200.h"
#include "nl_cuda.cuh"

namespace {

enum : int8_t { kNonLeaf = -1, kSurface = 0, kFeature = 1 };  // octree.h:5-10
constexpr int32_t kRest = INT_MAX;        // resting value of the per-node scratch word
constexpr uint32_t kNone = 0xffffffffu;   // empty entry of the pending dirty list
constexpr int64_t kMaxPoints = 1 << 23;   // keeps 8n * L (the first-visit sequence numbers) below 2^31
constexpr int kThreads = 256;

__host__ __device__ __forceinline__ uint64_t spread3(uint64_t v) {
    uint64_t x = v & 0x1fffffULL;
    x = (x | x << 32) & 0x1f00000000ffffULL;
    x = (x | x << 16) & 0x1f0000ff0000ffULL;
    x = (x | x << 8) & 0x100f00f00f00f00fULL;
    x = (x | x << 4) & 0x10c30c30c30c30c3ULL;
    x = (x | x << 2) & 0x1249249249249249ULL;
    return x;
}
__device__ __forceinline__ uint64_t squeeze3(uint64_t v) {
    uint64_t x = v & 0x1249249249249249ULL;
    x = (x | x >> 2) & 0x10c30c30c30c30c3ULL;
    x = (x | x >> 4) & 0x100f00f00f00f00fULL;
    x = (x | x >> 8) & 0x1f0000ff0000ffULL;
    x = (x | x >> 16) & 0x1f00000000ffffULL;
    x = (x | x >> 32) & 0x1fffffULL;
    return x;
}
__device__ __forceinline__ uint64_t morton(int x, int y, int z) {
    return spread3((uint64_t)x) | (spread3((uint64_t)y) << 1) | (spread3((uint64_t)z) << 2);
}
// first index in a[0, hi) with a[i] >= v
__device__ __forceinline__ int lower_bound(const uint64_t *__restrict__ a, int hi, uint64_t v) {
    int lo = 0;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ int find_node(const int32_t *__restrict__ child, int L, int size, int x, int y, int z) {  // octree.cpp:151-171
    int n = 0;
    unsigned edge = (unsigned)size >> 1;
    for (int d = 1; d <= L; ++d, edge >>= 1) {
        const int slot = ((x & edge) > 0) + 2 * ((y & edge) > 0) + 4 * ((z & edge) > 0);
        const int c = child[(size_t)n * 8 + slot];
        if (c < 0) return -1;
        n = c;
    }
    return n;
}
// existing nodes of the previous export whose row changes: appended once to the pending list
__device__ __forceinline__ void mark_dirty(int32_t id, int64_t base, int32_t *scratch, uint32_t *list, int64_t *counts) {
    if (id < base && atomicCAS(&scratch[id], kRest, 0) == kRest)
        list[atomicAdd((unsigned long long *)&counts[4], 1ull)] = (uint32_t)id;
}

int levels_of(int64_t grid_dim) {
    if (grid_dim < 2 || grid_dim > (1 << 20) || (grid_dim & (grid_dim - 1))) return -1;
    int L = 0;
    while ((int64_t(1) << L) < grid_dim) ++L;
    return L;
}

// Workspace layout for a batch of n points (everything is a function of n and L alone).
struct Layout {
    int L = 0, rank_bits = 0;
    int64_t n = 0, P = 0, T = 0, D = 0, M = 0, E = 0;
    // insert phase
    size_t keys_a, keys_b, vals_a, vals_b, dm, lo, enode, eparent, cnt, off, spos, par, pmin, surf, sid, k2a, k2b, v2a, v2b, tmp_ins;
    size_t tmp_ins_bytes = 0;
    // export phase (aliases the insert phase)
    size_t dsorted, sflag, sids, ns, rflag, rscan, tmp_exp;
    size_t tmp_exp_bytes = 0;
    size_t total = 0;
};

size_t take(size_t &at, size_t bytes) {
    const size_t o = (at + 255) & ~size_t(255);
    at = o + bytes;
    return o;
}

cudaError_t make_layout(int64_t n, int L, Layout &l) {
    l.L = L;
    l.n = n;
    l.P = 8 * n;
    l.T = 0;
    for (int d = 1; d <= L; ++d) l.T += (3 * d < 62 && (int64_t(1) << (3 * d)) < l.P) ? (int64_t(1) << (3 * d)) : l.P;
    l.D = l.P + 2 * n;
    l.M = l.T + l.D;
    l.E = 8 * n;
    const uint64_t seq_max = (uint64_t)l.P * (uint64_t)L;
    l.rank_bits = 1;
    while ((uint64_t(1) << l.rank_bits) <= seq_max) ++l.rank_bits;
    const int P = (int)l.P, T = (int)l.T, D = (int)l.D, M = (int)l.M, E = (int)l.E;
    size_t a = 0, b = 0, c = 0, d = 0, e = 0, f = 0;
    cudaError_t err;
    {
        cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
        cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
        if ((err = cub::DeviceRadixSort::SortPairs(nullptr, a, k, v, P, 0, 3 * L + 1)) != cudaSuccess) return err;
    }
    {
        cub::DoubleBuffer<uint32_t> k(nullptr, nullptr), v(nullptr, nullptr);
        if ((err = cub::DeviceRadixSort::SortPairs(nullptr, b, k, v, T, 0, l.rank_bits)) != cudaSuccess) return err;
        if ((err = cub::DeviceRadixSort::SortKeys(nullptr, d, k, D, 0, 32)) != cudaSuccess) return err;
    }
    if ((err = cub::DeviceScan::ExclusiveSum(nullptr, c, (const int32_t *)nullptr, (int32_t *)nullptr, P + 1)) != cudaSuccess) return err;
    if ((err = cub::DeviceSelect::Flagged(nullptr, e, (const int32_t *)nullptr, (const uint8_t *)nullptr, (int32_t *)nullptr,
                                          (int32_t *)nullptr, M)) != cudaSuccess)
        return err;
    if ((err = cub::DeviceScan::ExclusiveSum(nullptr, f, (const int32_t *)nullptr, (int32_t *)nullptr, E)) != cudaSuccess) return err;
    l.tmp_ins_bytes = std::max(std::max(a, b), c);
    l.tmp_exp_bytes = std::max(std::max(d, e), f);
    size_t at = 0;
    l.keys_a = take(at, 8 * (size_t)P); l.keys_b = take(at, 8 * (size_t)P);
    l.vals_a = take(at, 4 * (size_t)P); l.vals_b = take(at, 4 * (size_t)P);
    l.dm = take(at, (size_t)P); l.lo = take(at, (size_t)P);
    l.enode = take(at, 4 * (size_t)P); l.eparent = take(at, 4 * (size_t)P);
    l.cnt = take(at, 4 * (size_t)(P + 1)); l.off = take(at, 4 * (size_t)(P + 1));
    l.spos = take(at, 4 * (size_t)T); l.par = take(at, 4 * (size_t)T); l.pmin = take(at, 4 * (size_t)T);
    l.surf = take(at, (size_t)T); l.sid = take(at, 4 * (size_t)T);
    l.k2a = take(at, 4 * (size_t)T); l.k2b = take(at, 4 * (size_t)T); l.v2a = take(at, 4 * (size_t)T); l.v2b = take(at, 4 * (size_t)T);
    l.tmp_ins = take(at, l.tmp_ins_bytes);
    const size_t ins_end = at;
    at = 0;
    l.dsorted = take(at, 4 * (size_t)D);
    l.sflag = take(at, (size_t)M);
    l.sids = take(at, 4 * (size_t)n);
    l.ns = take(at, 4);
    l.rflag = take(at, 4 * (size_t)E); l.rscan = take(at, 4 * (size_t)E);
    l.tmp_exp = take(at, l.tmp_exp_bytes);
    l.total = std::max(ins_end, at);
    return cudaSuccess;
}

template <class T_>
T_ *at(void *ws, size_t off) { return reinterpret_cast<T_ *>(static_cast<char *>(ws) + off); }

int cuda_fail(const char *what, cudaError_t e) {
    char buf[256];
    std::snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
    return nl_set_error_code(NL_ERR_CUDA, buf);
}

// ---------------------------------------------------------------------------------------------------------------------------
__global__ void k_corners(int n, int L, int size, const int32_t *__restrict__ vox, const int32_t *__restrict__ child, uint64_t *keys,
                          uint32_t *vals, uint8_t *dm, int32_t *enode, int32_t *eparent, int64_t *counts) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= 8 * n) return;
    const int i = p >> 3, j = p & 7;
    const uint64_t none = uint64_t(1) << (3 * L);
    const int px = vox[3 * i], py = vox[3 * i + 1], pz = vox[3 * i + 2];
    vals[p] = (uint32_t)p;
    // (not `px + 1 >= size`: for px = INT32_MAX that overflows, and the point would pass and alias into the grid)
    if (px < 0 || py < 0 || pz < 0 || px >= size - 1 || py >= size - 1 || pz >= size - 1) {
        counts[0] = 1;                      // the batch is rejected after the read-back; nothing below modifies the tree
        keys[p] = none; dm[p] = (uint8_t)(L + 1); enode[p] = -1; eparent[p] = -1;
        return;
    }
    const int x = px + (j >> 2), y = py + ((j >> 1) & 1), z = pz + (j & 1);   // octree.cpp:12-14
    int node = 0, parent = -1, d = 1;
    unsigned edge = (unsigned)size >> 1;
    for (; d <= L; ++d, edge >>= 1) {
        const int slot = ((x & edge) > 0) + 2 * ((y & edge) > 0) + 4 * ((z & edge) > 0);
        const int c = child[(size_t)node * 8 + slot];
        if (c < 0) break;
        parent = node;
        node = c;
    }
    dm[p] = (uint8_t)d;
    enode[p] = node;        // deepest existing node on the path: the parent of the first new one, or the leaf
    eparent[p] = parent;
    keys[p] = d <= L ? morton(x, y, z) : none;
}

__global__ void k_count(int P, int L, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals, const uint8_t *__restrict__ dm,
                        uint8_t *lo, int32_t *cnt) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k > P) return;
    int c = 0, l = L + 1;
    if (k < P) {
        const uint64_t key = keys[k];
        if (key < (uint64_t(1) << (3 * L))) {
            int ds = 1;
            if (k > 0) {
                const uint64_t x = key ^ keys[k - 1];
                ds = x ? L - (63 - __clzll((long long)x)) / 3 : L + 1;   // first level whose 3d-bit prefix differs from the previous key
            }
            l = max((int)dm[vals[k]], ds);
            c = l <= L ? L - l + 1 : 0;
        }
        lo[k] = (uint8_t)l;
    }
    cnt[k] = c;
}

__global__ void k_store_new(int P, const int32_t *__restrict__ off, int64_t *counts) { counts[1] = off[P]; }

__global__ void k_slots(int P, int L, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals, const uint8_t *__restrict__ dm,
                        const uint8_t *__restrict__ lo, const int32_t *__restrict__ off, const int32_t *__restrict__ enode, int32_t *spos,
                        int32_t *par, uint32_t *pmin, uint8_t *surf) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P) return;
    const int l = lo[k];
    if (l > L) return;
    const uint64_t key = keys[k];
    const uint32_t p = vals[k];
    const int dmk = dm[p];
    for (int d = l; d <= L; ++d) {
        const int t = off[k] + d - l;
        spos[t] = k;
        pmin[t] = kNone;
        surf[t] = 0;
        if (d == dmk) {
            par[t] = -2 - enode[p];                  // existing parent, encoded
        } else if (d > l) {
            par[t] = t - 1;                          // same position, one level up
        } else {                                     // the parent's run started at an earlier position
            const int sh = 3 * (L - d + 1);
            const int s = lower_bound(keys, k, (key >> sh) << sh);
            par[t] = off[s] + (d - 1) - lo[s];
        }
    }
}

__global__ void k_pmin(int P, int L, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals, const uint8_t *__restrict__ lo,
                       const int32_t *__restrict__ off, const int32_t *__restrict__ par, uint32_t *pmin, uint8_t *surf) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P) return;
    const uint64_t key = keys[k];
    if (key >= (uint64_t(1) << (3 * L))) return;
    const uint32_t p = vals[k];
    if (k == 0 || keys[k - 1] != key) {              // leaf run start: the stable sort put its smallest p first
        int t = off[k] + L - lo[k];
        while (true) {
            const uint32_t old = atomicMin(&pmin[t], p);
            if (old <= p) break;
            t = par[t];
            if (t < 0) break;
        }
    }
    if ((p & 7) == 0) {                              // corner 0 visits its leaf: SURFACE (octree.cpp:94-106)
        const int s = lower_bound(keys, k + 1, key);
        surf[off[s] + L - lo[s]] = 1;
    }
}

__global__ void k_seq(int T, int L, const int32_t *__restrict__ spos, const int32_t *__restrict__ off, const uint8_t *__restrict__ lo,
                      const uint32_t *__restrict__ pmin, uint32_t *seq, uint32_t *slot) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const int k = spos[t];
    const int d = lo[k] + t - off[k];
    seq[t] = pmin[t] * (uint32_t)L + (uint32_t)(d - 1);
    slot[t] = (uint32_t)t;
}

__global__ void k_build(int T, int L, int64_t n0, const uint32_t *__restrict__ order, const int32_t *__restrict__ spos,
                        const int32_t *__restrict__ off, const uint8_t *__restrict__ lo, const uint64_t *__restrict__ keys,
                        const uint8_t *__restrict__ surf, int32_t *sid, int32_t *child, uint64_t *code, int8_t *type, uint8_t *level) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= T) return;
    const int t = (int)order[r];
    const int64_t id = n0 + r;
    sid[t] = (int32_t)id;
    const int k = spos[t];
    const int d = lo[k] + t - off[k];
    const int sh = 3 * (L - d);
    code[id] = (keys[k] >> sh) << sh;                // key & lvl_mask[d] (octree.cpp:79-80)
    type[id] = d < L ? kNonLeaf : (surf[t] ? kSurface : kFeature);
    level[id] = (uint8_t)d;
    int4 *c = reinterpret_cast<int4 *>(child + id * 8);
    c[0] = make_int4(-1, -1, -1, -1);
    c[1] = make_int4(-1, -1, -1, -1);
}

__global__ void k_link(int T, int L, int64_t base, const int32_t *__restrict__ spos, const int32_t *__restrict__ off,
                       const uint8_t *__restrict__ lo, const uint64_t *__restrict__ keys, const int32_t *__restrict__ par,
                       const int32_t *__restrict__ sid, int32_t *child, int32_t *scratch, uint32_t *list, int64_t *counts) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const int k = spos[t];
    const int d = lo[k] + t - off[k];
    const int q = par[t];
    const int32_t pid = q < 0 ? -2 - q : sid[q];
    child[(size_t)pid * 8 + ((keys[k] >> (3 * (L - d))) & 7)] = sid[t];   // slot = (x&edge>0) + 2(y&edge>0) + 4(z&edge>0)
    if (q < 0) mark_dirty(pid, base, scratch, list, counts);
}

__global__ void k_promote(int P, int L, int64_t base, const uint8_t *__restrict__ dm, const int32_t *__restrict__ enode,
                          const int32_t *__restrict__ eparent, int8_t *type, int32_t *scratch, uint32_t *list, int64_t *counts) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P || (p & 7) || dm[p] != L + 1) return;
    const int leaf = enode[p];
    if (leaf < 0 || type[leaf] != kFeature) return;
    type[leaf] = kSurface;                           // octree.cpp:102-106; concurrent writers store the same value
    mark_dirty(leaf, base, scratch, list, counts);
    mark_dirty(eparent[p], base, scratch, list, counts);
}

__global__ void k_dirty_tail(int n_list, int64_t n_new, int64_t base, const uint32_t *__restrict__ sorted, uint32_t *list, int32_t *scratch,
                             int32_t *ids, int64_t *counts) {
    const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t m_old = counts[4];
    if (o < n_list) {
        if (o < m_old) {
            const uint32_t id = sorted[o];
            ids[o] = (int32_t)id;
            scratch[id] = kRest;
        }
        list[o] = kNone;                             // (may alias `sorted`: each thread reads its own entry first)
    } else if (o < n_list + n_new) {
        const int64_t r = o - n_list;
        ids[m_old + r] = (int32_t)(base + r);
    }
    if (o == 0) counts[2] = m_old + n_new;
}

__global__ void k_reset_pending(int64_t *counts) { counts[4] = 0; }

// octree_host.cpp export_row: every output but vertex is optional (NULL = not written)
__global__ void k_export(int64_t rows, const int32_t *__restrict__ ids, const int64_t *__restrict__ count, int compact, int L, int size, float vs,
                         const int32_t *__restrict__ child, const uint64_t *__restrict__ code, const int8_t *__restrict__ type,
                         const uint8_t *__restrict__ level, float *voxels4, float *children_f, float *centres, int32_t *structure,
                         int32_t *vertex) {
    const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= rows || (count && o >= *count)) return;
    const int64_t id = ids ? ids[o] : o;
    const int64_t r = compact ? o : id;
    const int8_t ty = type[id];
    const bool visited = ty != kFeature;             // BFS reaches every non-FEATURE node (octree.cpp:330-338)
    float xyz[3] = {0.f, 0.f, 0.f}, sd = 0.f;
    if (visited) {
        const uint64_t c = code[id];
        xyz[0] = (float)(int)squeeze3(c);
        xyz[1] = (float)(int)squeeze3(c >> 1);
        xyz[2] = (float)(int)squeeze3(c >> 2);
        sd = (float)((unsigned)size >> level[id]);
    }
    if (voxels4) {
        for (int a = 0; a < 3; ++a) voxels4[r * 4 + a] = xyz[a];
        voxels4[r * 4 + 3] = sd;
    }
    const float h = sd / 2.0f;
    if (centres)
        for (int a = 0; a < 3; ++a) centres[r * 3 + a] = __fmul_rn(__fadd_rn(xyz[a], h), vs);   // mapping.py:322, all fp32
    for (int s = 0; s < 8; ++s) {
        const int32_t c = child[id * 8 + s];
        const int32_t v = (visited && c >= 0 && type[c] != kFeature) ? c : -1;
        if (structure) structure[r * 9 + s] = v;
        if (children_f) children_f[r * 8 + s] = (float)v;
    }
    if (structure) structure[r * 9 + 8] = (int32_t)sd;
    for (int k = 0; k < 8; ++k)
        vertex[r * 8 + k] = ty == kSurface ? find_node(child, L, size, (int)xyz[0] + (k >> 2), (int)xyz[1] + ((k >> 1) & 1), (int)xyz[2] + (k & 1)) : -1;
}

__global__ void k_sflag(int64_t rows, const int32_t *__restrict__ ids, const int64_t *__restrict__ counts, const int8_t *__restrict__ type,
                        uint8_t *flag) {
    const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= rows) return;
    flag[o] = o < counts[2] && type[ids[o]] == kSurface;
}

// the vertex of entry e of the SURFACE dirty rows, if it has no embedding row yet; else -1
__device__ __forceinline__ int new_vertex(int e, const int32_t *__restrict__ sids, const int32_t *__restrict__ ns, const int32_t *__restrict__ vertex,
                                          int64_t n_nodes, const int32_t *__restrict__ v2r) {
    if ((e >> 3) >= *ns) return -1;
    const int v = vertex[(size_t)sids[e >> 3] * 8 + (e & 7)];
    return (v >= 0 && v < n_nodes && v2r[v] < 0) ? v : -1;
}

__global__ void k_first(int E, const int32_t *__restrict__ sids, const int32_t *__restrict__ ns, const int32_t *__restrict__ vertex, int64_t n_nodes,
                        const int32_t *__restrict__ v2r, int32_t *scratch) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const int v = new_vertex(e, sids, ns, vertex, n_nodes, v2r);
    if (v >= 0) atomicMin(&scratch[v], e);
}

__global__ void k_rflag(int E, const int32_t *__restrict__ sids, const int32_t *__restrict__ ns, const int32_t *__restrict__ vertex, int64_t n_nodes,
                        const int32_t *__restrict__ v2r, const int32_t *__restrict__ scratch, int32_t *rflag) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const int v = new_vertex(e, sids, ns, vertex, n_nodes, v2r);
    rflag[e] = v >= 0 && scratch[v] == e;
}

__global__ void k_assign(int E, const int32_t *__restrict__ sids, const int32_t *__restrict__ ns, const int32_t *__restrict__ vertex,
                         const int32_t *__restrict__ rflag, const int32_t *__restrict__ rscan, int64_t n_emb, int32_t *v2r, int32_t *scratch) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E || !rflag[e]) return;
    const int v = vertex[(size_t)sids[e >> 3] * 8 + (e & 7)];
    v2r[v] = (int32_t)(n_emb + rscan[e]);
    scratch[v] = kRest;
}

__global__ void k_rows_total(int E, const int32_t *__restrict__ rflag, const int32_t *__restrict__ rscan, int64_t n_emb, int64_t *counts) {
    counts[3] = n_emb + (E ? rscan[E - 1] + rflag[E - 1] : 0);
}

__global__ void k_vox2row(int64_t rows, const int32_t *__restrict__ ids, const int64_t *__restrict__ counts, const int32_t *__restrict__ vertex,
                          int64_t n_nodes, const int32_t *__restrict__ v2r, int32_t *vox2row) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= rows * 8 || (e >> 3) >= counts[2]) return;
    const size_t i = (size_t)ids[e >> 3] * 8 + (e & 7);
    const int v = vertex[i];
    vox2row[i] = (v >= 0 && v < n_nodes) ? v2r[v] : -1;
}

__global__ void k_find(int64_t n, int L, int size, const int32_t *__restrict__ child, const int32_t *__restrict__ xyz, int32_t *out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    out[i] = (x < 0 || y < 0 || z < 0 || x >= size || y >= size || z >= size) ? -1 : find_node(child, L, size, x, y, z);
}

// ---------------------------------------------------------------------------------------------------------------------------
// Queries.  Preorder (get_voxels / get_leaf_voxels, octree.cpp:212-252): children are visited in slot order and the slot is the
// Morton digit of its level, so preorder is the order of (code, level); nodes with equal codes are an ancestor chain, created
// root first, so a stable sort of the codes with the node ids as values (ascending) is the preorder.
__global__ void k_pre_init(int N, const uint64_t *__restrict__ code, uint64_t *keys, uint32_t *vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    keys[i] = code[i];
    vals[i] = (uint32_t)i;
}

__global__ void k_pre_rows(int N, int size, const uint32_t *__restrict__ order, const uint64_t *__restrict__ code,
                           const uint8_t *__restrict__ level, float *out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    const uint32_t id = order[r];
    const uint64_t c = code[id];
    out[(size_t)r * 4 + 0] = (float)(int)squeeze3(c);
    out[(size_t)r * 4 + 1] = (float)(int)squeeze3(c >> 1);
    out[(size_t)r * 4 + 2] = (float)(int)squeeze3(c >> 2);
    out[(size_t)r * 4 + 3] = (float)((unsigned)size >> level[id]);
}

__global__ void k_pre_flag(int N, const uint32_t *__restrict__ order, const int8_t *__restrict__ type, uint8_t *flag) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < N) flag[r] = type[order[r]] == kSurface;   // SURFACE nodes are leaves: the walk lists them and returns
}

__global__ void k_leaf_rows(int N, const uint32_t *__restrict__ sel, const int64_t *__restrict__ count, const uint64_t *__restrict__ code,
                            float *out) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= N || o >= *count) return;
    const uint64_t c = code[sel[o]];
    out[(size_t)o * 3 + 0] = (float)(int)squeeze3(c);
    out[(size_t)o * 3 + 1] = (float)(int)squeeze3(c >> 1);
    out[(size_t)o * 3 + 2] = (float)(int)squeeze3(c >> 2);
}

// try_insert (octree_host.cpp nl_octree_try_insert, octree.cpp:113-149): |{(int32) k : k in keys, k a corner key}| / |keys| over
// the distinct corner keys of the batch.  The host's corner-key set is exactly the set of level-L node codes (every inserted
// corner creates its leaf, whose code is the corner's full key), so a key is a corner key iff it decodes to in-grid coordinates
// whose leaf exists.
__global__ void k_try_keys(int P, const int32_t *__restrict__ vox, uint64_t *keys) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int i = p >> 3, j = p & 7;
    // morton() keeps the low 21 bits of each coordinate: negative and out-of-grid corners alias exactly as on the host
    const uint64_t x = (uint32_t)vox[3 * i] + (uint32_t)(j >> 2), y = (uint32_t)vox[3 * i + 1] + (uint32_t)((j >> 1) & 1),
                   z = (uint32_t)vox[3 * i + 2] + (uint32_t)(j & 1);
    keys[p] = spread3(x) | (spread3(y) << 1) | (spread3(z) << 2);
}

// over the sorted keys: out[1] += distinct keys; low[k] = the low 32 bits of a distinct corner key, else bit 32 set
__global__ void k_try_match(int P, int L, int size, const int32_t *__restrict__ child, const uint64_t *__restrict__ keys, uint64_t *low,
                            int64_t *out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    int first = 0;
    if (k < P) {
        const uint64_t key = keys[k];
        uint64_t v = uint64_t(1) << 32;
        first = k == 0 || keys[k - 1] != key;
        if (first && (key >> (3 * L)) == 0 &&
            find_node(child, L, size, (int)squeeze3(key), (int)squeeze3(key >> 1), (int)squeeze3(key >> 2)) >= 0)
            v = key & 0xffffffffull;
        low[k] = v;
    }
    const int c = __syncthreads_count(first);
    if (threadIdx.x == 0 && c) atomicAdd((unsigned long long *)&out[1], (unsigned long long)c);
}

// over the sorted low words: out[0] += distinct low words of corner keys (octree.cpp:141-147 de-duplicates after truncation)
__global__ void k_try_distinct(int P, const uint64_t *__restrict__ low, int64_t *out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    int first = 0;
    if (k < P) {
        const uint64_t v = low[k];
        first = (v >> 32) == 0 && (k == 0 || low[k - 1] != v);
    }
    const int c = __syncthreads_count(first);
    if (threadIdx.x == 0 && c) atomicAdd((unsigned long long *)&out[0], (unsigned long long)c);
}

// ---------------------------------------------------------------------------------------------------------------------------
// Validation of uploaded node arrays (nl_octree_validate in octree_host.cpp, check for check).  Every block ORs its bits into one
// word, so the verdict is independent of the order in which blocks and atomics land.
__device__ __forceinline__ void or_bits(int bits, unsigned long long *word) {
    bits = __reduce_or_sync(0xffffffffu, bits);
    __shared__ int block_bits;
    if (threadIdx.x == 0) block_bits = 0;
    __syncthreads();
    if ((threadIdx.x & 31) == 0 && bits) atomicOr(&block_bits, bits);
    __syncthreads();
    if (threadIdx.x == 0 && block_bits) atomicOr(word, (unsigned long long)block_bits);
}

// one thread per (node i, slot s): the child id's range before anything is read at it, the link to the child, its parent count;
// slot 0 also checks the node's own fields
__global__ void k_val_tree(int64_t N, int L, const int32_t *__restrict__ child, const uint64_t *__restrict__ code, const int8_t *__restrict__ type,
                           const uint8_t *__restrict__ level, int32_t *parents, int64_t *out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = t < 8 * N;
    const int64_t i = t >> 3;
    const int s = (int)(t & 7);
    int bits = 0;
    bool has = false;
    if (live) {
        const int64_t c = child[t];
        has = c != -1;
        if (has) {
            if (c <= i || c >= N) {
                bits |= NL_TREE_RANGE;
            } else {
                atomicAdd(&parents[c], 1);
                const int lc = level[c], lv = level[i];
                if (lc != lv + 1 || lc > L) bits |= NL_TREE_LINK;
                else if (code[c] != (code[i] | (uint64_t)s << (3 * (L - lc)))) bits |= NL_TREE_LINK;
            }
        }
    }
    const unsigned any = __ballot_sync(0xffffffffu, has);            // blockDim % 32 == 0: a node's 8 slots share a warp
    if (live && s == 0) {
        const int ty = type[i], lv = level[i];
        if (i == 0 && (lv != 0 || code[0] != 0 || ty != kNonLeaf)) bits |= NL_TREE_ROOT;
        if (ty < kNonLeaf || ty > kFeature || lv > L) {
            bits |= NL_TREE_RANGE;
        } else {
            const bool has_child = (any >> (threadIdx.x & 24)) & 0xffu;
            if (code[i] & ((uint64_t(1) << (3 * (L - lv))) - 1)) bits |= NL_TREE_LINK;
            if ((ty == kNonLeaf) != (lv < L) || (ty == kNonLeaf && !has_child)) bits |= NL_TREE_SHAPE;
        }
    }
    if (t == 0 && N < 1) bits |= NL_TREE_ROOT;
    or_bits(bits, (unsigned long long *)&out[0]);
}

__global__ void k_val_parents(int64_t N, const int32_t *__restrict__ parents, int64_t *out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    or_bits(i >= 1 && i < N && parents[i] != 1 ? NL_TREE_PARENTS : 0, (unsigned long long *)&out[0]);
}

// rows and vertices, on a tree the structural pass found well-formed: a SURFACE node is then a level-L leaf with in-grid
// coordinates, and find_node's walk is bounded by L levels of range-checked ids
__global__ void k_val_rows(int64_t N, int L, int size, const int32_t *__restrict__ child, const uint64_t *__restrict__ code,
                           const int8_t *__restrict__ type, const uint8_t *__restrict__ level, const int32_t *__restrict__ v2r, int64_t n_rows,
                           int32_t *uses, int32_t *referenced, int64_t *out) {
    if (*(volatile int64_t *)&out[0] != 0) return;                // the structural verdict: never walk a malformed tree
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int bits = 0;
    if (i < N) {
        const int32_t r = v2r[i];
        if (r < -1 || r >= n_rows) {
            bits |= NL_TREE_ROWS;
        } else if (r >= 0) {
            if (level[i] != L) bits |= NL_TREE_ROWS;
            if (r < N) atomicAdd(&uses[r], 1);
        }
        if (type[i] == kSurface) {
            const uint64_t c = code[i];
            const int x = (int)squeeze3(c), y = (int)squeeze3(c >> 1), z = (int)squeeze3(c >> 2);
            for (int k = 0; k < 8; ++k) {
                const int cx = x + (k >> 2), cy = y + ((k >> 1) & 1), cz = z + (k & 1);
                const int v = (cx < size && cy < size && cz < size) ? find_node(child, L, size, cx, cy, cz) : -1;
                if (v < 0) bits |= NL_TREE_VERTICES;
                else referenced[v] = 1;                                 // idempotent store
            }
        }
    }
    if (i == 0 && n_rows > N) bits |= NL_TREE_ROWS;                  // a row per node at most
    or_bits(bits, (unsigned long long *)&out[1]);
}

__global__ void k_val_rows_sweep(int64_t N, const int32_t *__restrict__ v2r, int64_t n_rows, const int32_t *__restrict__ uses,
                                 const int32_t *__restrict__ referenced, int64_t *out) {
    if (*(volatile int64_t *)&out[0] != 0) return;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int bits = 0;
    if (i < N) {
        if (i < n_rows && uses[i] != 1) bits |= NL_TREE_ROWS;
        if ((v2r[i] >= 0) != (referenced[i] != 0)) bits |= NL_TREE_VERTICES;
    }
    or_bits(bits, (unsigned long long *)&out[1]);
}

// Query workspace: the preorder of N nodes and try_insert of n points (P = 8n corner keys) each use it from offset 0; the CUB
// scratch follows the larger of the two.  The arrays are pure arithmetic, so a short workspace is rejected before any CUDA call.
struct QueryLayout {
    int64_t N = 0, P = 0;
    size_t pk_a = 0, pk_b = 0, pv_a = 0, pv_b = 0, pflag = 0, psel = 0;   // preorder
    size_t tk_a = 0, tk_b = 0;                                           // try_insert
    size_t tmp = 0, tmp_bytes = 0, total = 0;
};

void query_arrays(int64_t N, int64_t n, QueryLayout &l) {
    l.N = N;
    l.P = 8 * n;
    size_t at = 0;
    l.pk_a = take(at, 8 * (size_t)N); l.pk_b = take(at, 8 * (size_t)N);
    l.pv_a = take(at, 4 * (size_t)N); l.pv_b = take(at, 4 * (size_t)N);
    l.pflag = take(at, (size_t)N); l.psel = take(at, 4 * (size_t)N);
    const size_t pre_end = at;
    at = 0;
    l.tk_a = take(at, 8 * (size_t)l.P); l.tk_b = take(at, 8 * (size_t)l.P);
    l.tmp = (std::max(pre_end, at) + 255) & ~size_t(255);
    l.total = l.tmp;
}

cudaError_t query_scratch(int L, QueryLayout &l) {
    size_t a = 0, b = 0, c = 0, d = 0;
    cudaError_t err;
    cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
    if (l.N > 0) {
        cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
        if ((err = cub::DeviceRadixSort::SortPairs(nullptr, a, k, v, (int)l.N, 0, 3 * L)) != cudaSuccess) return err;
        if ((err = cub::DeviceSelect::Flagged(nullptr, b, (const uint32_t *)nullptr, (const uint8_t *)nullptr, (uint32_t *)nullptr,
                                              (int64_t *)nullptr, (int)l.N)) != cudaSuccess)
            return err;
    }
    if (l.P > 0) {
        if ((err = cub::DeviceRadixSort::SortKeys(nullptr, c, k, (int)l.P, 0, 63)) != cudaSuccess) return err;
        if ((err = cub::DeviceRadixSort::SortKeys(nullptr, d, k, (int)l.P, 0, 33)) != cudaSuccess) return err;
    }
    l.tmp_bytes = std::max(std::max(a, b), std::max(c, d));
    l.total = l.tmp + l.tmp_bytes;
    return cudaSuccess;
}

int short_qws(const char *what, int64_t ws_bytes, size_t need) {
    char buf[192];
    std::snprintf(buf, sizeof(buf), "%s: workspace of %lld bytes, nl_devoctree_query_workspace_bytes asks for %lld", what, (long long)ws_bytes,
                  (long long)need);
    return nl_set_error(buf);
}

int check_qws(int64_t N, int64_t n, int L, const void *ws, int64_t ws_bytes, QueryLayout &l, const char *what) {
    query_arrays(N, n, l);
    if (ws_bytes < (int64_t)l.total) return short_qws(what, ws_bytes, l.total);            // the arrays alone do not fit
    if (((uintptr_t)ws & 255u) != 0) return nl_set_error("nl_devoctree: the workspace must be 256-byte aligned");
    const cudaError_t e = query_scratch(L, l);
    if (e != cudaSuccess) return cuda_fail(what, e);
    if (ws_bytes < (int64_t)l.total) return short_qws(what, ws_bytes, l.total);
    return NL_OK;
}

int check_ws(int64_t n, int L, const void *ws, int64_t ws_bytes, Layout &l, const char *what) {
    const cudaError_t e = make_layout(n, L, l);
    if (e != cudaSuccess) return cuda_fail(what, e);
    if (ws_bytes < (int64_t)l.total) {
        char buf[160];
        std::snprintf(buf, sizeof(buf), "%s: workspace of %lld bytes, nl_devoctree_workspace_bytes asks for %lld", what, (long long)ws_bytes,
                      (long long)l.total);
        return nl_set_error(buf);
    }
    if (((uintptr_t)ws & 255u) != 0) return nl_set_error("nl_devoctree: the workspace must be 256-byte aligned");
    return NL_OK;
}

}  // namespace

extern "C" {

int64_t nl_devoctree_workspace_bytes(int64_t n_points, int64_t grid_dim) {
    const int L = levels_of(grid_dim);
    if (n_points < 0 || n_points > kMaxPoints || L < 0) return nl_set_error("nl_devoctree_workspace_bytes: bad n_points or grid_dim");
    Layout l;
    const cudaError_t e = make_layout(n_points, L, l);
    if (e != cudaSuccess) return cuda_fail("nl_devoctree_workspace_bytes", e);
    return (int64_t)l.total;
}

int nl_devoctree_insert_count(int64_t grid_dim, const int32_t *d_child, const int32_t *d_vox, int64_t n, void *d_ws, int64_t ws_bytes,
                              int64_t *d_counts, void *stream) {
    const int L = levels_of(grid_dim);
    if (L < 0) return nl_set_error("nl_devoctree_insert_count: grid_dim must be a power of two in [2, 2^20]");
    if (n < 0 || n > kMaxPoints) return nl_set_error("nl_devoctree_insert_count: n must be in [0, 2^23]");
    if (!d_child || !d_counts || (n > 0 && (!d_vox || !d_ws))) return nl_set_error("nl_devoctree_insert_count: null pointer");
    Layout l;
    if (n > 0)
        if (int rc = check_ws(n, L, d_ws, ws_bytes, l, "nl_devoctree_insert_count")) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(d_counts, 0, 2 * sizeof(int64_t), s);
    if (e != cudaSuccess) return cuda_fail("nl_devoctree_insert_count", e);
    if (n == 0) return NL_OK;
    const int P = (int)l.P;
    uint64_t *ka = at<uint64_t>(d_ws, l.keys_a), *kb = at<uint64_t>(d_ws, l.keys_b);
    uint32_t *va = at<uint32_t>(d_ws, l.vals_a), *vb = at<uint32_t>(d_ws, l.vals_b);
    k_corners<<<nl_div_up(P, kThreads), kThreads, 0, s>>>((int)n, L, (int)grid_dim, d_vox, d_child, ka, va, at<uint8_t>(d_ws, l.dm),
                                                         at<int32_t>(d_ws, l.enode), at<int32_t>(d_ws, l.eparent), d_counts);
    NL_CHECK_LAUNCH("nl_devoctree_insert_count");
    cub::DoubleBuffer<uint64_t> dk(ka, kb);
    cub::DoubleBuffer<uint32_t> dv(va, vb);
    size_t tb = l.tmp_ins_bytes;
    if ((e = cub::DeviceRadixSort::SortPairs(at<void>(d_ws, l.tmp_ins), tb, dk, dv, P, 0, 3 * L + 1, s)) != cudaSuccess)
        return cuda_fail("nl_devoctree_insert_count: sort", e);
    if (dk.Current() != ka) {                        // keep the sorted corners at a fixed place for the commit
        cudaMemcpyAsync(ka, dk.Current(), 8 * (size_t)P, cudaMemcpyDeviceToDevice, s);
        cudaMemcpyAsync(va, dv.Current(), 4 * (size_t)P, cudaMemcpyDeviceToDevice, s);
    }
    int32_t *cnt = at<int32_t>(d_ws, l.cnt), *off = at<int32_t>(d_ws, l.off);
    k_count<<<nl_div_up(P + 1, kThreads), kThreads, 0, s>>>(P, L, ka, va, at<uint8_t>(d_ws, l.dm), at<uint8_t>(d_ws, l.lo), cnt);
    NL_CHECK_LAUNCH("nl_devoctree_insert_count");
    tb = l.tmp_ins_bytes;
    if ((e = cub::DeviceScan::ExclusiveSum(at<void>(d_ws, l.tmp_ins), tb, cnt, off, P + 1, s)) != cudaSuccess)
        return cuda_fail("nl_devoctree_insert_count: scan", e);
    k_store_new<<<1, 1, 0, s>>>(P, off, d_counts);
    NL_CHECK_LAUNCH("nl_devoctree_insert_count");
    return NL_OK;
}

int nl_devoctree_insert_commit(int64_t grid_dim, int64_t n_nodes, int64_t n_new, int64_t base, int32_t *d_child, uint64_t *d_code, int8_t *d_type,
                               uint8_t *d_level, int32_t *d_scratch, uint32_t *d_dirty_list, int64_t n, void *d_ws, int64_t ws_bytes,
                               int64_t *d_counts, void *stream) {
    const int L = levels_of(grid_dim);
    if (L < 0) return nl_set_error("nl_devoctree_insert_commit: grid_dim must be a power of two in [2, 2^20]");
    if (n < 0 || n > kMaxPoints || n_nodes < 1 || n_new < 0 || base < 0 || base > n_nodes || n_nodes + n_new > INT32_MAX)
        return nl_set_error("nl_devoctree_insert_commit: bad sizes");
    if (n == 0) return n_new == 0 ? NL_OK : nl_set_error("nl_devoctree_insert_commit: new nodes without points");
    if (!d_child || !d_code || !d_type || !d_level || !d_scratch || !d_dirty_list || !d_ws || !d_counts)
        return nl_set_error("nl_devoctree_insert_commit: null pointer");
    Layout l;
    if (int rc = check_ws(n, L, d_ws, ws_bytes, l, "nl_devoctree_insert_commit")) return rc;
    if (n_new > l.T) return nl_set_error("nl_devoctree_insert_commit: more new nodes than the batch can create");
    cudaStream_t s = (cudaStream_t)stream;
    const int P = (int)l.P, T = (int)n_new;
    const uint64_t *keys = at<uint64_t>(d_ws, l.keys_a);
    const uint32_t *vals = at<uint32_t>(d_ws, l.vals_a);
    const uint8_t *dm = at<uint8_t>(d_ws, l.dm), *lo = at<uint8_t>(d_ws, l.lo);
    const int32_t *off = at<int32_t>(d_ws, l.off), *enode = at<int32_t>(d_ws, l.enode), *eparent = at<int32_t>(d_ws, l.eparent);
    int32_t *spos = at<int32_t>(d_ws, l.spos), *par = at<int32_t>(d_ws, l.par), *sid = at<int32_t>(d_ws, l.sid);
    uint32_t *pmin = at<uint32_t>(d_ws, l.pmin);
    uint8_t *surf = at<uint8_t>(d_ws, l.surf);
    if (T > 0) {
        k_slots<<<nl_div_up(P, kThreads), kThreads, 0, s>>>(P, L, keys, vals, dm, lo, off, enode, spos, par, pmin, surf);
        k_pmin<<<nl_div_up(P, kThreads), kThreads, 0, s>>>(P, L, keys, vals, lo, off, par, pmin, surf);
        uint32_t *k2a = at<uint32_t>(d_ws, l.k2a), *k2b = at<uint32_t>(d_ws, l.k2b), *v2a = at<uint32_t>(d_ws, l.v2a), *v2b = at<uint32_t>(d_ws, l.v2b);
        k_seq<<<nl_div_up(T, kThreads), kThreads, 0, s>>>(T, L, spos, off, lo, pmin, k2a, v2a);
        NL_CHECK_LAUNCH("nl_devoctree_insert_commit");
        cub::DoubleBuffer<uint32_t> dk(k2a, k2b), dv(v2a, v2b);
        size_t tb = l.tmp_ins_bytes;
        const cudaError_t e = cub::DeviceRadixSort::SortPairs(at<void>(d_ws, l.tmp_ins), tb, dk, dv, T, 0, l.rank_bits, s);
        if (e != cudaSuccess) return cuda_fail("nl_devoctree_insert_commit: sort", e);
        k_build<<<nl_div_up(T, kThreads), kThreads, 0, s>>>(T, L, n_nodes, dv.Current(), spos, off, lo, keys, surf, sid, d_child, d_code, d_type, d_level);
        k_link<<<nl_div_up(T, kThreads), kThreads, 0, s>>>(T, L, base, spos, off, lo, keys, par, sid, d_child, d_scratch, d_dirty_list, d_counts);
    }
    k_promote<<<nl_div_up(P, kThreads), kThreads, 0, s>>>(P, L, base, dm, enode, eparent, d_type, d_scratch, d_dirty_list, d_counts);
    NL_CHECK_LAUNCH("nl_devoctree_insert_commit");
    return NL_OK;
}

int nl_devoctree_dirty_ids(int64_t grid_dim, int64_t n_nodes, int64_t base, int64_t n_list, uint32_t *d_dirty_list, int32_t *d_scratch, int32_t *d_ids,
                           int64_t n_points, void *d_ws, int64_t ws_bytes, int64_t *d_counts, void *stream) {
    const int L = levels_of(grid_dim);
    if (L < 0) return nl_set_error("nl_devoctree_dirty_ids: grid_dim must be a power of two in [2, 2^20]");
    if (n_nodes < 1 || base < 0 || base > n_nodes || n_list < 0 || n_points < 0 || n_points > kMaxPoints)
        return nl_set_error("nl_devoctree_dirty_ids: bad sizes");
    if (!d_scratch || !d_ids || !d_counts || (n_list > 0 && (!d_dirty_list || !d_ws))) return nl_set_error("nl_devoctree_dirty_ids: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t *sorted = d_dirty_list;
    if (n_list > 0) {
        Layout l;
        if (int rc = check_ws(n_points, L, d_ws, ws_bytes, l, "nl_devoctree_dirty_ids")) return rc;
        if (n_list > l.D) return nl_set_error("nl_devoctree_dirty_ids: pending list longer than n_points can fill");
        cub::DoubleBuffer<uint32_t> dk(d_dirty_list, at<uint32_t>(d_ws, l.dsorted));
        size_t tb = l.tmp_exp_bytes;
        const cudaError_t e = cub::DeviceRadixSort::SortKeys(at<void>(d_ws, l.tmp_exp), tb, dk, (int)n_list, 0, 32, s);
        if (e != cudaSuccess) return cuda_fail("nl_devoctree_dirty_ids: sort", e);
        sorted = dk.Current();
    }
    const int64_t rows = n_list + (n_nodes - base);
    k_dirty_tail<<<nl_div_up(std::max<int64_t>(rows, 1), kThreads), kThreads, 0, s>>>((int)n_list, n_nodes - base, base, sorted, d_dirty_list,
                                                                                     d_scratch, d_ids, d_counts);
    k_reset_pending<<<1, 1, 0, s>>>(d_counts);
    NL_CHECK_LAUNCH("nl_devoctree_dirty_ids");
    return NL_OK;
}

int nl_devoctree_export(int64_t grid_dim, double voxel_size, int64_t n_rows, const int32_t *d_ids, const int64_t *d_count, int compact,
                        const int32_t *d_child, const uint64_t *d_code, const int8_t *d_type, const uint8_t *d_level, float *d_centres,
                        int32_t *d_structure, int32_t *d_vertex, void *stream) {
    const int L = levels_of(grid_dim);
    if (L < 0) return nl_set_error("nl_devoctree_export: grid_dim must be a power of two in [2, 2^20]");
    if (n_rows < 0) return nl_set_error("nl_devoctree_export: negative n_rows");
    if (n_rows == 0) return NL_OK;
    if (!d_child || !d_code || !d_type || !d_level || !d_centres || !d_structure || !d_vertex) return nl_set_error("nl_devoctree_export: null pointer");
    k_export<<<nl_div_up(n_rows, kThreads), kThreads, 0, (cudaStream_t)stream>>>(n_rows, d_ids, d_count, compact, L, (int)grid_dim, (float)voxel_size,
                                                                                d_child, d_code, d_type, d_level, nullptr, nullptr, d_centres,
                                                                                d_structure, d_vertex);
    NL_CHECK_LAUNCH("nl_devoctree_export");
    return NL_OK;
}

int nl_devoctree_export_nodes(int64_t grid_dim, double voxel_size, int64_t n_rows, const int32_t *d_ids, const int64_t *d_count, int compact,
                              const int32_t *d_child, const uint64_t *d_code, const int8_t *d_type, const uint8_t *d_level, float *d_voxels4,
                              float *d_children_f, float *d_centres, int32_t *d_structure, int32_t *d_vertex, void *stream) {
    const int L = levels_of(grid_dim);
    if (L < 0) return nl_set_error("nl_devoctree_export_nodes: grid_dim must be a power of two in [2, 2^20]");
    if (n_rows < 0) return nl_set_error("nl_devoctree_export_nodes: negative n_rows");
    if (n_rows == 0) return NL_OK;
    if (!d_child || !d_code || !d_type || !d_level || !d_vertex) return nl_set_error("nl_devoctree_export_nodes: null pointer");
    k_export<<<nl_div_up(n_rows, kThreads), kThreads, 0, (cudaStream_t)stream>>>(n_rows, d_ids, d_count, compact, L, (int)grid_dim, (float)voxel_size,
                                                                                d_child, d_code, d_type, d_level, d_voxels4, d_children_f,
                                                                                d_centres, d_structure, d_vertex);
    NL_CHECK_LAUNCH("nl_devoctree_export_nodes");
    return NL_OK;
}

int64_t nl_devoctree_query_workspace_bytes(int64_t n_nodes, int64_t n_points, int64_t grid_dim) {
    const int L = levels_of(grid_dim);
    if (L < 0 || n_nodes < 0 || n_nodes > INT32_MAX || n_points < 0 || n_points > kMaxPoints)
        return nl_set_error("nl_devoctree_query_workspace_bytes: bad n_nodes, n_points or grid_dim");
    QueryLayout l;
    query_arrays(n_nodes, n_points, l);
    const cudaError_t e = query_scratch(L, l);
    if (e != cudaSuccess) return cuda_fail("nl_devoctree_query_workspace_bytes", e);
    return (int64_t)l.total;
}

int nl_devoctree_preorder(int64_t grid_dim, int64_t n_nodes, const uint64_t *d_code, const int8_t *d_type, const uint8_t *d_level, int leaves_only,
                          float *d_out, int64_t *d_count, void *d_ws, int64_t ws_bytes, void *stream) {
    const int L = levels_of(grid_dim);
    if (L < 0) return nl_set_error("nl_devoctree_preorder: grid_dim must be a power of two in [2, 2^20]");
    if (n_nodes < 1 || n_nodes > INT32_MAX || (leaves_only != 0 && leaves_only != 1)) return nl_set_error("nl_devoctree_preorder: bad sizes");
    if (!d_code || !d_type || !d_level || !d_out || !d_ws || (leaves_only && !d_count)) return nl_set_error("nl_devoctree_preorder: null pointer");
    QueryLayout l;
    if (int rc = check_qws(n_nodes, 0, L, d_ws, ws_bytes, l, "nl_devoctree_preorder")) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const int N = (int)n_nodes;
    uint64_t *ka = at<uint64_t>(d_ws, l.pk_a), *kb = at<uint64_t>(d_ws, l.pk_b);
    uint32_t *va = at<uint32_t>(d_ws, l.pv_a), *vb = at<uint32_t>(d_ws, l.pv_b);
    k_pre_init<<<nl_div_up(N, kThreads), kThreads, 0, s>>>(N, d_code, ka, va);
    NL_CHECK_LAUNCH("nl_devoctree_preorder");
    cub::DoubleBuffer<uint64_t> dk(ka, kb);
    cub::DoubleBuffer<uint32_t> dv(va, vb);
    size_t tb = l.tmp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(at<void>(d_ws, l.tmp), tb, dk, dv, N, 0, 3 * L, s);   // stable: equal codes keep id order
    if (e != cudaSuccess) return cuda_fail("nl_devoctree_preorder: sort", e);
    const uint32_t *order = dv.Current();
    if (!leaves_only) {
        k_pre_rows<<<nl_div_up(N, kThreads), kThreads, 0, s>>>(N, (int)grid_dim, order, d_code, d_level, d_out);
        NL_CHECK_LAUNCH("nl_devoctree_preorder");
        return NL_OK;
    }
    uint8_t *flag = at<uint8_t>(d_ws, l.pflag);
    uint32_t *sel = at<uint32_t>(d_ws, l.psel);
    k_pre_flag<<<nl_div_up(N, kThreads), kThreads, 0, s>>>(N, order, d_type, flag);
    NL_CHECK_LAUNCH("nl_devoctree_preorder");
    tb = l.tmp_bytes;
    if ((e = cub::DeviceSelect::Flagged(at<void>(d_ws, l.tmp), tb, order, flag, sel, d_count, N, s)) != cudaSuccess)   // keeps the order
        return cuda_fail("nl_devoctree_preorder: select", e);
    k_leaf_rows<<<nl_div_up(N, kThreads), kThreads, 0, s>>>(N, sel, d_count, d_code, d_out);
    NL_CHECK_LAUNCH("nl_devoctree_preorder");
    return NL_OK;
}

int nl_devoctree_try_insert(int64_t grid_dim, const int32_t *d_child, const int32_t *d_vox, int64_t n, void *d_ws, int64_t ws_bytes,
                            int64_t *d_out, void *stream) {
    const int L = levels_of(grid_dim);
    if (L < 0) return nl_set_error("nl_devoctree_try_insert: grid_dim must be a power of two in [2, 2^20]");
    if (n < 1 || n > kMaxPoints) return nl_set_error("nl_devoctree_try_insert: n must be in [1, 2^23]");
    if (!d_child || !d_vox || !d_ws || !d_out) return nl_set_error("nl_devoctree_try_insert: null pointer");
    QueryLayout l;
    if (int rc = check_qws(0, n, L, d_ws, ws_bytes, l, "nl_devoctree_try_insert")) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const int P = (int)(8 * n);
    cudaError_t e = cudaMemsetAsync(d_out, 0, 2 * sizeof(int64_t), s);
    if (e != cudaSuccess) return cuda_fail("nl_devoctree_try_insert", e);
    uint64_t *ka = at<uint64_t>(d_ws, l.tk_a), *kb = at<uint64_t>(d_ws, l.tk_b);
    k_try_keys<<<nl_div_up(P, kThreads), kThreads, 0, s>>>(P, d_vox, ka);
    NL_CHECK_LAUNCH("nl_devoctree_try_insert");
    cub::DoubleBuffer<uint64_t> dk(ka, kb);
    size_t tb = l.tmp_bytes;
    if ((e = cub::DeviceRadixSort::SortKeys(at<void>(d_ws, l.tmp), tb, dk, P, 0, 63, s)) != cudaSuccess)
        return cuda_fail("nl_devoctree_try_insert: sort", e);
    k_try_match<<<nl_div_up(P, kThreads), kThreads, 0, s>>>(P, L, (int)grid_dim, d_child, dk.Current(), dk.Alternate(), d_out);
    NL_CHECK_LAUNCH("nl_devoctree_try_insert");
    dk.selector ^= 1;                                // sort the matched keys' low words (bit 32 set = no match)
    tb = l.tmp_bytes;
    if ((e = cub::DeviceRadixSort::SortKeys(at<void>(d_ws, l.tmp), tb, dk, P, 0, 33, s)) != cudaSuccess)
        return cuda_fail("nl_devoctree_try_insert: sort", e);
    k_try_distinct<<<nl_div_up(P, kThreads), kThreads, 0, s>>>(P, dk.Current(), d_out);
    NL_CHECK_LAUNCH("nl_devoctree_try_insert");
    return NL_OK;
}

int nl_devoctree_validate(int64_t grid_dim, int64_t n_nodes, const int32_t *d_child, const uint64_t *d_code, const int8_t *d_type,
                          const uint8_t *d_level, const int32_t *d_vertex2row, int64_t n_rows, void *d_ws, int64_t ws_bytes, int64_t *d_out,
                          void *stream) {
    const int L = levels_of(grid_dim);
    if (L < 0) return nl_set_error("nl_devoctree_validate: grid_dim must be a power of two in [2, 2^20]");
    if (n_nodes < 0 || n_nodes > INT32_MAX || n_rows < 0) return nl_set_error("nl_devoctree_validate: bad sizes");
    if (!d_out || (n_nodes > 0 && (!d_child || !d_code || !d_type || !d_level || !d_ws))) return nl_set_error("nl_devoctree_validate: null pointer");
    size_t need = 0;
    const size_t parents = take(need, 4 * (size_t)n_nodes), uses = take(need, 4 * (size_t)n_nodes), referenced = take(need, 4 * (size_t)n_nodes);
    if (n_nodes > 0 && ws_bytes < (int64_t)need) {
        char buf[160];
        std::snprintf(buf, sizeof(buf), "nl_devoctree_validate: workspace of %lld bytes, needs %lld", (long long)ws_bytes, (long long)need);
        return nl_set_error(buf);
    }
    if (((uintptr_t)d_ws & 255u) != 0) return nl_set_error("nl_devoctree: the workspace must be 256-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(d_out, 0, 2 * sizeof(int64_t), s);
    if (e == cudaSuccess && n_nodes > 0) e = cudaMemsetAsync(d_ws, 0, need, s);
    if (e != cudaSuccess) return cuda_fail("nl_devoctree_validate", e);
    const int64_t nb = nl_div_up(std::max<int64_t>(8 * n_nodes, 1), kThreads);
    k_val_tree<<<nb, kThreads, 0, s>>>(n_nodes, L, d_child, d_code, d_type, d_level, at<int32_t>(d_ws, parents), d_out);
    if (n_nodes > 0) {
        const int64_t blocks = nl_div_up(n_nodes, kThreads);
        k_val_parents<<<blocks, kThreads, 0, s>>>(n_nodes, at<int32_t>(d_ws, parents), d_out);
        if (d_vertex2row) {
            k_val_rows<<<blocks, kThreads, 0, s>>>(n_nodes, L, (int)grid_dim, d_child, d_code, d_type, d_level, d_vertex2row, n_rows,
                                                   at<int32_t>(d_ws, uses), at<int32_t>(d_ws, referenced), d_out);
            k_val_rows_sweep<<<blocks, kThreads, 0, s>>>(n_nodes, d_vertex2row, n_rows, at<int32_t>(d_ws, uses), at<int32_t>(d_ws, referenced), d_out);
        }
    }
    NL_CHECK_LAUNCH("nl_devoctree_validate");
    return NL_OK;
}

int nl_devoctree_assign_rows(int64_t grid_dim, int64_t n_rows, const int32_t *d_ids, int64_t n_nodes, const int8_t *d_type, const int32_t *d_vertex,
                             int32_t *d_vertex2row, int32_t *d_scratch, int64_t n_emb_rows, int32_t *d_vox2row, int64_t n_points, void *d_ws,
                             int64_t ws_bytes, int64_t *d_counts, void *stream) {
    const int L = levels_of(grid_dim);
    if (L < 0) return nl_set_error("nl_devoctree_assign_rows: grid_dim must be a power of two in [2, 2^20]");
    if (n_rows < 0 || n_nodes < 1 || n_emb_rows < 0 || n_points < 0 || n_points > kMaxPoints) return nl_set_error("nl_devoctree_assign_rows: bad sizes");
    if (!d_counts || (n_rows > 0 && (!d_ids || !d_type || !d_vertex || !d_vertex2row || !d_scratch || !d_vox2row || !d_ws)))
        return nl_set_error("nl_devoctree_assign_rows: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    if (n_rows == 0 || n_points == 0) {              // no point inserted since the last export: no SURFACE row, no new vertex
        k_rows_total<<<1, 1, 0, s>>>(0, nullptr, nullptr, n_emb_rows, d_counts);
        if (n_rows > 0)
            k_vox2row<<<nl_div_up(n_rows * 8, kThreads), kThreads, 0, s>>>(n_rows, d_ids, d_counts, d_vertex, n_nodes, d_vertex2row, d_vox2row);
        NL_CHECK_LAUNCH("nl_devoctree_assign_rows");
        return NL_OK;
    }
    Layout l;
    if (int rc = check_ws(n_points, L, d_ws, ws_bytes, l, "nl_devoctree_assign_rows")) return rc;
    if (n_rows > l.M) return nl_set_error("nl_devoctree_assign_rows: more dirty rows than n_points can produce");
    uint8_t *sflag = at<uint8_t>(d_ws, l.sflag);
    int32_t *sids = at<int32_t>(d_ws, l.sids), *ns = at<int32_t>(d_ws, l.ns), *rflag = at<int32_t>(d_ws, l.rflag), *rscan = at<int32_t>(d_ws, l.rscan);
    const int E = (int)l.E;
    k_sflag<<<nl_div_up(n_rows, kThreads), kThreads, 0, s>>>(n_rows, d_ids, d_counts, d_type, sflag);
    NL_CHECK_LAUNCH("nl_devoctree_assign_rows");
    size_t tb = l.tmp_exp_bytes;
    cudaError_t e = cub::DeviceSelect::Flagged(at<void>(d_ws, l.tmp_exp), tb, d_ids, sflag, sids, ns, (int)n_rows, s);  // SURFACE rows, in order
    if (e != cudaSuccess) return cuda_fail("nl_devoctree_assign_rows: select", e);
    k_first<<<nl_div_up(E, kThreads), kThreads, 0, s>>>(E, sids, ns, d_vertex, n_nodes, d_vertex2row, d_scratch);
    k_rflag<<<nl_div_up(E, kThreads), kThreads, 0, s>>>(E, sids, ns, d_vertex, n_nodes, d_vertex2row, d_scratch, rflag);
    NL_CHECK_LAUNCH("nl_devoctree_assign_rows");
    tb = l.tmp_exp_bytes;
    if ((e = cub::DeviceScan::ExclusiveSum(at<void>(d_ws, l.tmp_exp), tb, rflag, rscan, E, s)) != cudaSuccess)
        return cuda_fail("nl_devoctree_assign_rows: scan", e);
    k_assign<<<nl_div_up(E, kThreads), kThreads, 0, s>>>(E, sids, ns, d_vertex, rflag, rscan, n_emb_rows, d_vertex2row, d_scratch);
    k_rows_total<<<1, 1, 0, s>>>(E, rflag, rscan, n_emb_rows, d_counts);
    k_vox2row<<<nl_div_up(n_rows * 8, kThreads), kThreads, 0, s>>>(n_rows, d_ids, d_counts, d_vertex, n_nodes, d_vertex2row, d_vox2row);
    NL_CHECK_LAUNCH("nl_devoctree_assign_rows");
    return NL_OK;
}

int nl_devoctree_find(int64_t grid_dim, const int32_t *d_child, const int32_t *d_xyz, int64_t n, int32_t *d_out, void *stream) {
    const int L = levels_of(grid_dim);
    if (L < 0) return nl_set_error("nl_devoctree_find: grid_dim must be a power of two in [2, 2^20]");
    if (n < 0) return nl_set_error("nl_devoctree_find: negative n");
    if (n == 0) return NL_OK;
    if (!d_child || !d_xyz || !d_out) return nl_set_error("nl_devoctree_find: null pointer");
    k_find<<<nl_div_up(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(n, L, (int)grid_dim, d_child, d_xyz, d_out);
    NL_CHECK_LAUNCH("nl_devoctree_find");
    return NL_OK;
}

}  // extern "C"
