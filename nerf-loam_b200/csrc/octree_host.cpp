// Host-side sparse voxel octree of the map-update step (SURVEY.md section 8 a-1 / a-14).
//
// Replaces the reference's pointer-based `svo` TorchScript class (third_party/sparse_octree) with a
// flat structure-of-arrays tree: a node is an index into parallel vectors, children are int32 ids,
// there is no per-node allocation and the export is a direct array pass (the reference walks a BFS
// queue and issues a torch dispatcher call per node, octree.cpp:293-342).
//
// Node ids are handed out in creation order exactly like Octant::index_ (octree.h:19, octree.cpp:68-109:
// point order x corner order incr_{x,y,z} x root->leaf), so the exported arrays are bit-identical to
// the reference's get_centres_and_children().  Duplicate points are skipped through a hash set: a
// repeated point can neither create a node nor change a type, so skipping it is exact.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <unordered_set>
#include <vector>

#include "../../include/nerfloam_b200.h"
#include "nl_error.h"

namespace {

enum : int8_t { kNonLeaf = -1, kSurface = 0, kFeature = 1 };  // octree.h:5-10

constexpr int kMaxBits = 21;  // utils.h:5

// Morton helpers: 21 bits per axis interleaved x | y<<1 | z<<2 (utils.h:64-109).
inline uint64_t spread3(uint64_t v) {
    uint64_t x = v & 0x1fffffULL;
    x = (x | x << 32) & 0x1f00000000ffffULL;
    x = (x | x << 16) & 0x1f0000ff0000ffULL;
    x = (x | x << 8) & 0x100f00f00f00f00fULL;
    x = (x | x << 4) & 0x10c30c30c30c30c3ULL;
    x = (x | x << 2) & 0x1249249249249249ULL;
    return x;
}
inline uint64_t squeeze3(uint64_t v) {
    uint64_t x = v & 0x1249249249249249ULL;
    x = (x | x >> 2) & 0x10c30c30c30c30c3ULL;
    x = (x | x >> 4) & 0x100f00f00f00f00fULL;
    x = (x | x >> 8) & 0x1f0000ff0000ffULL;
    x = (x | x >> 16) & 0x1f00000000ffffULL;
    x = (x | x >> 32) & 0x1fffffULL;
    return x;
}
inline uint64_t level_mask(int i) {  // utils.h:41-62 MASK[i]: top 3*(i+1) Morton bits below bit 63
    uint64_t m = 0;
    for (int k = 0; k <= i; ++k) m |= (0x7000000000000000ULL >> (3 * k));
    return m;
}
const uint64_t kAllLevels = level_mask(kMaxBits - 1);
inline uint64_t morton(int x, int y, int z) {
    return (spread3((uint64_t)(int64_t)x) | (spread3((uint64_t)(int64_t)y) << 1) | (spread3((uint64_t)(int64_t)z) << 2)) & kAllLevels;
}

const int kIncX[8] = {0, 0, 0, 0, 1, 1, 1, 1};  // octree.cpp:12-14: corner j = 4*dx + 2*dy + dz
const int kIncY[8] = {0, 0, 1, 1, 0, 0, 1, 1};
const int kIncZ[8] = {0, 1, 0, 1, 0, 1, 0, 1};

// Open-addressing set of 64-bit keys (linear probing, power-of-two capacity, load <= 1/2): membership tests are the inner loop of
// insertion -- every point of every scan asks "seen before?" -- and std::unordered_set's node chasing made that 2/3 of a map update.
struct KeySet {
    std::vector<uint64_t> slot;    // key + 1; 0 = empty (Morton keys never reach 2^64 - 1)
    size_t used = 0;
    KeySet() : slot(1024, 0) {}
    static size_t hash(uint64_t k) { return (size_t)((k * 0x9E3779B97F4A7C15ull) >> 20); }
    bool contains(uint64_t k) const {
        const size_t mask = slot.size() - 1;
        for (size_t i = hash(k) & mask;; i = (i + 1) & mask) {
            if (slot[i] == k + 1) return true;
            if (!slot[i]) return false;
        }
    }
    bool insert(uint64_t k) {      // true if the key was new
        if ((used + 1) * 2 > slot.size()) grow();
        const size_t mask = slot.size() - 1;
        for (size_t i = hash(k) & mask;; i = (i + 1) & mask) {
            if (slot[i] == k + 1) return false;
            if (!slot[i]) { slot[i] = k + 1; ++used; return true; }
        }
    }
    void grow() {
        std::vector<uint64_t> old(slot.size() * 2, 0);
        old.swap(slot);
        used = 0;
        for (uint64_t v : old)
            if (v) insert(v - 1);
    }
};

int32_t find_in(const int32_t *child, int size, int max_level, int x, int y, int z) {  // find_octant, octree.cpp:151-171
    int32_t n = 0;
    unsigned edge = (unsigned)size / 2;
    for (int d = 1; d <= max_level; edge /= 2, ++d) {
        int slot = ((x & edge) > 0) + 2 * ((y & edge) > 0) + 4 * ((z & edge) > 0);
        int32_t c = child[(size_t)n * 8 + slot];
        if (c < 0) return -1;
        n = c;
    }
    return n;
}

}  // namespace

struct nl_octree {
    int size = 0, max_level = 0;
    int64_t feat_dim = 0;
    double voxel_size = 0;
    std::vector<int32_t> child;   // [n][8], slot = (x&edge>0) + 2*(y&edge>0) + 4*(z&edge>0)  (octree.cpp:85)
    std::vector<uint64_t> code;   // Morton code of the min corner, truncated to the node's level
    std::vector<uint32_t> side;
    std::vector<int8_t> type;
    KeySet corner_keys;           // all_keys (octree.h:118) -- used by try_insert only
    KeySet seen_points;
    // Incremental export (nl_octree_export_dirty): ids of the nodes whose exported row may differ from the last export.  A row
    // changes only when the node is created, when one of its child slots is filled, when a FEATURE leaf becomes SURFACE (its
    // own row appears) or when one of its children does (the child id shows up in the parent's row, octree.cpp:333-337).
    std::vector<int32_t> dirty;
    std::vector<uint8_t> dirty_flag;

    void mark(int32_t id) {
        if (!dirty_flag[(size_t)id]) { dirty_flag[(size_t)id] = 1; dirty.push_back(id); }
    }
    int32_t new_node(uint64_t c, uint32_t s, int8_t t) {
        int32_t id = (int32_t)type.size();
        child.insert(child.end(), 8, -1);
        code.push_back(c);
        side.push_back(s);
        type.push_back(t);
        dirty_flag.push_back(0);
        mark(id);
        return id;
    }
    int32_t find(int x, int y, int z) const { return find_in(child.data(), size, max_level, x, y, z); }
};

extern "C" {

uint64_t nl_morton_encode(int x, int y, int z) { return morton(x, y, z); }

nl_octree *nl_octree_create(int64_t grid_dim, int64_t feat_dim, double voxel_size) {
    if (grid_dim < 2 || grid_dim > (1 << 20) || (grid_dim & (grid_dim - 1))) {
        nl_set_error("nl_octree_create: grid_dim must be a power of two in [2, 2^20]");
        return nullptr;
    }
    nl_octree *t = new nl_octree();
    t->size = (int)grid_dim;
    t->feat_dim = feat_dim;
    t->voxel_size = voxel_size;
    t->max_level = (int)std::log2((double)grid_dim);
    t->new_node(0, (uint32_t)grid_dim, kNonLeaf);  // root: id 0, code 0, side = size (octree.cpp:41-43)
    return t;
}

void nl_octree_destroy(nl_octree *t) { delete t; }

int nl_octree_insert(nl_octree *t, const int32_t *vox, int64_t n) {
    if (!t || (!vox && n > 0) || n < 0) return nl_set_error("nl_octree_insert: bad arguments");
    const unsigned shift = (unsigned)(kMaxBits - t->max_level - 1);  // octree.cpp:79
    std::vector<uint64_t> lvl_mask((size_t)t->max_level + 1);
    for (int d = 1; d <= t->max_level; ++d) lvl_mask[d] = level_mask(d + (int)shift);
    for (int64_t i = 0; i < n * 3; ++i) {
        // The reference silently wraps such coordinates through the bit masks; refuse the whole batch, before any point of it
        // changes the tree, instead of corrupting it.
        if (vox[i] < 0 || vox[i] >= t->size - 1)
            return nl_set_error("nl_octree_insert: voxel coordinate outside [0, grid_dim-2]; the batch was rejected and the tree is unchanged");
    }
    for (int64_t i = 0; i < n; ++i) {
        const int px = vox[i * 3 + 0], py = vox[i * 3 + 1], pz = vox[i * 3 + 2];
        if (!t->seen_points.insert(morton(px, py, pz))) continue;
        for (int j = 0; j < 8; ++j) {
            const int x = px + kIncX[j], y = py + kIncY[j], z = pz + kIncZ[j];
            const uint64_t key = morton(x, y, z);
            t->corner_keys.insert(key);
            int32_t node = 0;
            unsigned edge = (unsigned)t->size / 2;
            for (int d = 1; d <= t->max_level; edge /= 2, ++d) {
                const int slot = ((x & edge) > 0) + 2 * ((y & edge) > 0) + 4 * ((z & edge) > 0);
                int32_t c = t->child[(size_t)node * 8 + slot];
                if (c < 0) {
                    const bool leaf = (d == t->max_level);
                    c = t->new_node(key & lvl_mask[d], edge, leaf ? (j == 0 ? kSurface : kFeature) : kNonLeaf);
                    t->child[(size_t)node * 8 + slot] = c;
                    t->mark(node);
                } else if (j == 0 && t->type[c] == kFeature) {
                    t->type[c] = kSurface;  // octree.cpp:102-106
                    t->mark(c);
                    t->mark(node);
                }
                node = c;
            }
        }
    }
    return NL_OK;
}

double nl_octree_try_insert(nl_octree *t, const int32_t *vox, int64_t n) {
    if (!t || !vox || n <= 0) return -1.0;
    std::unordered_set<uint64_t> tmp;
    for (int64_t i = 0; i < n; ++i)
        for (int j = 0; j < 8; ++j) tmp.insert(morton(vox[i * 3] + kIncX[j], vox[i * 3 + 1] + kIncY[j], vox[i * 3 + 2] + kIncZ[j]));
    // octree.cpp:141-147 collects the intersection into a std::set<int>: keys are truncated to 32 bits
    // and de-duplicated after truncation; the ratio is reproduced with that quirk.
    std::unordered_set<int32_t> inter;
    for (uint64_t k : tmp)
        if (t->corner_keys.contains(k)) inter.insert((int32_t)k);
    return 1.0 * (double)inter.size() / (double)tmp.size();
}

int64_t nl_octree_count_nodes(const nl_octree *t) { return t ? (int64_t)t->type.size() : -1; }
int64_t nl_octree_count_export_nodes(const nl_octree *t) { return t ? (int64_t)t->type.size() : -1; }

int64_t nl_octree_count_leaf_nodes(const nl_octree *t) {
    if (!t) return -1;
    int64_t c = 0;
    for (int8_t ty : t->type) c += (ty == kSurface);
    return c;
}

int nl_octree_has_voxel(const nl_octree *t, const int32_t xyz[3]) {
    if (!t || !xyz) return 0;
    return t->find(xyz[0], xyz[1], xyz[2]) >= 0;
}

// exports node `i` into row `o` of the output arrays
static void export_row(const nl_octree *t, int64_t i, int64_t o, float *voxels4, float *children_f, int32_t *children_i9, float *centres,
                       int32_t *features);

static void export_rows(const nl_octree *t, float *voxels4, float *children_f, int32_t *children_i9, float *centres,
                        int32_t *features) {
    const int64_t n = (int64_t)t->type.size();
    for (int64_t i = 0; i < n; ++i) export_row(t, i, i, voxels4, children_f, children_i9, centres, features);
}

static void export_row(const nl_octree *t, int64_t i, int64_t o, float *voxels4, float *children_f, int32_t *children_i9, float *centres,
                       int32_t *features) {
    const float vs = (float)t->voxel_size;
    {
        const bool visited = t->type[i] != kFeature;  // BFS reaches every non-FEATURE node (octree.cpp:330-338)
        float xyz[3] = {0.f, 0.f, 0.f}, sd = 0.f;
        if (visited) {
            xyz[0] = (float)(int)squeeze3(t->code[i]);
            xyz[1] = (float)(int)squeeze3(t->code[i] >> 1);
            xyz[2] = (float)(int)squeeze3(t->code[i] >> 2);
            sd = (float)t->side[i];
        }
        if (voxels4) { voxels4[o * 4 + 0] = xyz[0]; voxels4[o * 4 + 1] = xyz[1]; voxels4[o * 4 + 2] = xyz[2]; voxels4[o * 4 + 3] = sd; }
        if (centres) {  // mapping.py:322: (voxels[:, :3] + voxels[:, -1:] / 2) * voxel_size, all fp32
            const float h = sd / 2.0f;
            for (int a = 0; a < 3; ++a) centres[o * 3 + a] = (xyz[a] + h) * vs;
        }
        for (int s = 0; s < 8; ++s) {
            const int32_t c = t->child[(size_t)i * 8 + s];
            const int32_t v = (visited && c >= 0 && t->type[c] != kFeature) ? c : -1;
            if (children_f) children_f[o * 8 + s] = (float)v;
            if (children_i9) children_i9[o * 9 + s] = v;
        }
        if (children_i9) children_i9[o * 9 + 8] = (int32_t)sd;  // mapping.py:323-326
        for (int k = 0; k < 8; ++k) {
            int32_t f = -1;
            if (t->type[i] == kSurface)
                f = t->find((int)(xyz[0] + (float)kIncX[k]), (int)(xyz[1] + (float)kIncY[k]), (int)(xyz[2] + (float)kIncZ[k]));
            features[o * 8 + k] = f;
        }
    }
}

int nl_octree_export(const nl_octree *t, float *voxels, float *children, int32_t *features) {
    if (!t || !voxels || !children || !features) return nl_set_error("nl_octree_export: null argument");
    export_rows(t, voxels, children, nullptr, nullptr, features);
    return NL_OK;
}

int nl_octree_export_map(const nl_octree *t, float *centres, int32_t *structure, int32_t *vertex) {
    if (!t || !centres || !structure || !vertex) return nl_set_error("nl_octree_export_map: null argument");
    export_rows(t, nullptr, nullptr, structure, centres, vertex);
    return NL_OK;
}

int64_t nl_octree_dirty_count(const nl_octree *t) { return t ? (int64_t)t->dirty.size() : -1; }

int nl_octree_export_dirty(nl_octree *t, int32_t *ids, float *centres, int32_t *structure, int32_t *vertex, int clear) {
    if (!t || !ids || !centres || !structure || !vertex) return nl_set_error("nl_octree_export_dirty: null argument");
    std::sort(t->dirty.begin(), t->dirty.end());       // ascending node id: the order in which a full export lists them
    for (size_t o = 0; o < t->dirty.size(); ++o) {
        ids[o] = t->dirty[o];
        export_row(t, t->dirty[o], (int64_t)o, nullptr, nullptr, structure, centres, vertex);
    }
    if (clear) {
        for (int32_t id : t->dirty) t->dirty_flag[(size_t)id] = 0;
        t->dirty.clear();
    }
    return NL_OK;
}

static void preorder(const nl_octree *t, int32_t n, bool leaves_only, std::vector<float> &out) {
    const float x = (float)(int)squeeze3(t->code[n]), y = (float)(int)squeeze3(t->code[n] >> 1), z = (float)(int)squeeze3(t->code[n] >> 2);
    if (leaves_only) {
        if (t->type[n] == kSurface) { out.insert(out.end(), {x, y, z}); return; }  // octree.cpp:233-237 (leaf && SURFACE)
    } else {
        out.insert(out.end(), {x, y, z, (float)t->side[n]});
    }
    for (int s = 0; s < 8; ++s) {
        int32_t c = t->child[(size_t)n * 8 + s];
        if (c >= 0) preorder(t, c, leaves_only, out);
    }
}

int64_t nl_octree_get_voxels(const nl_octree *t, float *out, int64_t cap_rows) {
    if (!t) return -1;
    std::vector<float> v;
    preorder(t, 0, false, v);
    int64_t rows = (int64_t)v.size() / 4;
    if (out && rows <= cap_rows) std::memcpy(out, v.data(), v.size() * sizeof(float));
    return rows;
}

int64_t nl_octree_get_leaf_voxels(const nl_octree *t, float *out, int64_t cap_rows) {
    if (!t) return -1;
    std::vector<float> v;
    preorder(t, 0, true, v);
    int64_t rows = (int64_t)v.size() / 3;
    if (out && rows <= cap_rows) std::memcpy(out, v.data(), v.size() * sizeof(float));
    return rows;
}

int64_t nl_assign_embedding_rows(const int32_t *vertex, int64_t n_nodes, int32_t *vertex2row, int64_t n_rows) {
    if (!vertex || !vertex2row || n_nodes < 0 || n_rows < 0) return nl_set_error("nl_assign_embedding_rows: bad arguments");
    for (int64_t i = 0; i < n_nodes * 8; ++i) {
        const int32_t v = vertex[i];
        if (v >= 0 && v < n_nodes && vertex2row[v] < 0) vertex2row[v] = (int32_t)n_rows++;
    }
    return n_rows;
}

int64_t nl_assign_embedding_rows_subset(const int32_t *vertex_rows, int64_t n_rows_in, int64_t n_nodes, int32_t *vertex2row, int64_t n_rows,
                                        int32_t *vox2row_rows) {
    if (!vertex_rows || !vertex2row || !vox2row_rows || n_rows_in < 0 || n_nodes < 0 || n_rows < 0)
        return nl_set_error("nl_assign_embedding_rows_subset: bad arguments");
    for (int64_t i = 0; i < n_rows_in * 8; ++i) {
        const int32_t v = vertex_rows[i];
        if (v >= 0 && v < n_nodes && vertex2row[v] < 0) vertex2row[v] = (int32_t)n_rows++;
        vox2row_rows[i] = (v >= 0 && v < n_nodes) ? vertex2row[v] : -1;
    }
    return n_rows;
}

// Node-array validation (header section 1, NL_TREE_*).  csrc/octree_dev.cu nl_devoctree_validate restates it check for check; the
// two must set the same bits for every input.
int64_t nl_octree_validate(int64_t grid_dim, int64_t n, const int32_t *child, const uint64_t *code, const int8_t *type, const uint8_t *level,
                           const int32_t *vertex2row, int64_t n_rows) {
    if (grid_dim < 2 || grid_dim > (1 << 20) || (grid_dim & (grid_dim - 1))) return nl_set_error("nl_octree_validate: grid_dim must be a power of two in [2, 2^20]");
    if (n < 0 || n > INT32_MAX || n_rows < 0) return nl_set_error("nl_octree_validate: bad sizes");
    if (n > 0 && (!child || !code || !type || !level)) return nl_set_error("nl_octree_validate: null pointer");
    if (n == 0) return NL_TREE_ROOT;
    int L = 0;
    while ((int64_t(1) << L) < grid_dim) ++L;
    int64_t bits = 0;
    if (level[0] != 0 || code[0] != 0 || type[0] != kNonLeaf) bits |= NL_TREE_ROOT;
    std::vector<int32_t> parents((size_t)n, 0);
    for (int64_t i = 0; i < n; ++i) {
        const int t = type[i], lv = level[i];
        bool has_child = false;
        for (int s = 0; s < 8; ++s) {
            const int64_t c = child[i * 8 + s];
            if (c == -1) continue;
            has_child = true;
            if (c <= i || c >= n) { bits |= NL_TREE_RANGE; continue; }   // never read at an unchecked id
            ++parents[(size_t)c];
            const int lc = level[c];
            if (lc != lv + 1 || lc > L) bits |= NL_TREE_LINK;
            else if (code[c] != (code[i] | (uint64_t)s << (3 * (L - lc)))) bits |= NL_TREE_LINK;
        }
        const bool t_ok = t >= kNonLeaf && t <= kFeature;
        if (!t_ok || lv > L) { bits |= NL_TREE_RANGE; continue; }
        if (code[i] & ((uint64_t(1) << (3 * (L - lv))) - 1)) bits |= NL_TREE_LINK;
        if ((t == kNonLeaf) != (lv < L) || (t == kNonLeaf && !has_child)) bits |= NL_TREE_SHAPE;
    }
    for (int64_t i = 1; i < n; ++i)
        if (parents[(size_t)i] != 1) bits |= NL_TREE_PARENTS;
    if (bits || !vertex2row) return bits;
    // rows: the tree is well-formed, so a SURFACE node is a level-L leaf with in-grid coordinates and find() stays in the tree
    const int size = (int)grid_dim;
    std::vector<int32_t> uses((size_t)std::min(n_rows, n), 0);
    std::vector<uint8_t> referenced((size_t)n, 0);
    if (n_rows > n) bits |= NL_TREE_ROWS;                          // a row per node at most
    for (int64_t i = 0; i < n; ++i) {
        const int32_t r = vertex2row[i];
        if (r < -1 || r >= n_rows) bits |= NL_TREE_ROWS;
        else if (r >= 0) {
            if (level[i] != L) bits |= NL_TREE_ROWS;
            if (r < n) ++uses[(size_t)r];
        }
        if (type[i] != kSurface) continue;
        const int x = (int)squeeze3(code[i]), y = (int)squeeze3(code[i] >> 1), z = (int)squeeze3(code[i] >> 2);
        for (int k = 0; k < 8; ++k) {
            const int cx = x + kIncX[k], cy = y + kIncY[k], cz = z + kIncZ[k];
            const int32_t v = (cx < size && cy < size && cz < size) ? find_in(child, size, L, cx, cy, cz) : -1;
            if (v < 0) bits |= NL_TREE_VERTICES;
            else referenced[(size_t)v] = 1;
        }
    }
    for (size_t r = 0; r < uses.size(); ++r)
        if (uses[r] != 1) bits |= NL_TREE_ROWS;
    for (int64_t i = 0; i < n; ++i)
        if ((vertex2row[i] >= 0) != (referenced[(size_t)i] != 0)) bits |= NL_TREE_VERTICES;
    return bits;
}

int nl_octree_nodes(const nl_octree *t, int32_t *child, uint64_t *code, int8_t *type, uint8_t *level) {
    if (!t || !child || !code || !type || !level) return nl_set_error("nl_octree_nodes: null argument");
    const size_t n = t->type.size();
    std::memcpy(child, t->child.data(), n * 8 * sizeof(int32_t));
    std::memcpy(code, t->code.data(), n * sizeof(uint64_t));
    std::memcpy(type, t->type.data(), n);
    for (size_t i = 0; i < n; ++i) level[i] = (uint8_t)(t->max_level - __builtin_ctz(t->side[i]));   // side = grid_dim >> level
    return NL_OK;
}

int nl_octree_restore(nl_octree *t, const int32_t *child, const uint64_t *code, const int8_t *type, const uint8_t *level, int64_t n) {
    if (!t || n < 0) return nl_set_error("nl_octree_restore: bad arguments");
    const int64_t bits = nl_octree_validate(t->size, n, child, code, type, level, nullptr, 0);
    if (bits != 0) return (int)bits;                              // < 0: bad arguments; > 0: the failed checks, tree untouched
    t->child.assign(child, child + n * 8);
    t->code.assign(code, code + n);
    t->type.assign(type, type + n);
    t->side.resize((size_t)n);
    t->corner_keys = KeySet();
    for (int64_t i = 0; i < n; ++i) {
        t->side[(size_t)i] = (uint32_t)t->size >> level[i];
        if (level[i] == t->max_level) t->corner_keys.insert(code[i]);   // the corner keys are exactly the level-L codes
    }
    t->dirty.clear();
    t->dirty_flag.assign((size_t)n, 0);
    // seen_points is a cache of inserted points: a repeated point only visits existing nodes and changes nothing, so the restored
    // tree starts with an empty one and inserts exactly like the tree it was saved from.
    t->seen_points = KeySet();
    return NL_OK;
}

}  // extern "C"
