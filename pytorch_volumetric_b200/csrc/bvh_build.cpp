// bvh_build.cpp -- host-side BVH4 construction for libpvb.so.
//
// Replaces the Embree scene build the reference triggers through
// RaycastingScene.add_triangles (reference src/pytorch_volumetric/sdf.py:115-118).
// Binned-SAH binary build -> greedy collapse to 4-wide nodes -> breadth-first
// layout (so the top of the tree is a contiguous prefix the query kernels stage
// into shared memory with one bulk copy) -> triangles emitted in leaf order.
#include "../../include/pvb.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <climits>
#include <queue>
#include <vector>

extern void pvb_set_error(const char *fmt, ...);

namespace {

struct Box {
    float lo[3], hi[3];
    void reset() { for (int k = 0; k < 3; ++k) { lo[k] = INFINITY; hi[k] = -INFINITY; } }
    void grow(const float *p) { for (int k = 0; k < 3; ++k) { lo[k] = std::min(lo[k], p[k]); hi[k] = std::max(hi[k], p[k]); } }
    void grow(const Box &b) { for (int k = 0; k < 3; ++k) { lo[k] = std::min(lo[k], b.lo[k]); hi[k] = std::max(hi[k], b.hi[k]); } }
    float half_area() const {
        const float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        if (!(dx >= 0.f)) return 0.f;
        return dx * dy + dy * dz + dz * dx;
    }
};

struct BinNode {
    Box box;
    int left = -1, right = -1;
    int start = 0, count = 0;
};

static int kLeafMax = 4;   // triangles per leaf, 1..4 (PVB_BVH_LEAF; the link encoding holds count-1 in 2 bits)
constexpr int kBins = 16;

struct Builder {
    const float *verts;
    const int32_t *faces;
    std::vector<Box> tbox;
    std::vector<float> cent;   // 3 per triangle
    std::vector<int32_t> order;
    std::vector<BinNode> nodes;
    bool force_median = false;   // balanced fallback when the SAH tree would be too deep for the traversal stack

    int build(int start, int count, int depth, int &max_depth) {
        const int id = (int)nodes.size();
        nodes.emplace_back();
        Box box, cbox;
        box.reset(); cbox.reset();
        for (int i = start; i < start + count; ++i) {
            box.grow(tbox[order[i]]);
            cbox.grow(&cent[3 * (size_t)order[i]]);
        }
        nodes[id].box = box;
        nodes[id].start = start;
        nodes[id].count = count;
        max_depth = std::max(max_depth, depth);
        if (count <= kLeafMax) return id;

        // binned SAH over the three axes
        int best_axis = -1, best_bin = -1;
        float best_cost = INFINITY;
        for (int ax = 0; ax < 3 && !force_median; ++ax) {
            const float ext = cbox.hi[ax] - cbox.lo[ax];
            if (!(ext > 0.f)) continue;
            Box bb[kBins]; int bc[kBins];
            for (int b = 0; b < kBins; ++b) { bb[b].reset(); bc[b] = 0; }
            const float scale = kBins / ext;
            for (int i = start; i < start + count; ++i) {
                const int t = order[i];
                int b = (int)((cent[3 * (size_t)t + ax] - cbox.lo[ax]) * scale);
                b = std::min(std::max(b, 0), kBins - 1);
                bb[b].grow(tbox[t]); bc[b]++;
            }
            float right_area[kBins]; int right_cnt[kBins];
            Box acc; acc.reset(); int cnt = 0;
            for (int b = kBins - 1; b > 0; --b) {
                acc.grow(bb[b]); cnt += bc[b];
                right_area[b] = acc.half_area(); right_cnt[b] = cnt;
            }
            acc.reset(); cnt = 0;
            for (int b = 0; b < kBins - 1; ++b) {
                acc.grow(bb[b]); cnt += bc[b];
                if (cnt == 0 || right_cnt[b + 1] == 0) continue;
                const float cost = acc.half_area() * cnt + right_area[b + 1] * right_cnt[b + 1];
                if (cost < best_cost) { best_cost = cost; best_axis = ax; best_bin = b; }
            }
        }
        int mid;
        if (best_axis >= 0) {
            const float ext = cbox.hi[best_axis] - cbox.lo[best_axis];
            const float scale = kBins / ext;
            const float lo = cbox.lo[best_axis];
            const int ax = best_axis, bin = best_bin;
            auto it = std::partition(order.begin() + start, order.begin() + start + count, [&](int32_t t) {
                int b = (int)((cent[3 * (size_t)t + ax] - lo) * scale);
                b = std::min(std::max(b, 0), kBins - 1);
                return b <= bin;
            });
            mid = (int)(it - order.begin());
        } else {
            mid = start;  // all centroids coincide: fall through to the median split
        }
        if (mid == start || mid == start + count || depth > 40) {
            // degenerate or too deep: median split on the longest axis
            int ax = 0;
            for (int k = 1; k < 3; ++k)
                if (cbox.hi[k] - cbox.lo[k] > cbox.hi[ax] - cbox.lo[ax]) ax = k;
            mid = start + count / 2;
            std::nth_element(order.begin() + start, order.begin() + mid, order.begin() + start + count,
                             [&](int32_t a, int32_t b) { return cent[3 * (size_t)a + ax] < cent[3 * (size_t)b + ax]; });
        }
        const int l = build(start, mid - start, depth + 1, max_depth);
        const int r = build(mid, start + count - mid, depth + 1, max_depth);
        nodes[id].left = l;
        nodes[id].right = r;
        return id;
    }
};

}  // namespace

// Collapse the binary tree to 4-wide nodes in breadth-first order; returns the depth of the wide tree.
static int collapse(const Builder &b, std::vector<pvb_bvh4_node> &wide) {

    std::vector<int> wide_depth;
    struct Item { int bin; int wide; };
    std::queue<Item> q;
    auto new_wide = [&](int depth) {
        pvb_bvh4_node n;
        for (int c = 0; c < 4; ++c) {
            n.lox[c] = n.loy[c] = n.loz[c] = INFINITY;
            n.hix[c] = n.hiy[c] = n.hiz[c] = -INFINITY;
            n.child[c] = INT32_MIN; n._pad[c] = 0;
        }
        wide.push_back(n); wide_depth.push_back(depth);
        return (int)wide.size() - 1;
    };
    int max_depth = 1;
    q.push({0, new_wide(1)});
    while (!q.empty()) {
        const Item it = q.front(); q.pop();
        const BinNode &root = b.nodes[(size_t)it.bin];
        int kids[4]; int nk = 0;
        if (root.left < 0) {
            kids[nk++] = it.bin;             // a leaf root (tiny mesh): single leaf child
        } else {
            kids[nk++] = root.left; kids[nk++] = root.right;
            while (nk < 4) {
                int pick = -1; float area = -1.f;
                for (int i = 0; i < nk; ++i) {
                    const BinNode &c = b.nodes[(size_t)kids[i]];
                    if (c.left >= 0 && c.box.half_area() > area) { area = c.box.half_area(); pick = i; }
                }
                if (pick < 0) break;
                const BinNode &c = b.nodes[(size_t)kids[pick]];
                kids[pick] = c.left; kids[nk++] = c.right;
            }
        }
        const int d = wide_depth[(size_t)it.wide];
        max_depth = std::max(max_depth, d);
        for (int i = 0; i < nk; ++i) {
            const BinNode &c = b.nodes[(size_t)kids[i]];
            // index into `wide` afresh each time: new_wide() may reallocate
            int32_t link;
            if (c.left < 0) {
                link = ~(int32_t)(((uint32_t)c.start << 2) | (uint32_t)(c.count - 1));
            } else {
                const int w = new_wide(d + 1);
                link = w;
                q.push({kids[i], w});
            }
            pvb_bvh4_node &n = wide[(size_t)it.wide];
            n.lox[i] = c.box.lo[0]; n.loy[i] = c.box.lo[1]; n.loz[i] = c.box.lo[2];
            n.hix[i] = c.box.hi[0]; n.hiy[i] = c.box.hi[1]; n.hiz[i] = c.box.hi[2];
            n.child[i] = link;
        }
    }
    return max_depth;
}

extern "C" int64_t pvb_bvh_max_nodes(int64_t n_faces) {
    // every wide node has >= 2 children, leaves hold >= 1 triangle
    return n_faces < 1 ? 1 : n_faces;
}

extern "C" int pvb_bvh_build(const float *verts, int64_t n_verts, const int32_t *faces, int64_t n_faces,
                             void *nodes_out, int64_t node_capacity, float *tris_out,
                             int64_t *n_nodes_out, int32_t *max_depth_out) {
    if (!verts || !faces || !nodes_out || !tris_out || n_faces < 1 || n_verts < 1) {
        pvb_set_error("pvb_bvh_build: null argument or empty mesh (n_verts=%lld n_faces=%lld)",
                      (long long)n_verts, (long long)n_faces);
        return PVB_ERR_INVALID;
    }
    if (n_faces >= (1ll << 29)) {
        pvb_set_error("pvb_bvh_build: too many faces (%lld)", (long long)n_faces);
        return PVB_ERR_INVALID;
    }
    for (int64_t i = 0; i < 3 * n_faces; ++i)
        if (faces[i] < 0 || faces[i] >= n_verts) {
            pvb_set_error("pvb_bvh_build: face index %d out of range [0,%lld)", faces[i], (long long)n_verts);
            return PVB_ERR_INVALID;
        }

    if (const char *e = getenv("PVB_BVH_LEAF")) {
        const int v = atoi(e);
        if (v >= 1 && v <= 4) kLeafMax = v;
    }
    Builder b;
    b.verts = verts; b.faces = faces;
    b.tbox.resize((size_t)n_faces);
    b.cent.resize(3 * (size_t)n_faces);
    b.order.resize((size_t)n_faces);
    for (int64_t t = 0; t < n_faces; ++t) {
        b.order[(size_t)t] = (int32_t)t;
        Box bx; bx.reset();
        for (int v = 0; v < 3; ++v) bx.grow(verts + 3 * (int64_t)faces[3 * t + v]);
        b.tbox[(size_t)t] = bx;
        for (int k = 0; k < 3; ++k) b.cent[3 * (size_t)t + k] = 0.5f * (bx.lo[k] + bx.hi[k]);
    }
    // The query kernels keep a fixed traversal stack: 3 * depth + 2 entries must fit (kMaxWideDepth).  SAH trees of
    // ordinary meshes are far below that; a pathological one is rebuilt with balanced median splits.
    constexpr int kMaxWideDepth = 20;
    std::vector<pvb_bvh4_node> wide;
    int max_depth = 1;
    for (int attempt = 0; attempt < 2; ++attempt) {
        b.force_median = attempt == 1;
        b.nodes.clear();
        b.nodes.reserve(2 * (size_t)n_faces);
        for (int64_t t = 0; t < n_faces; ++t) b.order[(size_t)t] = (int32_t)t;
        int bin_depth = 0;
        b.build(0, (int)n_faces, 0, bin_depth);
        wide.clear();
        max_depth = collapse(b, wide);
        if (max_depth <= kMaxWideDepth) break;
    }
    if (max_depth > kMaxWideDepth) {
        pvb_set_error("pvb_bvh_build: tree depth %d exceeds the traversal stack even with balanced splits", max_depth);
        return PVB_ERR_INVALID;
    }
    if ((int64_t)wide.size() > node_capacity) {
        pvb_set_error("pvb_bvh_build: node buffer too small (%lld > %lld)", (long long)wide.size(),
                      (long long)node_capacity);
        return PVB_ERR_CAPACITY;
    }
    std::memcpy(nodes_out, wide.data(), wide.size() * sizeof(pvb_bvh4_node));
    for (int64_t i = 0; i < n_faces; ++i) {
        const int32_t t = b.order[(size_t)i];
        float *o = tris_out + 12 * i;
        for (int v = 0; v < 3; ++v) {
            const float *p = verts + 3 * (int64_t)faces[3 * (int64_t)t + v];
            o[4 * v] = p[0]; o[4 * v + 1] = p[1]; o[4 * v + 2] = p[2]; o[4 * v + 3] = 0.f;
        }
        std::memcpy(&o[3], &t, sizeof(int32_t));   // original face index as int bits
    }
    if (n_nodes_out) *n_nodes_out = (int64_t)wide.size();
    if (max_depth_out) *max_depth_out = max_depth;
    return PVB_OK;
}
