// b2_scene_commit: the scene description flattened and precomputed (TriAccel, BVH, leaf records, MIP pyramids, CDFs) and uploaded to
// HBM as one DScene.  Each stage is one function that takes what it reads and returns what it makes; b2_scene_commit runs them in order.
#include "b2_host.h"
#include "bvh_builder.h"
#include "bvh_device.h"

#include <sched.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <thread>

struct H3 {
    float x, y, z;
};
static inline H3 sub3(const float *a, const float *b) { return {a[0] - b[0], a[1] - b[1], a[2] - b[2]}; }
static inline H3 cross3(const H3 &a, const H3 &b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
static inline float comp3(const H3 &a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }
// TriAccel::load, include/mitsuba/render/triaccel.h:61-94
static void triAccelLoad(const float *A, const float *B, const float *C, uint32_t words[12]) {
    static const int waldModulo[4] = {1, 2, 0, 1};
    memset(words, 0, 48);
    H3 b = sub3(C, A), c = sub3(B, A), N = cross3(c, b);
    uint32_t k = 0;
    for (int j = 0; j < 3; j++)
        if (std::fabs(comp3(N, j)) > std::fabs(comp3(N, k))) k = j;
    uint32_t u = waldModulo[k], v = waldModulo[k + 1];
    const float n_k = comp3(N, k), denom = comp3(b, u) * comp3(c, v) - comp3(b, v) * comp3(c, u);
    float f[12];
    memset(f, 0, sizeof(f));
    if (denom == 0) {
        k = 3;
    } else {
        f[1] = comp3(N, u) / n_k;
        f[2] = comp3(N, v) / n_k;
        f[3] = (A[0] * N.x + A[1] * N.y + A[2] * N.z) / n_k;
        f[6] = comp3(b, u) / denom;
        f[7] = -comp3(b, v) / denom;
        f[4] = A[u];
        f[5] = A[v];
        f[8] = comp3(c, v) / denom;
        f[9] = -comp3(c, u) / denom;
    }
    memcpy(words, f, 48);
    words[0] = k;
}
uint32_t materialFlags(const std::vector<b2_material_desc> &mats, int id) {
    const b2_material_desc &d = mats[id];
    const uint32_t EDiffuseReflection = 0x2, EGlossyReflection = 0x8, EGlossyTransmission = 0x10, EDeltaReflection = 0x20, EAnisotropic = 0x1000,
                   ENonSymmetric = 0x4000, EFrontSide = 0x8000, EBackSide = 0x10000, EUsesSampler = 0x20000;
    switch (d.type) {
        case 0: if (d.reflectance_texture > 0) return EDiffuseReflection | EFrontSide | 0x2000u /* ESpatiallyVarying */;
                return (std::max(std::max(d.reflectance[0], d.reflectance[1]), d.reflectance[2]) > 0) ? (EDiffuseReflection | EFrontSide) : 0; // diffuse.cpp:98-103
        case 1: return EGlossyReflection | EFrontSide | (d.alpha_u != d.alpha_v ? EAnisotropic : 0);
        case 2: return EGlossyReflection | EGlossyTransmission | EFrontSide | EBackSide | EUsesSampler | ENonSymmetric | (d.alpha_u != d.alpha_v ? EAnisotropic : 0);
        case 4: return 0x1u /* ENull */ | EFrontSide | EBackSide; // null.cpp:38-43
        case 5: return ((materialFlags(mats, d.nested) & ~EBackSide) | EFrontSide) | ((materialFlags(mats, d.nested2) & ~EFrontSide) | EBackSide); // twosided.cpp:96-102
        case 6: return EDeltaReflection | 0x40u /* EDeltaTransmission */ | EFrontSide | EBackSide | ENonSymmetric; // dielectric.cpp:190-194
        case 7: return EDeltaReflection | EFrontSide;                                                            // conductor.cpp:181-183
        case 8: return EDeltaReflection | EDiffuseReflection | EFrontSide;                                       // plastic.cpp:211-215
        default: return materialFlags(mats, d.nested) | EDeltaReflection | EFrontSide | EBackSide;
    }
}
// Threads the host-side build may use: hardware threads, capped by the scheduler affinity and the cgroup CPU quota (a 128-thread box
// leased with a 16-CPU quota runs 128 workers slower than 16)
static int usableThreads() {
    int n = (int) std::thread::hardware_concurrency();
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof(set), &set) == 0) n = std::min(n > 0 ? n : CPU_COUNT(&set), CPU_COUNT(&set));
    if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char quota[64]; long long period = 0;
        if (fscanf(f, "%63s %lld", quota, &period) == 2 && strcmp(quota, "max") != 0 && period > 0) {
            const long long q = atoll(quota);
            if (q > 0) n = std::min<long long>(n, std::max<long long>(1, (q + period - 1) / period));
        }
        fclose(f);
    }
    if (const char *e = getenv("B2_BUILD_THREADS")) n = atoi(e);
    return std::max(1, n);
}
// f(begin, end) over [0, n) in contiguous chunks, one per thread (per-element work that is independent and writes to its own slots)
template <typename F> static void parallelFor(size_t n, int threads, F f) {
    const int parts = (int) std::min<size_t>((size_t) std::max(1, threads), std::max<size_t>(1, n / 8192));
    if (parts <= 1) { f((size_t) 0, n); return; }
    std::vector<std::thread> th;
    for (int c = 1; c < parts; ++c) th.emplace_back([=]() { f(n * c / parts, n * (c + 1) / parts); });
    f((size_t) 0, n / parts);
    for (auto &t : th) t.join();
}
// B2_COMMIT_TIMING=1: host-side phase times of b2_scene_commit on stderr (where the seconds of a multi-million-triangle commit go)
struct CommitClock {
    bool on = getenv("B2_COMMIT_TIMING") != nullptr;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now(), last = t0;
    void mark(const char *what) {
        if (!on) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[b2 commit] %-28s %8.1f ms (total %8.1f ms)\n", what, std::chrono::duration<double, std::milli>(now - last).count(),
                std::chrono::duration<double, std::milli>(now - t0).count());
        last = now;
    }
};
// a binary-tree reference moved into merged node / leaf arrays
static int32_t shiftRef(int32_t r, uint32_t nodeBase, uint32_t leafBase) {
    if (r >= 0) return r + (int32_t) nodeBase;
    const uint32_t bits = ~(uint32_t) r;
    return (int32_t) ~(((bits & 0x0FFFFFFFu) + leafBase) | (bits & 0xF0000000u));
}
// gkdtree.h:1213-1220: a kd-tree box enlarged by a relative and an absolute epsilon (the max side uses the already-moved min, as in the
// reference)
static void enlargedBox(const float lo[3], const float hi[3], float mn[3], float mx[3]) {
    const float eps = 1e-3f;
    for (int a = 0; a < 3; ++a) {
        mn[a] = lo[a] - ((hi[a] - lo[a]) * eps + eps);
        mx[a] = hi[a] + ((hi[a] - mn[a]) * eps + eps);
    }
}
// ---- emitter order of Scene::m_emitters: emitters that are direct children of the scene (`constant`) are appended by Scene::addChild
// (scene.cpp:510-516); the area emitters of shapes only join in Scene::initialize -> addShape (scene.cpp:322-335, :570-571), i.e. behind
// them and in shape order, whatever the document order ----
struct EmitterOrder {
    std::vector<int> order, index; // device index -> emitter id, and the inverse
};
static EmitterOrder emitterOrder(const b2_scene *s) {
    EmitterOrder o;
    o.index.assign(s->emitters.size(), -1);
    for (size_t e = 0; e < s->emitters.size(); ++e) if (s->emitters[e].env) o.order.push_back((int) e);
    for (auto &m : s->meshes) if (m.emitter >= 0) o.order.push_back(m.emitter);
    for (size_t k = 0; k < o.order.size(); ++k) o.index[o.order[k]] = (int) k;
    return o;
}
// ---- flatten meshes: prim order = mesh order, triangle order (skdtree.cpp:68-72 m_shapeMap) ----
struct Flat {
    size_t nPrims = 0;
    std::vector<float4> verts, norms, texc; // 3 rows per prim (norms / texc empty when no mesh needs them)
    // candidate primitives (degenerate triangles excluded) per acceleration structure: bucket 0 = world, bucket g + 1 = shapegroup g
    std::vector<std::vector<PrimBox>> boxes;
    std::vector<std::vector<uint32_t>> ids;
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY}; // bounds of the world's triangles
};
// TriMesh::computeUVTangents, trimesh.cpp:683-735: dpdu, dpdv of triangle p0 p1 p2 with texture coordinates uv0 uv1 uv2 (left as they
// are for a triangle of zero area)
static void computeUVTangents(const float *p0, const float *p1, const float *p2, const float *uv0, const float *uv1, const float *uv2, float dpdu[3],
                              float dpdv[3]) {
    H3 dP1 = sub3(p1, p0), dP2 = sub3(p2, p0);
    float du1 = uv1[0] - uv0[0], dv1 = uv1[1] - uv0[1];
    float du2 = uv2[0] - uv0[0], dv2 = uv2[1] - uv0[1];
    H3 nn = cross3(dP1, dP2);
    float length = std::sqrt(nn.x * nn.x + nn.y * nn.y + nn.z * nn.z);
    if (length == 0) return;
    float determinant = du1 * dv2 - dv1 * du2;
    if (determinant == 0) {
        // coordinateSystem(n/length, dpdu, dpdv): util.cpp:592-601 -- dpdu is the `b` output
        float r = 1.0f / length;
        H3 a = {nn.x * r, nn.y * r, nn.z * r}, c;
        if (std::fabs(a.x) > std::fabs(a.y)) {
            float invLen = 1.0f / std::sqrt(a.x * a.x + a.z * a.z);
            c = {a.z * invLen, 0.0f, -a.x * invLen};
        } else {
            float invLen = 1.0f / std::sqrt(a.y * a.y + a.z * a.z);
            c = {0.0f, a.z * invLen, -a.y * invLen};
        }
        H3 b = cross3(c, a);
        dpdu[0] = b.x; dpdu[1] = b.y; dpdu[2] = b.z;
        dpdv[0] = c.x; dpdv[1] = c.y; dpdv[2] = c.z;
    } else {
        float invDet = 1.0f / determinant;
        dpdu[0] = (dv2 * dP1.x - dv1 * dP2.x) * invDet;
        dpdu[1] = (dv2 * dP1.y - dv1 * dP2.y) * invDet;
        dpdu[2] = (dv2 * dP1.z - dv1 * dP2.z) * invDet;
        dpdv[0] = (-du2 * dP1.x + du1 * dP2.x) * invDet;
        dpdv[1] = (-du2 * dP1.y + du1 * dP2.y) * invDet;
        dpdv[2] = (-du2 * dP1.z + du1 * dP2.z) * invDet;
    }
}
// Writes the prim-order TriAccel records straight into s->hTriAccelPrimOrder (b2_get_triaccel, and the source of the leaf rows).
static int flattenMeshes(b2_scene *s, const std::vector<int> &emIndex, int threads, Flat &f) {
    size_t nPrims = 0;
    for (auto &m : s->meshes) { m.primOffset = (uint32_t) nPrims; nPrims += m.idx.size() / 3; }
    if (nPrims >= (1u << 28)) return fail(s->ctx, B2_ERR_INVALID, "too many triangles (limit 2^28)");
    f.nPrims = nPrims;
    bool anyNorm = false;
    for (auto &m : s->meshes) anyNorm |= !m.N.empty() || !m.UV.empty();
    const bool anyTex = !s->textures.empty();
    f.verts.resize(3 * nPrims);
    f.norms.resize(anyNorm ? 3 * nPrims : 0);
    f.texc.resize(anyTex && anyNorm ? 3 * nPrims : 0);
    std::vector<float4> &triAccel = s->hTriAccelPrimOrder;
    triAccel.resize(3 * nPrims);
    f.boxes.resize(1 + (size_t) s->nGroups);
    f.ids.resize(1 + (size_t) s->nGroups);
    f.boxes[0].reserve(nPrims); f.ids[0].reserve(nPrims);
    std::vector<PrimBox> primBox(nPrims);          // per-prim boxes in prim order; compacted into the buckets (minus degenerates) below
    std::vector<uint8_t> primDegenerate(nPrims, 0);
    for (size_t mi = 0; mi < s->meshes.size(); ++mi) {
        const HostMesh &m = s->meshes[mi];
        const size_t nT = m.idx.size() / 3;
        parallelFor(nT, threads, [&](size_t jlo, size_t jhi) {
        for (size_t j = jlo; j < jhi; ++j) {
            const size_t p = m.primOffset + j;
            const uint32_t i0 = m.idx[3 * j], i1 = m.idx[3 * j + 1], i2 = m.idx[3 * j + 2];
            const float *p0 = &m.P[3 * i0], *p1 = &m.P[3 * i1], *p2 = &m.P[3 * i2];
            uint32_t tflags = (m.N.empty() ? 0u : 1u) | (m.UV.empty() ? 0u : 2u);
            int matBits = m.material, emBits = m.emitter >= 0 ? emIndex[m.emitter] : -1;
            float w0, w1, w2;
            memcpy(&w0, &matBits, 4); memcpy(&w1, &emBits, 4); memcpy(&w2, &tflags, 4);
            f.verts[3 * p] = make_float4(p0[0], p0[1], p0[2], w0);
            f.verts[3 * p + 1] = make_float4(p1[0], p1[1], p1[2], w1);
            f.verts[3 * p + 2] = make_float4(p2[0], p2[1], p2[2], w2);
            if (anyNorm) {
                float n[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, dpdu[3] = {0, 0, 0}, dpdv[3] = {0, 0, 0};
                if (!m.N.empty()) {
                    memcpy(n[0], &m.N[3 * i0], 12); memcpy(n[1], &m.N[3 * i1], 12); memcpy(n[2], &m.N[3 * i2], 12);
                }
                if (!m.UV.empty()) computeUVTangents(p0, p1, p2, &m.UV[2 * i0], &m.UV[2 * i1], &m.UV[2 * i2], dpdu, dpdv);
                f.norms[3 * p] = make_float4(n[0][0], n[0][1], n[0][2], dpdu[0]);
                f.norms[3 * p + 1] = make_float4(n[1][0], n[1][1], n[1][2], dpdu[1]);
                f.norms[3 * p + 2] = make_float4(n[2][0], n[2][1], n[2][2], dpdu[2]);
                if (!f.texc.empty() && !m.UV.empty()) { // texture coordinates of the three vertices + dpdv of computeUVTangents
                    f.texc[3 * p] = make_float4(m.UV[2 * i0], m.UV[2 * i0 + 1], dpdv[0], 0.0f);
                    f.texc[3 * p + 1] = make_float4(m.UV[2 * i1], m.UV[2 * i1 + 1], dpdv[1], 0.0f);
                    f.texc[3 * p + 2] = make_float4(m.UV[2 * i2], m.UV[2 * i2 + 1], dpdv[2], 0.0f);
                }
            }
            uint32_t wds[12];
            triAccelLoad(p0, p1, p2, wds);
            wds[10] = (uint32_t) p;       // global prim id (reference: shapeIndex)
            wds[11] = (uint32_t) j;       // primIndex within the mesh
            memcpy(&triAccel[3 * p], wds, 48);
            PrimBox pb;
            for (int a = 0; a < 3; ++a) {
                pb.lo[a] = std::min(std::min(p0[a], p1[a]), p2[a]);
                pb.hi[a] = std::max(std::max(p0[a], p1[a]), p2[a]);
            }
            primBox[p] = pb;
            primDegenerate[p] = wds[0] == 3; // k == 3: degenerate, never hit (triaccel.h:75-78): not a candidate of any tree
        }
        });
        std::vector<PrimBox> &bb = f.boxes[m.group + 1];
        std::vector<uint32_t> &bi = f.ids[m.group + 1];
        for (size_t j = 0; j < nT; ++j) {
            const size_t p = m.primOffset + j;
            const PrimBox &pb = primBox[p];
            if (m.group < 0) for (int a = 0; a < 3; ++a) { f.lo[a] = std::min(f.lo[a], pb.lo[a]); f.hi[a] = std::max(f.hi[a], pb.hi[a]); }
            if (!primDegenerate[p]) { bb.push_back(pb); bi.push_back((uint32_t) p); }
        }
    }
    return B2_OK;
}
// ---- acceleration structures ----
struct Accel {
    std::vector<uint32_t> leafPrims;  // leaf-ordered prim ids: world | shapegroups
    int32_t rootRef = -1, tlasRoot = -1;
    uint32_t rootCount = 0;           // > 0: no tree, the world is one flat leaf of this many triangles
    int depth = 0;                    // of the deepest world / shapegroup tree
    std::vector<DInstance> items;     // instanced scenes: in the order of the top-level leaves
    float lo[3], hi[3];               // bounds of the world triangles and the instances
    double ms = 0;                    // b2_stats::accel_build_ms: the world and shapegroup builds
    size_t uploadBytes = 0;           // the builds' share of b2_stats::bytes_uploaded
};
// A host-built tree moved to the device: its node arrays are uploaded on `st` (`h` may go at once; the caller synchronises `st` before
// the arrays are read elsewhere), its leaf order is taken over.
static cudaError_t uploadTree(BVHResult &h, cudaStream_t st, DeviceBVHResult &out) {
    out.leafPrims.swap(h.leafPrims);
    out.rootRef = h.rootRef; out.depth = h.depth; out.depth8 = h.depth8;
    out.nNodes = h.nodes.size(); out.nNodes8 = h.nodes8.size();
    DevBuf<BVHNode> nodes;
    DevBuf<BVH8Node> nodes8;
    cudaError_t e = nodes.upload(h.nodes, st);
    if (e == cudaSuccess) e = nodes8.upload(h.nodes8, st);
    out.nodes = nodes.detach(); out.nodes8 = nodes8.detach();
    return e;
}
// The world or a shapegroup tree, from the builder the scene chose; the only place that looks at it.  Host: buildBVH, then uploaded
// (out.ms = the wall time of buildBVH).  Device: buildBVHDevice.  a.uploadBytes counts the host build's binary nodes or the device
// build's boxes and ids.
static int buildTree(b2_scene *s, int threads, const std::vector<PrimBox> &boxes, const std::vector<uint32_t> &ids, int maxDepth, bool wide,
                     DeviceBVHResult &out, Accel &a) {
    b2_ctx *ctx = s->ctx;
    if (s->accelBuild == B2_ACCEL_BUILD_DEVICE) {
        const std::string e = buildBVHDevice(boxes, ids, 4, maxDepth, wide, ctx->stream, out);
        if (!e.empty()) return fail(ctx, B2_ERR_CUDA, e);
        a.uploadBytes += boxes.size() * (sizeof(PrimBox) + sizeof(uint32_t));
    } else {
        BVHResult h;
        const auto t0 = std::chrono::steady_clock::now();
        buildBVH(boxes, ids, 4, maxDepth, threads, h, wide);
        out.ms = (float) std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        a.uploadBytes += h.nodes.size() * sizeof(BVHNode);
        CK(ctx, uploadTree(h, ctx->stream, out));
    }
    a.ms += out.ms;
    if (out.depth8 > B2_STACK8_DEPTH - 1) { // deeper than the wide traversal's stack: binary tree only
        cudaFree(out.nodes8);
        out.nodes8 = nullptr; out.nNodes8 = 0;
    }
    return B2_OK;
}
// Builds the trees and lays out the scene's node and leaf arrays (s->dNodes, s->dNodes8, a.leafPrims).  Marks "BVH (world)" on `clk`.
static int buildAccel(b2_scene *s, int threads, const Flat &f, CommitClock &clk, Accel &a) {
    b2_ctx *ctx = s->ctx;
    const bool instanced = !s->instances.empty();
    const std::vector<uint32_t> &ids = f.ids[0];
    for (int k = 0; k < 3; ++k) { a.lo[k] = f.lo[k]; a.hi[k] = f.hi[k]; }
    // Merged arrays: nodes = world | shapegroups | top-level tree, leaves = world | shapegroups.  place() gives a tree its (nodeBase, leafBase)
    // and returns its root reference there; the top-level tree's leaves index items and keep their references (leafBase 0).
    struct Part { const DeviceBVHResult *tree; uint32_t nodeBase, leafBase; };
    std::vector<Part> parts;
    size_t nNodes = 0;
    auto place = [&](DeviceBVHResult &t, bool triangleLeaves) -> int32_t {
        const uint32_t nodeBase = (uint32_t) nNodes, leafBase = triangleLeaves ? (uint32_t) a.leafPrims.size() : 0u;
        if (triangleLeaves && a.leafPrims.empty()) a.leafPrims.swap(t.leafPrims);
        else if (triangleLeaves) a.leafPrims.insert(a.leafPrims.end(), t.leafPrims.begin(), t.leafPrims.end());
        nNodes += t.nNodes;
        parts.push_back({&t, nodeBase, leafBase});
        return shiftRef(t.rootRef, nodeBase, leafBase);
    };
    DeviceBVHResult world;
    // Tiny scenes skip the tree: the whole triangle list is one leaf, staged in shared memory and tested by all lanes
    // in lockstep (no divergence).  Break-even against the BVH2 walk measured on the Cornell scene, see DESIGN.md.
    const uint32_t flatLimit = 64;
    if (!instanced && !ids.empty() && ids.size() <= flatLimit) {
        a.leafPrims = ids;
        a.rootRef = -1; // ~0: leaf starting at triangle 0
        a.depth = 1;
        a.rootCount = (uint32_t) ids.size();
    } else {
        // non-instanced scenes also get the 8-wide compressed tree over the same leaves: that is what the ray-query kernels walk (the binary
        // tree stays for volpath's inline queries)
        if (int rc = buildTree(s, threads, f.boxes[0], ids, instanced ? 19 : B2_STACK_DEPTH - 2, !instanced, world, a)) return rc;
        a.depth = world.depth;
        a.rootRef = place(world, true);
    }
    clk.mark("BVH (world)");
    if (!instanced) { // the world tree's arrays become the scene's (none for the flat leaf)
        s->dNodes.adopt(world.nodes, world.nNodes);
        s->dNodes8.adopt(world.nodes8, world.nNodes8);
        world.nodes = nullptr; world.nodes8 = nullptr;
        CK(ctx, cudaStreamSynchronize(ctx->stream));
        return B2_OK;
    }
    // ---- instancing: one BVH per shapegroup, then a top-level BVH over the items (item 0 = the world triangles, item k = instance k - 1);
    //      stack budget: 9 (top) + 3 (leaf items) + 19 (bottom) < 32 ----
    struct GroupInfo { int rootRef = -1; float lo[3], hi[3]; bool empty = true; };
    std::vector<GroupInfo> gi((size_t) s->nGroups);
    std::vector<std::unique_ptr<DeviceBVHResult>> groups;
    for (int g = 0; g < s->nGroups; ++g) {
        const std::vector<PrimBox> &gb = f.boxes[g + 1];
        if (gb.empty()) continue;
        groups.emplace_back(new DeviceBVHResult());
        DeviceBVHResult &t = *groups.back();
        if (int rc = buildTree(s, threads, gb, f.ids[g + 1], 19, false, t, a)) return rc;
        a.depth = std::max(a.depth, t.depth);
        gi[g].rootRef = place(t, true);
        gi[g].empty = false;
        float l[3] = {INFINITY, INFINITY, INFINITY}, h[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (auto &b : gb) for (int k = 0; k < 3; ++k) { l[k] = std::min(l[k], b.lo[k]); h[k] = std::max(h[k], b.hi[k]); }
        enlargedBox(l, h, gi[g].lo, gi[g].hi); // the group's kd-tree box
    }
    if (a.leafPrims.size() >= (1u << 28)) return fail(ctx, B2_ERR_INVALID, "too many triangles (limit 2^28)");
    std::vector<DInstance> items;
    std::vector<PrimBox> itemBoxes;
    std::vector<uint32_t> itemIds;
    if (!ids.empty()) { // item: the world triangles, identity transform, no clipping
        DInstance it; memset(&it, 0, sizeof(it));
        it.identity = 1; it.rootRef = a.rootRef;
        PrimBox pb; for (int k = 0; k < 3; ++k) { pb.lo[k] = f.lo[k]; pb.hi[k] = f.hi[k]; }
        itemBoxes.push_back(pb); itemIds.push_back((uint32_t) items.size()); items.push_back(it);
    }
    for (size_t k = 0; k < s->instances.size(); ++k) {
        const auto &hi_ = s->instances[k];
        const GroupInfo &g = gi[hi_.group];
        if (g.empty) continue;
        DInstance it; memset(&it, 0, sizeof(it));
        for (int r = 0; r < 12; ++r) { it.M[r] = hi_.M[r]; it.Minv[r] = hi_.Minv[r]; }
        it.rootRef = g.rootRef; it.instance = (int32_t) k;
        memcpy(it.aabbMin, g.lo, 12); memcpy(it.aabbMax, g.hi, 12);
        PrimBox pb; for (int c = 0; c < 3; ++c) { pb.lo[c] = INFINITY; pb.hi[c] = -INFINITY; }
        for (int c = 0; c < 8; ++c) { // Instance::getAABB, instance.cpp:80-96
            const float q[3] = {(c & 1) ? g.hi[0] : g.lo[0], (c & 2) ? g.hi[1] : g.lo[1], (c & 4) ? g.hi[2] : g.lo[2]};
            for (int x = 0; x < 3; ++x) {
                const float w = hi_.M[4 * x] * q[0] + hi_.M[4 * x + 1] * q[1] + hi_.M[4 * x + 2] * q[2] + hi_.M[4 * x + 3];
                pb.lo[x] = std::min(pb.lo[x], w); pb.hi[x] = std::max(pb.hi[x], w);
            }
        }
        for (int x = 0; x < 3; ++x) { a.lo[x] = std::min(a.lo[x], pb.lo[x]); a.hi[x] = std::max(a.hi[x], pb.hi[x]); }
        itemBoxes.push_back(pb); itemIds.push_back((uint32_t) items.size()); items.push_back(it);
    }
    if (items.size() >= (1u << 20)) return fail(ctx, B2_ERR_INVALID, "too many instances (limit 2^20)");
    BVHResult topHost;
    buildBVH(itemBoxes, itemIds, 4, 9, 1, topHost);
    if (topHost.depth > 10) return fail(ctx, B2_ERR_INVALID, "instance hierarchy too deep for the traversal stack");
    a.items.resize(items.size());
    for (size_t k = 0; k < topHost.leafPrims.size(); ++k) a.items[k] = items[topHost.leafPrims[k]];
    DeviceBVHResult top;
    a.uploadBytes += topHost.nodes.size() * sizeof(BVHNode);
    CK(ctx, uploadTree(topHost, ctx->stream, top));
    a.tlasRoot = place(top, false);
    CK(ctx, s->dNodes.alloc(nNodes));
    for (const Part &p : parts) CK(ctx, appendTreeDevice(s->dNodes.p + p.nodeBase, p.tree->nodes, p.tree->nNodes, p.nodeBase, p.leafBase, ctx->stream));
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    s->dNodes8.release();
    return B2_OK;
}
// ---- leaf-ordered triangle rows: the TriAccel records gathered from prim order, and the plane form ----
// Plane form of triangle (a, b, c), evaluated in double: N = e1 x e2, U = (e2 x N)/|N|^2, V = (N x e1)/|N|^2;
// u(p) = U.p + du and v(p) = V.p + dv are the barycentrics of b and c
static void planeRows(const float4 &a, const float4 &b, const float4 &c, float4 *out) {
    const double p0[3] = {a.x, a.y, a.z}, e1[3] = {(double) b.x - a.x, (double) b.y - a.y, (double) b.z - a.z},
                 e2[3] = {(double) c.x - a.x, (double) c.y - a.y, (double) c.z - a.z};
    const double N[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
    const double nn = N[0] * N[0] + N[1] * N[1] + N[2] * N[2];
    const double U[3] = {(e2[1] * N[2] - e2[2] * N[1]) / nn, (e2[2] * N[0] - e2[0] * N[2]) / nn, (e2[0] * N[1] - e2[1] * N[0]) / nn};
    const double V[3] = {(N[1] * e1[2] - N[2] * e1[1]) / nn, (N[2] * e1[0] - N[0] * e1[2]) / nn, (N[0] * e1[1] - N[1] * e1[0]) / nn};
    // scale the t-plane so that |N| ~ 1 (keeps num/den well inside float range)
    const double inv = 1.0 / std::sqrt(nn);
    out[0] = make_float4((float) (N[0] * inv), (float) (N[1] * inv), (float) (N[2] * inv), (float) ((N[0] * p0[0] + N[1] * p0[1] + N[2] * p0[2]) * inv));
    out[1] = make_float4((float) U[0], (float) U[1], (float) U[2], (float) -(U[0] * p0[0] + U[1] * p0[1] + U[2] * p0[2]));
    out[2] = make_float4((float) V[0], (float) V[1], (float) V[2], (float) -(V[0] * p0[0] + V[1] * p0[1] + V[2] * p0[2]));
}
struct LeafRows {
    std::vector<float4> tri, plane; // 3 rows per leaf-ordered triangle
};
static LeafRows leafRows(const std::vector<uint32_t> &leafPrims, const std::vector<float4> &triAccel, const std::vector<float4> &verts, int threads) {
    LeafRows r;
    r.tri.resize(3 * leafPrims.size());
    r.plane.resize(3 * leafPrims.size());
    parallelFor(leafPrims.size(), threads, [&](size_t ilo, size_t ihi) {
        for (size_t i = ilo; i < ihi; ++i) {
            const size_t p = leafPrims[i];
            memcpy(&r.tri[3 * i], &triAccel[3 * p], 48);
            planeRows(verts[3 * p], verts[3 * p + 1], verts[3 * p + 2], &r.plane[3 * i]);
        }
    });
    return r;
}
// ---- flat leaf of the throughput build: coplanar triangle pairs share the plane test ----
// Two triangles with a common edge that lie in one plane are stored as ONE record: a parallelogram (3 rows: the
// lockstep test is 0 <= u,v <= 1 in the frame of the unshared corner) or a general coplanar pair (5 rows: one t and
// hit point, two (u,v) evaluations).  Everything else stays a single triangle.  Order: parallelograms, pairs, singles.
struct FlatLeaf {
    std::vector<float4> rec;
    std::vector<uint32_t> idx;     // 2 per record: leaf index of the first / second triangle
    uint32_t nP = 0, nC = 0, nS = 0; // two-wide steps of parallelograms, coplanar pairs, singles
};
// n = the flat leaf's triangle count (0: no flat leaf), lo / hi = the scene bounds
static FlatLeaf flatLeaf(uint32_t n, const std::vector<uint32_t> &leafPrims, const std::vector<float4> &verts, const std::vector<float4> &leafPlane,
                         const float lo[3], const float hi[3]) {
    FlatLeaf fl;
    if (!n) return fl;
    const double diag = std::sqrt((double) (hi[0] - lo[0]) * (hi[0] - lo[0]) + (double) (hi[1] - lo[1]) * (hi[1] - lo[1]) + (double) (hi[2] - lo[2]) * (hi[2] - lo[2]));
    const double tol = 1e-6 * std::max(diag, 1e-30);
    std::vector<int> mate(n, -1), kind(n, 0), cornerA(n, 0);
    auto V = [&](uint32_t leaf, int k) -> const float4 & { return verts[3 * (size_t) leafPrims[leaf] + k]; };
    auto same = [](const float4 &a, const float4 &b) { return a.x == b.x && a.y == b.y && a.z == b.z; };
    for (uint32_t i = 0; i < n; ++i) {
        if (mate[i] >= 0) continue;
        for (uint32_t j = i + 1; j < n && mate[i] < 0; ++j) {
            if (mate[j] >= 0) continue;
            int sharedA[3] = {0, 0, 0}, sharedB[3] = {0, 0, 0}, ns = 0;
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b)
                    if (!sharedA[a] && !sharedB[b] && same(V(i, a), V(j, b))) { sharedA[a] = sharedB[b] = 1; ++ns; }
            if (ns != 2) continue;
            int ka = !sharedA[0] ? 0 : (!sharedA[1] ? 1 : 2), kb = !sharedB[0] ? 0 : (!sharedB[1] ? 1 : 2);
            const float4 &pa = V(i, ka), &s0 = V(i, (ka + 1) % 3), &s1 = V(i, (ka + 2) % 3), &pb = V(j, kb);
            const double e[3] = {(double) s1.x - s0.x, (double) s1.y - s0.y, (double) s1.z - s0.z};
            const double fa[3] = {(double) pa.x - s0.x, (double) pa.y - s0.y, (double) pa.z - s0.z};
            const double fb[3] = {(double) pb.x - s0.x, (double) pb.y - s0.y, (double) pb.z - s0.z};
            const double na[3] = {e[1] * fa[2] - e[2] * fa[1], e[2] * fa[0] - e[0] * fa[2], e[0] * fa[1] - e[1] * fa[0]};
            const double nb[3] = {e[1] * fb[2] - e[2] * fb[1], e[2] * fb[0] - e[0] * fb[2], e[0] * fb[1] - e[1] * fb[0]};
            const double la = std::sqrt(na[0] * na[0] + na[1] * na[1] + na[2] * na[2]), lb = std::sqrt(nb[0] * nb[0] + nb[1] * nb[1] + nb[2] * nb[2]);
            if (!(la > 0) || !(lb > 0)) continue;
            if (na[0] * nb[0] + na[1] * nb[1] + na[2] * nb[2] >= 0) continue; // both on the same side of the common edge: overlap
            const double dist = (na[0] * fb[0] + na[1] * fb[1] + na[2] * fb[2]) / la; // distance of the 4th corner from the plane
            if (std::fabs(dist) > tol) continue;
            mate[i] = (int) j; mate[j] = (int) i;
            cornerA[i] = ka;
            const double q[3] = {(double) s0.x + s1.x - pa.x, (double) s0.y + s1.y - pa.y, (double) s0.z + s1.z - pa.z};
            const bool para = std::fabs(q[0] - pb.x) <= tol && std::fabs(q[1] - pb.y) <= tol && std::fabs(q[2] - pb.z) <= tol;
            kind[i] = para ? 1 : 2;
        }
    }
    // records per class, each as rows of float4: parallelogram / single = 3 rows (plane, U, V), coplanar pair = 5 rows (plane, U, V, U', V')
    std::vector<std::vector<float4>> recs[3];
    std::vector<std::pair<uint32_t, uint32_t>> recIdx[3];
    for (int pass = 1; pass <= 3; ++pass)
        for (uint32_t i = 0; i < n; ++i) {
            if (pass < 3) {
                if (mate[i] < (int) i || kind[i] != pass) continue; // each pair once, from its lower index
                const uint32_t j = (uint32_t) mate[i];
                std::vector<float4> rows;
                if (pass == 1) {
                    const int ka = cornerA[i];
                    rows.resize(3);
                    planeRows(V(i, ka), V(i, (ka + 1) % 3), V(i, (ka + 2) % 3), rows.data());
                } else {
                    rows.assign(&leafPlane[3 * i], &leafPlane[3 * i] + 3);
                    rows.insert(rows.end(), &leafPlane[3 * j + 1], &leafPlane[3 * j + 1] + 2);
                }
                recs[pass - 1].push_back(rows); recIdx[pass - 1].emplace_back(i, j);
            } else {
                if (mate[i] >= 0) continue;
                recs[2].push_back(std::vector<float4>(&leafPlane[3 * i], &leafPlane[3 * i] + 3));
                recIdx[2].emplace_back(i, i);
            }
        }
    // Two records wide (b2_trace.cuh traverseFlat: one packed FFMA2 evaluates both): row r of records 2j and 2j + 1 becomes the two
    // float4 (x, x', y, y') (z, z', w, w'); an odd count is padded with a plane that is never hit (N = 0, d0 = -1 -> t = -inf)
    for (int c = 0; c < 3; ++c) {
        const size_t rowsPer = c == 1 ? 5 : 3;
        if (recs[c].size() & 1) {
            std::vector<float4> pad(rowsPer, make_float4(0, 0, 0, 0));
            pad[0].w = -1.0f;
            recs[c].push_back(pad); recIdx[c].emplace_back(0u, 0u);
        }
        for (size_t j = 0; j + 1 < recs[c].size(); j += 2)
            for (size_t r = 0; r < rowsPer; ++r) {
                const float4 &a = recs[c][j][r], &b = recs[c][j + 1][r];
                fl.rec.push_back(make_float4(a.x, b.x, a.y, b.y));
                fl.rec.push_back(make_float4(a.z, b.z, a.w, b.w));
            }
        for (auto &ij : recIdx[c]) { fl.idx.push_back(ij.first); fl.idx.push_back(ij.second); }
        (c == 0 ? fl.nP : c == 1 ? fl.nC : fl.nS) = (uint32_t) (recs[c].size() / 2); // packed steps
    }
    return fl;
}
// ---- materials: the device table, the BSDF classes present (s->classPresent) and whether some BSDF transmits (s->hasTransmission) ----
static int uploadMaterials(b2_scene *s) {
    std::vector<DMaterial> dm(s->materials.size());
    for (int c = 0; c < B2_NCLASS; ++c) s->classPresent[c] = false;
    s->hasTransmission = false;
    for (size_t i = 0; i < s->materials.size(); ++i) {
        const b2_material_desc &m = s->materials[i];
        DMaterial &d = dm[i];
        memset(&d, 0, sizeof(d));
        d.type = m.type; d.distr = m.distr; d.sampleVisible = (m.distr == B2_DISTR_PHONG) ? 0 : m.sample_visible; d.nested = m.nested;
        d.alphaU = m.alpha_u; d.alphaV = m.alpha_v; d.eta = m.eta; d.thickness = m.thickness;
        memcpy(d.reflectance, m.reflectance, 12); memcpy(d.transmittance, m.transmittance, 12);
        memcpy(d.etaC, m.eta_c, 12); memcpy(d.kC, m.k_c, 12); memcpy(d.sigmaA, m.sigma_a, 12);
        d.flags = materialFlags(s->materials, (int) i);
        if (d.flags & 0x55u /* ETransmission incl. ENull */) s->hasTransmission = true;
        d.tex = m.reflectance_texture > 0 ? m.reflectance_texture - 1 : -1;
        d.nested2 = m.nested2; d.nonlinear = m.nonlinear; d.fdrInt = m.fdr_int;
        memcpy(d.diffuseReflectance, m.diffuse_reflectance, 12);
        if (m.type == B2_BSDF_PLASTIC) d.specSamplingWeight = m.spec_sampling_weight;
        if (m.type == B2_BSDF_COATING) { // coating.cpp:177-181
            float acc = 0.0f;
            for (int k = 0; k < 3; ++k) acc += (float) std::exp((double) (m.sigma_a[k] * (-2 * m.thickness)));
            float avgAbsorption = acc * (1.0f / 3.0f);
            d.specSamplingWeight = 1.0f / (avgAbsorption + 1.0f);
        }
    }
    for (auto &m : s->meshes) {
        const int t = s->materials[m.material].type;
        if (t >= B2_BSDF_NULL) {
            s->classPresent[B2_NCLASS - 1] = true; // types without a specialised kernel are shaded by the generic one (class queue 4)
            if (t == B2_BSDF_NULL && m.emitter >= 0)
                return fail(s->ctx, B2_ERR_INVALID, "Shape has an index-matched BSDF and an emitter attachment. This is not allowed!"); // shape.cpp:76-78
        } else s->classPresent[t] = true;
    }
    CK(s->ctx, s->dMaterials.upload(dm, s->ctx->stream));
    return B2_OK;
}
// ---- bitmap textures and the environment map: MIP pyramids (host, as the reference builds them at load time) on the device ----
// The device layout of a pyramid: its levels back to back, RGB texels padded to float4 (one 16-byte load per texel); fills d's level table.
static std::vector<float> packPyramid(const b2host::MipPyramid &mip, int channels, DTexture &d) {
    const int stride = channels == 3 ? 4 : 1;
    std::vector<float> packed;
    d.levels = (int) mip.level.size();
    size_t total = 0;
    for (int l = 0; l < d.levels; ++l) total += stride == 1 ? mip.level[l].size() : 4 * (size_t) mip.w[l] * mip.h[l];
    packed.reserve(total);
    for (int l = 0; l < d.levels; ++l) {
        d.lw[l] = mip.w[l]; d.lh[l] = mip.h[l];
        d.off[l] = (uint32_t) (packed.size() / stride);
        const std::vector<float> &src = mip.level[l];
        if (stride == 1) { packed.insert(packed.end(), src.begin(), src.end()); continue; }
        const size_t nTexel = (size_t) d.lw[l] * d.lh[l];
        for (size_t k = 0; k < nTexel; ++k) { packed.push_back(src[3 * k]); packed.push_back(src[3 * k + 1]); packed.push_back(src[3 * k + 2]); packed.push_back(0.0f); }
    }
    return packed;
}
static int uploadTextures(b2_scene *s) {
    b2_ctx *ctx = s->ctx;
    std::vector<DTexture> dtex(s->textures.size());
    s->dTexData.clear();
    for (size_t i = 0; i < s->textures.size(); ++i) {
        b2_scene::HostTexture &ht = s->textures[i];
        const b2_texture_desc &t = ht.desc;
        b2host::buildMipPyramid(ht.pixels.data(), t.width, t.height, t.channels, t.wrap_u, t.wrap_v, t.filter_type >= B2_TEX_TRILINEAR, ht.mip);
        if ((int) ht.mip.level.size() > B2_TEX_MAX_LEVELS) return fail(ctx, B2_ERR_INVALID, "texture has too many MIP levels");
        DTexture &d = dtex[i];
        memset(&d, 0, sizeof(d));
        d.channels = t.channels; d.filter = t.filter_type; d.wrapU = t.wrap_u; d.wrapV = t.wrap_v;
        d.maxAnisotropy = t.max_anisotropy; d.uoffset = t.uoffset; d.voffset = t.voffset; d.uscale = t.uscale; d.vscale = t.vscale;
        d.bsdfScale = ht.mip.maximum > 1.0f ? 0.99f * (1.0f / ht.mip.maximum) : 1.0f; // bsdf.cpp:93-107
        s->dTexData.emplace_back(new DevBuf<float>());
        const std::vector<float> packed = packPyramid(ht.mip, t.channels, d);
        CK(ctx, s->dTexData.back()->upload(packed, ctx->stream));
        d.data = s->dTexData.back()->p;
    }
    CK(ctx, s->dTextures.upload(dtex, ctx->stream));
    return B2_OK;
}
// Environment map: pyramid (half-rounded floats, RGB padded to float4) + the tables of EnvironmentMap::configure (envmap.cpp:260-329).
// Its CDFs have no `sum > 0` guard, unlike the emitter and triangle CDFs: a black row normalises by inf, as in envmap.cpp.
static int uploadEnvmap(b2_scene *s) {
    b2_ctx *ctx = s->ctx;
    b2_scene::HostEnvMap &he = *s->envmap;
    b2host::buildMipPyramid(he.pixels.data(), he.w, he.h, 3, B2_WRAP_REPEAT, B2_WRAP_CLAMP, true, he.mip, std::numeric_limits<float>::infinity());
    if ((int) he.mip.level.size() > B2_TEX_MAX_LEVELS) return fail(ctx, B2_ERR_INVALID, "environment map has too many MIP levels");
    DEnvMap de;
    memset(&de, 0, sizeof(de));
    DTexture &d = de.tex;
    d.channels = 3; d.filter = B2_TEX_EWA; d.wrapU = B2_WRAP_REPEAT; d.wrapV = B2_WRAP_CLAMP;
    d.maxAnisotropy = 10.0f; d.uscale = d.vscale = 1.0f; d.bsdfScale = 1.0f; // envmap.cpp:139-142
    const std::vector<float> packed = packPyramid(he.mip, 3, d);
    const int w = he.w, h = he.h;
    std::vector<float> cdfCols((size_t) (w + 1) * h), cdfRows((size_t) h + 1), rowWeights((size_t) h);
    size_t colPos = 0, rowPos = 0;
    float rowSum = 0.0f;
    const float kPi = 3.14159265358979323846f;
    const std::vector<float> &base = he.mip.level[0];
    cdfRows[rowPos++] = 0;
    for (int y = 0; y < h; ++y) {
        float colSum = 0;
        cdfCols[colPos++] = 0;
        for (int x = 0; x < w; ++x) {
            const float *px = &base[3 * ((size_t) y * w + x)];
            colSum += px[0] * 0.212671f + px[1] * 0.715160f + px[2] * 0.072169f; // spectrum.h:725-727
            cdfCols[colPos++] = colSum;
        }
        const float normalization = 1.0f / colSum;
        for (int x = 1; x < w; ++x) cdfCols[colPos - x - 1] *= normalization;
        cdfCols[colPos - 1] = 1.0f;
        const float weight = std::sin((y + 0.5f) * kPi / h);
        rowWeights[y] = weight;
        rowSum += colSum * weight;
        cdfRows[rowPos++] = rowSum;
    }
    const float normalization = 1.0f / rowSum;
    for (int y = 1; y < h; ++y) cdfRows[rowPos - y - 1] *= normalization;
    cdfRows[rowPos - 1] = 1.0f;
    if (rowSum == 0) return fail(ctx, B2_ERR_INVALID, "The environment map is completely black -- this is not allowed.");
    if (!std::isfinite(rowSum)) return fail(ctx, B2_ERR_INVALID, "The environment map contains an invalid floating point value (nan/inf) -- giving up.");
    de.normalization = 1.0f / (rowSum * (2 * kPi / w) * (kPi / h));
    de.pixelSizeX = 2 * kPi / w; de.pixelSizeY = kPi / h;
    de.scale = he.scale; de.w = w; de.h = h;
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { de.toWorld[3 * r + c] = he.toWorld[4 * r + c]; de.toLocal[3 * r + c] = he.toLocal[4 * r + c]; }
    CK(ctx, s->dEnvTexels.upload(packed, ctx->stream));
    CK(ctx, s->dEnvCdfRows.upload(cdfRows, ctx->stream)); CK(ctx, s->dEnvCdfCols.upload(cdfCols, ctx->stream)); CK(ctx, s->dEnvRowWeights.upload(rowWeights, ctx->stream));
    d.data = s->dEnvTexels.p;
    de.cdfRows = s->dEnvCdfRows.p; de.cdfCols = s->dEnvCdfCols.p; de.rowWeights = s->dEnvRowWeights.p;
    CK(ctx, s->dEnvMap.upload(std::vector<DEnvMap>(1, de), ctx->stream));
    return B2_OK;
}
// ---- media (volpath): the media table and the per-prim (interior, exterior) ids, none when no mesh borders a medium ----
static int uploadMedia(b2_scene *s, size_t nPrims) {
    std::vector<DMedium> dmed(s->media.size());
    s->dDensity.clear();
    for (size_t i = 0; i < s->media.size(); ++i) {
        const b2_medium_desc &m = s->media[i].desc;
        DMedium &d = dmed[i];
        memset(&d, 0, sizeof(d));
        d.type = m.type; d.phase = m.phase; d.g = m.g; d.strategy = m.strategy;
        memcpy(d.sigmaA, m.sigma_a, 12); memcpy(d.sigmaS, m.sigma_s, 12);
        d.samplingDensity = m.sampling_density; d.mediumSamplingWeight = m.medium_sampling_weight;
        d.scale = m.scale; d.invMaxDensity = 1.0f / (m.scale * 1.0f); // heterogeneous.cpp:239-243, gridvolume.cpp:583-585
        memcpy(d.albedo, m.albedo, 12); memcpy(d.res, m.res, 12); memcpy(d.worldToGrid, m.world_to_grid, 48);
        memcpy(d.aabbMin, m.aabb_min, 12); memcpy(d.aabbMax, m.aabb_max, 12);
        s->dDensity.emplace_back(new DevBuf<float>());
        CK(s->ctx, s->dDensity.back()->upload(s->media[i].density, s->ctx->stream));
        d.density = s->dDensity.back()->p;
    }
    std::vector<int2> primMedia;
    bool anyMedia = false;
    for (auto &m : s->meshes) anyMedia |= m.interior >= 0 || m.exterior >= 0;
    if (anyMedia) {
        primMedia.resize(nPrims);
        for (auto &m : s->meshes)
            for (size_t j = 0; j < m.idx.size() / 3; ++j) primMedia[m.primOffset + j] = make_int2(m.interior, m.exterior);
    }
    CK(s->ctx, s->dMedia.upload(dmed, s->ctx->stream));
    CK(s->ctx, s->dPrimMedia.upload(primMedia, s->ctx->stream));
    return B2_OK;
}
// ---- emitters in device order, their CDF and the triangle CDF of each area emitter: scene.cpp:375-380, trimesh.cpp:388-403, pmf.h.
// emNorm = DiscreteDistribution::getNormalization of the emitter CDF ----
static int uploadEmitters(b2_scene *s, const std::vector<int> &emOrder, float &emNorm) {
    std::vector<DEmitter> de(s->emitters.size());
    std::vector<float> emCdf(1, 0.0f), triCdf;
    emNorm = 0.0f;
    for (size_t e = 0; e < s->emitters.size(); ++e) {
        const HostEmitter &he = s->emitters[emOrder[e]];
        DEmitter &d = de[e];
        memcpy(d.radiance, he.radiance, 12);
        d.samplingWeight = he.samplingWeight;
        if (he.env) { // constant.cpp: no mesh, no area distribution
            d.cdfOffset = 0; d.nTri = 0; d.primOffset = 0; d.invSurfaceArea = 0;
            emCdf.push_back(emCdf.back() + he.samplingWeight);
            continue;
        }
        const HostMesh &m = s->meshes[he.mesh];
        d.cdfOffset = (uint32_t) triCdf.size();
        d.nTri = (uint32_t) (m.idx.size() / 3);
        d.primOffset = m.primOffset;
        size_t base = triCdf.size();
        triCdf.push_back(0.0f);
        for (uint32_t j = 0; j < d.nTri; ++j) {
            const float *p0 = &m.P[3 * m.idx[3 * j]], *p1 = &m.P[3 * m.idx[3 * j + 1]], *p2 = &m.P[3 * m.idx[3 * j + 2]];
            H3 n = cross3(sub3(p1, p0), sub3(p2, p0));
            float area = 0.5f * std::sqrt(n.x * n.x + n.y * n.y + n.z * n.z); // triangle.cpp:64-70
            triCdf.push_back(triCdf.back() + area);
        }
        float sum = triCdf.back();
        if (sum > 0) {
            float normalization = 1.0f / sum;
            for (size_t k = base + 1; k < triCdf.size(); ++k) triCdf[k] *= normalization;
            triCdf.back() = 1.0f;
        }
        d.invSurfaceArea = 1.0f / sum;
        emCdf.push_back(emCdf.back() + he.samplingWeight);
    }
    if (!s->emitters.empty()) {
        float sum = emCdf.back();
        if (sum > 0) {
            emNorm = 1.0f / sum;
            for (size_t k = 1; k < emCdf.size(); ++k) emCdf[k] *= emNorm;
            emCdf.back() = 1.0f;
        }
    }
    CK(s->ctx, s->dEmitters.upload(de, s->ctx->stream));
    CK(s->ctx, s->dEmitterCdf.upload(emCdf, s->ctx->stream));
    CK(s->ctx, s->dTriCdf.upload(triCdf, s->ctx->stream));
    return B2_OK;
}
// ---- camera ----
static void fillCamera(const b2_scene *s, DCamera &cam) {
    memcpy(cam.camToWorld, s->camToWorld, 64);
    memcpy(cam.sampleToCamera, s->sampleToCamera, 64);
    cam.nearClip = s->nearClip; cam.farClip = s->farClip;
    cam.invResX = 1.0f / (float) s->W; cam.invResY = 1.0f / (float) s->H; // sensor.cpp:104-107
    cam.origin[0] = s->camToWorld[3]; cam.origin[1] = s->camToWorld[7]; cam.origin[2] = s->camToWorld[11];
    cam.W = s->W; cam.H = s->H;
    cam.apertureRadius = s->apertureRadius; cam.focusDistance = s->focusDistance;
    // m_dx, m_dy (perspective.cpp:160-163): sampleToCamera(Point(invRes.x, 0, 0)) - sampleToCamera(Point(0)), likewise y
    auto s2c = [&](float px, float py, float out[3]) { // Transform::operator()(Point), transform.h:108-125
        const float *M = s->sampleToCamera;
        const float x = M[0] * px + M[1] * py + M[2] * 0.0f + M[3], y = M[4] * px + M[5] * py + M[6] * 0.0f + M[7],
                    z = M[8] * px + M[9] * py + M[10] * 0.0f + M[11], w = M[12] * px + M[13] * py + M[14] * 0.0f + M[15];
        if (w != 1.0f) { const float r = 1.0f / w; out[0] = x * r; out[1] = y * r; out[2] = z * r; }
        else { out[0] = x; out[1] = y; out[2] = z; }
    };
    float z0[3], ax[3], ay[3];
    s2c(0.0f, 0.0f, z0); s2c(cam.invResX, 0.0f, ax); s2c(0.0f, cam.invResY, ay);
    for (int k = 0; k < 3; ++k) { cam.dx[k] = ax[k] - z0[k]; cam.dy[k] = ay[k] - z0[k]; }
}
// ---- the device scene: the remaining uploads, DScene over the scene's device arrays, launch configurations, b2_stats ----
static int assembleScene(b2_scene *s, const Flat &f, const Accel &a, const LeafRows &rows, const FlatLeaf &fl, const std::vector<int> &emIndex, float emNorm) {
    b2_ctx *ctx = s->ctx;
    CK(ctx, s->dTriAccel.upload(rows.tri, ctx->stream));
    CK(ctx, s->dTriPlane.upload(rows.plane, ctx->stream));
    CK(ctx, s->dLeafPrim.upload(a.leafPrims, ctx->stream));
    CK(ctx, s->dFlatRec.upload(fl.rec, ctx->stream));
    CK(ctx, s->dFlatIdx.upload(fl.idx, ctx->stream));
    CK(ctx, s->dVerts.upload(f.verts, ctx->stream));
    CK(ctx, s->dNorms.upload(f.norms, ctx->stream));
    CK(ctx, s->dTexc.upload(f.texc, ctx->stream));
    CK(ctx, s->dInstances.upload(a.items, ctx->stream));
    const size_t nPrims = f.nPrims, nNodes = s->dNodes.n, nNodes8 = s->dNodes8.n;
    DScene &ds = s->ds;
    memset(&ds, 0, sizeof(ds));
    ds.triAccel = s->dTriAccel.p; ds.triPlane = s->dTriPlane.p; ds.leafPrim = s->dLeafPrim.p; ds.nLeafTris = (uint32_t) a.leafPrims.size();
    // environment emitter: index + constant.cpp:67-70 bounding sphere of (acceleration-structure box U sensor position) (scene.cpp:386-399)
    ds.envEmitter = -1;
    ds.envmap = s->envmap ? s->dEnvMap.p : nullptr;
    for (size_t e = 0; e < s->emitters.size(); ++e) if (s->emitters[e].env) ds.envEmitter = emIndex[e];
    {
        float l[3], h[3], mn[3], mx[3], bl[3], bh[3];
        for (int k = 0; k < 3; ++k) { l[k] = nPrims ? a.lo[k] : 0.0f; h[k] = nPrims ? a.hi[k] : 0.0f; }
        enlargedBox(l, h, mn, mx);
        for (int k = 0; k < 3; ++k) {
            const float camP = s->camToWorld[4 * k + 3];
            bl[k] = std::min(mn[k], camP); bh[k] = std::max(mx[k], camP);
        }
        float c[3];
        for (int k = 0; k < 3; ++k) { c[k] = (bh[k] + bl[k]) * 0.5f; ds.bsCenter[k] = c[k]; }
        const float dx = c[0] - bh[0], dy = c[1] - bh[1], dz = c[2] - bh[2];
        ds.bsRadius = std::max(1e-4f, std::sqrt(dx * dx + dy * dy + dz * dz) * 1.5f);
    }
    ds.items = s->dInstances.p; ds.nItems = (uint32_t) a.items.size(); ds.tlasRoot = a.tlasRoot;
    ds.media = s->dMedia.p; ds.primMedia = s->dPrimMedia.p; ds.nMedia = (uint32_t) s->dMedia.n;
    ds.nodes8 = nNodes8 ? s->dNodes8.p : nullptr; ds.nNodes8 = (uint32_t) nNodes8;
    ds.nodes = s->dNodes.p; ds.nNodes = (uint32_t) nNodes; ds.rootRef = a.rootRef; ds.rootCount = a.rootCount;
    ds.flatRec = s->dFlatRec.p; ds.flatIdx = (const uint2 *) s->dFlatIdx.p; ds.flatP = fl.nP; ds.flatC = fl.nC; ds.flatS = fl.nS;
    ds.flatBytes = (uint32_t) (fl.rec.size() * 16);
    {   // enlarged scene box
        float l[3] = {a.lo[0], a.lo[1], a.lo[2]}, h[3] = {a.hi[0], a.hi[1], a.hi[2]};
        if (nPrims == 0 || !(l[0] <= h[0])) for (int k = 0; k < 3; ++k) { l[k] = 0; h[k] = 0; }
        enlargedBox(l, h, ds.aabbMin, ds.aabbMax);
    }
    ds.verts = s->dVerts.p; ds.norms = s->dNorms.p; ds.nPrims = (uint32_t) nPrims;
    ds.materials = s->dMaterials.p; ds.nMaterials = (uint32_t) s->dMaterials.n;
    ds.textures = s->dTextures.p; ds.nTextures = (uint32_t) s->dTextures.n; ds.texc = s->dTexc.p; ds.ewaLut = s->dEwaLut.p;
    ds.emitters = s->dEmitters.p; ds.nEmitters = (uint32_t) s->dEmitters.n;
    ds.emitterCdf = s->dEmitterCdf.p; ds.emitterNormalization = emNorm; ds.triCdf = s->dTriCdf.p;
    fillCamera(s, ds.cam);
    ds.sobolM32 = ctx->dM32; ds.sobolVdc = ctx->dVdc; ds.sobolInv = ctx->dInv; ds.sobolNib = ctx->dNib;
    // shared-memory staging budget: up to 256 nodes (16 KB) and 256 triangles (12 KB) per CTA
    ds.stageNodes = std::min<uint32_t>(ds.nNodes, 256u);
    ds.stageNodes8 = std::min<uint32_t>(ds.nNodes8, 192u); // 15 KB: the root, its children and most of the third level
    ds.stageTris = a.rootCount; // a BVH's leaf-ordered head is arbitrary: only the flat leaf is worth staging
    ds.stageTriBytes = std::max(ds.stageTris * 48u, (ds.flatBytes + 15u) & ~15u);
    ds.refill = 16; // measured sweep 8..32 on the material-ball and 1M-triangle scenes (DESIGN.md)
    ds.leafVote = 8;
    // rays that leave the scene are binned into the first BSDF class that has a shading kernel launched for it (a scene without a
    // diffuse mesh launches no class-0 kernel: its escaped paths must still be retired)
    ds.missClass = 0;
    for (int c = B2_NCLASS - 1; c >= 0; --c)
        if (s->classPresent[c]) ds.missClass = (uint32_t) c;
    for (bool ieee : {true, false}) {
        const Kernels kn = kernelsFor(s, ieee);
        kn.set.init(kn.cfg, ds, ctx->numSMs);
    }
    CK(ctx, cudaGetLastError());
    CK(ctx, s->dCounters.alloc(CTR_COUNT));
    memset(&s->stats, 0, sizeof(s->stats));
    s->stats.n_triangles = nPrims;
    s->stats.n_bvh_nodes = nNodes8 ? nNodes8 : nNodes;
    s->stats.bvh_node_bytes = nNodes8 ? sizeof(BVH8Node) : sizeof(BVHNode);
    s->stats.accel_build_ms = (float) a.ms;
    s->stats.accel_build_mode = s->accelBuild;
    s->stats.bytes_uploaded = rows.tri.size() * 16 + rows.plane.size() * 16 + a.leafPrims.size() * 4 + f.verts.size() * 16 + f.norms.size() * 16 +
                              a.uploadBytes + s->dMaterials.n * sizeof(DMaterial) + s->dEmitters.n * sizeof(DEmitter) + (s->dEmitterCdf.n + s->dTriCdf.n) * 4;
    return B2_OK;
}
extern "C" int b2_scene_commit(b2_scene *s) {
    if (!s) return fail(nullptr, B2_ERR_INVALID, "b2_scene_commit: null scene");
    b2_ctx *ctx = s->ctx;
    if (!s->hasCamera) return fail(ctx, B2_ERR_INVALID, "scene has no sensor");
    CK(ctx, cudaSetDevice(ctx->device));
    CommitClock clk;
    for (size_t e = 0; e < s->emitters.size(); ++e)
        if (s->emitters[e].mesh < 0 && !s->emitters[e].env) return fail(ctx, B2_ERR_INVALID, "area emitter without a parent shape");
    const int threads = usableThreads();
    const EmitterOrder emo = emitterOrder(s);
    Flat flat;
    if (int rc = flattenMeshes(s, emo.index, threads, flat)) return rc;
    clk.mark("flatten + TriAccel");
    Accel acc;
    if (int rc = buildAccel(s, threads, flat, clk, acc)) return rc;
    const LeafRows rows = leafRows(acc.leafPrims, s->hTriAccelPrimOrder, flat.verts, threads);
    clk.mark("instancing / leaf order");
    const FlatLeaf fl = flatLeaf(acc.rootCount, acc.leafPrims, flat.verts, rows.plane, acc.lo, acc.hi);
    if (getenv("B2_VERBOSE"))
        fprintf(stderr, "[b2mts] commit: %zu triangles, flat leaf %u (two-wide steps: parallelograms %u, coplanar pairs %u, singles %u), bvh nodes %zu depth %d\n",
                flat.nPrims, acc.rootCount, fl.nP, fl.nC, fl.nS, s->dNodes.n, acc.depth);
    clk.mark("leaf records");
    if (int rc = uploadMaterials(s)) return rc;
    if (int rc = uploadTextures(s)) return rc;
    if (s->envmap)
        if (int rc = uploadEnvmap(s)) return rc;
    if (!s->textures.empty() || s->envmap) {
        std::vector<float> lut(64);
        b2host::ewaWeightTable(lut.data());
        CK(ctx, s->dEwaLut.upload(lut, ctx->stream));
    }
    if (int rc = uploadMedia(s, flat.nPrims)) return rc;
    clk.mark("materials / textures / media");
    float emNorm;
    if (int rc = uploadEmitters(s, emo.order, emNorm)) return rc;
    clk.mark("emitters");
    if (int rc = assembleScene(s, flat, acc, rows, fl, emo.index, emNorm)) return rc;
    CK(ctx, cudaStreamSynchronize(ctx->stream)); // the uploads of the stages above
    clk.mark("upload");
    s->committed = true;
    return B2_OK;
}
