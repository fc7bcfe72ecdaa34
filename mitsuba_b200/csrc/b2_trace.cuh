// Ray queries on the device: ShapeKDTree::rayIntersect semantics (src/librender/skdtree.cpp:112-226:
// scene-box clip, adaptive epsilon, closest / any hit) over a BVH2 instead of the SAH kd-tree, with the
// reference's TriAccel test (include/mitsuba/render/triaccel.h:96-158) as the only arithmetic that
// decides a hit.  The returned (t,u,v,prim) is argmin_t over TriAccel tests -- identical to what the
// Havran kd-tree traversal (sahkdtree3.h:178-308) returns, except for exact-t ties.
//
// Per-lane traversal stack lives in shared memory (interleaved: entry k of thread i at
// stack[k * blockDim + i], conflict free); the leading part of the node / triangle arrays is staged
// into shared memory by a TMA bulk copy (see b2_kernels.inl: stageScene).
#pragma once
#include "b2_math.cuh"
#include "b2_types.h"

namespace b2 {


struct TraceMem {
    const float4 *gNodes8;  // wide tree: global, 5 x float4 per node; sNodes8: shared copy of the first stageNodes8 nodes
    const float4 *sNodes8;
    uint32_t stageNodes8;
    uint2 *stack8;          // this thread's column of the shared stack of the wide traversal (B2_STACK8_DEPTH entries)
    const float4 *gNodes;   // global: 4 x float4 per node
    const float4 *gTris;    // global: 3 x float4 per leaf-ordered triangle
    const float4 *sNodes;   // shared copies of the first stageNodes / stageTris records
    const float4 *sTris;
    uint32_t stageNodes, stageTris;
    uint32_t *stack;        // this thread's column of the shared stack
    uint32_t stride;        // blockDim.x
};

struct HitRec {
    float t, u, v;
    uint32_t prim;
    uint32_t leaf;   // leaf-ordered index of the triangle (into triAccel / triPlane); valid when prim is
};

// (t, u, v, prim) of a miss (leaf is not set)
B2_DEV HitRec missHit() {
    HitRec h;
    h.t = B2_INF; h.u = 0; h.v = 0; h.prim = 0xFFFFFFFFu;
    return h;
}
// the pool's hit record (DPool::hit): (t, u, v, prim)
B2_DEV float4 packHit(const HitRec &h) { return make_float4(h.t, h.u, h.v, __uint_as_float(h.prim)); }
B2_DEV HitRec unpackHit(const float4 &r) {
    HitRec h;
    h.t = r.x; h.u = r.y; h.v = r.z; h.prim = __float_as_uint(r.w);
    return h;
}

// triaccel.h:96-158
B2_DEV bool triAccelIntersect(const float4 &q0, const float4 &q1, const float4 &q2, const V3 &o, const V3 &d, float mint,
                              float maxt, float &u, float &v, float &t) {
    const uint32_t k = __float_as_uint(q0.x);
    float o_u, o_v, o_k, d_u, d_v, d_k;
    if (k == 0) { o_u = o.y; o_v = o.z; o_k = o.x; d_u = d.y; d_v = d.z; d_k = d.x; }
    else if (k == 1) { o_u = o.z; o_v = o.x; o_k = o.y; d_u = d.z; d_v = d.x; d_k = d.y; }
    else if (k == 2) { o_u = o.x; o_v = o.y; o_k = o.z; d_u = d.x; d_v = d.y; d_k = d.z; }
    else return false;
    const float n_u = q0.y, n_v = q0.z, n_d = q0.w;
    t = (n_d - o_u * n_u - o_v * n_v - o_k) / (d_u * n_u + d_v * n_v + d_k);
    if (t < mint || t > maxt) return false;
    const float hu = o_u + t * d_u - q1.x;
    const float hv = o_v + t * d_v - q1.y;
    u = hv * q1.z + hu * q1.w;
    v = hu * q2.x + hv * q2.y;
    return u >= 0 && v >= 0 && u + v <= 1.0f;
}

// Throughput build: the same triangle as three planes; branch free, no component permutation, reciprocal instead of an
// IEEE division.  t, u, v agree with the TriAccel arithmetic to a few ulp (DESIGN.md "fast build").
B2_DEV bool triPlaneIntersect(const float4 &q0, const float4 &q1, const float4 &q2, const V3 &o, const V3 &d, float mint, float maxt,
                              float &u, float &v, float &t) {
    const float den = q0.x * d.x + q0.y * d.y + q0.z * d.z;
    const float num = q0.w - (q0.x * o.x + q0.y * o.y + q0.z * o.z);
    t = __fdividef(num, den);
    const float px = o.x + t * d.x, py = o.y + t * d.y, pz = o.z + t * d.z;
    u = q1.x * px + q1.y * py + q1.z * pz + q1.w;
    v = q2.x * px + q2.y * py + q2.z * pz + q2.w;
    return (t >= mint) & (t <= maxt) & (u >= 0.0f) & (v >= 0.0f) & (u + v <= 1.0f);
}

#ifdef B2_FAST_TRI
#define B2_TRI_TEST triPlaneIntersect
#else
#define B2_TRI_TEST triAccelIntersect
#endif

// include/mitsuba/core/aabb.h:308-338
B2_DEV bool aabbRayIntersect(const float *bmin, const float *bmax, const V3 &o, const V3 &d, const V3 &dRcp, float &nearT, float &farT) {
    nearT = -B2_INF; farT = B2_INF;
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const float origin = comp(o, i), minVal = bmin[i], maxVal = bmax[i];
        const float di = comp(d, i);
        if (di == 0) {
            if (origin < minVal || origin > maxVal) return false;
        } else {
            float t1 = (minVal - origin) * comp(dRcp, i);
            float t2 = (maxVal - origin) * comp(dRcp, i);
            if (t1 > t2) { float tmp = t1; t1 = t2; t2 = tmp; }
            nearT = fmaxf(t1, nearT);
            farT = fminf(t2, farT);
            if (!(nearT <= farT)) return false;
        }
    }
    return true;
}

// skdtree.cpp:124-133 (closest) / :211-218 (occlusion): clip to the scene box and apply the adaptive epsilon
template <bool SHADOW> B2_DEV bool clipRay(const DScene &sc, const V3 &o, const V3 &d, float rayMint, float rayMaxt, float &mint, float &maxt) {
    const V3 dRcp(1.0f / d.x, 1.0f / d.y, 1.0f / d.z); // ray.h:83-84
    if (!aabbRayIntersect(sc.aabbMin, sc.aabbMax, o, d, dRcp, mint, maxt)) return false;
    float rayMinT = rayMint;
    if (rayMinT == B2_EPSILON) {
        float m = fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fabsf(o.z));
        if (!SHADOW) m = fmaxf(m, B2_EPSILON);
        rayMinT *= m;
    }
    if (rayMinT > mint) mint = rayMinT;
    if (rayMaxt < maxt) maxt = rayMaxt;
    return maxt > mint;
}

B2_DEV void slabSetup(const V3 &o, const V3 &d, V3 &idir, V3 &ood) {
    const float tiny = 1e-20f;
    const float dx = fabsf(d.x) > tiny ? d.x : copysignf(tiny, d.x), dy = fabsf(d.y) > tiny ? d.y : copysignf(tiny, d.y),
                dz = fabsf(d.z) > tiny ? d.z : copysignf(tiny, d.z);
    idir = V3(1.0f / dx, 1.0f / dy, 1.0f / dz);
    ood = V3(o.x * idir.x, o.y * idir.y, o.z * idir.z);
}

// slab test against one child box; conservative (boxes are padded at build time, far side scaled by 1+2ulp)
B2_DEV bool boxHit(float bx0, float by0, float bz0, float bx1, float by1, float bz1, const V3 &ood, const V3 &idir, float mint, float maxt,
                   float &tEntry) {
    // (b - o) * idir evaluated as b * idir - o * idir: one FMA per plane (boxes are padded, the test stays conservative)
    float tx0 = fmaf(bx0, idir.x, -ood.x), tx1 = fmaf(bx1, idir.x, -ood.x);
    float ty0 = fmaf(by0, idir.y, -ood.y), ty1 = fmaf(by1, idir.y, -ood.y);
    float tz0 = fmaf(bz0, idir.z, -ood.z), tz1 = fmaf(bz1, idir.z, -ood.z);
    float tmin = fmaxf(fmaxf(fminf(tx0, tx1), fminf(ty0, ty1)), fmaxf(fminf(tz0, tz1), mint));
    float tmax = fminf(fminf(fmaxf(tx0, tx1), fmaxf(ty0, ty1)), fminf(fmaxf(tz0, tz1), maxt));
    tEntry = tmin;
    return tmin <= tmax * 1.0000003f;
}

// Tiny scenes (DScene::rootCount > 0): every lane tests the whole shared-memory resident triangle list in lockstep.
#ifdef B2_FAST_TRI
// Throughput build: the list holds paired records (b2_host.cpp "flat leaf of the throughput build"): a coplanar pair of
// triangles costs one plane test + one hit point; a parallelogram additionally shares (u, v).
//
// The leaf is stored TWO RECORDS WIDE: element k of record 2j sits next to element k of record 2j + 1, so one float4 load
// feeds the same step of two records and the two independent FMA chains interleave (the loop is FP32-issue bound).  Odd
// counts are padded with a record that can never be hit (N = 0, d0 = -1: t = -inf).  Hopper has no packed FP32 arithmetic:
// each pair operation is two scalar round-to-nearest, flush-to-zero instructions (the same rounding element by element as
// a packed f32x2 instruction would give).
struct F2 { float x, y; };
B2_DEV float fmaFtz(float a, float b, float c) { float r; asm("fma.rn.ftz.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c)); return r; }
B2_DEV float mulFtz(float a, float b) { float r; asm("mul.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
B2_DEV float subFtz(float a, float b) { float r; asm("sub.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
B2_DEV F2 fma2(const F2 &a, const F2 &b, const F2 &c) { F2 r; r.x = fmaFtz(a.x, b.x, c.x); r.y = fmaFtz(a.y, b.y, c.y); return r; }
B2_DEV F2 mul2(const F2 &a, const F2 &b) { F2 r; r.x = mulFtz(a.x, b.x); r.y = mulFtz(a.y, b.y); return r; }
B2_DEV F2 sub2(const F2 &a, const F2 &b) { F2 r; r.x = subFtz(a.x, b.x); r.y = subFtz(a.y, b.y); return r; }
B2_DEV F2 lo2(const float4 &v) { F2 r; r.x = v.x; r.y = v.y; return r; }
B2_DEV F2 hi2(const float4 &v) { F2 r; r.x = v.z; r.y = v.w; return r; }
B2_DEV F2 dup2(float v) { F2 r; r.x = v; r.y = v; return r; }

struct FlatRay2 { F2 ox, oy, oz, dx, dy, dz; };
// plane test of two records: rows r0 = (Nx, Nx', Ny, Ny'), r1 = (Nz, Nz', d0, d0') -> t of both, hit point of both
B2_DEV void flatPlane2(const FlatRay2 &r, const float4 &r0, const float4 &r1, F2 &t, F2 &px, F2 &py, F2 &pz) {
    F2 den = mul2(lo2(r0), r.dx); den = fma2(hi2(r0), r.dy, den); den = fma2(lo2(r1), r.dz, den);
    F2 nd = mul2(lo2(r0), r.ox); nd = fma2(hi2(r0), r.oy, nd); nd = fma2(lo2(r1), r.oz, nd);
    const F2 num = sub2(hi2(r1), nd);
    t.x = __fdividef(num.x, den.x); t.y = __fdividef(num.y, den.y);
    px = fma2(t, r.dx, r.ox); py = fma2(t, r.dy, r.oy); pz = fma2(t, r.dz, r.oz);
}
// one barycentric of two records: rows a = (Ux, Ux', Uy, Uy'), b = (Uz, Uz', du, du')
B2_DEV F2 flatCoord2(const float4 &a, const float4 &b, const F2 &px, const F2 &py, const F2 &pz) {
    F2 u = fma2(lo2(a), px, hi2(b)); u = fma2(hi2(a), py, u); u = fma2(lo2(b), pz, u);
    return u;
}

template <bool SHADOW, bool COUNT> B2_DEV bool traverseFlat(const DScene &sc, const TraceMem &tm, const V3 &o, const V3 &d, float mint, float maxt,
                                                             HitRec &hit, uint32_t &primTests) {
    // record numbering (index into flatIdx): parallelograms [0, 2 nP2), coplanar pairs [2 nP2, 2 nP2 + 2 nC2), singles behind them
    const uint32_t nP2 = sc.flatP, nC2 = sc.flatC, nS2 = sc.flatS; // packed steps (two records each)
    int best = -1;
    bool second = false;
    FlatRay2 r;
    r.ox = dup2(o.x); r.oy = dup2(o.y); r.oz = dup2(o.z); r.dx = dup2(d.x); r.dy = dup2(d.y); r.dz = dup2(d.z);
    const float4 *p = tm.sTris;
#pragma unroll 2
    for (uint32_t i = 0; i < nP2; ++i, p += 6) {
        F2 t, px, py, pz;
        flatPlane2(r, p[0], p[1], t, px, py, pz);
        const F2 u = flatCoord2(p[2], p[3], px, py, pz), v = flatCoord2(p[4], p[5], px, py, pz);
        if ((t.x >= mint) & (t.x <= maxt) & (u.x >= 0.0f) & (v.x >= 0.0f) & (u.x <= 1.0f) & (v.x <= 1.0f)) {
            if (SHADOW) return true;
            hit.t = t.x; hit.u = u.x; hit.v = v.x; best = (int) (2 * i);
            maxt = t.x;
        }
        if ((t.y >= mint) & (t.y <= maxt) & (u.y >= 0.0f) & (v.y >= 0.0f) & (u.y <= 1.0f) & (v.y <= 1.0f)) {
            if (SHADOW) return true;
            hit.t = t.y; hit.u = u.y; hit.v = v.y; best = (int) (2 * i + 1);
            maxt = t.y;
        }
    }
    for (uint32_t i = 0; i < nC2; ++i, p += 10) {
        F2 t, px, py, pz;
        flatPlane2(r, p[0], p[1], t, px, py, pz);
        const F2 uA = flatCoord2(p[2], p[3], px, py, pz), vA = flatCoord2(p[4], p[5], px, py, pz);
        const F2 uB = flatCoord2(p[6], p[7], px, py, pz), vB = flatCoord2(p[8], p[9], px, py, pz);
        {
            const bool hA = (uA.x >= 0.0f) & (vA.x >= 0.0f) & (uA.x + vA.x <= 1.0f), hB = (uB.x >= 0.0f) & (vB.x >= 0.0f) & (uB.x + vB.x <= 1.0f);
            if ((t.x >= mint) & (t.x <= maxt) & (hA | hB)) {
                if (SHADOW) return true;
                hit.t = t.x; hit.u = hB ? uB.x : uA.x; hit.v = hB ? vB.x : vA.x; best = (int) (2 * (nP2 + i)); second = hB;
                maxt = t.x;
            }
        }
        {
            const bool hA = (uA.y >= 0.0f) & (vA.y >= 0.0f) & (uA.y + vA.y <= 1.0f), hB = (uB.y >= 0.0f) & (vB.y >= 0.0f) & (uB.y + vB.y <= 1.0f);
            if ((t.y >= mint) & (t.y <= maxt) & (hA | hB)) {
                if (SHADOW) return true;
                hit.t = t.y; hit.u = hB ? uB.y : uA.y; hit.v = hB ? vB.y : vA.y; best = (int) (2 * (nP2 + i) + 1); second = hB;
                maxt = t.y;
            }
        }
    }
    for (uint32_t i = 0; i < nS2; ++i, p += 6) {
        F2 t, px, py, pz;
        flatPlane2(r, p[0], p[1], t, px, py, pz);
        const F2 u = flatCoord2(p[2], p[3], px, py, pz), v = flatCoord2(p[4], p[5], px, py, pz);
        if ((t.x >= mint) & (t.x <= maxt) & (u.x >= 0.0f) & (v.x >= 0.0f) & (u.x + v.x <= 1.0f)) {
            if (SHADOW) return true;
            hit.t = t.x; hit.u = u.x; hit.v = v.x; best = (int) (2 * (nP2 + nC2 + i)); second = false;
            maxt = t.x;
        }
        if ((t.y >= mint) & (t.y <= maxt) & (u.y >= 0.0f) & (v.y >= 0.0f) & (u.y + v.y <= 1.0f)) {
            if (SHADOW) return true;
            hit.t = t.y; hit.u = u.y; hit.v = v.y; best = (int) (2 * (nP2 + nC2 + i) + 1); second = false;
            maxt = t.y;
        }
    }
    if (COUNT) primTests += sc.rootCount;
    if (best < 0) return false;
    const uint2 id = __ldg(sc.flatIdx + best);
    uint32_t leaf = id.x;
    if ((uint32_t) best < 2 * nP2) {
        // the record's frame starts at the unshared corner of the first triangle: pick the half, then evaluate that
        // triangle's own barycentrics at the hit point
        if (hit.u + hit.v > 1.0f) leaf = id.y;
        const float4 r1 = __ldg(sc.triPlane + 3 * leaf + 1), r2 = __ldg(sc.triPlane + 3 * leaf + 2);
        const float px = o.x + hit.t * d.x, py = o.y + hit.t * d.y, pz = o.z + hit.t * d.z;
        hit.u = r1.x * px + r1.y * py + r1.z * pz + r1.w;
        hit.v = r2.x * px + r2.y * py + r2.z * pz + r2.w;
    } else if (second) leaf = id.y;
    hit.leaf = leaf;
    hit.prim = __ldg(sc.leafPrim + leaf);
    return true;
}
#else
template <bool SHADOW, bool COUNT> B2_DEV bool traverseFlat(const DScene &sc, const TraceMem &tm, const V3 &o, const V3 &d, float mint, float maxt,
                                                             HitRec &hit, uint32_t &primTests) {
    const uint32_t n = sc.rootCount;
    bool found = false;
    uint32_t best = 0;
    const float4 *p = tm.sTris;
#pragma unroll 4
    for (uint32_t i = 0; i < n; ++i, p += 3) {
        const float4 q0 = p[0], q1 = p[1], q2 = p[2];
        float tu, tv, tt;
        if (B2_TRI_TEST(q0, q1, q2, o, d, mint, maxt, tu, tv, tt)) {
            if (SHADOW) return true;
            hit.t = tt; hit.u = tu; hit.v = tv; best = i;
            maxt = tt;
            found = true;
        }
    }
    if (COUNT) primTests += n;
    if (found) { hit.leaf = best; hit.prim = __ldg(sc.leafPrim + best); }
    return found;
}
#endif

// Returns true if something was hit.  Closest: fills `hit`; SHADOW: returns at the first hit.
template <bool SHADOW, bool COUNT> B2_DEV bool traverse(const DScene &sc, const TraceMem &tm, const V3 &o, const V3 &d, float mint, float maxt,
                                                         HitRec &hit, uint32_t &nodeVisits, uint32_t &primTests) {
    if (sc.rootCount) return traverseFlat<SHADOW, COUNT>(sc, tm, o, d, mint, maxt, hit, primTests);
    // reciprocal for the slab test only; |d| below 1e-20 is clamped so o * idir stays finite (conservative: boxes are padded)
    V3 idir, ood;
    slabSetup(o, d, idir, ood);
    bool found = false;
    uint32_t best = 0xFFFFFFFFu;
    int sp = 0;
    int ref = sc.rootRef;
    const uint32_t stride = tm.stride;
    while (true) {
        if (ref >= 0) {
            float4 a, b, c, e;
            if ((uint32_t) ref < tm.stageNodes) {
                const float4 *p = tm.sNodes + 4 * ref;
                a = p[0]; b = p[1]; c = p[2]; e = p[3];
            } else {
                const float4 *p = tm.gNodes + 4 * (size_t) ref;
                a = __ldg(p); b = __ldg(p + 1); c = __ldg(p + 2); e = __ldg(p + 3);
            }
            if (COUNT) ++nodeVisits;
            float tL, tR;
            bool hL = boxHit(a.x, a.y, a.z, a.w, b.x, b.y, ood, idir, mint, maxt, tL);
            bool hR = boxHit(b.z, b.w, c.x, c.y, c.z, c.w, ood, idir, mint, maxt, tR);
            int lref = __float_as_int(e.x), rref = __float_as_int(e.y);
            if (hL && hR) {
                int nearRef = lref, farRef = rref;
                if (tR < tL) { nearRef = rref; farRef = lref; }
                tm.stack[sp * stride] = (uint32_t) farRef;
                ++sp;
                ref = nearRef;
                continue;
            } else if (hL) { ref = lref; continue; }
            else if (hR) { ref = rref; continue; }
        } else {
            uint32_t bits = ~(uint32_t) ref;
            uint32_t start = bits & 0x0FFFFFFFu, count = bits >> 28;
            for (uint32_t i = 0; i < count; ++i) {
                uint32_t ti = start + i;
                float4 q0, q1, q2;
                if (ti < tm.stageTris) {
                    const float4 *p = tm.sTris + 3 * ti;
                    q0 = p[0]; q1 = p[1]; q2 = p[2];
                } else {
                    const float4 *p = tm.gTris + 3 * (size_t) ti;
                    q0 = __ldg(p); q1 = __ldg(p + 1); q2 = __ldg(p + 2);
                }
                if (COUNT) ++primTests;
                float tu, tv, tt;
                if (B2_TRI_TEST(q0, q1, q2, o, d, mint, maxt, tu, tv, tt)) {
                    if (SHADOW) return true;
                    hit.t = tt; hit.u = tu; hit.v = tv; best = ti;
                    maxt = tt;
                    found = true;
                }
            }
        }
        if (sp == 0) break;
        --sp;
        ref = (int) tm.stack[sp * stride];
    }
    if (found) { hit.leaf = best; hit.prim = __ldg(sc.leafPrim + best); }
    return found;
}

// One ray traced inline by the calling thread: clip to the scene box with the epsilon of a closest (CLIP_SHADOW = false) or an
// occlusion query, then a closest or any-hit (SHADOW) walk of the flat leaf (FLAT) or of whichever of the flat leaf and the binary
// tree the scene has.  Returns whether something was hit; otherwise `hit` is the miss record.
template <bool SHADOW, bool CLIP_SHADOW, bool FLAT>
B2_DEV bool traceRay(const DScene &sc, const TraceMem &tm, const V3 &o, const V3 &d, float rayMint, float rayMaxt, HitRec &hit) {
    hit = missHit();
    float mint, maxt;
    uint32_t nv = 0, pt = 0;
    if (!clipRay<CLIP_SHADOW>(sc, o, d, rayMint, rayMaxt, mint, maxt)) return false;
    return FLAT ? traverseFlat<SHADOW, false>(sc, tm, o, d, mint, maxt, hit, pt) : traverse<SHADOW, false>(sc, tm, o, d, mint, maxt, hit, nv, pt);
}

// ------------------------------------------------------------------------------------------------------------
// Instanced scenes (src/shapes/{shapegroup,instance}.cpp): a top-level BVH over items (the world triangles, each `instance`),
// below it the shapegroup's own BVH in object space.  Entering an item transforms the ray with the instance's inverse
// (transform.h:262-278: o and d, t keeps its meaning), clips [mint, maxt] against the group's box like the nested query of
// skdtree.h:430-458, and remembers the stack height; when the stack falls back to that height the world ray is restored.
// ------------------------------------------------------------------------------------------------------------
B2_DEV V3 xfPoint(const float *M, const V3 &p) { return V3(M[0] * p.x + M[1] * p.y + M[2] * p.z + M[3], M[4] * p.x + M[5] * p.y + M[6] * p.z + M[7], M[8] * p.x + M[9] * p.y + M[10] * p.z + M[11]); }
B2_DEV V3 xfVector(const float *M, const V3 &v) { return V3(M[0] * v.x + M[1] * v.y + M[2] * v.z, M[4] * v.x + M[5] * v.y + M[6] * v.z, M[8] * v.x + M[9] * v.y + M[10] * v.z); }
B2_DEV V3 xfNormal(const float *Minv, const V3 &n) { return V3(Minv[0] * n.x + Minv[4] * n.y + Minv[8] * n.z, Minv[1] * n.x + Minv[5] * n.y + Minv[9] * n.z, Minv[2] * n.x + Minv[6] * n.y + Minv[10] * n.z); }

template <bool SHADOW, bool COUNT> B2_DEV bool traverseTop(const DScene &sc, const TraceMem &tm, const V3 &o, const V3 &d, float mint, float maxt, HitRec &hit,
                                                            uint32_t &item, uint32_t &nodeVisits, uint32_t &primTests) {
    V3 co = o, cd = d, idir, ood;
    slabSetup(co, cd, idir, ood);
    bool found = false;
    uint32_t best = 0xFFFFFFFFu;
    int sp = 0, ref = sc.tlasRoot;
    int blasBase = -1;        // stack height at which the current item was entered; -1: in the top-level tree
    uint32_t curItem = 0;
    float lo = mint, hiClip = B2_INF; // [lo, min(maxt, hiClip)]: valid range inside the current item
    const uint32_t stride = tm.stride;
    while (true) {
        bool pop = true;
        if (ref >= 0) {
            const float4 *p = tm.gNodes + 4 * (size_t) ref;
            const float4 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 2), e = __ldg(p + 3);
            if (COUNT) ++nodeVisits;
            float tL, tR;
            const float hi = fminf(maxt, hiClip);
            const bool hL = boxHit(a.x, a.y, a.z, a.w, b.x, b.y, ood, idir, lo, hi, tL);
            const bool hR = boxHit(b.z, b.w, c.x, c.y, c.z, c.w, ood, idir, lo, hi, tR);
            const int lref = __float_as_int(e.x), rref = __float_as_int(e.y);
            if (hL && hR) {
                int nearRef = lref, farRef = rref;
                if (tR < tL) { nearRef = rref; farRef = lref; }
                tm.stack[sp * stride] = (uint32_t) farRef;
                ++sp;
                ref = nearRef; pop = false;
            } else if (hL) { ref = lref; pop = false; }
            else if (hR) { ref = rref; pop = false; }
        } else {
            const uint32_t bits = ~(uint32_t) ref;
            const uint32_t start = bits & 0x0FFFFFFFu, count = bits >> 28;
            if (blasBase < 0) { // top-level leaf: items; all but the first go back on the stack as single-item leaves
                if (count > 0) {
                    for (uint32_t k = 1; k < count; ++k) { tm.stack[sp * stride] = ~((start + k) | (1u << 28)); ++sp; }
                    const DInstance &in = sc.items[start];
                    bool enter = true;
                    if (in.identity) { co = o; cd = d; lo = mint; hiClip = B2_INF; }
                    else {
                        co = xfPoint(in.Minv, o); cd = xfVector(in.Minv, d);
                        const V3 dRcp(1.0f / cd.x, 1.0f / cd.y, 1.0f / cd.z);
                        float m0, m1;
                        enter = aabbRayIntersect(in.aabbMin, in.aabbMax, co, cd, dRcp, m0, m1);
                        if (enter) {
                            if (mint > m0) m0 = mint;
                            if (maxt < m1) m1 = maxt;
                            enter = m1 > m0;
                            lo = m0; hiClip = m1;
                        }
                    }
                    if (enter) {
                        slabSetup(co, cd, idir, ood);
                        blasBase = sp; curItem = start;
                        ref = in.rootRef; pop = false;
                    } else { co = o; cd = d; lo = mint; hiClip = B2_INF; slabSetup(co, cd, idir, ood); }
                }
            } else {
                const float hi = fminf(maxt, hiClip);
                for (uint32_t i = 0; i < count; ++i) {
                    const uint32_t ti = start + i;
                    const float4 *p = tm.gTris + 3 * (size_t) ti;
                    const float4 q0 = __ldg(p), q1 = __ldg(p + 1), q2 = __ldg(p + 2);
                    if (COUNT) ++primTests;
                    float tu, tv, tt;
                    if (B2_TRI_TEST(q0, q1, q2, co, cd, lo, fminf(maxt, hi), tu, tv, tt)) {
                        if (SHADOW) return true;
                        hit.t = tt; hit.u = tu; hit.v = tv; best = ti; item = curItem;
                        maxt = tt;
                        found = true;
                    }
                }
            }
        }
        if (!pop) continue;
        if (blasBase >= 0 && sp == blasBase) { // the item is exhausted: back to the world ray
            blasBase = -1;
            co = o; cd = d; lo = mint; hiClip = B2_INF;
            slabSetup(co, cd, idir, ood);
        }
        if (sp == 0) break;
        --sp;
        ref = (int) tm.stack[sp * stride];
    }
    if (found) { hit.leaf = best; hit.prim = __ldg(sc.leafPrim + best); }
    return found;
}

// ------------------------------------------------------------------------------------------------------------
// Persistent traversal with per-lane ray replacement: a warp keeps walking while its lanes finish at different times;
// when REFILL or more lanes are idle they commit their results and pull the next rays from a global ticket counter
// (one atomic per refill), so lanes do not idle until the slowest ray of a 32-ray batch is done.
//   fetch(idx, o, d, mint, maxt) -> 0: nothing to do for this item, 1: ray misses the scene box (commit a miss), 2: traverse
//   commit(idx, found, hit, item): `hit` is the miss record unless something was found; `item`: the instance that was hit
//   (traverseTop), else 0xFFFFFFFF
// The ticket protocol lives in refillQueue alone.  A walker hands it start(lane), which sets up the walker's own state for the
// lane's new ray, and walk(lane, exhausted), which advances the warp's lanes until enough of them finish; a finished lane sets
// active = false and pending = true.
// ------------------------------------------------------------------------------------------------------------
struct QueueLane {
    bool active, pending, found;
    uint32_t best; // leaf-ordered index of the closest hit so far
    V3 o, d, idir, ood;
    float mint, maxt;
    HitRec hit;
};

template <typename Fetch, typename Commit, typename Start, typename Walk>
B2_DEV void refillQueue(const DScene &sc, uint32_t n, unsigned long long *ticket, Fetch fetch, Commit commit, Start start, Walk walk) {
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    QueueLane q;
    q.active = false; q.pending = false; q.found = false; q.best = 0;
    q.o = V3(0.0f); q.d = V3(0.0f); q.idir = V3(0.0f); q.ood = V3(0.0f);
    q.mint = 0; q.maxt = 0;
    q.hit = missHit();
    bool exhausted = false;
    uint32_t idx = 0;
    const int refill = (int) sc.refill;
    // tickets a warp reserves per atomic: 128 for big launches, down to 32 so that small launches still spread over the grid
    const unsigned warpsInGrid = gridDim.x * (blockDim.x >> 5);
    const unsigned long long CHUNK = (unsigned long long) min(128u, max(32u, (n / (4u * warpsInGrid)) & ~31u));
    unsigned long long chunkNext = 0, chunkEnd = 0; // warp-uniform: locally reserved ticket range
    while (true) {
        const unsigned idle = __ballot_sync(FULL, !q.active);
        if (idle == FULL || (!exhausted && __popc(idle) >= refill)) {
            if (q.pending) {
                if (q.found) { q.hit.leaf = q.best; q.hit.prim = __ldg(sc.leafPrim + q.best); }
                commit(idx, q.found, q.hit, 0xFFFFFFFFu);
                q.pending = false;
            }
            if (!exhausted) {
                const unsigned need = (unsigned) __popc(idle);
                const unsigned rank = (unsigned) __popc(idle & ((1u << lane) - 1u));
                // tickets come from a warp-local reservation; a new chunk is reserved (one atomic) when it runs dry
                const unsigned long long have = chunkEnd - chunkNext;
                unsigned long long base2 = 0;
                if (have < need) {
                    if (lane == 0) base2 = atomicAdd(ticket, (unsigned long long) CHUNK);
                    base2 = __shfl_sync(FULL, base2, 0);
                }
                unsigned long long my;
                if (rank < have) my = chunkNext + rank;
                else my = base2 + (rank - have);
                if (have < need) { chunkNext = base2 + (need - have); chunkEnd = base2 + CHUNK; }
                else chunkNext += need;
                if (!q.active && my < n) {
                    idx = (uint32_t) my;
                    q.found = false;
                    q.hit = missHit();
                    const int r = fetch(idx, q.o, q.d, q.mint, q.maxt);
                    if (r == 2) {
                        q.active = true;
                        slabSetup(q.o, q.d, q.idir, q.ood);
                        start(q);
                    } else if (r == 1) q.pending = true;
                }
                if (chunkNext >= n) exhausted = true; // every later ticket of this warp is out of range
            }
            if (__ballot_sync(FULL, q.active) == 0) {
                if (exhausted) {
                    if (q.pending) commit(idx, q.found, q.hit, 0xFFFFFFFFu);
                    break;
                }
                continue;
            }
        }
        walk(q, exhausted);
    }
}

template <bool SHADOW, bool COUNT, typename Fetch, typename Commit>
B2_DEV void traverseQueue(const DScene &sc, const TraceMem &tm, uint32_t n, unsigned long long *ticket, Fetch fetch, Commit commit,
                          uint32_t &nodeVisits, uint32_t &primTests) {
    const unsigned FULL = 0xffffffffu;
    const uint32_t stride = tm.stride;
    int sp = 0, ref = 0;
    const int refill = (int) sc.refill;
    const int leafVote = (int) sc.leafVote;
    auto start = [&](const QueueLane &) { sp = 0; ref = sc.rootRef; };
    auto walk = [&](QueueLane &q, bool exhausted) {
        // ---- node phase ("while-while" with a vote): lanes standing on an inner node keep descending; lanes that reached
        // a leaf wait, so that the leaf code below runs with many lanes instead of 2-3.  The phase ends when enough lanes
        // wait at a leaf, nobody is on a node any more, or enough lanes went idle to make a refill worthwhile.
        while (true) {
            const bool atNode = q.active && ref >= 0;
            const unsigned nm = __ballot_sync(FULL, atNode);
            if (nm == 0) break;
            const unsigned lm = __ballot_sync(FULL, q.active && ref < 0);
            if (__popc(lm) >= leafVote) break;
            if (!exhausted && __popc(~(nm | lm)) >= refill) break;
            if (atNode) {
                float4 a, b, c, e;
                if ((uint32_t) ref < tm.stageNodes) {
                    const float4 *p = tm.sNodes + 4 * ref;
                    a = p[0]; b = p[1]; c = p[2]; e = p[3];
                } else {
                    const float4 *p = tm.gNodes + 4 * (size_t) ref;
                    a = __ldg(p); b = __ldg(p + 1); c = __ldg(p + 2); e = __ldg(p + 3);
                }
                if (COUNT) ++nodeVisits;
                float tL, tR;
                const bool hL = boxHit(a.x, a.y, a.z, a.w, b.x, b.y, q.ood, q.idir, q.mint, q.maxt, tL);
                const bool hR = boxHit(b.z, b.w, c.x, c.y, c.z, c.w, q.ood, q.idir, q.mint, q.maxt, tR);
                const int lref = __float_as_int(e.x), rref = __float_as_int(e.y);
                if (hL && hR) {
                    int nearRef = lref, farRef = rref;
                    if (tR < tL) { nearRef = rref; farRef = lref; }
                    tm.stack[sp * stride] = (uint32_t) farRef;
                    ++sp;
                    ref = nearRef;
                } else if (hL) ref = lref;
                else if (hR) ref = rref;
                else if (sp == 0) { q.active = false; q.pending = true; }
                else { --sp; ref = (int) tm.stack[sp * stride]; }
            }
        }
        // ---- leaf phase
        if (q.active && ref < 0) {
            const uint32_t bits = ~(uint32_t) ref;
            const uint32_t first = bits & 0x0FFFFFFFu, count = bits >> 28;
            for (uint32_t i = 0; i < count; ++i) {
                const uint32_t ti = first + i;
                const float4 *p = tm.gTris + 3 * (size_t) ti;
                const float4 q0 = __ldg(p), q1 = __ldg(p + 1), q2 = __ldg(p + 2);
                if (COUNT) ++primTests;
                float tu, tv, tt;
                if (B2_TRI_TEST(q0, q1, q2, q.o, q.d, q.mint, q.maxt, tu, tv, tt)) {
                    q.found = true;
                    if (SHADOW) break;
                    q.hit.t = tt; q.hit.u = tu; q.hit.v = tv; q.best = ti;
                    q.maxt = tt;
                }
            }
            if ((SHADOW && q.found) || sp == 0) { q.active = false; q.pending = true; }
            else { --sp; ref = (int) tm.stack[sp * stride]; }
        }
    };
    refillQueue(sc, n, ticket, fetch, commit, start, walk);
}

// ------------------------------------------------------------------------------------------------------------
// Wide (8-ary, quantised) tree: persistent traversal with per-lane ray replacement, same protocol as traverseQueue.
//
// A lane holds one "group": the node index of the first internal child of some node plus a bit field -- bits 24..31 the children of
// that node that were hit and still have to be visited, in visiting order (bit 24 + (slot ^ octFlip): the highest bit is the nearest
// child for this ray's direction octant), bits 0..7 the node's internal-child mask (child node = base + number of internal children
// in lower slots).  Visiting a node tests its eight quantised child boxes (t = q * (2^e * idir) + (p - o) * idir, the near / far byte
// planes picked by the direction signs), tests the triangles of the leaf children that were hit at once, and makes the hit internal
// children the new group; the rest of the old group goes on the stack (one entry per level).
// ------------------------------------------------------------------------------------------------------------
B2_DEV float byteF(uint32_t w, int k) { return (float) ((w >> (8 * k)) & 0xFFu); }

template <bool SHADOW, bool COUNT, typename Fetch, typename Commit>
B2_DEV void traverseQueue8(const DScene &sc, const TraceMem &tm, uint32_t n, unsigned long long *ticket, Fetch fetch, Commit commit,
                           uint32_t &nodeVisits, uint32_t &primTests) {
    const uint32_t stride = tm.stride;
    int sp = 0;
    uint32_t cur = 0, grpBase = 0, grpBits = 0, octFlip = 0;
    auto start = [&](const QueueLane &q) {
        sp = 0; cur = 0; grpBits = 0;
        octFlip = 7u ^ ((q.d.x < 0 ? 1u : 0u) | (q.d.y < 0 ? 2u : 0u) | (q.d.z < 0 ? 4u : 0u));
    };
    auto walk = [&](QueueLane &q, bool) {
        // per-lane results of the node visit: hit internal children (visiting order), triangles of the hit leaf children
        uint32_t hmask = 0, tmask = 0, triBase = 0, imaskN = 0, childBaseN = 0;
        if (q.active) {
            // ---- node: eight quantised child boxes ----
            float4 n0, n1, n2, n3, n4;
            if (cur < tm.stageNodes8) {
                const float4 *p = tm.sNodes8 + 5 * cur;
                n0 = p[0]; n1 = p[1]; n2 = p[2]; n3 = p[3]; n4 = p[4];
            } else {
                const float4 *p = tm.gNodes8 + 5 * (size_t) cur;
                n0 = __ldg(p); n1 = __ldg(p + 1); n2 = __ldg(p + 2); n3 = __ldg(p + 3); n4 = __ldg(p + 4);
            }
            if (COUNT) ++nodeVisits;
            const uint32_t ew = __float_as_uint(n0.w);
            const uint32_t imask = ew >> 24;
            const float ax = __uint_as_float((uint32_t) ((int) (int8_t) (ew & 0xFFu) + 127) << 23) * q.idir.x;
            const float ay = __uint_as_float((uint32_t) ((int) (int8_t) ((ew >> 8) & 0xFFu) + 127) << 23) * q.idir.y;
            const float az = __uint_as_float((uint32_t) ((int) (int8_t) ((ew >> 16) & 0xFFu) + 127) << 23) * q.idir.z;
            const float bx = fmaf(n0.x, q.idir.x, -q.ood.x), by = fmaf(n0.y, q.idir.y, -q.ood.y), bz = fmaf(n0.z, q.idir.z, -q.ood.z);
            // byte planes: near = lo for a positive direction component, hi otherwise
            const bool px = q.idir.x >= 0, py = q.idir.y >= 0, pz = q.idir.z >= 0;
            const uint32_t nx0 = __float_as_uint(px ? n2.x : n3.z), nx1 = __float_as_uint(px ? n2.y : n3.w);
            const uint32_t fx0 = __float_as_uint(px ? n3.z : n2.x), fx1 = __float_as_uint(px ? n3.w : n2.y);
            const uint32_t ny0 = __float_as_uint(py ? n2.z : n4.x), ny1 = __float_as_uint(py ? n2.w : n4.y);
            const uint32_t fy0 = __float_as_uint(py ? n4.x : n2.z), fy1 = __float_as_uint(py ? n4.y : n2.w);
            const uint32_t nz0 = __float_as_uint(pz ? n3.x : n4.z), nz1 = __float_as_uint(pz ? n3.y : n4.w);
            const uint32_t fz0 = __float_as_uint(pz ? n4.z : n3.x), fz1 = __float_as_uint(pz ? n4.w : n3.y);
            const uint32_t meta0 = __float_as_uint(n1.z), meta1 = __float_as_uint(n1.w);
#pragma unroll
            for (int s = 0; s < 8; ++s) {
                const int k = s & 3;
                const float tnx = fmaf(byteF(s < 4 ? nx0 : nx1, k), ax, bx), tfx = fmaf(byteF(s < 4 ? fx0 : fx1, k), ax, bx);
                const float tny = fmaf(byteF(s < 4 ? ny0 : ny1, k), ay, by), tfy = fmaf(byteF(s < 4 ? fy0 : fy1, k), ay, by);
                const float tnz = fmaf(byteF(s < 4 ? nz0 : nz1, k), az, bz), tfz = fmaf(byteF(s < 4 ? fz0 : fz1, k), az, bz);
                const float tmin = fmaxf(fmaxf(tnx, tny), fmaxf(tnz, q.mint));
                const float tmax = fminf(fminf(tfx, tfy), fminf(tfz, q.maxt));
                const uint32_t m = ((s < 4 ? meta0 : meta1) >> (8 * k)) & 0xFFu;
                if (tmin <= tmax * 1.0000003f) {
                    if ((imask >> s) & 1u) hmask |= 1u << (24u + ((uint32_t) s ^ octFlip));
                    else tmask |= ((1u << (m >> 5)) - 1u) << (m & 31u); // an empty slot has m == 0: no bits
                }
            }
            triBase = __float_as_uint(n1.y); imaskN = imask; childBaseN = __float_as_uint(n1.x);
            // ---- the triangles of the leaf children that were hit ----
            // ncu (round 2, 10 M triangles, 1.60 Grays/s): this per-lane loop runs at 3 of 32 lanes (10 M warp-level passes against 2.1 M
            // node passes at 23 lanes) and 37 % of the stall samples sit on the first use of a freshly loaded triangle.  Four remedies were
            // implemented and measured on the same workload; all were SLOWER and are not kept: next-triangle prefetch + prefetch.global.L2
            // of the hit children 1.51; postponing the triangles until 8 lanes of the warp wait 1.51; binning the tickets by entry cell x
            // direction cell 1.41; a warp-cooperative pass (prefix-sum numbered (lane, triangle) pairs, every lane tests one pair
            // with the owner's ray fetched by shuffles, closest hit by a 64-bit shared-memory atomicMin) 1.21.
            while (tmask) {
                const uint32_t ti = triBase + (uint32_t) (__ffs((int) tmask) - 1);
                tmask &= tmask - 1u;
                const float4 *p = tm.gTris + 3 * (size_t) ti;
                const float4 q0 = __ldg(p), q1 = __ldg(p + 1), q2 = __ldg(p + 2);
                if (COUNT) ++primTests;
                float tu, tv, tt;
                if (B2_TRI_TEST(q0, q1, q2, q.o, q.d, q.mint, q.maxt, tu, tv, tt)) {
                    q.found = true;
                    if (SHADOW) break;
                    q.hit.t = tt; q.hit.u = tu; q.hit.v = tv; q.best = ti;
                    q.maxt = tt;
                }
            }
            // ---- next node ----
            if (SHADOW && q.found) { q.active = false; q.pending = true; }
            else {
                if (hmask) {
                    if (grpBits >> 24) { tm.stack8[sp * stride] = make_uint2(grpBase, grpBits); ++sp; }
                    grpBase = childBaseN; grpBits = hmask | imaskN;
                }
                if (!(grpBits >> 24)) {
                    if (sp == 0) { q.active = false; q.pending = true; }
                    else { --sp; const uint2 g = tm.stack8[sp * stride]; grpBase = g.x; grpBits = g.y; }
                }
                if (q.active) {
                    const uint32_t b = 31u - (uint32_t) __clz((int) grpBits);
                    grpBits &= ~(1u << b);
                    const uint32_t slot = (b - 24u) ^ octFlip;
                    cur = grpBase + (uint32_t) __popc(grpBits & 0xFFu & ((1u << slot) - 1u));
                }
            }
        }
    };
    refillQueue(sc, n, ticket, fetch, commit, start, walk);
}

// The tree the ray-query kernels (k_extend, k_occluded, k_trace_rays) walk, which also fixes their shared-memory layout: the 8-wide tree
// of a non-instanced BVH scene when the commit kept it (it drops it when it is too deep for the wide stack), else the binary layout (the
// binary tree, the two levels of an instanced scene, the flat leaf).  The flat-leaf kernels and volpath name their walker themselves.
enum Walker { WALK_FLAT, WALK_BINARY, WALK_WIDE };
B2_DEV Walker traceWalker(const DScene &sc) { return sc.nodes8 != nullptr && !sc.rootCount && !sc.nItems ? WALK_WIDE : WALK_BINARY; }

// The ray queries of a launch: items [0, n), each traced with the fetch / commit contract above.  BVH scenes take the queue of their
// tree; instanced scenes and the flat leaf take a static grid-stride loop (per-lane tickets were slower for instanced scenes,
// DESIGN.md §8c).
template <bool SHADOW, bool COUNT, typename Fetch, typename Commit>
B2_DEV void traceQueue(const DScene &sc, const TraceMem &tm, uint32_t n, unsigned long long *ticket, Fetch fetch, Commit commit,
                       uint32_t &nodeVisits, uint32_t &primTests) {
    if (traceWalker(sc) == WALK_WIDE) traverseQueue8<SHADOW, COUNT>(sc, tm, n, ticket, fetch, commit, nodeVisits, primTests);
    else if (!sc.rootCount && !sc.nItems) traverseQueue<SHADOW, COUNT>(sc, tm, n, ticket, fetch, commit, nodeVisits, primTests);
    else
        for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
            const uint32_t i = base + threadIdx.x;
            V3 o, d;
            float mint, maxt;
            const int r = i < n ? fetch(i, o, d, mint, maxt) : 0;
            if (r == 0) continue;
            HitRec h = missHit();
            uint32_t item = 0xFFFFFFFFu;
            bool found = false;
            if (r == 2)
                found = sc.nItems ? traverseTop<SHADOW, COUNT>(sc, tm, o, d, mint, maxt, h, item, nodeVisits, primTests)
                                  : traverseFlat<SHADOW, COUNT>(sc, tm, o, d, mint, maxt, h, primTests);
            commit(i, found, h, item);
        }
}

} // namespace b2
