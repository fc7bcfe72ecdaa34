// Device-side binned-SAH build: the trees of bvh_builder.cpp, byte for byte, built in HBM.
//
// The host builder is deterministic and every float step in it is a plain IEEE + - * / (this unit is compiled with -fmad=false), a
// min / max or an integer count, so the device can make the same decisions from the same data:
//   1. Top-down, one level at a time, over the open nodes with more than kSmall primitives: bounds (block reductions, then one atomic
//      per block on order-preserving integer keys), 3 x 16 bins (shared-memory privatised), the host's SAH sweep (one thread per node),
//      a stable partition (block scans + a scan over the blocks of each node) and, where the host takes its object median, a segmented
//      sort by (centroid, id).  Nodes of at most kSmall primitives get their whole subtree built by one thread running the host's loop.
//      Node ids of this phase are arbitrary (atomic allocation): the layouts below only follow the tree's structure.
//   2. Binary BFS numbering, level by level: the index of an inner node is a scan of "is inner" over its level, which is exactly the
//      order the host's std::queue visits them in.
//   3. 8-wide collapse, level by level: one thread per wide node runs the host's greedy opening, slot assignment and quantisation;
//      childBase / triBase are scans over the level of (internal children) and (leaf triangles), carried over from the levels before.
//
// Signed zeros: an integer-keyed atomic min keeps -0 where the host's std::min keeps whichever zero came first.  No output byte depends
// on it: raw box coordinates only reach the nodes through padBox (x - (|x| * 4e-7 + tiny), tiny > 0, equal for +0 and -0), through a
// difference with a non-zero value, or through a comparison, where +0 == -0.
#include "bvh_device.h"
#include <cub/cub.cuh>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace b2 {
namespace {

constexpr int NB = 16;               // bins per axis (bvh_builder.cpp Builder::NB)
constexpr uint32_t kSmall = 128;     // nodes with at most this many primitives: the whole subtree on one thread
constexpr uint32_t kChunk = 4096;    // primitives per block in the level passes
constexpr int kThreads = 256;
constexpr int kBinWords = 3 * NB * 7; // per node: 3 axes x 16 bins x (lo xyz, hi xyz, count)

struct Ref { float lo[3], hi[3]; uint32_t id; };                                  // Builder::Ref
struct TNode { float lo[3], hi[3]; int32_t left, right; uint32_t start, count; int32_t depth; }; // TmpNode
struct Open { int32_t node; uint32_t start, count; int32_t depth; };
enum { kSAH = 0, kMedian = 1 };
struct Work { float clo[3], scale[3], ext[3]; int32_t axis, mode, bestAxis, bestBin; uint32_t nLeft; };

// std::min / std::max: the first argument wins a tie
__device__ __forceinline__ float hmin(float a, float b) { return b < a ? b : a; }
__device__ __forceinline__ float hmax(float a, float b) { return a < b ? b : a; }
// order-preserving integer key of a float (for atomic min / max and sort keys)
__host__ __device__ __forceinline__ uint32_t fkey(uint32_t u) { return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ uint32_t fkey(float f) { return fkey(__float_as_uint(f)); }
__device__ __forceinline__ float fdec(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }
constexpr uint32_t kKeyPInf = 0xFF800000u, kKeyNInf = 0x007FFFFFu; // fkey(+inf), fkey(-inf)

__device__ __forceinline__ float centroid(const Ref &r, int a) { return 0.5f * (r.lo[a] + r.hi[a]); }
__device__ __forceinline__ int binOf(float c, float lo, float scale) { return min(max((int) ((c - lo) * scale), 0), NB - 1); }
__device__ __forceinline__ float area(const float *lo, const float *hi) {
    const float d0 = hi[0] - lo[0], d1 = hi[1] - lo[1], d2 = hi[2] - lo[2];
    if (d0 < 0) return 0;
    return 2.0f * (d0 * d1 + d1 * d2 + d0 * d2);
}
__device__ __forceinline__ void resetBox(float *lo, float *hi) { for (int a = 0; a < 3; ++a) { lo[a] = INFINITY; hi[a] = -INFINITY; } }
__device__ __forceinline__ void grow(float *lo, float *hi, const float *l, const float *h) {
    for (int a = 0; a < 3; ++a) { lo[a] = hmin(lo[a], l[a]); hi[a] = hmax(hi[a], h[a]); }
}
__device__ __forceinline__ void padBox(const float *blo, const float *bhi, float tiny, float *lo, float *hi) {
    for (int i = 0; i < 3; ++i) {
        lo[i] = blo[i] - (fabsf(blo[i]) * 4e-7f + tiny);
        hi[i] = bhi[i] + (fabsf(bhi[i]) * 4e-7f + tiny);
    }
}
// depth cap of Builder::build: the remaining levels can only just hold a balanced tree
__device__ __forceinline__ bool forceMedianAt(uint32_t count, int depth, int maxLeaf, int maxDepth) {
    const int remaining = maxDepth - depth;
    const uint32_t leaves = (count + (uint32_t) maxLeaf - 1) / (uint32_t) maxLeaf;
    int need = 0;
    while ((1u << need) < leaves) ++need;
    return need + 1 >= remaining;
}
__device__ __forceinline__ int widestAxis(const float *ext) {
    int axis = 0;
    if (ext[1] > ext[axis]) axis = 1;
    if (ext[2] > ext[axis]) axis = 2;
    return axis;
}
// the object-median order of the host's nth_element: (centroid, id), +0 == -0
__device__ __forceinline__ bool medianLess(const Ref &a, const Ref &b, int axis) {
    const float ca = centroid(a, axis), cb = centroid(b, axis);
    return ca < cb || (ca == cb && a.id < b.id);
}
__device__ __forceinline__ int32_t leafRefOf(uint32_t start, uint32_t count) { return (int32_t) ~(start | (count << 28)); }

// ---- phase 1: binned SAH -----------------------------------------------------------------------------------------------------------
__global__ void k_init(const PrimBox *boxes, uint32_t n, Ref *refs) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Ref r;
    for (int a = 0; a < 3; ++a) { r.lo[a] = boxes[i].lo[a]; r.hi[a] = boxes[i].hi[a]; }
    r.id = i;
    refs[i] = r;
}

__global__ void k_accInit(uint32_t nL, uint32_t *acc, uint32_t *bins) {
    const size_t stride = (size_t) gridDim.x * blockDim.x;
    for (size_t j = blockIdx.x * (size_t) blockDim.x + threadIdx.x; j < 12 * (size_t) nL; j += stride)
        acc[j] = (j % 12) % 6 < 3 ? kKeyPInf : kKeyNInf; // box lo, box hi, centroid lo, centroid hi
    for (size_t j = blockIdx.x * (size_t) blockDim.x + threadIdx.x; j < (size_t) kBinWords * nL; j += stride) {
        const int m = (int) (j % 7);
        bins[j] = m < 3 ? kKeyPInf : (m < 6 ? kKeyNInf : 0u);
    }
}

// block b covers primitives [chunk, chunk + kChunk) of node blk[b].x
__device__ __forceinline__ void chunkRange(const Open &o, uint32_t chunk, uint32_t &beg, uint32_t &end) {
    beg = o.start + chunk;
    end = o.start + min(o.count, chunk + kChunk);
}

__global__ void __launch_bounds__(kThreads) k_bounds(const Ref *refs, const Open *open, const uint2 *blk, uint32_t *acc) {
    const uint2 b = blk[blockIdx.x];
    const Open o = open[b.x];
    uint32_t beg, end;
    chunkRange(o, b.y, beg, end);
    uint32_t k[12];
    for (int j = 0; j < 12; ++j) k[j] = (j % 6) < 3 ? 0xFFFFFFFFu : 0u;
    for (uint32_t i = beg + threadIdx.x; i < end; i += kThreads) {
        const Ref r = refs[i];
        for (int a = 0; a < 3; ++a) {
            k[a] = min(k[a], fkey(r.lo[a]));
            k[3 + a] = max(k[3 + a], fkey(r.hi[a]));
            const uint32_t c = fkey(centroid(r, a));
            k[6 + a] = min(k[6 + a], c);
            k[9 + a] = max(k[9 + a], c);
        }
    }
    __shared__ uint32_t sm[kThreads / 32][12];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j = 0; j < 12; ++j) {
        const uint32_t v = (j % 6) < 3 ? __reduce_min_sync(0xFFFFFFFFu, k[j]) : __reduce_max_sync(0xFFFFFFFFu, k[j]);
        if (lane == 0) sm[warp][j] = v;
    }
    __syncthreads();
    if (threadIdx.x < 12) {
        const int j = threadIdx.x;
        const bool isMin = (j % 6) < 3;
        uint32_t v = sm[0][j];
        for (int w = 1; w < kThreads / 32; ++w) v = isMin ? min(v, sm[w][j]) : max(v, sm[w][j]);
        if (isMin) atomicMin(&acc[12 * (size_t) b.x + j], v); else atomicMax(&acc[12 * (size_t) b.x + j], v);
    }
}

// per node: box into the tree, the depth cap, the split axis, the binning grid
__global__ void k_decide(uint32_t nL, const Open *open, const uint32_t *acc, TNode *pool, Work *work, int maxLeaf, int maxDepth) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nL) return;
    const Open o = open[k];
    const uint32_t *A = acc + 12 * (size_t) k;
    TNode &t = pool[o.node];
    float clo[3], chi[3];
    for (int a = 0; a < 3; ++a) {
        t.lo[a] = fdec(A[a]); t.hi[a] = fdec(A[3 + a]);
        clo[a] = fdec(A[6 + a]); chi[a] = fdec(A[9 + a]);
    }
    t.start = o.start; t.count = o.count; t.depth = o.depth;
    // these nodes hold more than kSmall > maxLeaf primitives: never a leaf
    const bool forceMedian = forceMedianAt(o.count, o.depth, maxLeaf, maxDepth);
    Work w;
    for (int a = 0; a < 3; ++a) { w.clo[a] = clo[a]; w.ext[a] = chi[a] - clo[a]; }
    w.axis = widestAxis(w.ext);
    for (int a = 0; a < 3; ++a) w.scale[a] = w.ext[a] > 0 ? NB / w.ext[a] : 0.0f;
    w.mode = (!forceMedian && w.ext[w.axis] > 0) ? kSAH : kMedian;
    w.bestAxis = -1; w.bestBin = -1; w.nLeft = o.count / 2;
    work[k] = w;
}

__global__ void __launch_bounds__(kThreads) k_bins(const Ref *refs, const Open *open, const uint2 *blk, const Work *work, uint32_t *bins) {
    const uint2 b = blk[blockIdx.x];
    const Work w = work[b.x];
    if (w.mode != kSAH) return;
    __shared__ uint32_t sb[kBinWords];
    for (int j = threadIdx.x; j < kBinWords; j += kThreads) { const int m = j % 7; sb[j] = m < 3 ? kKeyPInf : (m < 6 ? kKeyNInf : 0u); }
    __syncthreads();
    const Open o = open[b.x];
    uint32_t beg, end;
    chunkRange(o, b.y, beg, end);
    for (uint32_t i = beg + threadIdx.x; i < end; i += kThreads) {
        const Ref r = refs[i];
        for (int a = 0; a < 3; ++a) {
            if (!(w.ext[a] > 0)) continue;
            uint32_t *s = sb + (a * NB + binOf(centroid(r, a), w.clo[a], w.scale[a])) * 7;
            for (int c = 0; c < 3; ++c) { atomicMin(&s[c], fkey(r.lo[c])); atomicMax(&s[3 + c], fkey(r.hi[c])); }
            atomicAdd(&s[6], 1u);
        }
    }
    __syncthreads();
    uint32_t *g = bins + (size_t) kBinWords * b.x;
    for (int j = threadIdx.x; j < 3 * NB; j += kThreads) {
        const uint32_t *s = sb + 7 * j;
        if (!s[6]) continue;
        for (int c = 0; c < 3; ++c) { atomicMin(&g[7 * j + c], s[c]); atomicMax(&g[7 * j + 3 + c], s[3 + c]); }
        atomicAdd(&g[7 * j + 6], s[6]);
    }
}

// the host's sweep over the merged bins (Builder::build): right-to-left areas, then left-to-right, first minimum wins
__device__ void sahSweep(const float (*bbl)[NB][3], const float (*bbh)[NB][3], const uint32_t (*bc)[NB], const float *ext, float &bestCost,
                         int &bestAxis, int &bestBin) {
    bestCost = INFINITY; bestAxis = -1; bestBin = -1;
    for (int a = 0; a < 3; ++a) {
        if (!(ext[a] > 0)) continue;
        float rightArea[NB];
        uint32_t rightCount[NB];
        float lo[3], hi[3];
        resetBox(lo, hi);
        uint32_t cnt = 0;
        for (int k = NB - 1; k > 0; --k) {
            if (bc[a][k]) grow(lo, hi, bbl[a][k], bbh[a][k]);
            cnt += bc[a][k];
            rightArea[k] = area(lo, hi);
            rightCount[k] = cnt;
        }
        resetBox(lo, hi);
        cnt = 0;
        for (int k = 0; k < NB - 1; ++k) {
            if (bc[a][k]) grow(lo, hi, bbl[a][k], bbh[a][k]);
            cnt += bc[a][k];
            if (cnt == 0 || rightCount[k + 1] == 0) continue;
            const float cost = area(lo, hi) * cnt + rightArea[k + 1] * rightCount[k + 1];
            if (cost < bestCost) { bestCost = cost; bestAxis = a; bestBin = k; }
        }
    }
}

__global__ void k_sah(uint32_t nL, const uint32_t *bins, Work *work) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nL) return;
    Work w = work[k];
    if (w.mode != kSAH) return;
    const uint32_t *g = bins + (size_t) kBinWords * k;
    float bbl[3][NB][3], bbh[3][NB][3];
    uint32_t bc[3][NB];
    for (int a = 0; a < 3; ++a)
        for (int j = 0; j < NB; ++j) {
            const uint32_t *s = g + 7 * (a * NB + j);
            for (int c = 0; c < 3; ++c) { bbl[a][j][c] = fdec(s[c]); bbh[a][j][c] = fdec(s[3 + c]); }
            bc[a][j] = s[6];
        }
    float bestCost;
    sahSweep(bbl, bbh, bc, w.ext, bestCost, w.bestAxis, w.bestBin);
    // more than maxLeaf primitives: the split is taken whatever its cost; without one the host falls back to the median
    if (w.bestAxis < 0) w.mode = kMedian;
    else {
        uint32_t l = 0;
        for (int j = 0; j <= w.bestBin; ++j) l += bc[w.bestAxis][j];
        w.nLeft = l;
    }
    work[k] = w;
}

__device__ __forceinline__ bool goesLeft(const Ref &r, const Work &w) {
    return binOf(centroid(r, w.bestAxis), w.clo[w.bestAxis], w.scale[w.bestAxis]) <= w.bestBin;
}

__global__ void __launch_bounds__(kThreads) k_flags(const Ref *refs, const Open *open, const uint2 *blk, const Work *work, uint32_t *blockLeft) {
    const uint2 b = blk[blockIdx.x];
    const Work w = work[b.x];
    if (w.mode != kSAH) { if (threadIdx.x == 0) blockLeft[blockIdx.x] = 0; return; }
    const Open o = open[b.x];
    uint32_t beg, end;
    chunkRange(o, b.y, beg, end);
    uint32_t c = 0;
    for (uint32_t i = beg + threadIdx.x; i < end; i += kThreads) c += goesLeft(refs[i], w) ? 1u : 0u;
    c = __reduce_add_sync(0xFFFFFFFFu, c);
    __shared__ uint32_t sm[kThreads / 32];
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0;
        for (int j = 0; j < kThreads / 32; ++j) s += sm[j];
        blockLeft[blockIdx.x] = s;
    }
}

// stable partition into `scratch`: left-hand primitives at [start, start + nLeft), right-hand ones after, both in their old order
__global__ void __launch_bounds__(kThreads) k_scatter(const Ref *refs, Ref *scratch, const Open *open, const uint2 *blk, const Work *work,
                                                      const uint32_t *blockLeftEx, const uint32_t *firstBlock) {
    const uint2 b = blk[blockIdx.x];
    const Work w = work[b.x];
    if (w.mode != kSAH) return;
    const Open o = open[b.x];
    uint32_t beg, end;
    chunkRange(o, b.y, beg, end);
    const uint32_t leftBase = blockLeftEx[blockIdx.x] - blockLeftEx[firstBlock[b.x]], rightBase = b.y - leftBase;
    typedef cub::BlockScan<uint32_t, kThreads> BlockScan;
    __shared__ typename BlockScan::TempStorage ts;
    uint32_t carry = 0;
    for (uint32_t off = 0; beg + off < end; off += kThreads) {
        const uint32_t li = off + threadIdx.x;
        const bool valid = beg + li < end;
        Ref r;
        uint32_t f = 0;
        if (valid) { r = refs[beg + li]; f = goesLeft(r, w) ? 1u : 0u; }
        uint32_t pos, agg;
        BlockScan(ts).ExclusiveSum(f, pos, agg);
        if (valid) {
            if (f) scratch[o.start + leftBase + carry + pos] = r;
            else scratch[o.start + w.nLeft + rightBase + (li - carry - pos)] = r;
        }
        carry += agg;
        __syncthreads();
    }
}

__global__ void k_medianKeys(const Ref *refs, const Open *open, const uint2 *blk, const Work *work, unsigned long long *keys, uint32_t *vals) {
    const uint2 b = blk[blockIdx.x];
    const Work w = work[b.x];
    if (w.mode != kMedian) return;
    const Open o = open[b.x];
    uint32_t beg, end;
    chunkRange(o, b.y, beg, end);
    for (uint32_t i = beg + threadIdx.x; i < end; i += blockDim.x) {
        const Ref r = refs[i];
        float c = centroid(r, w.axis);
        if (c == 0.0f) c = 0.0f; // -0 sorts with +0, as the host's float comparison has it
        keys[i] = ((unsigned long long) fkey(c) << 32) | r.id;
        vals[i] = i;
    }
}

__global__ void k_medianGather(const Ref *refs, Ref *scratch, const Open *open, const uint2 *blk, const Work *work, const uint32_t *vals) {
    const uint2 b = blk[blockIdx.x];
    if (work[b.x].mode != kMedian) return;
    const Open o = open[b.x];
    uint32_t beg, end;
    chunkRange(o, b.y, beg, end);
    for (uint32_t i = beg + threadIdx.x; i < end; i += blockDim.x) scratch[i] = refs[vals[i]];
}

__global__ void k_copyBack(Ref *refs, const Ref *scratch, const Open *open, const uint2 *blk) {
    const uint2 b = blk[blockIdx.x];
    const Open o = open[b.x];
    uint32_t beg, end;
    chunkRange(o, b.y, beg, end);
    for (uint32_t i = beg + threadIdx.x; i < end; i += blockDim.x) refs[i] = scratch[i];
}

__global__ void k_children(uint32_t nL, const Open *open, const Work *work, TNode *pool, uint32_t *counters, Open *next, Open *small) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nL) return;
    const Open o = open[k];
    const uint32_t mid = work[k].nLeft; // the partition's left count, or count / 2 for the median
    const int32_t idx = (int32_t) atomicAdd(&counters[0], 2u);
    pool[o.node].left = idx;
    pool[o.node].right = idx + 1;
    for (int c = 0; c < 2; ++c) {
        Open ch;
        ch.node = idx + c;
        ch.start = c ? o.start + mid : o.start;
        ch.count = c ? o.count - mid : mid;
        ch.depth = o.depth + 1;
        TNode &t = pool[ch.node];
        t.left = t.right = -1;
        if (ch.count > kSmall) next[atomicAdd(&counters[1], 1u)] = ch;
        else small[atomicAdd(&counters[2], 1u)] = ch;
    }
}

// one thread builds the subtree of a small node exactly as Builder::build does with one thread (smaller child first: the stack stays
// within log2(kSmall) + 1 pending nodes)
__global__ void __launch_bounds__(128) k_small(uint32_t nS, const Open *small, Ref *refs, Ref *scratch, TNode *pool, uint32_t *counters,
                                               int maxLeaf, int maxDepth) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nS) return;
    const Open root = small[k];
    int32_t next = root.count >= 2 ? (int32_t) atomicAdd(&counters[0], 2 * root.count - 2) : 0; // at most 2 count - 1 nodes below
    Open stack[24];
    int sp = 0;
    stack[sp++] = root;
    float bbl[3][NB][3], bbh[3][NB][3];
    uint32_t bc[3][NB];
    while (sp) {
        const Open o = stack[--sp];
        const uint32_t start = o.start, count = o.count;
        TNode t;
        resetBox(t.lo, t.hi);
        float clo[3], chi[3];
        resetBox(clo, chi);
        for (uint32_t i = start; i < start + count; ++i) {
            const Ref r = refs[i];
            grow(t.lo, t.hi, r.lo, r.hi);
            const float c3[3] = {centroid(r, 0), centroid(r, 1), centroid(r, 2)};
            grow(clo, chi, c3, c3);
        }
        t.left = t.right = -1; t.start = start; t.count = count; t.depth = o.depth;
        pool[o.node] = t;
        if (count == 1) continue;
        const bool canLeaf = (int) count <= maxLeaf;
        const bool forceMedian = forceMedianAt(count, o.depth, maxLeaf, maxDepth);
        if (canLeaf && (forceMedian || maxDepth - o.depth <= 1)) continue;
        float ext[3] = {chi[0] - clo[0], chi[1] - clo[1], chi[2] - clo[2]};
        const int axis = widestAxis(ext);
        uint32_t mid = count / 2;
        bool done = false;
        if (!forceMedian && ext[axis] > 0) {
            float scale[3];
            for (int a = 0; a < 3; ++a) scale[a] = ext[a] > 0 ? NB / ext[a] : 0.0f;
            for (int a = 0; a < 3; ++a) for (int j = 0; j < NB; ++j) { resetBox(bbl[a][j], bbh[a][j]); bc[a][j] = 0; }
            for (uint32_t i = start; i < start + count; ++i) {
                const Ref r = refs[i];
                for (int a = 0; a < 3; ++a) {
                    if (!(ext[a] > 0)) continue;
                    const int j = binOf(centroid(r, a), clo[a], scale[a]);
                    grow(bbl[a][j], bbh[a][j], r.lo, r.hi);
                    bc[a][j]++;
                }
            }
            float bestCost;
            int bestAxis, bestBin;
            sahSweep(bbl, bbh, bc, ext, bestCost, bestAxis, bestBin);
            if (bestAxis >= 0) {
                const float leafCost = area(t.lo, t.hi) * count;
                const float splitCost = 1.0f * area(t.lo, t.hi) + bestCost;
                if (splitCost < leafCost || !canLeaf) {
                    Work w;
                    w.bestAxis = bestAxis; w.bestBin = bestBin; w.clo[bestAxis] = clo[bestAxis]; w.scale[bestAxis] = scale[bestAxis];
                    uint32_t l = start, r = 0;
                    for (uint32_t i = start; i < start + count; ++i) {
                        const Ref p = refs[i];
                        if (goesLeft(p, w)) refs[l++] = p; else scratch[start + r++] = p;
                    }
                    for (uint32_t i = 0; i < r; ++i) refs[l + i] = scratch[start + i];
                    mid = l - start;
                    done = mid > 0 && mid < count;
                }
            }
        }
        if (!done && canLeaf) continue;
        if (!done) { // object median: sort the range by (centroid, id), lower half left
            for (uint32_t i = start + 1; i < start + count; ++i) {
                const Ref x = refs[i];
                uint32_t j = i;
                while (j > start && medianLess(x, refs[j - 1], axis)) { refs[j] = refs[j - 1]; --j; }
                refs[j] = x;
            }
            mid = count / 2;
        }
        pool[o.node].left = next;
        pool[o.node].right = next + 1;
        const Open L = {next, start, mid, o.depth + 1}, R = {next + 1, start + mid, count - mid, o.depth + 1};
        next += 2;
        if (L.count <= R.count) { stack[sp++] = R; stack[sp++] = L; }
        else { stack[sp++] = L; stack[sp++] = R; }
    }
}

// ---- phase 2: binary BFS numbering ---------------------------------------------------------------------------------------------------
__global__ void k_innerCount(uint32_t nL, const int32_t *cur, const TNode *pool, uint32_t *cnt) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nL) return;
    const TNode t = pool[cur[k]];
    cnt[k] = (pool[t.left].left >= 0 ? 1u : 0u) + (pool[t.right].left >= 0 ? 1u : 0u);
}

__global__ void k_innerNext(uint32_t nL, const int32_t *cur, const TNode *pool, const uint32_t *ex, uint32_t nextBase, int32_t *innerIndex,
                            int32_t *next) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nL) return;
    const TNode t = pool[cur[k]];
    uint32_t j = ex[k];
    for (int side = 0; side < 2; ++side) {
        const int32_t c = side ? t.right : t.left;
        if (pool[c].left >= 0) { innerIndex[c] = (int32_t) (nextBase + j); next[j++] = c; }
    }
}

__global__ void k_binaryNodes(uint32_t nPool, const TNode *pool, const int32_t *innerIndex, const uint32_t *leafStart, float tiny, BVHNode *nodes) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= nPool) return;
    const int32_t ii = innerIndex[p];
    if (ii < 0) return;
    const TNode t = pool[p];
    const TNode L = pool[t.left], R = pool[t.right];
    BVHNode nd;
    padBox(L.lo, L.hi, tiny, nd.lmin, nd.lmax);
    padBox(R.lo, R.hi, tiny, nd.rmin, nd.rmax);
    nd.left = L.left >= 0 ? innerIndex[t.left] : leafRefOf(leafStart ? leafStart[t.left] : L.start, L.count);
    nd.right = R.left >= 0 ? innerIndex[t.right] : leafRefOf(leafStart ? leafStart[t.right] : R.start, R.count);
    nd.pad0 = nd.pad1 = 0;
    nodes[ii] = nd;
}

__global__ void k_leafGather(uint32_t n, const Ref *refs, const uint32_t *ids, uint32_t *leafPrims) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) leafPrims[i] = ids[refs[i].id];
}

// ---- phase 3: 8-wide collapse (WideBuild::run / quantise) ----------------------------------------------------------------------------
__global__ void k_widePlan(uint32_t nL, const int32_t *cur, const TNode *pool, float tiny, int32_t *plans, uint32_t *nInner, uint32_t *nTris) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nL) return;
    const TNode tn = pool[cur[k]];
    int ch[8], n = 0;
    ch[n++] = tn.left; ch[n++] = tn.right;
    while (n < 8) {
        int best = -1;
        float bestArea = -1.0f;
        for (int j = 0; j < n; ++j) {
            const TNode c = pool[ch[j]];
            if (c.left >= 0 && area(c.lo, c.hi) > bestArea) { bestArea = area(c.lo, c.hi); best = j; }
        }
        if (best < 0) break;
        const int t = ch[best];
        ch[best] = pool[t].left; ch[n++] = pool[t].right;
    }
    float nlo[3], nhi[3];
    resetBox(nlo, nhi);
    for (int j = 0; j < n; ++j) {
        const TNode c = pool[ch[j]];
        float clo[3], chi[3];
        padBox(c.lo, c.hi, tiny, clo, chi);
        grow(nlo, nhi, clo, chi);
    }
    float score[8][8];
    for (int j = 0; j < n; ++j) {
        const TNode c = pool[ch[j]];
        for (int s = 0; s < 8; ++s) {
            float v = 0;
            for (int a = 0; a < 3; ++a) {
                const float d = 0.5f * (c.lo[a] + c.hi[a]) - 0.5f * (nlo[a] + nhi[a]);
                v += ((s >> a) & 1) ? d : -d;
            }
            score[j][s] = v;
        }
    }
    int slotOf[8], used = 0;
    bool done[8] = {false, false, false, false, false, false, false, false};
    for (int round = 0; round < n; ++round) {
        int bk = -1, bs = -1;
        float bv = -INFINITY;
        for (int j = 0; j < n; ++j) {
            if (done[j]) continue;
            for (int s = 0; s < 8; ++s)
                if (!((used >> s) & 1) && score[j][s] > bv) { bv = score[j][s]; bk = j; bs = s; }
        }
        done[bk] = true; used |= 1 << bs; slotOf[bk] = bs;
    }
    int32_t *pl = plans + 8 * (size_t) k;
    for (int s = 0; s < 8; ++s) pl[s] = -1;
    for (int j = 0; j < n; ++j) pl[slotOf[j]] = ch[j];
    uint32_t ni = 0, nt = 0;
    for (int j = 0; j < n; ++j) {
        const TNode c = pool[ch[j]];
        if (c.left >= 0) ++ni; else nt += c.count;
    }
    nInner[k] = ni;
    nTris[k] = nt;
}

// the smallest e with 255 * 2^e >= ext, within [-100, 100]: what the host's ceil(log2(ext / 255)) and its correction loop give
__device__ int quantExponent(double ext) {
    if (!(ext > 0)) return -100;
    int e = ilogb(ext) - 7;
    while (ldexp(255.0, e) < ext) ++e;
    while (ldexp(255.0, e - 1) >= ext) --e;
    return max(-100, min(100, e));
}

__global__ void k_wideEmit(uint32_t nL, const int32_t *plans, const uint32_t *exInner, const uint32_t *exTris, uint32_t levelBase, uint32_t triCarry,
                           const TNode *pool, const Ref *refs, const uint32_t *ids, float tiny, BVH8Node *nodes8, int32_t *next,
                           uint32_t *leafStart, uint32_t *leafPrims) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nL) return;
    const int32_t *pl = plans + 8 * (size_t) k;
    float nlo[3], nhi[3], clo[8][3], chi[8][3];
    resetBox(nlo, nhi);
    for (int s = 0; s < 8; ++s)
        if (pl[s] >= 0) { const TNode c = pool[pl[s]]; padBox(c.lo, c.hi, tiny, clo[s], chi[s]); grow(nlo, nhi, clo[s], chi[s]); }
    BVH8Node nd;
    memset(&nd, 0, sizeof(nd));
    double scale[3];
    for (int a = 0; a < 3; ++a) {
        nd.p[a] = nlo[a];
        const int e = quantExponent((double) nhi[a] - (double) nlo[a]);
        nd.e[a] = (int8_t) e;
        scale[a] = ldexp(1.0, e);
    }
    nd.childBase = levelBase + nL + exInner[k];
    nd.triBase = triCarry + exTris[k];
    uint32_t triOff = 0, inner = 0;
    for (int s = 0; s < 8; ++s) {
        if (pl[s] < 0) continue;
        const TNode c = pool[pl[s]];
        for (int a = 0; a < 3; ++a) {
            int lo = (int) floor(((double) clo[s][a] - (double) nd.p[a]) / scale[a]);
            int hi = (int) ceil(((double) chi[s][a] - (double) nd.p[a]) / scale[a]);
            lo = max(0, min(255, lo)); hi = max(0, min(255, hi));
            while (lo > 0 && (float) ((double) nd.p[a] + lo * scale[a]) > clo[s][a]) --lo;
            while (hi < 255 && (float) ((double) nd.p[a] + hi * scale[a]) < chi[s][a]) ++hi;
            nd.qlo[a][s] = (uint8_t) lo; nd.qhi[a][s] = (uint8_t) hi;
        }
        if (c.left >= 0) {
            nd.imask |= (uint8_t) (1u << s);
            next[exInner[k] + inner++] = pl[s];
        } else {
            nd.meta[s] = (uint8_t) ((c.count << 5) | triOff);
            leafStart[pl[s]] = nd.triBase + triOff;
            for (uint32_t q = 0; q < c.count; ++q) leafPrims[nd.triBase + triOff + q] = ids[refs[c.start + q].id];
            triOff += c.count;
        }
    }
    nodes8[levelBase + k] = nd;
}

__global__ void k_appendTree(BVHNode *dst, const BVHNode *src, size_t n, uint32_t nodeBase, uint32_t leafBase) {
    const size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
    if (i >= n) return;
    BVHNode nd = src[i];
    for (int side = 0; side < 2; ++side) {
        int32_t &r = side ? nd.right : nd.left;
        if (r >= 0) r += (int32_t) nodeBase;
        else { const uint32_t bits = ~(uint32_t) r; r = (int32_t) ~(((bits & 0x0FFFFFFFu) + leafBase) | (bits & 0xF0000000u)); }
    }
    dst[i] = nd;
}

template <typename T> struct Buf {
    T *p = nullptr;
    size_t n = 0;
    Buf() = default;
    Buf(const Buf &) = delete;
    ~Buf() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t count) {
        if (p && count <= n) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; n = 0;
        const cudaError_t e = cudaMalloc((void **) &p, std::max<size_t>(count, 1) * sizeof(T));
        if (e == cudaSuccess) n = count;
        return e;
    }
    T *release() { T *q = p; p = nullptr; n = 0; return q; }
};

inline unsigned blocksFor(size_t n, int threads) { return (unsigned) std::max<size_t>(1, (n + threads - 1) / threads); }

// B2_COMMIT_TIMING=1: the device phases on stderr, from CUDA events
struct PhaseEvents {
    bool on = getenv("B2_COMMIT_TIMING") != nullptr;
    std::vector<std::pair<const char *, cudaEvent_t>> ev;
    ~PhaseEvents() { for (auto &e : ev) cudaEventDestroy(e.second); }
    cudaError_t mark(const char *what, cudaStream_t st) {
        cudaEvent_t e;
        cudaError_t r = cudaEventCreate(&e);
        if (r != cudaSuccess) return r;
        ev.emplace_back(what, e);
        return cudaEventRecord(e, st);
    }
    float total() const { float ms = 0; if (ev.size() >= 2) cudaEventElapsedTime(&ms, ev.front().second, ev.back().second); return ms; }
    void print() const {
        if (!on) return;
        for (size_t i = 1; i < ev.size(); ++i) {
            float ms = 0;
            cudaEventElapsedTime(&ms, ev[i - 1].second, ev[i].second);
            fprintf(stderr, "[b2 commit]   bvh (device): %-22s %8.1f ms\n", ev[i].first, ms);
        }
    }
};

} // namespace

#define DCK(call)                                                                                            \
    do {                                                                                                     \
        const cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) return std::string("device BVH build: ") + #call + ": " + cudaGetErrorString(e_); \
    } while (0)

cudaError_t appendTreeDevice(BVHNode *dst, const BVHNode *src, size_t n, uint32_t nodeBase, uint32_t leafBase, cudaStream_t st) {
    if (!n) return cudaSuccess;
    k_appendTree<<<blocksFor(n, 256), 256, 0, st>>>(dst, src, n, nodeBase, leafBase);
    return cudaGetLastError();
}

std::string buildBVHDevice(const std::vector<PrimBox> &boxes, const std::vector<uint32_t> &ids, int maxLeaf, int maxDepth, bool wide,
                           cudaStream_t st, DeviceBVHResult &out) {
    if (wide) maxLeaf = std::min(maxLeaf, 3); // a leaf child of the wide node holds at most 3 triangles
    const uint32_t n = (uint32_t) boxes.size();
    if (n == 0) return std::string();
    PhaseEvents ph;
    DCK(ph.mark("start", st));
    Buf<PrimBox> dBoxes;
    Buf<uint32_t> dIds, counters;
    Buf<Ref> refs, scratch;
    Buf<TNode> pool;
    DCK(dBoxes.alloc(n)); DCK(dIds.alloc(n)); DCK(refs.alloc(n)); DCK(scratch.alloc(n));
    DCK(pool.alloc(2 * (size_t) n)); // a binary tree over n primitives has at most 2n - 1 nodes; small subtrees reserve that bound
    DCK(counters.alloc(3));          // pool nodes in use, next level's large nodes, small nodes
    DCK(cudaMemcpyAsync(dBoxes.p, boxes.data(), (size_t) n * sizeof(PrimBox), cudaMemcpyHostToDevice, st));
    DCK(cudaMemcpyAsync(dIds.p, ids.data(), (size_t) n * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    DCK(ph.mark("upload", st));
    k_init<<<blocksFor(n, 256), 256, 0, st>>>(dBoxes.p, n, refs.p);
    DCK(cudaGetLastError());

    // ---- phase 1 ----
    const size_t capL = n / (kSmall + 1) + 2; // open nodes above kSmall at one level
    Buf<Open> cur, nxt, small;
    DCK(cur.alloc(capL)); DCK(nxt.alloc(capL)); DCK(small.alloc(n));
    Buf<uint32_t> acc, bins, blockLeft, blockLeftEx, firstBlock;
    Buf<Work> work;
    Buf<uint2> blk;
    Buf<unsigned char> cubTmp;
    Buf<unsigned long long> keys, keys2;
    Buf<uint32_t> vals, vals2;
    Buf<uint32_t> segBeg, segEnd;
    std::vector<Open> hCur(1);
    hCur[0] = Open{0, 0u, n, 0};
    uint32_t hCounters[3] = {1u, 0u, 0u};
    {
        TNode root;
        memset(&root, 0, sizeof(root));
        root.left = root.right = -1;
        DCK(cudaMemcpyAsync(pool.p, &root, sizeof(root), cudaMemcpyHostToDevice, st));
    }
    if (n <= kSmall) { DCK(cudaMemcpyAsync(small.p, hCur.data(), sizeof(Open), cudaMemcpyHostToDevice, st)); hCur.clear(); hCounters[2] = 1; }
    DCK(cudaMemcpyAsync(counters.p, hCounters, sizeof(hCounters), cudaMemcpyHostToDevice, st));
    if (!hCur.empty()) DCK(cudaMemcpyAsync(cur.p, hCur.data(), sizeof(Open), cudaMemcpyHostToDevice, st));
    std::vector<uint2> hBlk;
    std::vector<uint32_t> hFirst;
    std::vector<Work> hWork;
    while (!hCur.empty()) {
        const uint32_t nL = (uint32_t) hCur.size();
        hBlk.clear(); hFirst.resize(nL);
        for (uint32_t k = 0; k < nL; ++k) {
            hFirst[k] = (uint32_t) hBlk.size();
            for (uint32_t off = 0; off < hCur[k].count; off += kChunk) hBlk.push_back(make_uint2(k, off));
        }
        const uint32_t nB = (uint32_t) hBlk.size();
        DCK(blk.alloc(nB)); DCK(firstBlock.alloc(nL)); DCK(blockLeft.alloc(nB)); DCK(blockLeftEx.alloc(nB));
        DCK(acc.alloc(12 * (size_t) nL)); DCK(bins.alloc((size_t) kBinWords * nL)); DCK(work.alloc(nL));
        DCK(cudaMemcpyAsync(blk.p, hBlk.data(), nB * sizeof(uint2), cudaMemcpyHostToDevice, st));
        DCK(cudaMemcpyAsync(firstBlock.p, hFirst.data(), nL * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        k_accInit<<<blocksFor((size_t) kBinWords * nL, 256), 256, 0, st>>>(nL, acc.p, bins.p);
        k_bounds<<<nB, kThreads, 0, st>>>(refs.p, cur.p, blk.p, acc.p);
        k_decide<<<blocksFor(nL, 128), 128, 0, st>>>(nL, cur.p, acc.p, pool.p, work.p, maxLeaf, maxDepth);
        k_bins<<<nB, kThreads, 0, st>>>(refs.p, cur.p, blk.p, work.p, bins.p);
        k_sah<<<blocksFor(nL, 64), 64, 0, st>>>(nL, bins.p, work.p);
        k_flags<<<nB, kThreads, 0, st>>>(refs.p, cur.p, blk.p, work.p, blockLeft.p);
        DCK(cudaGetLastError());
        size_t tmpBytes = 0;
        DCK(cub::DeviceScan::ExclusiveSum(nullptr, tmpBytes, blockLeft.p, blockLeftEx.p, (int) nB, st));
        DCK(cubTmp.alloc(tmpBytes));
        DCK(cub::DeviceScan::ExclusiveSum(cubTmp.p, tmpBytes, blockLeft.p, blockLeftEx.p, (int) nB, st));
        k_scatter<<<nB, kThreads, 0, st>>>(refs.p, scratch.p, cur.p, blk.p, work.p, blockLeftEx.p, firstBlock.p);
        DCK(cudaGetLastError());
        // object medians (all centroids equal on the split axis, or the depth cap): segmented sort by (centroid, id)
        hWork.resize(nL);
        DCK(cudaMemcpyAsync(hWork.data(), work.p, nL * sizeof(Work), cudaMemcpyDeviceToHost, st));
        DCK(cudaStreamSynchronize(st));
        std::vector<uint32_t> hBeg, hEnd;
        for (uint32_t k = 0; k < nL; ++k)
            if (hWork[k].mode == kMedian) { hBeg.push_back(hCur[k].start); hEnd.push_back(hCur[k].start + hCur[k].count); }
        if (!hBeg.empty()) {
            DCK(keys.alloc(n)); DCK(keys2.alloc(n)); DCK(vals.alloc(n)); DCK(vals2.alloc(n));
            DCK(segBeg.alloc(hBeg.size())); DCK(segEnd.alloc(hEnd.size()));
            DCK(cudaMemcpyAsync(segBeg.p, hBeg.data(), hBeg.size() * 4, cudaMemcpyHostToDevice, st));
            DCK(cudaMemcpyAsync(segEnd.p, hEnd.data(), hEnd.size() * 4, cudaMemcpyHostToDevice, st));
            k_medianKeys<<<nB, kThreads, 0, st>>>(refs.p, cur.p, blk.p, work.p, keys.p, vals.p);
            DCK(cudaGetLastError());
            size_t sortBytes = 0;
            DCK(cub::DeviceSegmentedSort::SortPairs(nullptr, sortBytes, keys.p, keys2.p, vals.p, vals2.p, (int) n, (int) hBeg.size(), segBeg.p,
                                                    segEnd.p, st));
            DCK(cubTmp.alloc(sortBytes));
            DCK(cub::DeviceSegmentedSort::SortPairs(cubTmp.p, sortBytes, keys.p, keys2.p, vals.p, vals2.p, (int) n, (int) hBeg.size(), segBeg.p,
                                                    segEnd.p, st));
            k_medianGather<<<nB, kThreads, 0, st>>>(refs.p, scratch.p, cur.p, blk.p, work.p, vals2.p);
            DCK(cudaGetLastError());
        }
        k_copyBack<<<nB, kThreads, 0, st>>>(refs.p, scratch.p, cur.p, blk.p);
        DCK(cudaMemsetAsync(counters.p + 1, 0, 4, st));
        k_children<<<blocksFor(nL, 128), 128, 0, st>>>(nL, cur.p, work.p, pool.p, counters.p, nxt.p, small.p);
        DCK(cudaGetLastError());
        uint32_t hc[3];
        DCK(cudaMemcpyAsync(hc, counters.p, sizeof(hc), cudaMemcpyDeviceToHost, st));
        DCK(cudaStreamSynchronize(st));
        hCounters[2] = hc[2]; // small nodes accumulate over the levels
        hCur.resize(hc[1]);
        if (hc[1]) DCK(cudaMemcpyAsync(hCur.data(), nxt.p, hc[1] * sizeof(Open), cudaMemcpyDeviceToHost, st));
        DCK(cudaStreamSynchronize(st));
        std::swap(cur.p, nxt.p);
    }
    if (hCounters[2]) {
        k_small<<<blocksFor(hCounters[2], 128), 128, 0, st>>>(hCounters[2], small.p, refs.p, scratch.p, pool.p, counters.p, maxLeaf, maxDepth);
        DCK(cudaGetLastError());
    }
    DCK(cudaMemcpyAsync(hCounters, counters.p, 4, cudaMemcpyDeviceToHost, st));
    TNode hRoot;
    DCK(cudaMemcpyAsync(&hRoot, pool.p, sizeof(TNode), cudaMemcpyDeviceToHost, st));
    DCK(ph.mark("binned SAH (binary)", st));
    DCK(cudaStreamSynchronize(st));
    const uint32_t nPool = hCounters[0];
    float diag = 0; // scene scale for the padding
    for (int i = 0; i < 3; ++i) diag = std::max(diag, hRoot.hi[i] - hRoot.lo[i]);
    const float tiny = diag * 1e-7f + 1e-30f;

    Buf<uint32_t> leafPrims;
    DCK(leafPrims.alloc(n));
    out.leafPrims.resize(n);
    if (hRoot.left < 0) { // the root is a leaf
        k_leafGather<<<blocksFor(n, 256), 256, 0, st>>>(n, refs.p, dIds.p, leafPrims.p);
        DCK(cudaGetLastError());
        DCK(cudaMemcpyAsync(out.leafPrims.data(), leafPrims.p, (size_t) n * 4, cudaMemcpyDeviceToHost, st));
        DCK(cudaStreamSynchronize(st));
        out.rootRef = (int32_t) ~(0u | (hRoot.count << 28));
        out.depth = 1;
        DCK(ph.mark("leaf order readback", st));
        DCK(cudaStreamSynchronize(st));
        out.ms = ph.total();
        ph.print();
        return std::string();
    }

    // ---- phase 2: binary BFS numbering ----
    Buf<int32_t> innerIndex, lvA, lvB;
    Buf<uint32_t> cnt, ex, cnt2, ex2;
    DCK(innerIndex.alloc(nPool)); DCK(lvA.alloc(n)); DCK(lvB.alloc(n)); DCK(cnt.alloc(n)); DCK(ex.alloc(n));
    DCK(cudaMemsetAsync(innerIndex.p, 0xFF, (size_t) nPool * 4, st));
    DCK(cudaMemsetAsync(innerIndex.p, 0, 4, st)); // the root is inner node 0
    DCK(cudaMemsetAsync(lvA.p, 0, 4, st));
    auto exclusiveSum = [&](const uint32_t *in, uint32_t *outp, uint32_t count) -> cudaError_t {
        size_t bytes = 0;
        cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, outp, (int) count, st);
        if (e == cudaSuccess) e = cubTmp.alloc(bytes);
        if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(cubTmp.p, bytes, in, outp, (int) count, st);
        return e;
    };
    auto lastSum = [&](const uint32_t *exArr, const uint32_t *cntArr, uint32_t count, uint32_t &total) -> cudaError_t {
        uint32_t h[2];
        cudaError_t e = cudaMemcpyAsync(&h[0], exArr + count - 1, 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(&h[1], cntArr + count - 1, 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        total = h[0] + h[1];
        return e;
    };
    uint32_t nInner = 0, levels = 0;
    {
        int32_t *curL = lvA.p, *nextL = lvB.p;
        uint32_t nL = 1;
        while (nL) {
            k_innerCount<<<blocksFor(nL, 256), 256, 0, st>>>(nL, curL, pool.p, cnt.p);
            DCK(cudaGetLastError());
            DCK(exclusiveSum(cnt.p, ex.p, nL));
            k_innerNext<<<blocksFor(nL, 256), 256, 0, st>>>(nL, curL, pool.p, ex.p, nInner + nL, innerIndex.p, nextL);
            DCK(cudaGetLastError());
            uint32_t total;
            DCK(lastSum(ex.p, cnt.p, nL, total));
            nInner += nL;
            ++levels;
            nL = total;
            std::swap(curL, nextL);
        }
    }
    out.depth = (int) levels + 1; // deepest inner node's depth + 2
    DCK(ph.mark("binary BFS numbering", st));

    // ---- phase 3: 8-wide collapse ----
    Buf<uint32_t> leafStart;
    Buf<BVH8Node> nodes8;
    if (wide) {
        DCK(leafStart.alloc(nPool)); DCK(nodes8.alloc(nInner)); // one wide node per binary inner node at most
        Buf<int32_t> plans;
        DCK(plans.alloc(8 * (size_t) nInner)); DCK(cnt2.alloc(n)); DCK(ex2.alloc(n));
        int32_t *curL = lvA.p, *nextL = lvB.p;
        DCK(cudaMemsetAsync(curL, 0, 4, st));
        uint32_t nL = 1, levelBase = 0, triCarry = 0, levels8 = 0;
        while (nL) {
            k_widePlan<<<blocksFor(nL, 128), 128, 0, st>>>(nL, curL, pool.p, tiny, plans.p, cnt.p, cnt2.p);
            DCK(cudaGetLastError());
            DCK(exclusiveSum(cnt.p, ex.p, nL));
            DCK(exclusiveSum(cnt2.p, ex2.p, nL));
            k_wideEmit<<<blocksFor(nL, 128), 128, 0, st>>>(nL, plans.p, ex.p, ex2.p, levelBase, triCarry, pool.p, refs.p, dIds.p, tiny, nodes8.p,
                                                           nextL, leafStart.p, leafPrims.p);
            DCK(cudaGetLastError());
            uint32_t totalInner, totalTris;
            DCK(lastSum(ex.p, cnt.p, nL, totalInner));
            DCK(lastSum(ex2.p, cnt2.p, nL, totalTris));
            levelBase += nL;
            triCarry += totalTris;
            ++levels8;
            nL = totalInner;
            std::swap(curL, nextL);
        }
        out.nNodes8 = levelBase;
        out.depth8 = (int) levels8;
        DCK(ph.mark("8-wide collapse", st));
    } else {
        k_leafGather<<<blocksFor(n, 256), 256, 0, st>>>(n, refs.p, dIds.p, leafPrims.p);
        DCK(cudaGetLastError());
    }
    Buf<BVHNode> nodes;
    DCK(nodes.alloc(nInner));
    k_binaryNodes<<<blocksFor(nPool, 256), 256, 0, st>>>(nPool, pool.p, innerIndex.p, wide ? leafStart.p : nullptr, tiny, nodes.p);
    DCK(cudaGetLastError());
    DCK(ph.mark("binary relayout", st));
    DCK(cudaMemcpyAsync(out.leafPrims.data(), leafPrims.p, (size_t) n * 4, cudaMemcpyDeviceToHost, st));
    DCK(ph.mark("leaf order readback", st));
    DCK(cudaStreamSynchronize(st));
    out.ms = ph.total();
    ph.print();
    out.rootRef = 0;
    out.nNodes = nInner;
    out.nodes = nodes.release();
    out.nodes8 = wide ? nodes8.release() : nullptr;
    return std::string();
}

} // namespace b2
