// Plain data shared by the host side (scene commit, render loop) and the kernels: the layout of the
// scene in HBM and of the wavefront path pool.  DESIGN.md "data layout" documents every array.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

// per-lane traversal stack entries in shared memory; the BVH builder caps the tree depth below this
#define B2_STACK_DEPTH 32

namespace b2 {

// One BSDF node, device copy of b2_material_desc plus values precomputed once on the host
struct DMaterial {
    int32_t type, distr, sampleVisible, nested;
    float alphaU, alphaV, eta, thickness;
    float reflectance[3], transmittance[3], etaC[3], kC[3], sigmaA[3];
    uint32_t flags;        // BSDF type flags (bsdf.h:224-285) incl. nested, as BSDF::configure ORs them
    float specSamplingWeight; // coating.cpp:177-181; plastic.cpp:199-202
    int32_t nested2;       // twosided: back-side BSDF
    int32_t nonlinear;     // plastic.cpp:161
    float diffuseReflectance[3]; // plastic
    float fdrInt;          // plastic.cpp:194 (fdrExt is only used by getDiffuseReflectance)
    int32_t tex;           // diffuse: index into DScene::textures of the `bitmap` texture bound to `reflectance`, -1 = constant
};

// One `bitmap` texture (src/textures/bitmap.cpp + include/mitsuba/render/mipmap.h): the MIP pyramid built by the host at commit
// (Lanczos-2 resampling as the reference does), texels as float4 (RGB, channels == 3) or float (luminance, channels == 1)
#define B2_TEX_MAX_LEVELS 17   // 65535 texels on a side (the largest environment map, envmap.cpp:160-162) -> 17 levels
struct DTexture {
    int32_t levels, channels;
    int32_t filter;            // 0 nearest, 1 bilinear, 2 trilinear, 3 ewa (bitmap.cpp:213-230)
    int32_t wrapU, wrapV;      // 0 repeat, 1 clamp, 2 mirror, 3 zero, 4 one (bitmap.cpp:324-338)
    float maxAnisotropy;       // bitmap.cpp:232-235
    float uoffset, voffset, uscale, vscale; // texture.cpp:82-95
    float bsdfScale;           // BSDF::ensureEnergyConservation (bsdf.cpp:88-111): 0.99 / max when the image exceeds 1
    int32_t lw[B2_TEX_MAX_LEVELS], lh[B2_TEX_MAX_LEVELS];
    uint32_t off[B2_TEX_MAX_LEVELS]; // first texel of each level inside `data`
    const void *data;
};

// `envmap` emitter (src/emitters/envmap.cpp): the pyramid as a texture (repeat / clamp, EWA, maxAnisotropy 10, RGB texels padded to
// float4, values half-representable), the sampling tables of configure() (envmap.cpp:260-329) and the 3x3 parts of toWorld / its inverse
struct DEnvMap {
    DTexture tex;
    const float *cdfRows;      // h + 1
    const float *cdfCols;      // h rows of w + 1
    const float *rowWeights;   // h: sin(theta) of the row centres
    float normalization, scale, pixelSizeX, pixelSizeY;
    float toWorld[9], toLocal[9];
    int32_t w, h;
};

// One participating medium + its phase function (device copy of b2_medium_desc; SURVEY.md 8f-1)
struct DMedium {
    int32_t type, phase;      // 0 homogeneous / 1 heterogeneous (Woodcock); 0 isotropic / 1 hg
    float g;
    int32_t strategy;         // homogeneous.cpp:186-222: 0 balance, 1 single, 2 manual
    float sigmaA[3], sigmaS[3];
    float samplingDensity, mediumSamplingWeight;
    float scale, invMaxDensity; // heterogeneous.cpp:185,239-243 (gridvolume maximum value 1)
    float albedo[3];
    int32_t res[3];
    float worldToGrid[12];    // gridvolume.cpp:186-193
    float aabbMin[3], aabbMax[3]; // world box of the density grid (gridvolume.cpp:197-199)
    const float *density;     // res.x * res.y * res.z, x fastest
};

// One item of the top-level BVH of an instanced scene: the world triangles (identity) or one `instance` shape
// (src/shapes/instance.cpp): affine object-to-world rows, its inverse, the root of the shapegroup's BVH and the group's box
struct DInstance {
    float M[12], Minv[12];
    int32_t rootRef;
    int32_t identity;      // 1: world triangles, no transform, no clipping
    int32_t instance;      // index of the instance (statistics / debugging)
    int32_t pad;
    float aabbMin[3], aabbMax[3]; // the group's enlarged kd-tree box in object space (skdtree.h:430-458 clips against it)
    float pad2[2];
};

// Area emitter + its mesh's area distribution (area.cpp, trimesh.cpp:388-403)
struct DEmitter {
    float radiance[3];
    float samplingWeight;
    float invSurfaceArea;
    uint32_t cdfOffset;    // into triCdf (nTri + 1 floats, cdf[0] = 0)
    uint32_t nTri;         // 0: environment emitter, no mesh: `constant` (src/emitters/constant.cpp) or, when DScene::envmap is set, `envmap`
    uint32_t primOffset;   // global prim index of the mesh's first triangle
};

// 64-byte BVH2 node: both children's boxes + child references.
// ref >= 0: inner node index; ref < 0: leaf, bits = ~ref, start = bits & 0x0FFFFFFF (into the
// leaf-ordered TriAccel array), count = bits >> 28.
struct BVHNode {
    float lmin[3], lmax[3], rmin[3], rmax[3];
    int32_t left, right, pad0, pad1;
};
static_assert(sizeof(BVHNode) == 64, "BVHNode must be 64 bytes");

// 80-byte node of the 8-wide tree (after Ylitie, Karras, Laine: "Efficient Incoherent Ray Traversal on GPUs Through Compressed Wide
// BVHs", HPG 2017, restated): the eight child boxes are 8-bit offsets from `p` in units of 2^e per axis (conservative: lo rounded down,
// hi rounded up), internal children are consecutive nodes starting at childBase (in slot order), the <= 3 triangles of each leaf child
// sit at triBase + offset in the leaf-ordered triangle array.  Slot s holds the child that lies towards (s&1 ? +x : -x, s&2 ? +y : -y,
// s&4 ? +z : -z) of the node centre, so a ray with direction octant o visits the hit children in the order of decreasing s ^ (7 ^ o).
struct BVH8Node {
    float p[3];
    int8_t e[3];
    uint8_t imask;        // bit s: child s is an internal node
    uint32_t childBase;   // first internal child
    uint32_t triBase;     // first triangle of this node's leaf children
    uint8_t meta[8];      // leaf child: (triangle count 1..3) << 5 | offset (0..23) from triBase; 0: empty slot or internal child
    uint8_t qlo[3][8], qhi[3][8];
};
static_assert(sizeof(BVH8Node) == 80, "BVH8Node must be 80 bytes");
#define B2_NCLASS 5          // class queues of the material-sorted dispatch: diffuse, roughconductor, roughdielectric, coating, everything else
#define B2_STACK8_DEPTH 28   // uint2 entries per lane of the wide traversal (one pending child group per level)

struct DCamera {
    float camToWorld[16];
    float sampleToCamera[16];
    float nearClip, farClip;
    float invResX, invResY;
    float origin[3];
    int32_t W, H;
    float apertureRadius, focusDistance; // > 0: `thinlens` sensor (src/sensors/thinlens.cpp); 0: pinhole
    float dx[3], dy[3];        // m_dx, m_dy (perspective.cpp:160-163): camera-space offset of one pixel on the near plane
};

// Scene resident in HBM
struct DScene {
    // leaf-ordered TriAccel records, 3 x float4 each (triaccel.h:37-59; word 10 = global prim id)
    const float4 *triAccel;
    // same triangles as three planes (N, d0), (U, -U.p0), (V, -V.p0): branch-free test used by the throughput build
    // (t = (d0 - N.o) / N.d, u = U.P + du, v = V.P + dv); leafPrim maps the leaf-ordered index to the prim id
    const float4 *triPlane;
    const uint32_t *leafPrim;
    // throughput build, flat leaf only: paired records stored TWO WIDE for the packed FP32 instructions (b2_trace.cuh traverseFlat):
    // flatP steps of two parallelograms (6 rows), flatC steps of two coplanar pairs (10 rows), flatS steps of two single triangles
    // (6 rows), in this order; flatIdx[r] = leaf indices of record r's first / second triangle
    const float4 *flatRec;
    const uint2 *flatIdx;
    uint32_t flatP, flatC, flatS, flatBytes;
    uint32_t nLeafTris;
    const DInstance *items;    // instanced scenes only (nItems > 0): top-level items in the order of the top-level leaves
    uint32_t nItems;
    int32_t tlasRoot;          // root reference of the top-level BVH (leaf refs there index `items`)
    int32_t envEmitter;        // index of the environment emitter or -1 (Scene::getEnvironmentEmitter)
    const DEnvMap *envmap;     // non-null: that emitter is an `envmap` (else `constant`)
    float bsCenter[3], bsRadius; // constant.cpp:67-70 m_sceneBSphere: sphere of the scene box (incl. the sensor position), radius x 1.5
    // participating media (volpath): media table and per-prim (interior, exterior) ids, -1 = vacuum; null without media
    const DMedium *media;
    const int2 *primMedia;
    uint32_t nMedia;
    const BVHNode *nodes;
    uint32_t nNodes;
    const BVH8Node *nodes8;    // wide tree of non-instanced BVH scenes (null otherwise): what k_extend / k_occluded / b2_trace walk
    uint32_t nNodes8, stageNodes8;
    int32_t rootRef;           // root child reference (leaf-only scenes: a leaf ref)
    uint32_t rootCount;        // > 0: the whole scene is one flat leaf of rootCount triangles (tiny scenes, tested in lockstep)
    float aabbMin[3], aabbMax[3]; // enlarged scene box (gkdtree.h:1213-1220)
    // per-prim shading data in prim order: verts[3*p+k] = (position k, w = {material id, emitter id, flags} as int bits)
    const float4 *verts;
    // optional: norms[3*p+k] = (vertex normal k, w = dpdu component k); flags bit0 = has normals, bit1 = has dpdu
    const float4 *norms;
    uint32_t nPrims;
    const DMaterial *materials;
    uint32_t nMaterials;
    // bitmap textures (null / 0 without): table, per-prim texc[3*p+k] = (u_k, v_k, dpdv component k, 0), EWA weight table (64 entries)
    const DTexture *textures;
    uint32_t nTextures;
    const float4 *texc;
    const float *ewaLut;
    const DEmitter *emitters;
    uint32_t nEmitters;
    const float *emitterCdf;   // nEmitters + 1
    float emitterNormalization; // DiscreteDistribution::getNormalization (pmf.h)
    const float *triCdf;
    DCamera cam;
    // Sobol tables (sobolseq.h:31-38)
    const uint32_t *sobolM32;  // [1024][52]
    const uint64_t *sobolVdc;  // [25][52]
    const uint64_t *sobolInv;  // [26][52]
    const uint32_t *sobolNib;  // [1024][13][16]: XOR of the 4 columns of nibble p selected by v (b2_host.cpp: buildSobolNibbles)
    // staging limits for shared memory (number of leading BVH nodes / TriAccel records copied by TMA)
    uint32_t stageNodes, stageTris;
    uint32_t stageTriBytes;    // shared memory reserved for the staged triangles: max(stageTris * 48, flatBytes) (the two-wide flat leaf pads odd counts)
    uint32_t leafVote;         // persistent traversal: run the leaf code once this many lanes wait at a leaf (8, set by b2_scene_commit)
    uint32_t missClass;        // material-sorted dispatch: the class queue that takes rays which left the scene (first class present)
    uint32_t refill;           // persistent traversal: refill a warp when at least this many lanes are idle (16, set by b2_scene_commit)
};

struct DFilter {
    float values[32];
    float radius, scaleFactor;
    int32_t borderSize, kind;
};

// Path flags
enum : uint32_t {
    PF_ALIVE = 1u << 0,       // slot holds a path that still needs work
    PF_DONE = 1u << 1,        // path finished: Li must be splatted, slot can be regenerated
    PF_FRESH = 1u << 2,       // ray is the camera ray (EEmittedRadiance still set, depth == 1)
    PF_SCATTERED = 1u << 3,
    PF_DELTA = 1u << 4,       // last sampled lobe was EDelta (path.cpp:261)
    PF_REFN_OK = 1u << 5,     // dot(wo, refN) >= 0 for the pending emitter-hit MIS test (area.cpp:178)
    PF_ALPHA = 1u << 6,       // camera ray hit something
    PF_CAMRAY = 1u << 7,      // volpath: the current segment is still the sensor ray (it carries ray differentials, volpath.cpp:89 / ray.h:150-157)
};

// Wavefront pool: structure of arrays, one entry per in-flight path ("slot"), 16-byte records
struct DPool {
    uint32_t capacity;
    // 32-byte records (one full DRAM sector each, also when slots are written in scattered order by k_generate):
    float4 *ray;       // [2i] = o.xyz, mint ; [2i+1] = d.xyz, w  (w = maxt for the camera ray, else the pdf of the pending BSDF sample; maxt = inf)
    float4 *st;        // [2i] = throughput rgb, eta ; [2i+1] = Li rgb, -
    float4 *hit;       // t, u, v, prim (bits)
    uint2 *smp;        // sampler state: Sobol' index / stream key (lo, hi)
    float2 *pos;       // samplePos (film coordinates of the sample; read again only when the path is splatted)
    uint32_t *pix;     // pixel (y << 16 | x)
    uint32_t *flags;   // PF_* | depth << 8 | sampler dimension << 20
    uint32_t *inst;    // instanced scenes only: item index of the hit (0xFFFFFFFF = none)
    uint2 *vol;        // volpath only: (current medium id or -1, sampler dimension); null for `path`
    // shadow queue (compacted by warp ballot): 48-byte records, everything k_occluded needs
    float4 *shO;       // o.xyz, -
    float4 *shD;       // d.xyz, maxt
    float4 *shC;       // contribution rgb, slot (bits)
    // material-class queues
    uint32_t *matQueue;   // [B2_NCLASS][capacity]: four specialised BSDF classes + the generic one
    // finished-path queues, double buffered: k_shade of iteration k appends to doneQueue[k & 1], k_generate of
    // iteration k + 1 drains it (splat + refill) with full warps
    uint32_t *doneQueue;  // [2][capacity]
    // counters (device, u64): see CTR_*
    unsigned long long *counters;
};

// [CTR_DONE0, CTR_SHADOW, CTR_CLASS0..3, CTR_DONE1] is zeroed per iteration as one 48-byte window that slides by one
// entry with the iteration parity (even: DONE0..CLASS3, odd: SHADOW..DONE1)
enum { CTR_DONE0 = 0, CTR_SHADOW = 1, CTR_CLASS0 = 2, /* 2..5 */ CTR_DONE1 = 6, CTR_NEXT = 7, CTR_ACTIVE = 8, CTR_RAYS = 9, CTR_SHADOWRAYS = 10,
       CTR_PATHLEN = 11, CTR_SAMPLES = 12, CTR_BAD = 13, CTR_DIMOVF = 14, CTR_NODEVIS = 15, CTR_PRIMTESTS = 16,
       CTR_ITER = 17,   // host-loop iteration, advanced on the device by k_publish (one graph serves every iteration)
       CTR_UNOCCLUDED = 18,
       CTR_TICKET_EXT = 19, CTR_TICKET_OCC = 20, // work tickets of the persistent traversal loops (zeroed by k_publish)
       CTR_CLASSG = 21,  // fifth class queue: hits on BSDFs without a specialised shading kernel (null, twosided, dielectric, conductor, plastic)
       // set by k_publish: QUIET, no path alive and every work item handed out; IDLE, QUIET held at the previous iteration, so nothing is
       // left to splat either and k_generate<SLOTS> / k_bounce_flat return at once (the host queues iterations ahead of the end it sees)
       CTR_QUIET = 22, CTR_IDLE = 23,
       CTR_COUNT = 24 };

// progress ring in mapped pinned host memory, written by k_publish: {sequence = iteration + 1, live paths, next work item, -}
#define B2_RING 64
// per-launch device time stamps (%globaltimer): [iteration][stage]{min start, max end}
#define B2_MAX_STAMPS (1u << 17)
enum { STAGE_GENERATE = 0, STAGE_EXTEND = 1, STAGE_SHADE = 2, STAGE_OCCLUDED = 3 };

struct DRender {
    int32_t spp, sampler;
    uint64_t scramble;       // sobol: after the TEA step (sobol.cpp:96-102); independent: seed
    int32_t maxDepth, rrDepth, strictNormals, hideEmitters;
    int32_t sampleLo, sampleHi;
    int32_t integrator;      // 0 path, 1 volpath
    float diffScale;         // 1/sqrt(sampleCount): RayDifferential::scaleDifferential factor (integrator.cpp:144-145,181)
    uint32_t logRes;         // sobol m_logResolution
    float resolution;        // sobol m_resolution
    uint64_t totalWork;      // W*H*(hi-lo)
    uint32_t roundSpp;       // samples every tile receives per round of the work enumeration (divides hi - lo; workItemPixel)
    uint32_t tilesX, tilesY; // whole 8x8 tiles of the film (W / 8, H / 8); the remaining strips are enumerated pixel by pixel
    int32_t drainSlots;      // k_bounce_flat's route: k_generate drains the pool in slot order, no finished-path queue (b2_render)
    float4 *filmRGBA;        // H*W float4 accumulators (r, g, b, weight * alpha)
    float *filmW;            // H*W accumulators of weight * (1 - alpha): touched only by samples whose camera ray missed
    const uint64_t *lookupNib; // [2][13][16] nibble tables of sobol look_up for this render's m: [0] vdc (delta), [1] inv
    uint32_t indexNibbles;   // nibbles needed to cover the largest Sobol' index of this render (<= 13)
    uint32_t frameNibbles, bNibbles; // nibbles of the sample index / of the 2m-bit pixel code in look_up
    unsigned long long *ring;       // device pointer of the mapped host progress ring (B2_RING x 4 words)
    unsigned long long *pixStats;   // null unless per-pixel path diagnostics were requested (flags bit5): [pixel] += (len^2 << 32) | len
    unsigned long long *pathTrace;  // null unless per-sample event traces were requested (flags bit6): [pixel * nS + s] gets one event byte per bounce
    unsigned long long *stampStart; // null unless per-launch timing was requested (b2_render_params.flags bit2)
    unsigned long long *stampEnd;
    int32_t emitterSamples, bsdfSamples; // direct: sample counts of the two strategies (direct.cpp:93-108)
};

} // namespace b2
