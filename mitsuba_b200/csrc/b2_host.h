// Definitions shared by the units of the C-ABI (include/b2mts.h): b2_host.cpp (scene description, render loop, component entry points)
// and b2_commit.cpp (b2_scene_commit).  Private to the library.
#pragma once
#include "../../include/b2mts.h"
#include "b2_types.h"
#include "b2_launch.h"
#include "../host/mipmap.h"

#include <cuda_runtime.h>
#include <atomic>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

using namespace b2;

struct RenderStore;
struct b2_ctx {
    RenderStore *store = nullptr; // render-time buffers (path pool, film accumulators, progress ring) shared by the scenes of this context
    int device = 0;
    int numSMs = 0;
    cudaStream_t stream = nullptr;
    std::string lastError;
    // Sobol tables on the device
    uint32_t *dM32 = nullptr, *dNib = nullptr;
    uint64_t *dVdc = nullptr, *dInv = nullptr;
    std::vector<uint64_t> hVdc, hInv; // host copies: per-render look_up nibble tables are derived from them
    bool tablesLoaded = false;
    int accelBuild = B2_ACCEL_BUILD_HOST; // builder of the scenes created from now on (b2_context_set_accel_build)
};

// Records `msg` as the last error (of `ctx` and of the library) and returns `code`.
int fail(b2_ctx *ctx, int code, const std::string &msg);
#define CK(ctx, call)                                                                                          \
    do {                                                                                                       \
        cudaError_t e_ = (call);                                                                               \
        if (e_ != cudaSuccess)                                                                                 \
            return fail(ctx, B2_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));                 \
    } while (0)

struct HostMesh {
    std::vector<float> P, N, UV;
    std::vector<uint32_t> idx;
    int material = -1, emitter = -1;
    int interior = -1, exterior = -1; // media ids (shape.h:427-435), -1 = vacuum
    int group = -1;                   // >= 0: member of that shapegroup (object space), src/shapes/shapegroup.cpp
    uint32_t primOffset = 0;
};
struct HostEmitter {
    float radiance[3];
    float samplingWeight;
    int mesh = -1;
    bool env = false; // `constant` environment emitter (no parent shape)
};

// Stream rule: every upload and memset the library issues goes on the context stream (b2_ctx::stream), and a host read of device
// memory comes after a synchronise of that stream.  The stream is non-blocking, so it does not wait for the legacy
// default stream that a synchronous cudaMemcpy uses: a kernel on it is only ordered after copies queued on it.  A pageable source may
// go out of scope as soon as cudaMemcpyAsync returns: the copy stages it first.
template <typename T> struct DevBuf {
    T *p = nullptr;
    size_t n = 0;
    ~DevBuf() { release(); }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
    // takes over a cudaMalloc'd array of `count` elements
    void adopt(T *q, size_t count) { release(); p = q; n = count; }
    // gives the array up to the caller, who frees it
    T *detach() { T *q = p; p = nullptr; n = 0; return q; }
    cudaError_t alloc(size_t count) {
        if (count == n && p) return cudaSuccess;
        release();
        n = count;
        if (count == 0) return cudaSuccess;
        return cudaMalloc((void **) &p, count * sizeof(T));
    }
    cudaError_t upload(const std::vector<T> &v, cudaStream_t st) {
        cudaError_t e = alloc(v.size());
        if (e != cudaSuccess || v.empty()) return e;
        return cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, st);
    }
};

// Render-time buffers live in the context, not in the scene: a 4 Mi-path pool is ~0.6 GB, and allocating / freeing it around every
// scene costs tens to hundreds of milliseconds (cudaFree synchronises) -- more than committing a small scene.  One render at a
// time per context (renderMutex); scenes refresh their DPool pointers from here at the start of every b2_render.
struct RenderStore {
    std::mutex renderMutex;
    uint32_t capacity = 0;
    DevBuf<float4> pRay, pSt, pHit, pShO, pShD, pShC;
    DevBuf<uint2> pSmp, pVol;
    DevBuf<uint32_t> pInst;
    DevBuf<float2> pPos;
    DevBuf<uint32_t> pPix, pFlags;
    DevBuf<uint32_t> pMatQueue, pDoneQueue;
    DevBuf<float4> dFilmRGBA;
    DevBuf<float> dFilmW, dFilmOut;
    unsigned long long *hRing = nullptr, *dRing = nullptr; // mapped pinned progress ring written by k_publish
    DevBuf<unsigned long long> dStampStart, dStampEnd;      // per-launch %globaltimer stamps (flags bit2)
    DevBuf<unsigned long long> dPixStats;                   // per-pixel path-length sums (flags bit5)
    DevBuf<unsigned long long> dPathTrace;                  // per-sample event traces (flags bit6)
    ~RenderStore() { if (hRing) cudaFreeHost(hRing); }
};

struct b2_scene {
    b2_ctx *ctx = nullptr;
    std::vector<b2_material_desc> materials;
    std::vector<HostEmitter> emitters;
    std::vector<HostMesh> meshes;
    struct HostMedium { b2_medium_desc desc; std::vector<float> density; };
    struct HostInstance { int group; float M[16], Minv[16]; };
    std::vector<HostInstance> instances;
    int nGroups = 0;
    std::vector<HostMedium> media;
    struct HostTexture { b2_texture_desc desc; std::vector<float> pixels; b2host::MipPyramid mip; };
    std::vector<HostTexture> textures;
    // <emitter type="envmap">: the decoded image and its placement; pyramid + sampling tables are derived at commit
    struct HostEnvMap { int w = 0, h = 0; std::vector<float> pixels; float scale = 1; float toWorld[16], toLocal[16]; b2host::MipPyramid mip; };
    std::unique_ptr<HostEnvMap> envmap;
    DevBuf<float> dEnvTexels, dEnvCdfRows, dEnvCdfCols, dEnvRowWeights;
    DevBuf<DEnvMap> dEnvMap;
    // camera
    float camToWorld[16];
    float sampleToCamera[16];
    float xfov = 0, nearClip = 1e-2f, farClip = 1e4f;
    float apertureRadius = 0, focusDistance = 0;
    int W = 0, H = 0;                 // the film the integrator sees = the crop window (Film::getCropSize)
    int filmW = 0, filmH = 0, cropX = 0, cropY = 0; // full film and crop offset (film.cpp:36-47)
    bool hasCamera = false, committed = false;
    // device scene
    DScene ds{};
    DevBuf<float4> dTriAccel, dTriPlane, dVerts, dNorms;
    DevBuf<uint32_t> dLeafPrim, dFlatIdx;
    DevBuf<float4> dFlatRec;
    DevBuf<BVHNode> dNodes;
    DevBuf<BVH8Node> dNodes8;
    DevBuf<DMaterial> dMaterials;
    DevBuf<DEmitter> dEmitters;
    DevBuf<float> dEmitterCdf, dTriCdf;
    DevBuf<DMedium> dMedia;
    DevBuf<DInstance> dInstances;
    DevBuf<int2> dPrimMedia;
    std::vector<std::unique_ptr<DevBuf<float>>> dDensity;
    DevBuf<DTexture> dTextures;
    std::vector<std::unique_ptr<DevBuf<float>>> dTexData;
    DevBuf<float4> dTexc;
    DevBuf<float> dEwaLut;
    bool hasTransmission = false;  // some BSDF transmits (ETransmission): `path` renders of such scenes use the IEEE kernels (b2_render)
    std::vector<float4> hTriAccelPrimOrder; // for b2_get_triaccel
    LaunchCfg cfgParity, cfgFast;
    bool classPresent[B2_NCLASS] = {false, false, false, false, false}; // [4]: BSDF types without a specialised shading kernel
    // pool
    DPool pool{};
    DevBuf<uint64_t> dLookupNib;
    DevBuf<unsigned long long> dCounters;
    std::vector<cudaEvent_t> timingEvents;                  // per-launch CUDA events (flags bit3)
    std::atomic<int> cancel{0};
    b2_stats stats{};
    int accelBuild = B2_ACCEL_BUILD_HOST;
};

// The kernel build that runs a render or a component call: the IEEE build (b2::parity, -fmad=false) or the throughput build
// (b2::fast), with the launch configuration b2_scene_commit computed for it.
struct Kernels {
    const KernelSet &set;
    LaunchCfg &cfg;
};
inline Kernels kernelsFor(b2_scene *s, bool ieee) {
    if (ieee) return {parity::kernels, s->cfgParity};
    return {fast::kernels, s->cfgFast};
}

// Combined BSDF flags of material `id` (as BSDF::configure ORs the components' types)
uint32_t materialFlags(const std::vector<b2_material_desc> &mats, int id);
