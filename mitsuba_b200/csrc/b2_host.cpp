// C-ABI implementation (include/b2mts.h): scene commit (TriAccel precompute, BVH, CDFs, upload to HBM),
// the wavefront render loop, film handling and the component entry points.
#include "../../include/b2mts.h"
#include "b2_types.h"
#include "b2_launch.h"
#include "bvh_builder.h"
#include "../host/mipmap.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <sched.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <limits>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

using namespace b2;

namespace {
std::string g_lastError;
std::mutex g_errMutex;
}

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
};

static int fail(b2_ctx *ctx, int code, const std::string &msg) {
    {
        std::lock_guard<std::mutex> g(g_errMutex);
        g_lastError = msg;
    }
    if (ctx) ctx->lastError = msg;
    return code;
}
extern "C" int b2_set_error_(b2_ctx *ctx, int code, const char *msg) { return fail(ctx, code, msg ? msg : ""); }
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

template <typename T> struct DevBuf {
    T *p = nullptr;
    size_t n = 0;
    ~DevBuf() { release(); }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
    cudaError_t alloc(size_t count) {
        if (count == n && p) return cudaSuccess;
        release();
        n = count;
        if (count == 0) return cudaSuccess;
        return cudaMalloc((void **) &p, count * sizeof(T));
    }
    cudaError_t upload(const std::vector<T> &v) {
        cudaError_t e = alloc(v.size());
        if (e != cudaSuccess || v.empty()) return e;
        return cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
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
    bool hasNullBsdf = false;
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
    uint32_t nPrims = 0;
    int bvhDepth = 0;
};

// ------------------------------------------------------------------------------------------------
// lifetime
// ------------------------------------------------------------------------------------------------
extern "C" const char *b2_version(void) { return "b2mts 0.1 (sm_90a wavefront path tracer)"; }
extern "C" int b2_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}
extern "C" const char *b2_last_error(b2_ctx *ctx) {
    if (ctx) return ctx->lastError.c_str();
    return g_lastError.c_str();
}

static std::string dataDir() {
    const char *env = getenv("B2MTS_DATA");
    if (env) return env;
    // <dir>/libb2mts.so -> <dir>/data
    Dl_info info;
    if (dladdr((const void *) &b2_version, &info) && info.dli_fname) {
        std::string p(info.dli_fname);
        size_t k = p.find_last_of('/');
        return (k == std::string::npos ? std::string(".") : p.substr(0, k)) + "/data";
    }
    return "data";
}
extern "C" const char *b2_data_dir_(void) { // the data directory, for the scene-file front end (conductor presets)
    static std::string dir = dataDir();
    return dir.c_str();
}
template <typename T> static bool readFile(const std::string &path, std::vector<T> &out, size_t expect) {
    std::ifstream f(path, std::ios::binary);
    if (!f) return false;
    out.resize(expect);
    f.read((char *) out.data(), (std::streamsize) (expect * sizeof(T)));
    return (size_t) f.gcount() == expect * sizeof(T);
}

extern "C" int b2_context_create(int device, b2_ctx **out) {
    if (!out) return fail(nullptr, B2_ERR_INVALID, "b2_context_create: null out pointer");
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0)
        return fail(nullptr, B2_ERR_NO_DEVICE, "no CUDA device available (this library has no CPU fallback)");
    if (device < 0 || device >= n) return fail(nullptr, B2_ERR_INVALID, "device index out of range");
    b2_ctx *ctx = new b2_ctx();
    ctx->store = new RenderStore();
    ctx->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { delete ctx->store; delete ctx; return fail(nullptr, B2_ERR_CUDA, "cudaSetDevice failed"); }
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    ctx->numSMs = prop.multiProcessorCount;
    if (prop.major != 9 || prop.minor != 0) { // sm_90a code runs on compute capability 9.0 only
        delete ctx->store; delete ctx;
        return fail(nullptr, B2_ERR_NO_DEVICE, "device is not compute capability 9.0; kernels are built for sm_90a only");
    }
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx->store; delete ctx; return fail(nullptr, B2_ERR_CUDA, "stream create failed"); }
    // Sobol tables
    std::vector<uint32_t> m32;
    std::vector<uint64_t> vdc, inv;
    std::string dir = dataDir();
    if (!readFile(dir + "/sobol_matrices32.bin", m32, 1024 * 52) || !readFile(dir + "/sobol_vdc.bin", vdc, 25 * 52) ||
        !readFile(dir + "/sobol_vdc_inv.bin", inv, 26 * 52)) {
        cudaStreamDestroy(ctx->stream);
        delete ctx->store; delete ctx;
        return fail(nullptr, B2_ERR_IO, "cannot read Sobol tables from " + dir + " (set B2MTS_DATA)");
    }
    vdc.resize(26 * 52, 0);
    ctx->hVdc = vdc; ctx->hInv = inv;
    {   // nibble-sliced direction matrices: nib[d][p][v] = XOR_{k in bits(v)} m32[d][4p + k]  (b2_sampler.cuh: sobolSampleNib)
        std::vector<uint32_t> nib((size_t) 1024 * 13 * 16, 0u);
        for (int d = 0; d < 1024; ++d)
            for (int p = 0; p < 13; ++p)
                for (int v = 0; v < 16; ++v) {
                    uint32_t x = 0;
                    for (int k = 0; k < 4; ++k)
                        if ((v >> k) & 1) x ^= m32[(size_t) d * 52 + 4 * p + k];
                    nib[((size_t) d * 13 + p) * 16 + v] = x;
                }
        if (cudaMalloc((void **) &ctx->dNib, nib.size() * 4) != cudaSuccess ||
            cudaMemcpy(ctx->dNib, nib.data(), nib.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
            b2_context_destroy(ctx);
            return fail(nullptr, B2_ERR_CUDA, "b2_context_create: upload of the Sobol' nibble tables failed");
        }
    }
    if (cudaMalloc((void **) &ctx->dM32, m32.size() * 4) != cudaSuccess || cudaMalloc((void **) &ctx->dVdc, vdc.size() * 8) != cudaSuccess ||
        cudaMalloc((void **) &ctx->dInv, inv.size() * 8) != cudaSuccess ||
        cudaMemcpy(ctx->dM32, m32.data(), m32.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(ctx->dVdc, vdc.data(), vdc.size() * 8, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(ctx->dInv, inv.data(), inv.size() * 8, cudaMemcpyHostToDevice) != cudaSuccess) {
        b2_context_destroy(ctx);
        return fail(nullptr, B2_ERR_CUDA, "b2_context_create: upload of the Sobol' tables failed");
    }
    ctx->tablesLoaded = true;
    *out = ctx;
    return B2_OK;
}
extern "C" void b2_context_destroy(b2_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->dM32) cudaFree(ctx->dM32);
    if (ctx->dNib) cudaFree(ctx->dNib);
    if (ctx->dVdc) cudaFree(ctx->dVdc);
    if (ctx->dInv) cudaFree(ctx->dInv);
    delete ctx->store;
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}
extern "C" int b2_scene_create(b2_ctx *ctx, b2_scene **out) {
    if (!ctx || !out) return fail(ctx, B2_ERR_INVALID, "b2_scene_create: null argument");
    b2_scene *s = new b2_scene();
    s->ctx = ctx;
    *out = s;
    return B2_OK;
}
extern "C" void b2_scene_destroy(b2_scene *s) {
    if (!s) return;
    cudaSetDevice(s->ctx->device);
    for (auto e : s->timingEvents) cudaEventDestroy(e);
    delete s;
}

// ------------------------------------------------------------------------------------------------
// scene description
// ------------------------------------------------------------------------------------------------
static void mat4mul(const double *a, const double *b, double *c) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double s = 0;
            for (int k = 0; k < 4; ++k) s += a[i * 4 + k] * b[k * 4 + j];
            c[i * 4 + j] = s;
        }
}
static bool mat4inv(const double *m, double *inv) {
    double a[4][8];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) { a[i][j] = m[i * 4 + j]; a[i][4 + j] = i == j ? 1.0 : 0.0; }
    for (int c = 0; c < 4; ++c) {
        int piv = c;
        for (int r = c + 1; r < 4; ++r)
            if (std::fabs(a[r][c]) > std::fabs(a[piv][c])) piv = r;
        if (std::fabs(a[piv][c]) < 1e-300) return false;
        if (piv != c)
            for (int j = 0; j < 8; ++j) std::swap(a[piv][j], a[c][j]);
        double d = a[c][c];
        for (int j = 0; j < 8; ++j) a[c][j] /= d;
        for (int r = 0; r < 4; ++r)
            if (r != c) {
                double f = a[r][c];
                if (f != 0)
                    for (int j = 0; j < 8; ++j) a[r][j] -= f * a[c][j];
            }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) inv[i * 4 + j] = a[i][4 + j];
    return true;
}

// perspective.cpp:133-153 evaluated in double, rounded once: cameraToSample = scale(1/relSize) * translate(-relOffset) *
// scale(-0.5, -0.5*aspect, 1) * translate(-1, -1/aspect, 0) * perspective(xfov, near, far), aspect from the FULL film
static bool deriveSampleToCamera(b2_scene *s) {
    const double aspect = (double) s->filmW / (double) s->filmH;
    const double recip = 1.0 / ((double) s->farClip - (double) s->nearClip);
    const double cot = 1.0 / std::tan(((double) s->xfov / 2.0) * (M_PI / 180.0));
    const double relSX = (double) s->W / s->filmW, relSY = (double) s->H / s->filmH, relOX = (double) s->cropX / s->filmW, relOY = (double) s->cropY / s->filmH;
    double persp[16] = {cot, 0, 0, 0, 0, cot, 0, 0, 0, 0, s->farClip * recip, -(double) s->nearClip * s->farClip * recip, 0, 0, 1, 0};
    double tr[16] = {1, 0, 0, -1, 0, 1, 0, -1.0 / aspect, 0, 0, 1, 0, 0, 0, 0, 1};
    double sc[16] = {-0.5, 0, 0, 0, 0, -0.5 * aspect, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    double ctr[16] = {1, 0, 0, -relOX, 0, 1, 0, -relOY, 0, 0, 1, 0, 0, 0, 0, 1};
    double csc[16] = {1.0 / relSX, 0, 0, 0, 0, 1.0 / relSY, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    double t1[16], t2[16], t3[16], c2s[16], s2c[16];
    mat4mul(tr, persp, t1);
    mat4mul(sc, t1, t2);
    mat4mul(ctr, t2, t3);
    mat4mul(csc, t3, c2s);
    if (!mat4inv(c2s, s2c)) return false;
    for (int i = 0; i < 16; ++i) s->sampleToCamera[i] = (float) s2c[i];
    return true;
}

extern "C" int b2_scene_set_camera(b2_scene *s, const float to_world[16], float xfov_deg, float near_clip, float far_clip, int width,
                                   int height) {
    if (!s || !to_world) return fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_scene_set_camera: null argument");
    if (width <= 0 || height <= 0 || width > 65535 || height > 65535) return fail(s->ctx, B2_ERR_INVALID, "film size must be in [1, 65535]");
    if (near_clip <= 0) return fail(s->ctx, B2_ERR_INVALID, "The 'nearClip' parameter must be greater than zero!");   // sensor.cpp:164-165
    if (near_clip >= far_clip) return fail(s->ctx, B2_ERR_INVALID, "The 'nearClip' parameter must be smaller than 'farClip'."); // :166-167
    memcpy(s->camToWorld, to_world, 64);
    s->xfov = xfov_deg; s->nearClip = near_clip; s->farClip = far_clip;
    s->filmW = width; s->filmH = height;
    s->cropX = 0; s->cropY = 0; s->W = width; s->H = height;
    if (!deriveSampleToCamera(s)) return fail(s->ctx, B2_ERR_INVALID, "singular camera matrix");
    s->hasCamera = true;
    s->committed = false;
    return B2_OK;
}
// Film crop window (film.cpp:36-47): the render covers crop_width x crop_height pixels whose upper left corner sits at
// (crop_offset_x, crop_offset_y) of the full film given to b2_scene_set_camera.  As in the reference the cropped film IS the film the
// integrator sees from then on (Film::getCropSize: sample positions, the Sobol' resolution, blocks and the output buffer are relative
// to the crop window); only the sensor's sampleToCamera changes (perspective.cpp:133-153, relSize / relOffset).
extern "C" int b2_scene_set_crop(b2_scene *s, int crop_offset_x, int crop_offset_y, int crop_width, int crop_height) {
    if (!s) return fail(nullptr, B2_ERR_INVALID, "b2_scene_set_crop: null scene");
    if (!s->hasCamera) return fail(s->ctx, B2_ERR_INVALID, "b2_scene_set_crop: set the camera first");
    if (crop_offset_x < 0 || crop_offset_y < 0 || crop_width <= 0 || crop_height <= 0 || crop_offset_x + crop_width > s->filmW ||
        crop_offset_y + crop_height > s->filmH)
        return fail(s->ctx, B2_ERR_INVALID, "Invalid crop window specification!"); // film.cpp:44-48
    s->cropX = crop_offset_x; s->cropY = crop_offset_y; s->W = crop_width; s->H = crop_height;
    if (!deriveSampleToCamera(s)) return fail(s->ctx, B2_ERR_INVALID, "singular camera matrix");
    s->committed = false;
    return B2_OK;
}
// <sensor type="thinlens">: apertureRadius (required there, thinlens.cpp:132-142) and focusDistance (sensor.cpp:162, default farClip);
// call after b2_scene_set_camera.  aperture_radius = 0 returns to the pinhole camera.
extern "C" int b2_scene_set_thinlens(b2_scene *s, float aperture_radius, float focus_distance) {
    if (!s) return fail(nullptr, B2_ERR_INVALID, "b2_scene_set_thinlens: null scene");
    if (!s->hasCamera) return fail(s->ctx, B2_ERR_INVALID, "b2_scene_set_thinlens: set the camera first");
    if (aperture_radius < 0) return fail(s->ctx, B2_ERR_INVALID, "thinlens: 'apertureRadius' must be non-negative");
    if (aperture_radius > 0 && !(focus_distance > 0)) return fail(s->ctx, B2_ERR_INVALID, "thinlens: 'focusDistance' must be positive");
    s->apertureRadius = aperture_radius; s->focusDistance = focus_distance;
    s->committed = false;
    return B2_OK;
}
extern "C" int b2_scene_get_sample_to_camera(b2_scene *s, float out[16]) {
    if (!s || !s->hasCamera) return fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "camera not set");
    memcpy(out, s->sampleToCamera, 64);
    return B2_OK;
}
extern "C" int b2_scene_film_size(b2_scene *s, int *width, int *height) {
    if (!s || !s->hasCamera || !width || !height) return fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "camera not set");
    *width = s->W; *height = s->H;
    return B2_OK;
}
static uint32_t materialFlags(const std::vector<b2_material_desc> &mats, int id);
extern "C" int b2_scene_add_material(b2_scene *s, const b2_material_desc *m) {
    if (!s || !m) { fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_scene_add_material: null argument"); return -1; }
    if (m->type < 0 || m->type > B2_BSDF_PLASTIC) { fail(s->ctx, B2_ERR_INVALID, "unknown BSDF type"); return -1; }
    if (m->type == B2_BSDF_COATING) {
        if (m->nested < 0 || m->nested >= (int) s->materials.size()) { fail(s->ctx, B2_ERR_INVALID, "coating: A child BSDF instance is required"); return -1; }
        if (s->materials[m->nested].type == B2_BSDF_COATING) { fail(s->ctx, B2_ERR_INVALID, "coating over coating is not supported on the device"); return -1; }
    }
    if (m->type == B2_BSDF_TWOSIDED) { // twosided.cpp:87-107
        const int n0 = m->nested, n1 = m->nested2;
        if (n0 < 0 || n0 >= (int) s->materials.size()) { fail(s->ctx, B2_ERR_INVALID, "A nested one-sided material is required!"); return -1; }
        if (n1 < 0 || n1 >= (int) s->materials.size()) { fail(s->ctx, B2_ERR_INVALID, "twosided: invalid back-side material id"); return -1; }
        for (int n : {n0, n1}) {
            const int t = s->materials[n].type;
            if (t == B2_BSDF_TWOSIDED) { fail(s->ctx, B2_ERR_INVALID, "twosided inside twosided is not supported on the device"); return -1; }
            if (materialFlags(s->materials, n) & 0x55u /* ETransmission */) { fail(s->ctx, B2_ERR_INVALID, "Only materials without a transmission component can be nested!"); return -1; }
        }
    }
    if (m->type == B2_BSDF_COATING && s->materials[m->nested].type == B2_BSDF_TWOSIDED) { fail(s->ctx, B2_ERR_INVALID, "coating over twosided is not supported on the device"); return -1; }
    if ((m->type == B2_BSDF_DIELECTRIC || m->type == B2_BSDF_PLASTIC) && m->eta <= 0) { fail(s->ctx, B2_ERR_INVALID, "The interior and exterior indices of refraction must be positive!"); return -1; }
    if ((m->type == B2_BSDF_ROUGHDIELECTRIC || m->type == B2_BSDF_COATING) && (m->eta <= 0 || m->eta == 1.0f)) {
        fail(s->ctx, B2_ERR_INVALID, "The interior and exterior indices of refraction must be positive and differ!"); // roughdielectric.cpp:196-198
        return -1;
    }
    if (m->reflectance_texture != 0) {
        if (m->type != B2_BSDF_DIFFUSE && m->type != B2_BSDF_PLASTIC && m->type != B2_BSDF_ROUGHCONDUCTOR && m->type != B2_BSDF_CONDUCTOR) { fail(s->ctx, B2_ERR_INVALID, "bitmap textures are supported on the 'reflectance' of diffuse, the 'specularReflectance' of roughconductor / conductor and the 'diffuseReflectance' of plastic only"); return -1; }
        if (m->reflectance_texture < 0 || m->reflectance_texture > (int) s->textures.size()) { fail(s->ctx, B2_ERR_INVALID, "invalid texture id"); return -1; }
    }
    s->materials.push_back(*m);
    s->committed = false;
    return (int) s->materials.size() - 1;
}
// Texture plugin instance -> id (>= 0) or -1
extern "C" int b2_scene_add_texture(b2_scene *s, const b2_texture_desc *t) {
    if (!s || !t || !t->pixels) { fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_scene_add_texture: null argument"); return -1; }
    if (t->width <= 0 || t->height <= 0 || (t->channels != 1 && t->channels != 3)) { fail(s->ctx, B2_ERR_INVALID, "The input image has an unsupported pixel format!"); return -1; } // bitmap.cpp:276-278
    if (t->filter_type < B2_TEX_NEAREST || t->filter_type > B2_TEX_EWA) { fail(s->ctx, B2_ERR_INVALID, "Invalid filter type, must be 'ewa', 'trilinear', or 'nearest'!"); return -1; } // bitmap.cpp:228-230
    for (int w : {t->wrap_u, t->wrap_v})
        if (w < B2_WRAP_REPEAT || w > B2_WRAP_ONE) { fail(s->ctx, B2_ERR_INVALID, "Invalid wrap mode, must be 'repeat', 'clamp', 'black', or 'white'!"); return -1; } // bitmap.cpp:335-337
    if ((uint64_t) t->width * (uint64_t) t->height > (1ull << 28)) { fail(s->ctx, B2_ERR_INVALID, "texture too large"); return -1; }
    b2_scene::HostTexture ht;
    ht.desc = *t;
    ht.pixels.assign(t->pixels, t->pixels + (size_t) t->width * t->height * t->channels);
    ht.desc.pixels = nullptr;
    if (ht.desc.filter_type != B2_TEX_EWA) ht.desc.max_anisotropy = 1.0f; // bitmap.cpp:234-235
    s->textures.push_back(std::move(ht));
    s->committed = false;
    return (int) s->textures.size() - 1;
}
extern "C" int b2_scene_add_area_emitter(b2_scene *s, const float radiance[3], float sampling_weight) {
    if (!s || !radiance) { fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_scene_add_area_emitter: null argument"); return -1; }
    HostEmitter e;
    memcpy(e.radiance, radiance, 12);
    e.samplingWeight = sampling_weight;
    s->emitters.push_back(e);
    s->committed = false;
    return (int) s->emitters.size() - 1;
}
// <emitter type="constant"> (src/emitters/constant.cpp:47-52); one environment emitter per scene (scene.cpp:510-514)
extern "C" int b2_scene_add_constant_emitter(b2_scene *s, const float radiance[3], float sampling_weight) {
    if (!s || !radiance) { fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_scene_add_constant_emitter: null argument"); return -1; }
    for (auto &e : s->emitters)
        if (e.env) { fail(s->ctx, B2_ERR_INVALID, "The scene may only contain one environment emitter"); return -1; }
    HostEmitter e;
    memcpy(e.radiance, radiance, 12);
    e.samplingWeight = sampling_weight;
    e.env = true;
    s->emitters.push_back(e);
    s->committed = false;
    return (int) s->emitters.size() - 1;
}
// <emitter type="envmap"> (src/emitters/envmap.cpp:106-181): `pixels` = the decoded image, linear float RGB, row-major, top row first
extern "C" int b2_scene_add_envmap_emitter(b2_scene *s, int width, int height, const float *pixels, float scale, const float *to_world, const float *to_local,
                                           float sampling_weight) {
    if (!s || !pixels) { fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_scene_add_envmap_emitter: null argument"); return -1; }
    if ((to_world == nullptr) != (to_local == nullptr)) { fail(s->ctx, B2_ERR_INVALID, "b2_scene_add_envmap_emitter: to_world and to_local go together"); return -1; }
    for (auto &e : s->emitters)
        if (e.env) { fail(s->ctx, B2_ERR_INVALID, "The scene may only contain one environment emitter"); return -1; } // scene.cpp:510-514
    if (width <= 0 || height <= 0) { fail(s->ctx, B2_ERR_INVALID, "b2_scene_add_envmap_emitter: empty image"); return -1; }
    if (std::max(width, height) > 0xFFFF) { fail(s->ctx, B2_ERR_INVALID, "Environment maps images must be smaller than 65536  pixels in width and height"); return -1; } // envmap.cpp:160-162
    std::unique_ptr<b2_scene::HostEnvMap> em(new b2_scene::HostEnvMap());
    em->w = width; em->h = height; em->scale = scale;
    em->pixels.assign(pixels, pixels + (size_t) width * height * 3);
    static const float I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    memcpy(em->toWorld, to_world ? to_world : I, 64); memcpy(em->toLocal, to_local ? to_local : I, 64);
    // the checks of configure() (envmap.cpp:311-315) need the luminance sum; a cheap pass over the image tells the same
    double sum = 0;
    for (float v : em->pixels) { if (!std::isfinite(v)) { fail(s->ctx, B2_ERR_INVALID, "The environment map contains an invalid floating point value (nan/inf) -- giving up."); return -1; } sum += std::max(v, 0.0f); }
    if (sum == 0) { fail(s->ctx, B2_ERR_INVALID, "The environment map is completely black -- this is not allowed."); return -1; }
    s->envmap = std::move(em);
    HostEmitter e;
    e.radiance[0] = e.radiance[1] = e.radiance[2] = 0.0f;
    e.samplingWeight = sampling_weight;
    e.env = true;
    s->emitters.push_back(e);
    s->committed = false;
    return (int) s->emitters.size() - 1;
}
extern "C" int b2_scene_add_mesh(b2_scene *s, const float *P, const float *N, const float *UV, uint32_t nV, const uint32_t *idx, uint32_t nT,
                                 int material_id, int emitter_id) {
    if (!s || !P || !idx) { fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_scene_add_mesh: null argument"); return -1; }
    if (nT == 0) { fail(s->ctx, B2_ERR_INVALID, "Encountered an empty triangle mesh!"); return -1; } // trimesh.cpp:389-392
    if (material_id < 0 || material_id >= (int) s->materials.size()) { fail(s->ctx, B2_ERR_INVALID, "invalid material id"); return -1; }
    if (emitter_id >= (int) s->emitters.size()) { fail(s->ctx, B2_ERR_INVALID, "invalid emitter id"); return -1; }
    if (emitter_id >= 0 && s->emitters[emitter_id].env) { fail(s->ctx, B2_ERR_INVALID, "an environment emitter cannot be attached to a shape"); return -1; }
    if (emitter_id >= 0 && s->emitters[emitter_id].mesh >= 0) { fail(s->ctx, B2_ERR_INVALID, "An area light cannot be parent of multiple shapes"); return -1; } // area.cpp:190-192
    for (uint32_t i = 0; i < 3 * nT; ++i)
        if (idx[i] >= nV) { fail(s->ctx, B2_ERR_INVALID, "triangle index out of range"); return -1; }
    HostMesh m;
    m.P.assign(P, P + 3 * (size_t) nV);
    if (N) m.N.assign(N, N + 3 * (size_t) nV);
    if (UV) m.UV.assign(UV, UV + 2 * (size_t) nV);
    m.idx.assign(idx, idx + 3 * (size_t) nT);
    m.material = material_id;
    m.emitter = emitter_id;
    if (emitter_id >= 0) s->emitters[emitter_id].mesh = (int) s->meshes.size();
    s->meshes.push_back(std::move(m));
    s->committed = false;
    return (int) s->meshes.size() - 1;
}

// Medium plugin instance + phase function (src/medium/{homogeneous,heterogeneous}.cpp, src/phase/{isotropic,hg}.cpp)
extern "C" int b2_scene_add_medium(b2_scene *s, const b2_medium_desc *m) {
    if (!s || !m) { fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_scene_add_medium: null argument"); return -1; }
    if (m->type != B2_MEDIUM_HOMOGENEOUS && m->type != B2_MEDIUM_HETEROGENEOUS) { fail(s->ctx, B2_ERR_INVALID, "unknown medium type"); return -1; }
    if (m->phase != B2_PHASE_ISOTROPIC && m->phase != B2_PHASE_HG) { fail(s->ctx, B2_ERR_INVALID, "unknown phase function"); return -1; }
    b2_scene::HostMedium hm;
    hm.desc = *m;
    if (m->type == B2_MEDIUM_HETEROGENEOUS) {
        if (!m->density) { fail(s->ctx, B2_ERR_INVALID, "No density specified!"); return -1; } // heterogeneous.cpp:230
        if (m->res[0] < 2 || m->res[1] < 2 || m->res[2] < 2) { fail(s->ctx, B2_ERR_INVALID, "density grid needs at least 2 samples per axis"); return -1; }
        if (!(m->scale > 0)) { fail(s->ctx, B2_ERR_INVALID, "heterogeneous medium: 'scale' must be positive"); return -1; }
        const size_t n = (size_t) m->res[0] * m->res[1] * m->res[2];
        hm.density.assign(m->density, m->density + n);
    } else {
        if (m->strategy < 0 || m->strategy > 2) { fail(s->ctx, B2_ERR_INVALID, "Specified an unknown sampling strategy"); return -1; } // homogeneous.cpp:220
    }
    hm.desc.density = nullptr;
    s->media.push_back(std::move(hm));
    s->committed = false;
    return (int) s->media.size() - 1;
}
// <ref name="interior"/"exterior"> children of a shape (shape.cpp:160-176)
extern "C" int b2_scene_set_mesh_media(b2_scene *s, int mesh, int interior, int exterior) {
    if (!s) return fail(nullptr, B2_ERR_INVALID, "b2_scene_set_mesh_media: null scene");
    if (mesh < 0 || mesh >= (int) s->meshes.size()) return fail(s->ctx, B2_ERR_INVALID, "invalid mesh id");
    if (interior >= (int) s->media.size() || exterior >= (int) s->media.size()) return fail(s->ctx, B2_ERR_INVALID, "invalid medium id");
    s->meshes[mesh].interior = interior < 0 ? -1 : interior;
    s->meshes[mesh].exterior = exterior < 0 ? -1 : exterior;
    s->committed = false;
    return B2_OK;
}

// <shape type="shapegroup"> / <shape type="instance"> (src/shapes/{shapegroup,instance}.cpp)
extern "C" int b2_scene_add_shapegroup(b2_scene *s) {
    if (!s) { fail(nullptr, B2_ERR_INVALID, "b2_scene_add_shapegroup: null scene"); return -1; }
    s->committed = false;
    return s->nGroups++;
}
extern "C" int b2_scene_set_mesh_group(b2_scene *s, int mesh, int group) {
    if (!s) return fail(nullptr, B2_ERR_INVALID, "b2_scene_set_mesh_group: null scene");
    if (mesh < 0 || mesh >= (int) s->meshes.size() || group < 0 || group >= s->nGroups) return fail(s->ctx, B2_ERR_INVALID, "invalid mesh or shapegroup id");
    if (s->meshes[mesh].emitter >= 0) return fail(s->ctx, B2_ERR_INVALID, "Instancing of emitters is not supported"); // shapegroup.cpp:115-116
    s->meshes[mesh].group = group;
    s->committed = false;
    return B2_OK;
}
extern "C" int b2_scene_add_instance(b2_scene *s, int group, const float to_world[16], const float to_object[16]) {
    if (!s || !to_world || !to_object) { fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_scene_add_instance: null argument"); return -1; }
    if (group < 0 || group >= s->nGroups) { fail(s->ctx, B2_ERR_INVALID, "A reference to a 'shapegroup' must be specified!"); return -1; } // instance.cpp:75-78
    b2_scene::HostInstance in;
    in.group = group;
    memcpy(in.M, to_world, 64); memcpy(in.Minv, to_object, 64);
    s->instances.push_back(in);
    s->committed = false;
    return (int) s->instances.size() - 1;
}

// ------------------------------------------------------------------------------------------------
// commit
// ------------------------------------------------------------------------------------------------
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

static uint32_t materialFlags(const std::vector<b2_material_desc> &mats, int id) {
    // combined BSDF type as BSDF::configure ORs the components
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
extern "C" int b2_scene_commit(b2_scene *s) {
    if (!s) return fail(nullptr, B2_ERR_INVALID, "b2_scene_commit: null scene");
    b2_ctx *ctx = s->ctx;
    if (!s->hasCamera) return fail(ctx, B2_ERR_INVALID, "scene has no sensor");
    CK(ctx, cudaSetDevice(ctx->device));
    CommitClock clk;
    for (size_t e = 0; e < s->emitters.size(); ++e)
        if (s->emitters[e].mesh < 0 && !s->emitters[e].env) return fail(ctx, B2_ERR_INVALID, "area emitter without a parent shape");
    // ---- emitter order of Scene::m_emitters: emitters that are direct children of the scene (`constant`) are appended by
    // Scene::addChild (scene.cpp:510-516); the area emitters of shapes only join in Scene::initialize -> addShape (scene.cpp:322-335,
    // :570-571), i.e. behind them and in shape order, whatever the document order.  emOrder: device index -> id, emIndex: the inverse ----
    std::vector<int> emOrder, emIndex(s->emitters.size(), -1);
    for (size_t e = 0; e < s->emitters.size(); ++e) if (s->emitters[e].env) emOrder.push_back((int) e);
    for (auto &m : s->meshes) if (m.emitter >= 0) emOrder.push_back(m.emitter);
    for (size_t k = 0; k < emOrder.size(); ++k) emIndex[emOrder[k]] = (int) k;
    // ---- flatten meshes: prim order = mesh order, triangle order (skdtree.cpp:68-72 m_shapeMap) ----
    size_t nPrims = 0;
    for (auto &m : s->meshes) { m.primOffset = (uint32_t) nPrims; nPrims += m.idx.size() / 3; }
    if (nPrims >= (1u << 28)) return fail(ctx, B2_ERR_INVALID, "too many triangles (limit 2^28)");
    s->nPrims = (uint32_t) nPrims;
    bool anyNorm = false;
    for (auto &m : s->meshes) anyNorm |= !m.N.empty() || !m.UV.empty();
    const bool anyTex = !s->textures.empty();
    std::vector<float4> verts(3 * nPrims), norms(anyNorm ? 3 * nPrims : 0), triAccel(3 * nPrims), texc(anyTex && anyNorm ? 3 * nPrims : 0);
    // candidate primitives per acceleration structure: bucket 0 = world, bucket g + 1 = shapegroup g
    const bool instanced = !s->instances.empty();
    std::vector<std::vector<PrimBox>> bBoxes(1 + (size_t) s->nGroups);
    std::vector<std::vector<uint32_t>> bIds(1 + (size_t) s->nGroups);
    std::vector<PrimBox> &boxes = bBoxes[0];
    std::vector<uint32_t> &ids = bIds[0];
    boxes.reserve(nPrims); ids.reserve(nPrims);
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    const int hostThreads = usableThreads();
    std::vector<PrimBox> primBox(nPrims);          // per-prim boxes in prim order; compacted into the buckets (minus degenerates) below
    std::vector<uint8_t> primDegenerate(nPrims, 0);
    for (size_t mi = 0; mi < s->meshes.size(); ++mi) {
        const HostMesh &m = s->meshes[mi];
        const size_t nT = m.idx.size() / 3;
        parallelFor(nT, hostThreads, [&](size_t jlo, size_t jhi) {
        for (size_t j = jlo; j < jhi; ++j) {
            const size_t p = m.primOffset + j;
            const uint32_t i0 = m.idx[3 * j], i1 = m.idx[3 * j + 1], i2 = m.idx[3 * j + 2];
            const float *p0 = &m.P[3 * i0], *p1 = &m.P[3 * i1], *p2 = &m.P[3 * i2];
            uint32_t tflags = (m.N.empty() ? 0u : 1u) | (m.UV.empty() ? 0u : 2u);
            int matBits = m.material, emBits = m.emitter >= 0 ? emIndex[m.emitter] : -1;
            float w0, w1, w2;
            memcpy(&w0, &matBits, 4); memcpy(&w1, &emBits, 4); memcpy(&w2, &tflags, 4);
            verts[3 * p] = make_float4(p0[0], p0[1], p0[2], w0);
            verts[3 * p + 1] = make_float4(p1[0], p1[1], p1[2], w1);
            verts[3 * p + 2] = make_float4(p2[0], p2[1], p2[2], w2);
            if (anyNorm) {
                float n[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, dpdu[3] = {0, 0, 0}, dpdv[3] = {0, 0, 0};
                if (!m.N.empty()) {
                    memcpy(n[0], &m.N[3 * i0], 12); memcpy(n[1], &m.N[3 * i1], 12); memcpy(n[2], &m.N[3 * i2], 12);
                }
                if (!m.UV.empty()) { // TriMesh::computeUVTangents, trimesh.cpp:683-735
                    H3 dP1 = sub3(p1, p0), dP2 = sub3(p2, p0);
                    float du1 = m.UV[2 * i1] - m.UV[2 * i0], dv1 = m.UV[2 * i1 + 1] - m.UV[2 * i0 + 1];
                    float du2 = m.UV[2 * i2] - m.UV[2 * i0], dv2 = m.UV[2 * i2 + 1] - m.UV[2 * i0 + 1];
                    H3 nn = cross3(dP1, dP2);
                    float length = std::sqrt(nn.x * nn.x + nn.y * nn.y + nn.z * nn.z);
                    if (length != 0) {
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
                }
                norms[3 * p] = make_float4(n[0][0], n[0][1], n[0][2], dpdu[0]);
                norms[3 * p + 1] = make_float4(n[1][0], n[1][1], n[1][2], dpdu[1]);
                norms[3 * p + 2] = make_float4(n[2][0], n[2][1], n[2][2], dpdu[2]);
                if (!texc.empty() && !m.UV.empty()) { // texture coordinates of the three vertices + dpdv of computeUVTangents
                    texc[3 * p] = make_float4(m.UV[2 * i0], m.UV[2 * i0 + 1], dpdv[0], 0.0f);
                    texc[3 * p + 1] = make_float4(m.UV[2 * i1], m.UV[2 * i1 + 1], dpdv[1], 0.0f);
                    texc[3 * p + 2] = make_float4(m.UV[2 * i2], m.UV[2 * i2 + 1], dpdv[2], 0.0f);
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
        std::vector<PrimBox> &bb = bBoxes[m.group + 1];
        std::vector<uint32_t> &bi = bIds[m.group + 1];
        for (size_t j = 0; j < nT; ++j) {
            const size_t p = m.primOffset + j;
            const PrimBox &pb = primBox[p];
            if (m.group < 0) for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], pb.lo[a]); hi[a] = std::max(hi[a], pb.hi[a]); }
            if (!primDegenerate[p]) { bb.push_back(pb); bi.push_back((uint32_t) p); }
        }
    }
    std::vector<PrimBox>().swap(primBox);
    s->hTriAccelPrimOrder = triAccel;
    clk.mark("flatten + TriAccel");
    // ---- BVH ----
    BVHResult bvh;
    int threads = usableThreads();
    // Tiny scenes skip the tree: the whole triangle list is one leaf, staged in shared memory and tested by all lanes
    // in lockstep (no divergence).  Break-even against the BVH2 walk measured on the Cornell scene, see DESIGN.md.
    uint32_t flatLimit = 64;
    if (const char *e = getenv("B2_FLAT_LIMIT")) flatLimit = (uint32_t) atoi(e);
    uint32_t rootCount = 0;
    if (!instanced && !ids.empty() && ids.size() <= flatLimit) {
        bvh.leafPrims = ids;
        bvh.rootRef = -1; // ~0: leaf starting at triangle 0
        bvh.depth = 1;
        rootCount = (uint32_t) ids.size();
    } else {
        // non-instanced scenes also get the 8-wide compressed tree over the same leaves: that is what the ray-query kernels walk (the binary
        // tree stays for volpath's inline queries)
        const bool wide = !instanced && !getenv("B2_NO_WIDE");
        buildBVH(boxes, ids, 4, instanced ? 19 : B2_STACK_DEPTH - 2, threads > 0 ? threads : 1, bvh, wide);
        if (bvh.depth8 > B2_STACK8_DEPTH - 1) bvh.nodes8.clear(); // deeper than the wide traversal's stack: binary tree only
    }
    clk.mark("BVH (world)");
    // ---- instancing: one BVH per shapegroup appended to the node / leaf arrays, then a top-level BVH over the items
    //      (item 0 = the world triangles, item k = instance k - 1); stack budget: 9 (top) + 3 (leaf items) + 19 (bottom) < 32 ----
    std::vector<DInstance> items;
    int tlasRoot = -1;
    float topLo[3] = {lo[0], lo[1], lo[2]}, topHi[3] = {hi[0], hi[1], hi[2]};
    if (instanced) {
        struct GroupInfo { int rootRef = -1; float lo[3], hi[3]; bool empty = true; };
        std::vector<GroupInfo> gi((size_t) s->nGroups);
        auto appendTree = [&](BVHResult &g) -> int { // returns the root reference inside the merged arrays
            const uint32_t nodeBase = (uint32_t) bvh.nodes.size(), leafBase = (uint32_t) bvh.leafPrims.size();
            auto fix = [&](int32_t r) -> int32_t {
                if (r >= 0) return r + (int32_t) nodeBase;
                const uint32_t bits = ~(uint32_t) r;
                return (int32_t) ~(((bits & 0x0FFFFFFFu) + leafBase) | (bits & 0xF0000000u));
            };
            for (auto nd : g.nodes) { nd.left = fix(nd.left); nd.right = fix(nd.right); bvh.nodes.push_back(nd); }
            bvh.leafPrims.insert(bvh.leafPrims.end(), g.leafPrims.begin(), g.leafPrims.end());
            return fix(g.rootRef);
        };
        for (int g = 0; g < s->nGroups; ++g) {
            if (bIds[g + 1].empty()) continue;
            BVHResult r;
            buildBVH(bBoxes[g + 1], bIds[g + 1], 4, 19, threads > 0 ? threads : 1, r);
            gi[g].rootRef = appendTree(r);
            gi[g].empty = false;
            float l[3] = {INFINITY, INFINITY, INFINITY}, h[3] = {-INFINITY, -INFINITY, -INFINITY};
            for (auto &b : bBoxes[g + 1]) for (int a = 0; a < 3; ++a) { l[a] = std::min(l[a], b.lo[a]); h[a] = std::max(h[a], b.hi[a]); }
            const float eps = 1e-3f; // the group's kd-tree box, enlarged (gkdtree.h:1213-1220)
            for (int a = 0; a < 3; ++a) { gi[g].lo[a] = l[a] - ((h[a] - l[a]) * eps + eps); gi[g].hi[a] = h[a] + ((h[a] - gi[g].lo[a]) * eps + eps); }
            bvh.depth = std::max(bvh.depth, r.depth);
        }
        if (bvh.leafPrims.size() >= (1u << 28)) return fail(ctx, B2_ERR_INVALID, "too many triangles (limit 2^28)");
        std::vector<PrimBox> itemBoxes;
        std::vector<uint32_t> itemIds;
        if (!ids.empty()) { // item: the world triangles, identity transform, no clipping
            DInstance it; memset(&it, 0, sizeof(it));
            it.identity = 1; it.rootRef = bvh.rootRef;
            PrimBox pb; for (int a = 0; a < 3; ++a) { pb.lo[a] = lo[a]; pb.hi[a] = hi[a]; }
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
            PrimBox pb; for (int a = 0; a < 3; ++a) { pb.lo[a] = INFINITY; pb.hi[a] = -INFINITY; }
            for (int c = 0; c < 8; ++c) { // Instance::getAABB, instance.cpp:80-96
                const float q[3] = {(c & 1) ? g.hi[0] : g.lo[0], (c & 2) ? g.hi[1] : g.lo[1], (c & 4) ? g.hi[2] : g.lo[2]};
                for (int a = 0; a < 3; ++a) {
                    const float w = hi_.M[4 * a] * q[0] + hi_.M[4 * a + 1] * q[1] + hi_.M[4 * a + 2] * q[2] + hi_.M[4 * a + 3];
                    pb.lo[a] = std::min(pb.lo[a], w); pb.hi[a] = std::max(pb.hi[a], w);
                }
            }
            for (int a = 0; a < 3; ++a) { topLo[a] = std::min(topLo[a], pb.lo[a]); topHi[a] = std::max(topHi[a], pb.hi[a]); }
            itemBoxes.push_back(pb); itemIds.push_back((uint32_t) items.size()); items.push_back(it);
        }
        if (items.size() >= (1u << 20)) return fail(ctx, B2_ERR_INVALID, "too many instances (limit 2^20)");
        BVHResult top;
        buildBVH(itemBoxes, itemIds, 4, 9, 1, top);
        if (top.depth > 10) return fail(ctx, B2_ERR_INVALID, "instance hierarchy too deep for the traversal stack");
        // top-level leaves reference items, not triangles: keep their refs apart from the triangle leaf array
        const uint32_t nodeBase = (uint32_t) bvh.nodes.size();
        std::vector<uint32_t> order = top.leafPrims; // item order of the top-level leaves
        std::vector<DInstance> sorted(items.size());
        for (size_t k = 0; k < order.size(); ++k) sorted[k] = items[order[k]];
        items.swap(sorted);
        for (auto nd : top.nodes) {
            if (nd.left >= 0) nd.left += (int32_t) nodeBase;
            if (nd.right >= 0) nd.right += (int32_t) nodeBase;
            bvh.nodes.push_back(nd);
        }
        tlasRoot = top.rootRef >= 0 ? top.rootRef + (int32_t) nodeBase : top.rootRef;
        lo[0] = topLo[0]; lo[1] = topLo[1]; lo[2] = topLo[2]; hi[0] = topHi[0]; hi[1] = topHi[1]; hi[2] = topHi[2];
    }
    s->bvhDepth = bvh.depth;
    std::vector<float4> leafTri(3 * bvh.leafPrims.size()), leafPlane(3 * bvh.leafPrims.size());
    // plane form of triangle (a, b, c), evaluated in double: N = e1 x e2, U = (e2 x N)/|N|^2, V = (N x e1)/|N|^2;
    // u(p) = U.p + du and v(p) = V.p + dv are the barycentrics of b and c
    auto planeRows = [](const float4 &a, const float4 &b, const float4 &c, float4 *out) {
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
    };
    parallelFor(bvh.leafPrims.size(), usableThreads(), [&](size_t ilo, size_t ihi) {
        for (size_t i = ilo; i < ihi; ++i) {
            const size_t p = bvh.leafPrims[i];
            memcpy(&leafTri[3 * i], &triAccel[3 * p], 48);
            planeRows(verts[3 * p], verts[3 * p + 1], verts[3 * p + 2], &leafPlane[3 * i]);
        }
    });
    clk.mark("instancing / leaf order");
    // ---- flat leaf of the throughput build: coplanar triangle pairs share the plane test ----
    // Two triangles with a common edge that lie in one plane are stored as ONE record: a parallelogram (3 rows: the
    // lockstep test is 0 <= u,v <= 1 in the frame of the unshared corner) or a general coplanar pair (5 rows: one t and
    // hit point, two (u,v) evaluations).  Everything else stays a single triangle.  Order: parallelograms, pairs, singles.
    std::vector<float4> flatRec;
    std::vector<uint32_t> flatIdx; // 2 per record: leaf index of the first / second triangle
    uint32_t flatP = 0, flatC = 0, flatS = 0;
    if (rootCount) {
        const uint32_t n = rootCount;
        const double diag = std::sqrt((double) (hi[0] - lo[0]) * (hi[0] - lo[0]) + (double) (hi[1] - lo[1]) * (hi[1] - lo[1]) + (double) (hi[2] - lo[2]) * (hi[2] - lo[2]));
        const double tol = 1e-6 * std::max(diag, 1e-30);
        std::vector<int> mate(n, -1), kind(n, 0), cornerA(n, 0);
        auto V = [&](uint32_t leaf, int k) -> const float4 & { return verts[3 * (size_t) bvh.leafPrims[leaf] + k]; };
        auto same = [](const float4 &a, const float4 &b) { return a.x == b.x && a.y == b.y && a.z == b.z; };
        if (!getenv("B2_NO_QUADS"))
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
                    flatRec.push_back(make_float4(a.x, b.x, a.y, b.y));
                    flatRec.push_back(make_float4(a.z, b.z, a.w, b.w));
                }
            for (auto &ij : recIdx[c]) { flatIdx.push_back(ij.first); flatIdx.push_back(ij.second); }
            (c == 0 ? flatP : c == 1 ? flatC : flatS) = (uint32_t) (recs[c].size() / 2); // packed steps
        }
    }
    if (getenv("B2_VERBOSE"))
        fprintf(stderr, "[b2mts] commit: %zu triangles, flat leaf %u (two-wide steps: parallelograms %u, coplanar pairs %u, singles %u), bvh nodes %zu depth %d\n", nPrims, rootCount,
                flatP, flatC, flatS, bvh.nodes.size(), bvh.depth);
    clk.mark("leaf records");
    // ---- materials ----
    std::vector<DMaterial> dm(s->materials.size());
    for (int c = 0; c < B2_NCLASS; ++c) s->classPresent[c] = false;
    for (size_t i = 0; i < s->materials.size(); ++i) {
        const b2_material_desc &m = s->materials[i];
        DMaterial &d = dm[i];
        memset(&d, 0, sizeof(d));
        d.type = m.type; d.distr = m.distr; d.sampleVisible = (m.distr == B2_DISTR_PHONG) ? 0 : m.sample_visible; d.nested = m.nested;
        d.alphaU = m.alpha_u; d.alphaV = m.alpha_v; d.eta = m.eta; d.thickness = m.thickness;
        memcpy(d.reflectance, m.reflectance, 12); memcpy(d.transmittance, m.transmittance, 12);
        memcpy(d.etaC, m.eta_c, 12); memcpy(d.kC, m.k_c, 12); memcpy(d.sigmaA, m.sigma_a, 12);
        d.flags = materialFlags(s->materials, (int) i);
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
    s->hasNullBsdf = false;
    s->hasTransmission = false;
    for (size_t i = 0; i < s->materials.size(); ++i)
        if (materialFlags(s->materials, (int) i) & 0x55u /* ETransmission incl. ENull */) s->hasTransmission = true;
    for (auto &m : s->meshes) {
        const int t = s->materials[m.material].type;
        if (t >= B2_BSDF_NULL) {
            s->hasNullBsdf = true; // types without a specialised kernel are shaded by the generic one (class queue 4)
            s->classPresent[B2_NCLASS - 1] = true;
            if (t == B2_BSDF_NULL && m.emitter >= 0)
                return fail(ctx, B2_ERR_INVALID, "Shape has an index-matched BSDF and an emitter attachment. This is not allowed!"); // shape.cpp:76-78
        } else s->classPresent[t] = true;
    }
    // ---- bitmap textures: MIP pyramids (host, as the reference builds them at load time) -> one device array per texture ----
    std::vector<DTexture> dtex(s->textures.size());
    s->dTexData.clear();
    for (size_t i = 0; i < s->textures.size(); ++i) {
        b2_scene::HostTexture &ht = s->textures[i];
        const b2_texture_desc &t = ht.desc;
        b2host::buildMipPyramid(ht.pixels.data(), t.width, t.height, t.channels, t.wrap_u, t.wrap_v, t.filter_type >= B2_TEX_TRILINEAR, ht.mip);
        if ((int) ht.mip.level.size() > B2_TEX_MAX_LEVELS) return fail(ctx, B2_ERR_INVALID, "texture has too many MIP levels");
        DTexture &d = dtex[i];
        memset(&d, 0, sizeof(d));
        d.levels = (int) ht.mip.level.size(); d.channels = t.channels; d.filter = t.filter_type; d.wrapU = t.wrap_u; d.wrapV = t.wrap_v;
        d.maxAnisotropy = t.max_anisotropy; d.uoffset = t.uoffset; d.voffset = t.voffset; d.uscale = t.uscale; d.vscale = t.vscale;
        d.bsdfScale = ht.mip.maximum > 1.0f ? 0.99f * (1.0f / ht.mip.maximum) : 1.0f; // bsdf.cpp:93-107
        const int stride = t.channels == 3 ? 4 : 1; // RGB texels are padded to float4 (one 16-byte load per texel)
        std::vector<float> packed;
        for (int l = 0; l < d.levels; ++l) {
            d.lw[l] = ht.mip.w[l]; d.lh[l] = ht.mip.h[l];
            d.off[l] = (uint32_t) (packed.size() / stride);
            const std::vector<float> &src = ht.mip.level[l];
            const size_t nTexel = (size_t) d.lw[l] * d.lh[l];
            if (stride == 1) packed.insert(packed.end(), src.begin(), src.end());
            else for (size_t k = 0; k < nTexel; ++k) { packed.push_back(src[3 * k]); packed.push_back(src[3 * k + 1]); packed.push_back(src[3 * k + 2]); packed.push_back(0.0f); }
        }
        s->dTexData.emplace_back(new DevBuf<float>());
        CK(ctx, s->dTexData.back()->upload(packed));
        d.data = s->dTexData.back()->p;
    }
    CK(ctx, s->dTextures.upload(dtex));
    CK(ctx, s->dTexc.upload(texc));
    // ---- environment map: pyramid (half-rounded floats, RGB padded to float4) + the tables of EnvironmentMap::configure (envmap.cpp:260-329) ----
    if (s->envmap) {
        b2_scene::HostEnvMap &he = *s->envmap;
        b2host::buildMipPyramid(he.pixels.data(), he.w, he.h, 3, B2_WRAP_REPEAT, B2_WRAP_CLAMP, true, he.mip, std::numeric_limits<float>::infinity());
        if ((int) he.mip.level.size() > B2_TEX_MAX_LEVELS) return fail(ctx, B2_ERR_INVALID, "environment map has too many MIP levels");
        DEnvMap de;
        memset(&de, 0, sizeof(de));
        DTexture &d = de.tex;
        d.levels = (int) he.mip.level.size(); d.channels = 3; d.filter = B2_TEX_EWA; d.wrapU = B2_WRAP_REPEAT; d.wrapV = B2_WRAP_CLAMP;
        d.maxAnisotropy = 10.0f; d.uscale = d.vscale = 1.0f; d.bsdfScale = 1.0f; // envmap.cpp:139-142
        std::vector<float> packed;
        for (int l = 0; l < d.levels; ++l) {
            d.lw[l] = he.mip.w[l]; d.lh[l] = he.mip.h[l];
            d.off[l] = (uint32_t) (packed.size() / 4);
            const std::vector<float> &src = he.mip.level[l];
            const size_t nTexel = (size_t) d.lw[l] * d.lh[l];
            packed.reserve(packed.size() + 4 * nTexel);
            for (size_t k = 0; k < nTexel; ++k) { packed.push_back(src[3 * k]); packed.push_back(src[3 * k + 1]); packed.push_back(src[3 * k + 2]); packed.push_back(0.0f); }
        }
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
        CK(ctx, s->dEnvTexels.upload(packed));
        CK(ctx, s->dEnvCdfRows.upload(cdfRows)); CK(ctx, s->dEnvCdfCols.upload(cdfCols)); CK(ctx, s->dEnvRowWeights.upload(rowWeights));
        d.data = s->dEnvTexels.p;
        de.cdfRows = s->dEnvCdfRows.p; de.cdfCols = s->dEnvCdfCols.p; de.rowWeights = s->dEnvRowWeights.p;
        CK(ctx, s->dEnvMap.upload(std::vector<DEnvMap>(1, de)));
    }
    if (anyTex || s->envmap) {
        std::vector<float> lut(64);
        b2host::ewaWeightTable(lut.data());
        CK(ctx, s->dEwaLut.upload(lut));
    }
    // ---- media (volpath) ----
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
        CK(ctx, s->dDensity.back()->upload(s->media[i].density));
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
    clk.mark("materials / textures / media");
    // ---- emitters: scene.cpp:375-380, trimesh.cpp:388-403, pmf.h ----
    std::vector<DEmitter> de(s->emitters.size());
    std::vector<float> emCdf(1, 0.0f), triCdf;
    float emNorm = 0.0f;
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
    clk.mark("emitters");
    // ---- upload ----
    CK(ctx, s->dTriAccel.upload(leafTri));
    CK(ctx, s->dTriPlane.upload(leafPlane));
    CK(ctx, s->dLeafPrim.upload(bvh.leafPrims));
    CK(ctx, s->dFlatRec.upload(flatRec));
    CK(ctx, s->dFlatIdx.upload(flatIdx));
    CK(ctx, s->dVerts.upload(verts));
    CK(ctx, s->dNorms.upload(norms));
    CK(ctx, s->dNodes.upload(bvh.nodes));
    CK(ctx, s->dNodes8.upload(bvh.nodes8));
    CK(ctx, s->dMaterials.upload(dm));
    CK(ctx, s->dEmitters.upload(de));
    CK(ctx, s->dEmitterCdf.upload(emCdf));
    CK(ctx, s->dTriCdf.upload(triCdf));
    CK(ctx, s->dMedia.upload(dmed));
    CK(ctx, s->dInstances.upload(items));
    CK(ctx, s->dPrimMedia.upload(primMedia));
    DScene &ds = s->ds;
    memset(&ds, 0, sizeof(ds));
    ds.triAccel = s->dTriAccel.p; ds.triPlane = s->dTriPlane.p; ds.leafPrim = s->dLeafPrim.p; ds.nLeafTris = (uint32_t) bvh.leafPrims.size();
    // environment emitter: index + constant.cpp:67-70 bounding sphere of (acceleration-structure box U sensor position) (scene.cpp:386-399)
    ds.envEmitter = -1;
    ds.envmap = s->envmap ? s->dEnvMap.p : nullptr;
    for (size_t e = 0; e < s->emitters.size(); ++e) if (s->emitters[e].env) ds.envEmitter = emIndex[e];
    {
        float bl[3], bh[3];
        for (int a = 0; a < 3; ++a) {
            const float eps = 1e-3f;
            float l = nPrims ? lo[a] : 0.0f, h = nPrims ? hi[a] : 0.0f;
            float mn = l - ((h - l) * eps + eps), mx = h + ((h - mn) * eps + eps); // gkdtree.h:1213-1220 (as ds.aabbMin/Max below)
            const float camP = s->camToWorld[4 * a + 3];
            bl[a] = std::min(mn, camP); bh[a] = std::max(mx, camP);
        }
        float c[3], r2 = 0;
        for (int a = 0; a < 3; ++a) { c[a] = (bh[a] + bl[a]) * 0.5f; ds.bsCenter[a] = c[a]; }
        const float dx = c[0] - bh[0], dy = c[1] - bh[1], dz = c[2] - bh[2];
        r2 = dx * dx + dy * dy + dz * dz;
        ds.bsRadius = std::max(1e-4f, std::sqrt(r2) * 1.5f);
    }
    ds.items = s->dInstances.p; ds.nItems = (uint32_t) items.size(); ds.tlasRoot = tlasRoot;
    ds.media = s->dMedia.p; ds.primMedia = anyMedia ? s->dPrimMedia.p : nullptr; ds.nMedia = (uint32_t) dmed.size();
    ds.nodes8 = bvh.nodes8.empty() ? nullptr : s->dNodes8.p; ds.nNodes8 = (uint32_t) bvh.nodes8.size();
    ds.nodes = s->dNodes.p; ds.nNodes = (uint32_t) bvh.nodes.size(); ds.rootRef = bvh.rootRef; ds.rootCount = rootCount;
    ds.flatRec = s->dFlatRec.p; ds.flatIdx = (const uint2 *) s->dFlatIdx.p; ds.flatP = flatP; ds.flatC = flatC; ds.flatS = flatS;
    ds.flatBytes = (uint32_t) (flatRec.size() * 16);
    // gkdtree.h:1213-1220: enlarged scene box (the max side uses the already-moved min, as in the reference)
    if (nPrims == 0 || !(lo[0] <= hi[0])) { for (int a = 0; a < 3; ++a) { lo[a] = 0; hi[a] = 0; } }
    const float eps = 1e-3f;
    for (int a = 0; a < 3; ++a) {
        float mn = lo[a] - ((hi[a] - lo[a]) * eps + eps);
        float mx = hi[a] + ((hi[a] - mn) * eps + eps);
        ds.aabbMin[a] = mn; ds.aabbMax[a] = mx;
    }
    ds.verts = s->dVerts.p; ds.norms = s->dNorms.p; ds.nPrims = (uint32_t) nPrims;
    ds.materials = s->dMaterials.p; ds.nMaterials = (uint32_t) dm.size();
    ds.textures = s->dTextures.p; ds.nTextures = (uint32_t) dtex.size(); ds.texc = s->dTexc.p; ds.ewaLut = s->dEwaLut.p;
    ds.emitters = s->dEmitters.p; ds.nEmitters = (uint32_t) de.size();
    ds.emitterCdf = s->dEmitterCdf.p; ds.emitterNormalization = emNorm; ds.triCdf = s->dTriCdf.p;
    memcpy(ds.cam.camToWorld, s->camToWorld, 64);
    memcpy(ds.cam.sampleToCamera, s->sampleToCamera, 64);
    ds.cam.nearClip = s->nearClip; ds.cam.farClip = s->farClip;
    ds.cam.invResX = 1.0f / (float) s->W; ds.cam.invResY = 1.0f / (float) s->H; // sensor.cpp:104-107
    ds.cam.origin[0] = s->camToWorld[3]; ds.cam.origin[1] = s->camToWorld[7]; ds.cam.origin[2] = s->camToWorld[11];
    ds.cam.W = s->W; ds.cam.H = s->H;
    ds.cam.apertureRadius = s->apertureRadius; ds.cam.focusDistance = s->focusDistance;
    { // m_dx, m_dy (perspective.cpp:160-163): sampleToCamera(Point(invRes.x, 0, 0)) - sampleToCamera(Point(0)), likewise y
        auto s2c = [&](float px, float py, float out[3]) { // Transform::operator()(Point), transform.h:108-125
            const float *M = s->sampleToCamera;
            const float x = M[0] * px + M[1] * py + M[2] * 0.0f + M[3], y = M[4] * px + M[5] * py + M[6] * 0.0f + M[7],
                        z = M[8] * px + M[9] * py + M[10] * 0.0f + M[11], w = M[12] * px + M[13] * py + M[14] * 0.0f + M[15];
            if (w != 1.0f) { const float r = 1.0f / w; out[0] = x * r; out[1] = y * r; out[2] = z * r; }
            else { out[0] = x; out[1] = y; out[2] = z; }
        };
        float z0[3], ax[3], ay[3];
        s2c(0.0f, 0.0f, z0); s2c(ds.cam.invResX, 0.0f, ax); s2c(0.0f, ds.cam.invResY, ay);
        for (int k = 0; k < 3; ++k) { ds.cam.dx[k] = ax[k] - z0[k]; ds.cam.dy[k] = ay[k] - z0[k]; }
    }
    ds.sobolM32 = ctx->dM32; ds.sobolVdc = ctx->dVdc; ds.sobolInv = ctx->dInv; ds.sobolNib = ctx->dNib;
    // shared-memory staging budget: up to 256 nodes (16 KB) and 256 triangles (12 KB) per CTA
    ds.stageNodes = std::min<uint32_t>(ds.nNodes, 256u);
    ds.stageNodes8 = std::min<uint32_t>(ds.nNodes8, 192u); // 15 KB: the root, its children and most of the third level
    ds.stageTris = rootCount ? rootCount : 0u; // a BVH's leaf-ordered head is arbitrary: only the flat leaf is worth staging
    ds.stageTriBytes = std::max(ds.stageTris * 48u, (ds.flatBytes + 15u) & ~15u);
    ds.refill = 16; // measured sweep 8..32 on the material-ball and 1M-triangle scenes (DESIGN.md)
    if (const char *e = getenv("B2_REFILL")) ds.refill = (uint32_t) std::max(1, std::min(32, atoi(e)));
    ds.leafVote = 8;
    // rays that leave the scene are binned into the first BSDF class that has a shading kernel launched for it (a scene without a
    // diffuse mesh launches no class-0 kernel: its escaped paths must still be retired)
    ds.missClass = 0;
    for (int c = B2_NCLASS - 1; c >= 0; --c)
        if (s->classPresent[c]) ds.missClass = (uint32_t) c;
    if (const char *e = getenv("B2_LEAFVOTE")) ds.leafVote = (uint32_t) std::max(1, std::min(32, atoi(e)));
    parity::KernelSet_init(s->cfgParity, ds, ctx->numSMs);
    fast::KernelSet_init(s->cfgFast, ds, ctx->numSMs);
    CK(ctx, cudaGetLastError());
    CK(ctx, s->dCounters.alloc(CTR_COUNT));
    memset(&s->stats, 0, sizeof(s->stats));
    s->stats.n_triangles = nPrims;
    s->stats.n_bvh_nodes = bvh.nodes8.empty() ? bvh.nodes.size() : bvh.nodes8.size();
    s->stats.bvh_node_bytes = bvh.nodes8.empty() ? sizeof(BVHNode) : sizeof(BVH8Node);
    s->stats.bytes_uploaded = leafTri.size() * 16 + leafPlane.size() * 16 + bvh.leafPrims.size() * 4 + verts.size() * 16 + norms.size() * 16 + bvh.nodes.size() * sizeof(BVHNode) +
                              dm.size() * sizeof(DMaterial) + de.size() * sizeof(DEmitter) + (emCdf.size() + triCdf.size()) * 4;
    clk.mark("upload");
    s->committed = true;
    return B2_OK;
}

extern "C" int b2_get_triaccel(b2_scene *s, float *out) {
    if (!s || !s->committed || !out) return fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "scene not committed");
    memcpy(out, s->hTriAccelPrimOrder.data(), s->hTriAccelPrimOrder.size() * sizeof(float4));
    return B2_OK;
}

// ------------------------------------------------------------------------------------------------
// filter table: rfilter.cpp:37-57, box.cpp:41-45, gaussian.cpp:35-57
// ------------------------------------------------------------------------------------------------
static int makeFilter(b2_ctx *ctx, int kind, float param, DFilter &f) {
    if (kind != B2_RFILTER_BOX && kind != B2_RFILTER_GAUSSIAN) return fail(ctx, B2_ERR_INVALID, "unknown reconstruction filter");
    float radius = kind == B2_RFILTER_BOX ? param + 1e-5f : 4 * param;
    if (!(radius > 0) || radius > 30) return fail(ctx, B2_ERR_INVALID, "reconstruction filter radius out of range");
    float sum = 0.0f;
    for (int i = 0; i < 31; ++i) {
        float x = (radius * i) / 31, value;
        if (kind == B2_RFILTER_BOX) value = std::fabs(x) <= radius ? 1.0f : 0.0f;
        else {
            float alpha = -1.0f / (2.0f * param * param);
            value = std::max(0.0f, (float) std::exp((double) (alpha * x * x)) - (float) std::exp((double) (alpha * radius * radius)));
        }
        f.values[i] = value;
        sum += value;
    }
    f.values[31] = 0.0f;
    f.scaleFactor = 31 / radius;
    f.borderSize = (int) std::ceil(radius - 0.5f);
    sum *= 2 * radius / 31;
    float normalization = 1.0f / sum;
    for (int i = 0; i < 31; ++i) f.values[i] *= normalization;
    f.radius = radius;
    f.kind = kind;
    return B2_OK;
}

// ------------------------------------------------------------------------------------------------
// render
// ------------------------------------------------------------------------------------------------
static uint64_t teaHost(uint32_t v0, uint32_t v1, int rounds = 4) { // qmc.h:146-156
    uint32_t sum = 0;
    for (int i = 0; i < rounds; ++i) {
        sum += 0x9e3779b9u;
        v0 += ((v1 << 4) + 0xA341316Cu) ^ (v1 + sum) ^ ((v1 >> 5) + 0xC8013EA4u);
        v1 += ((v0 << 4) + 0xAD90777Du) ^ (v0 + sum) ^ ((v0 >> 5) + 0x7E95761Eu);
    }
    return ((uint64_t) v1 << 32) + v0;
}
static uint32_t roundToPowerOfTwo(uint32_t i) {
    i--; i |= i >> 1; i |= i >> 2; i |= i >> 4; i |= i >> 8; i |= i >> 16;
    return i + 1;
}

static int fillRender(b2_scene *s, const b2_render_params *p, DRender &r) {
    b2_ctx *ctx = s->ctx;
    if (p->spp <= 0) return fail(ctx, B2_ERR_INVALID, "sampleCount must be positive");
    if (p->rr_depth <= 0) return fail(ctx, B2_ERR_INVALID, "'rrDepth' must be set to a value greater than zero!"); // integrator.cpp:218-219
    if (p->max_depth <= 0 && p->max_depth != -1)
        return fail(ctx, B2_ERR_INVALID, "'maxDepth' must be set to -1 (infinite) or a value greater than zero!"); // :221-222
    if (p->sampler != B2_SAMPLER_SOBOL && p->sampler != B2_SAMPLER_INDEPENDENT) return fail(ctx, B2_ERR_INVALID, "unknown sampler");
    memset(&r, 0, sizeof(r));
    r.spp = p->spp; r.sampler = p->sampler;
    r.maxDepth = p->max_depth; r.rrDepth = p->rr_depth; r.strictNormals = p->strict_normals; r.hideEmitters = p->hide_emitters;
    r.sampleLo = p->sample_lo; r.sampleHi = p->sample_hi > 0 ? p->sample_hi : p->spp;
    if (p->integrator != B2_INTEGRATOR_PATH && p->integrator != B2_INTEGRATOR_VOLPATH) return fail(ctx, B2_ERR_INVALID, "unknown integrator");
    if (p->integrator == B2_INTEGRATOR_VOLPATH && s->ds.nItems) return fail(ctx, B2_ERR_INVALID, "volpath with instanced geometry is not supported");
    if (p->integrator == B2_INTEGRATOR_VOLPATH && s->ds.nTextures) return fail(ctx, B2_ERR_INVALID, "volpath with bitmap textures is not supported");
    r.integrator = p->integrator;
    r.diffScale = 1.0f / std::sqrt((float) p->spp); // integrator.cpp:144-145
    if (r.sampleLo < 0 || r.sampleHi > p->spp || r.sampleLo >= r.sampleHi) return fail(ctx, B2_ERR_INVALID, "invalid sample range");
    if (p->sampler == B2_SAMPLER_SOBOL) {
        r.scramble = p->seed ? teaHost((uint32_t) p->seed, (uint32_t) (p->seed >> 32)) : 0; // sobol.cpp:96-102
        uint32_t res = roundToPowerOfTwo((uint32_t) std::max(s->W, s->H));                  // sobol.cpp:147-158
        r.resolution = (float) res;
        uint32_t lg = 0;
        while ((1u << lg) < res) ++lg;
        r.logRes = lg;
    } else {
        r.scramble = p->seed;
    }
    // work items = exactly the W*H*(hi-lo) (pixel, sample) pairs: whole 8x8 tiles first (tile-major, then sample, then pixel), then
    // the pixels of the right / bottom strips that no whole tile covers (sample-major).  No item is ever invalid, so a pool slot is
    // never consumed by a pixel outside the film (workItemPixel in b2_kernels.inl).
    r.tilesX = (uint32_t) s->W / 8; r.tilesY = (uint32_t) s->H / 8;
    { // samples per tile visit: the largest divisor of the sample count that does not exceed B2_ROUND_SPP (0 = all samples at once).
      // A 5 x 5 gaussian splat wants the in-flight paths spread over many pixels (the L2 serialises atomics per address), a 1-pixel box
      // splat does not.
        const uint32_t nS = (uint32_t) (r.sampleHi - r.sampleLo);
        uint32_t want = p->rfilter == B2_RFILTER_GAUSSIAN ? 8 : 0;
        if (const char *e = getenv("B2_ROUND_SPP")) want = (uint32_t) atoi(e);
        r.roundSpp = nS;
        if (want > 0 && want < nS)
            for (uint32_t d = want; d >= 1; --d)
                if (nS % d == 0) { r.roundSpp = d; break; }
    }
    r.totalWork = (uint64_t) s->W * (uint64_t) s->H * (uint64_t) (r.sampleHi - r.sampleLo);
    // nibble tables of sobol::look_up for this m (sobolseq.h:104-133) and the nibble counts that cover the indices
    auto bitsOf = [](uint64_t v) { uint32_t b = 0; while (v) { ++b; v >>= 1; } return b; };
    const uint32_t frameBits = std::max(1u, bitsOf((uint64_t) r.sampleHi - 1));
    r.frameNibbles = (frameBits + 3) / 4;
    r.bNibbles = (2 * r.logRes + 3) / 4;
    const uint32_t indexBits = (p->sampler == B2_SAMPLER_SOBOL && r.logRes > 1) ? frameBits + 2 * r.logRes : frameBits;
    if (indexBits > 52) return fail(ctx, B2_ERR_INVALID, "sample index exceeds the 52-bit range of the Sobol' tables");
    r.indexNibbles = std::max(8u, (indexBits + 3) / 4);
    if (p->sampler == B2_SAMPLER_SOBOL && r.logRes > 1) {
        if (r.logRes > 25) return fail(ctx, B2_ERR_INVALID, "film resolution too large for the Sobol' look_up tables");
        std::vector<uint64_t> lut((size_t) 2 * 13 * 16, 0ull);
        const uint64_t *vrow = ctx->hVdc.data() + (size_t) (r.logRes - 1) * 52, *irow = ctx->hInv.data() + (size_t) (r.logRes - 1) * 52;
        for (int q = 0; q < 13; ++q)
            for (int v = 0; v < 16; ++v) {
                uint64_t a = 0, b = 0;
                for (int k = 0; k < 4; ++k)
                    if ((v >> k) & 1) { a ^= vrow[4 * q + k]; b ^= irow[4 * q + k]; }
                lut[(size_t) q * 16 + v] = a;
                lut[(size_t) (13 + q) * 16 + v] = b;
            }
        if (s->dLookupNib.alloc(lut.size()) != cudaSuccess) return fail(ctx, B2_ERR_CUDA, "cudaMalloc(lookup tables) failed");
        if (cudaMemcpy(s->dLookupNib.p, lut.data(), lut.size() * 8, cudaMemcpyHostToDevice) != cudaSuccess) return fail(ctx, B2_ERR_CUDA, "upload of lookup tables failed");
        r.lookupNib = s->dLookupNib.p;
    }
    return B2_OK;
}

static int ensurePool(b2_scene *s, uint32_t Q, bool vol) {
    b2_ctx *ctx = s->ctx;
    RenderStore &R = *ctx->store;
    if (R.capacity != Q) {
        CK(ctx, R.pRay.alloc((size_t) 2 * Q)); CK(ctx, R.pSt.alloc((size_t) 2 * Q)); CK(ctx, R.pHit.alloc(Q));
        CK(ctx, R.pShO.alloc(Q)); CK(ctx, R.pShD.alloc(Q)); CK(ctx, R.pShC.alloc(Q)); CK(ctx, R.pSmp.alloc(Q)); CK(ctx, R.pPos.alloc(Q));
        CK(ctx, R.pPix.alloc(Q)); CK(ctx, R.pFlags.alloc(Q));
        CK(ctx, R.pMatQueue.alloc((size_t) B2_NCLASS * Q)); CK(ctx, R.pDoneQueue.alloc((size_t) 2 * Q));
        R.pVol.release(); R.pInst.release();
        R.capacity = Q;
    }
    if (vol && R.pVol.n != Q) CK(ctx, R.pVol.alloc(Q));
    if (s->ds.nItems && R.pInst.n != Q) CK(ctx, R.pInst.alloc(Q));
    DPool &p = s->pool;
    p.capacity = Q;
    p.ray = R.pRay.p; p.st = R.pSt.p; p.hit = R.pHit.p; p.smp = R.pSmp.p; p.pos = R.pPos.p; p.pix = R.pPix.p; p.flags = R.pFlags.p;
    p.shO = R.pShO.p; p.shD = R.pShD.p; p.shC = R.pShC.p; p.matQueue = R.pMatQueue.p;
    p.doneQueue = R.pDoneQueue.p;
    p.counters = s->dCounters.p;
    p.vol = R.pVol.p;
    p.inst = R.pInst.p;
    return B2_OK;
}

extern "C" int b2_render(b2_scene *s, const b2_render_params *p, float *film) {
    if (!s || !p || !film) return fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_render: null argument");
    b2_ctx *ctx = s->ctx;
    if (!s->committed) return fail(ctx, B2_ERR_INVALID, "b2_render: scene not committed");
    CK(ctx, cudaSetDevice(ctx->device));
    RenderStore &R = *ctx->store;
    std::lock_guard<std::mutex> renderLock(R.renderMutex);
    cudaStream_t st = ctx->stream;
    DRender r;
    int rc = fillRender(s, p, r);
    if (rc) return rc;
    DFilter filt;
    rc = makeFilter(ctx, p->rfilter, p->rfilter_param, filt);
    if (rc) return rc;
    // Which kernel set renders?  parity_mode 1: the IEEE build (-fmad=false, accurate division / sqrt / sincos, TriAccel).  parity_mode 0: the
    // throughput build -- EXCEPT for `path` renders of scenes with a transmissive BSDF.  A path that bounces inside a glass ball amplifies
    // ulp-level differences chaotically: under FMA contraction alone a few in 1e5 of such paths leave the reference's path (different hit,
    // other lobe, other ending -- not fast-math, not the plane-form triangle test), each an unrelated sample of a heavy-tailed estimator,
    // i.e. above 1e-3 relative L2 at 1024^2 @ 512 spp whatever else the kernels do.  Shading such scenes
    // with the IEEE kernels and keeping only the traversal fast ("hybrid", tried: exact TriAccel (t,u,v) of the winning triangle) removes
    // a third of the flips -- the fast traversal still picks the neighbouring triangle at shared edges -- so those scenes get the IEEE
    // build as a whole (BVH traversal dominates BASELINE config 3, so the IEEE shading costs little there).  flags bit8 forces the throughput kernels.
    const bool autoIeee = s->hasTransmission && p->integrator == B2_INTEGRATOR_PATH && !(p->flags & 256);
    const bool parityMode = p->parity_mode != 0 || autoIeee;
    const LaunchCfg &cfg = parityMode ? s->cfgParity : s->cfgFast;
    uint32_t Q = p->pool_size > 0 ? (uint32_t) p->pool_size : (1u << 22); // 4M paths (~0.6 GB)
    Q = std::max<uint32_t>(Q, 1024u);
    Q = (uint32_t) std::min<uint64_t>(Q, std::max<uint64_t>(1024u, r.totalWork));
    Q = (Q + 255u) & ~255u;
    const bool volpath = p->integrator == B2_INTEGRATOR_VOLPATH;
    rc = ensurePool(s, Q, volpath);
    if (rc) return rc;
    const size_t nPix = (size_t) s->W * s->H;
    CK(ctx, R.dFilmRGBA.alloc(nPix));
    CK(ctx, R.dFilmW.alloc(nPix));
    r.filmRGBA = R.dFilmRGBA.p; r.filmW = R.dFilmW.p;
    if (!R.hRing) {
        CK(ctx, cudaHostAlloc((void **) &R.hRing, sizeof(unsigned long long) * 4 * B2_RING, cudaHostAllocMapped));
        CK(ctx, cudaHostGetDevicePointer((void **) &R.dRing, R.hRing, 0));
    }
    memset(R.hRing, 0, sizeof(unsigned long long) * 4 * B2_RING);
    r.ring = R.dRing;
    const bool timing = (p->flags & 4) != 0;      // per-launch device time stamps (%globaltimer inside the kernels)
    const bool useEvents = (p->flags & 8) != 0;   // no graph: plain launches bracketed by CUDA events (cross-check path)
    if (timing) {
        CK(ctx, R.dStampStart.alloc((size_t) B2_MAX_STAMPS * 4));
        CK(ctx, R.dStampEnd.alloc((size_t) B2_MAX_STAMPS * 4));
        CK(ctx, cudaMemsetAsync(R.dStampStart.p, 0xFF, (size_t) B2_MAX_STAMPS * 4 * 8, st));
        CK(ctx, cudaMemsetAsync(R.dStampEnd.p, 0, (size_t) B2_MAX_STAMPS * 4 * 8, st));
        r.stampStart = R.dStampStart.p; r.stampEnd = R.dStampEnd.p;
    }
    if (p->flags & 32) { // per-pixel path diagnostics: sum of path lengths (low word) and of their squares (high word)
        CK(ctx, R.dPixStats.alloc(nPix));
        CK(ctx, cudaMemsetAsync(R.dPixStats.p, 0, nPix * sizeof(unsigned long long), st));
        r.pixStats = R.dPixStats.p;
    }
    if (p->flags & 64) { // per-sample event traces (diagnostics; Sobol' sampler, film resolution > 2): one byte per bounce, eight bounces
        if (p->sampler != B2_SAMPLER_SOBOL || r.logRes <= 1) return fail(ctx, B2_ERR_INVALID, "path traces (flags bit6) need the sobol sampler and a film larger than 2 pixels");
        const size_t nTr = nPix * (size_t) (r.sampleHi - r.sampleLo);
        CK(ctx, R.dPathTrace.alloc(nTr));
        CK(ctx, cudaMemsetAsync(R.dPathTrace.p, 0, nTr * sizeof(unsigned long long), st));
        r.pathTrace = R.dPathTrace.p;
    }
    CK(ctx, cudaMemsetAsync(R.dFilmRGBA.p, 0, nPix * sizeof(float4), st));
    CK(ctx, cudaMemsetAsync(R.dFilmW.p, 0, nPix * sizeof(float), st));
    CK(ctx, cudaMemsetAsync(s->dCounters.p, 0, CTR_COUNT * sizeof(unsigned long long), st));
    CK(ctx, cudaMemsetAsync(R.pFlags.p, 0, (size_t) Q * sizeof(uint32_t), st));
    int nClasses = 0, onlyClass = -1;
    for (int c = 0; c < B2_NCLASS; ++c)
        if (s->classPresent[c]) { ++nClasses; onlyClass = c == B2_NCLASS - 1 ? -1 : c; }
    // more than one class: k_extend bins the hits by BSDF class and every class gets its own shading launch over its queue -- the four
    // specialised instances, and the generic instance for the rest (null, twosided, dielectric, conductor, plastic); scenes with bitmap
    // textures or an environment map use the TEX instances of the same classes (launch_shade)
    bool sorted = nClasses > 1;
    if (p->flags & 2) sorted = false;
    s->cancel.store(0);
    // every early return below leaves the stream idle and releases the events / the captured graph
    struct RenderGuard {
        cudaStream_t st;
        cudaEvent_t a = nullptr, b = nullptr;
        cudaGraph_t *graph = nullptr;
        cudaGraphExec_t *exec = nullptr;
        ~RenderGuard() {
            cudaStreamSynchronize(st);
            if (exec && *exec) cudaGraphExecDestroy(*exec);
            if (graph && *graph) cudaGraphDestroy(*graph);
            if (a) cudaEventDestroy(a);
            if (b) cudaEventDestroy(b);
        }
    } guard{st};
    cudaEvent_t evStart, evStop;
    CK(ctx, cudaEventCreate(&evStart));
    guard.a = evStart;
    CK(ctx, cudaEventCreate(&evStop));
    guard.b = evStop;
    CK(ctx, cudaEventRecord(evStart, st));
    uint64_t iter = 0, checked = 0, launches = 0;
    bool finished = false;
    int status = B2_OK;
    std::vector<std::pair<int, size_t>> timed; // (stage, index of the start event) -- events path only
    size_t evUsed = 0;
    auto tick = [&](int stage) {
        if (!useEvents) return;
        if (evUsed == s->timingEvents.size()) { cudaEvent_t e; cudaEventCreate(&e); s->timingEvents.push_back(e); }
        cudaEventRecord(s->timingEvents[evUsed], st);
        if (stage >= 0) timed.emplace_back(stage, evUsed);
        ++evUsed;
    };
    int launchesPerIter = 0;
    // one iteration = generate (+publish) -> extend -> shade (per material class) -> occluded
    auto enqueueIteration = [&]() {
        launchesPerIter = 0;
#define ITER(nsS, cfgS, nsT, cfgT) /* nsS: generate + shade (+ volpath); nsT: the ray queries */                                            \
        do {                                                                                                   \
            tick(0); nsS::launch_generate(cfgS, s->ds, s->pool, r, filt, st); tick(-1);                        \
            if (volpath) { /* volpath: every ray of an iteration is cast inline by k_volstep */                 \
                tick(2); nsS::launch_volstep(cfgS, s->ds, s->pool, r, st); tick(-1);                           \
                launchesPerIter = 3;                                                                           \
                break;                                                                                         \
            }                                                                                                  \
            tick(1); nsT::launch_extend(cfgT, s->ds, s->pool, r, sorted, st); tick(-1); ++launchesPerIter;     \
            tick(2);                                                                                           \
            if (sorted) {                                                                                      \
                for (int c = 0; c < B2_NCLASS; ++c)                                                            \
                    if (s->classPresent[c]) { nsS::launch_shade(cfgS, s->ds, s->pool, r, c, true, st); ++launchesPerIter; } \
            } else {                                                                                           \
                nsS::launch_shade(cfgS, s->ds, s->pool, r, nClasses == 1 ? onlyClass : -1, false, st);         \
                ++launchesPerIter;                                                                             \
            }                                                                                                  \
            tick(-1);                                                                                          \
            tick(3); nsT::launch_occluded(cfgT, s->ds, s->pool, r, st); tick(-1); ++launchesPerIter;           \
            launchesPerIter += 2;                                                                              \
        } while (0)
        if (parityMode) ITER(parity, s->cfgParity, parity, s->cfgParity);
        else ITER(fast, s->cfgFast, fast, s->cfgFast);
#undef ITER
    };
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t graphExec = nullptr;
    guard.graph = &graph; guard.exec = &graphExec;
    if (!useEvents) {
        if (volpath || s->ds.nTextures || s->ds.envmap) {
            // k_volstep (and the textured k_shade) have a deep local-memory frame: their first launch may have to grow the context's
            // local-memory pool, which is not allowed inside a stream capture.  The first iteration therefore runs as plain launches.
            enqueueIteration();
            launches += launchesPerIter;
            ++iter;
        }
        // the iteration index lives on the device (CTR_ITER, advanced by k_publish): one captured graph replays for every iteration
        CK(ctx, cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        enqueueIteration();
        {
            cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
            cudaStreamIsCapturing(st, &cs);
            const cudaError_t le = cudaPeekAtLastError();
            if (cs != cudaStreamCaptureStatusActive || le != cudaSuccess) {
                cudaStreamEndCapture(st, &graph);
                cudaGetLastError();
                return fail(ctx, B2_ERR_CUDA, std::string("graph capture of the iteration failed: ") + cudaGetErrorString(le) +
                                              (volpath ? " (volpath)" : " (path)") + ", grid " + std::to_string(cfg.gridVolstep) + ", smem " + std::to_string(cfg.traceSmem));
            }
        }
        CK(ctx, cudaStreamEndCapture(st, &graph));
        CK(ctx, cudaGraphInstantiate(&graphExec, graph, 0));
    }
    volatile unsigned long long *ring = R.hRing;
    while (!finished) {
        if (s->cancel.load()) { status = B2_ERR_CANCELLED; break; }
        // consume published progress; never run more than B2_RING - 1 iterations ahead of the device
        for (;;) {
            while (checked < iter && ring[(checked % B2_RING) * 4] == checked + 1) {
                const unsigned long long active = ring[(checked % B2_RING) * 4 + 1], next = ring[(checked % B2_RING) * 4 + 2];
                ++checked;
                if (active == 0 && next >= r.totalWork) { finished = true; break; }
            }
            if (finished || iter - checked < (uint64_t) B2_RING - 1) break;
            if (cudaStreamQuery(st) != cudaErrorNotReady && ring[(checked % B2_RING) * 4] != checked + 1) {
                cudaError_t e = cudaStreamSynchronize(st);
                if (ring[(checked % B2_RING) * 4] != checked + 1) {
                    status = fail(ctx, B2_ERR_CUDA, std::string("render loop: device made no progress: ") + cudaGetErrorString(e == cudaSuccess ? cudaGetLastError() : e));
                    finished = true;
                    break;
                }
            }
        }
        if (finished) break;
        if (useEvents) enqueueIteration();
        else if (cudaGraphLaunch(graphExec, st) != cudaSuccess) { status = fail(ctx, B2_ERR_CUDA, "cudaGraphLaunch failed"); break; }
        launches += launchesPerIter;
        ++iter;
        if (iter > 100000000ull) { status = fail(ctx, B2_ERR_CUDA, "render loop did not terminate"); break; }
    }
    // pack + copy out (the guard destroys the graph and the events when this function returns)
    CK(ctx, cudaEventRecord(evStop, st));
    if (status == B2_OK) {
        float *dOut = film;
        if (!p->film_on_device) {
            CK(ctx, R.dFilmOut.alloc(nPix * 5));
            dOut = R.dFilmOut.p;
        }
        if (parityMode) parity::launch_film_pack(cfg, R.dFilmRGBA.p, R.dFilmW.p, dOut, nPix, st);
        else fast::launch_film_pack(cfg, R.dFilmRGBA.p, R.dFilmW.p, dOut, nPix, st);
        if (!p->film_on_device) CK(ctx, cudaMemcpyAsync(film, dOut, nPix * 5 * sizeof(float), cudaMemcpyDeviceToHost, st));
    }
    CK(ctx, cudaStreamSynchronize(st));
    CK(ctx, cudaGetLastError());
    std::vector<unsigned long long> ctr(CTR_COUNT);
    CK(ctx, cudaMemcpy(ctr.data(), s->dCounters.p, CTR_COUNT * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    float ms = 0;
    cudaEventElapsedTime(&ms, evStart, evStop);
    b2_stats &t = s->stats;
    t.ms_generate = t.ms_extend = t.ms_shade = t.ms_occluded = 0;
    t.n_generate = t.n_extend = t.n_shade = t.n_occluded = 0;
    for (auto &te : timed) {
        float e = 0;
        cudaEventElapsedTime(&e, s->timingEvents[te.second], s->timingEvents[te.second + 1]);
        switch (te.first) {
            case 0: t.ms_generate += e; ++t.n_generate; break;
            case 1: t.ms_extend += e; ++t.n_extend; break;
            case 2: t.ms_shade += e; ++t.n_shade; break;
            default: t.ms_occluded += e; ++t.n_occluded; break;
        }
    }
    if (timing && !useEvents) {
        const size_t nIt = (size_t) std::min<uint64_t>(iter, B2_MAX_STAMPS);
        std::vector<unsigned long long> a(nIt * 4), b(nIt * 4);
        if (nIt) {
            CK(ctx, cudaMemcpy(a.data(), R.dStampStart.p, nIt * 4 * 8, cudaMemcpyDeviceToHost));
            CK(ctx, cudaMemcpy(b.data(), R.dStampEnd.p, nIt * 4 * 8, cudaMemcpyDeviceToHost));
        }
        float *ms[4] = {&t.ms_generate, &t.ms_extend, &t.ms_shade, &t.ms_occluded};
        uint64_t *cnt[4] = {&t.n_generate, &t.n_extend, &t.n_shade, &t.n_occluded};
        double acc[4] = {0, 0, 0, 0};
        for (size_t i = 0; i < nIt; ++i)
            for (int k = 0; k < 4; ++k)
                if (b[i * 4 + k] > a[i * 4 + k] && a[i * 4 + k] != ~0ull) { acc[k] += (double) (b[i * 4 + k] - a[i * 4 + k]) * 1e-6; ++*cnt[k]; }
        for (int k = 0; k < 4; ++k) *ms[k] = (float) acc[k];
    }
    t.pool_size = Q;
    t.unoccluded_shadow_rays = ctr[CTR_UNOCCLUDED];
    t.samples = ctr[CTR_SAMPLES]; t.rays = ctr[CTR_RAYS]; t.shadow_rays = ctr[CTR_SHADOWRAYS]; t.path_length_sum = ctr[CTR_PATHLEN];
    t.bad_samples = ctr[CTR_BAD]; t.dim_overflow = ctr[CTR_DIMOVF]; t.iterations = iter; t.kernel_launches = launches + 1;
    t.ms_total = ms;
    return status;
}

// Per-pixel path diagnostics of the last b2_render that ran with flags bit5: out[y * W + x] = (sum of squared path lengths << 32) |
// sum of path lengths over the samples of that pixel (both modulo 2^32).  Two renders of the same scene and sampler that differ in
// one path of a pixel differ in that pixel's word: the fraction of differing words bounds the fraction of flipped paths from below.
extern "C" int b2_get_pixel_stats(b2_scene *s, uint64_t *out) {
    if (!s || !out) return fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_get_pixel_stats: null argument");
    b2_ctx *ctx = s->ctx;
    RenderStore &R = *ctx->store;
    std::lock_guard<std::mutex> renderLock(R.renderMutex);
    const size_t nPix = (size_t) s->W * s->H;
    if (R.dPixStats.n != nPix) return fail(ctx, B2_ERR_INVALID, "b2_get_pixel_stats: the last render did not collect pixel statistics (flags bit5)");
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, cudaMemcpy(out, R.dPixStats.p, nPix * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return B2_OK;
}
// Per-sample event traces of the last b2_render that ran with flags bit6 (diagnostics): out[(y * W + x) * n_samples + s] holds one event
// byte per bounce k (bits 8k .. 8k+7, k < 8): bits 0-2 material id of the hit (7 = the ray left the scene), bit 3 a shadow ray was emitted,
// bits 4-5 how the vertex ended (0 continues, 1 Russian roulette, 2 zero BSDF sample / strict normals, 3 depth limit or miss),
// bit 6 the sampled lobe transmits, bit 7 always set.  Two builds that disagree on a path disagree in its word.
extern "C" int b2_get_path_traces(b2_scene *s, uint64_t n_words, uint64_t *out) {
    if (!s || !out) return fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_get_path_traces: null argument");
    b2_ctx *ctx = s->ctx;
    RenderStore &R = *ctx->store;
    std::lock_guard<std::mutex> renderLock(R.renderMutex);
    if (R.dPathTrace.n != n_words || !n_words) return fail(ctx, B2_ERR_INVALID, "b2_get_path_traces: size does not match the last traced render (flags bit6)");
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, cudaMemcpy(out, R.dPathTrace.p, n_words * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return B2_OK;
}
extern "C" int b2_cancel(b2_scene *s) {
    if (!s) return B2_ERR_INVALID;
    s->cancel.store(1);
    return B2_OK;
}
extern "C" int b2_get_stats(b2_scene *s, b2_stats *out) {
    if (!s || !out) return B2_ERR_INVALID;
    *out = s->stats;
    return B2_OK;
}
extern "C" int b2_film_develop(const float *film, int W, int H, float *rgb) { // fmtconv.cpp:979-990
    if (!film || !rgb || W <= 0 || H <= 0) return fail(nullptr, B2_ERR_INVALID, "b2_film_develop: invalid argument");
    for (size_t i = 0; i < (size_t) W * H; ++i) {
        float weight = film[5 * i + 4], invWeight = (weight != 0) ? 1 / weight : weight;
        for (int k = 0; k < 3; ++k) rgb[3 * i + k] = film[5 * i + k] * invWeight;
    }
    return B2_OK;
}

// ------------------------------------------------------------------------------------------------
// component entry points
// ------------------------------------------------------------------------------------------------
struct TmpDev {
    std::vector<void *> ptrs;
    ~TmpDev() { for (void *p : ptrs) cudaFree(p); }
    template <typename T> T *alloc(size_t n) {
        void *p = nullptr;
        if (cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) return nullptr;
        ptrs.push_back(p);
        return (T *) p;
    }
    template <typename T> T *upload(const T *h, size_t n) {
        T *d = alloc<T>(n);
        if (d && n) cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice);
        return d;
    }
};
#define NEED_COMMIT(s) if (!(s) || !(s)->committed) return fail((s) ? (s)->ctx : nullptr, B2_ERR_INVALID, "scene not committed")

extern "C" int b2_trace_device(b2_scene *s, uint64_t n, const float *d_rays, int mode, int parity_mode, float *d_tuvp, float *ms_kernel) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    CK(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const bool count = (mode & 2) != 0;
    const bool shadow = (mode & 1) != 0;
    if (n > 0xFFFFFFFFull) return fail(ctx, B2_ERR_INVALID, "b2_trace: at most 2^32-1 rays per call");
    struct EventPair { cudaEvent_t a = nullptr, b = nullptr; ~EventPair() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); } } ev;
    CK(ctx, cudaEventCreate(&ev.a));
    CK(ctx, cudaEventCreate(&ev.b));
    cudaEvent_t a = ev.a, b = ev.b;
    if (count) cudaMemsetAsync(s->dCounters.p + CTR_NODEVIS, 0, 16, st);
    cudaMemsetAsync(s->dCounters.p + CTR_TICKET_EXT, 0, 8, st);
    // B2_BIN=1 (experiment): tickets binned by (entry cell, direction cell) first -- inside the timed region
    TmpDev tmp;
    uint32_t *order = nullptr;
    const bool bin = s->ds.nodes8 && !s->ds.rootCount && !s->ds.nItems && n >= (1u << 16) && getenv("B2_BIN"); // A/B switch: measured 12 % slower
    uint32_t *keys = nullptr, *hist = nullptr;
    if (bin) {
        keys = tmp.alloc<uint32_t>(n); hist = tmp.alloc<uint32_t>(B2_NBINS + 1); order = tmp.alloc<uint32_t>(n);
        if (!keys || !hist || !order) return fail(ctx, B2_ERR_CUDA, "b2_trace: device allocation failed");
    }
    cudaEventRecord(a, st);
    if (bin) {
        if (parity_mode) parity::launch_bin(s->cfgParity, s->ds, s->pool, (const float4 *) d_rays, (uint32_t) n, keys, hist, order, st);
        else fast::launch_bin(s->cfgFast, s->ds, s->pool, (const float4 *) d_rays, (uint32_t) n, keys, hist, order, st);
    }
    if (parity_mode) parity::launch_trace(s->cfgParity, s->ds, (const float4 *) d_rays, (float4 *) d_tuvp, n, shadow, count, s->dCounters.p, order, st);
    else fast::launch_trace(s->cfgFast, s->ds, (const float4 *) d_rays, (float4 *) d_tuvp, n, shadow, count, s->dCounters.p, order, st);
    cudaEventRecord(b, st);
    CK(ctx, cudaStreamSynchronize(st));
    CK(ctx, cudaGetLastError());
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    if (ms_kernel) *ms_kernel = ms;
    if (count) {
        unsigned long long c[2];
        cudaMemcpy(c, s->dCounters.p + CTR_NODEVIS, 16, cudaMemcpyDeviceToHost);
        s->stats.node_visits = c[0]; s->stats.prim_tests = c[1];
    }
    return B2_OK;
}
extern "C" int b2_trace(b2_scene *s, uint64_t n, const float *rays, int mode, int parity_mode, float *t, float *u, float *v, uint32_t *prim,
                        float *ms_kernel) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    CK(ctx, cudaSetDevice(ctx->device));
    TmpDev tmp;
    float *dR = tmp.upload(rays, 8 * n);
    float *dO = tmp.alloc<float>(4 * n);
    if (!dR || !dO) return fail(ctx, B2_ERR_CUDA, "b2_trace: device allocation failed");
    int rc = b2_trace_device(s, n, dR, mode, parity_mode, dO, ms_kernel);
    if (rc) return rc;
    std::vector<float> h(4 * n);
    CK(ctx, cudaMemcpy(h.data(), dO, 4 * n * sizeof(float), cudaMemcpyDeviceToHost));
    for (uint64_t i = 0; i < n; ++i) {
        if (t) t[i] = h[4 * i];
        if (u) u[i] = h[4 * i + 1];
        if (v) v[i] = h[4 * i + 2];
        if (prim) memcpy(&prim[i], &h[4 * i + 3], 4);
    }
    return B2_OK;
}
extern "C" int b2_bsdf_eval(b2_scene *s, int mat, uint64_t n, const float *wi, const float *wo, int parity_mode, float *out_rgb, float *out_pdf) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    if (mat < 0 || mat >= (int) s->materials.size()) return fail(ctx, B2_ERR_INVALID, "invalid material id");
    CK(ctx, cudaSetDevice(ctx->device));
    TmpDev tmp;
    float *dWi = tmp.upload(wi, 3 * n), *dWo = tmp.upload(wo, 3 * n), *dRgb = tmp.alloc<float>(3 * n), *dPdf = tmp.alloc<float>(n);
    if (parity_mode) parity::launch_bsdf_eval(s->cfgParity, s->ds, mat, n, dWi, dWo, dRgb, dPdf, ctx->stream);
    else fast::launch_bsdf_eval(s->cfgFast, s->ds, mat, n, dWi, dWo, dRgb, dPdf, ctx->stream);
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(out_rgb, dRgb, 3 * n * sizeof(float), cudaMemcpyDeviceToHost));
    CK(ctx, cudaMemcpy(out_pdf, dPdf, n * sizeof(float), cudaMemcpyDeviceToHost));
    return B2_OK;
}
extern "C" int b2_bsdf_sample(b2_scene *s, int mat, uint64_t n, const float *wi, const float *samples, int parity_mode, float *out) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    if (mat < 0 || mat >= (int) s->materials.size()) return fail(ctx, B2_ERR_INVALID, "invalid material id");
    CK(ctx, cudaSetDevice(ctx->device));
    TmpDev tmp;
    float *dWi = tmp.upload(wi, 3 * n), *dS = tmp.upload(samples, 3 * n), *dO = tmp.alloc<float>(10 * n);
    if (parity_mode) parity::launch_bsdf_sample(s->cfgParity, s->ds, mat, n, dWi, dS, dO, ctx->stream);
    else fast::launch_bsdf_sample(s->cfgFast, s->ds, mat, n, dWi, dS, dO, ctx->stream);
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(out, dO, 10 * n * sizeof(float), cudaMemcpyDeviceToHost));
    return B2_OK;
}
extern "C" int b2_sample_emitter_direct(b2_scene *s, uint64_t n, const float *ref, const float *samples, int parity_mode, float *out) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    if (s->emitters.empty()) return fail(ctx, B2_ERR_INVALID, "scene has no emitters");
    CK(ctx, cudaSetDevice(ctx->device));
    TmpDev tmp;
    float *dR = tmp.upload(ref, 6 * n), *dS = tmp.upload(samples, 2 * n), *dO = tmp.alloc<float>(12 * n);
    if (parity_mode) parity::launch_emitter_direct(s->cfgParity, s->ds, n, dR, dS, dO, ctx->stream);
    else fast::launch_emitter_direct(s->cfgFast, s->ds, n, dR, dS, dO, ctx->stream);
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    CK(ctx, cudaGetLastError());
    std::vector<float> h(12 * n);
    CK(ctx, cudaMemcpy(h.data(), dO, 12 * n * sizeof(float), cudaMemcpyDeviceToHost));
    // fold the visibility test (scene.cpp:838-843) into `visible` with the occlusion kernel
    std::vector<float> rays(8 * n);
    for (uint64_t i = 0; i < n; ++i) {
        float *r = &rays[8 * i];
        r[0] = ref[6 * i]; r[1] = ref[6 * i + 1]; r[2] = ref[6 * i + 2]; r[3] = 1e-4f;
        r[4] = h[12 * i]; r[5] = h[12 * i + 1]; r[6] = h[12 * i + 2]; r[7] = h[12 * i + 3] * (1 - 1e-3f);
    }
    std::vector<uint32_t> occ(n);
    int rc = b2_trace(s, n, rays.data(), 1, parity_mode, nullptr, nullptr, nullptr, occ.data(), nullptr);
    if (rc) return rc;
    for (uint64_t i = 0; i < n; ++i) {
        if (h[12 * i + 8] != 0 && occ[i]) { h[12 * i + 8] = 0; h[12 * i + 4] = 0; h[12 * i + 5] = h[12 * i + 6] = h[12 * i + 7] = 0; }
        else if (h[12 * i + 8] == 0) { h[12 * i + 4] = 0; }
    }
    memcpy(out, h.data(), 12 * n * sizeof(float));
    return B2_OK;
}
// Medium component probe (parity tests): what = 0 evalTransmittance (in: n x 8 ray floats, out n x 3), 1 sampleDistance (out n x 12),
// 2 density lookup (in n x 3, out n), 3 phase sample (in n x 5: wi, two uniforms; out n x 5: wo, pdf, eval)
extern "C" int b2_medium_probe(b2_scene *s, int medium, int what, uint64_t n, const float *in, uint64_t seed, int parity_mode, float *out) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    if (medium < 0 || medium >= (int) s->media.size()) return fail(ctx, B2_ERR_INVALID, "invalid medium id");
    if (what < 0 || what > 3 || !in || !out) return fail(ctx, B2_ERR_INVALID, "b2_medium_probe: invalid argument");
    static const int inW[4] = {8, 8, 3, 5}, outW[4] = {3, 12, 1, 5};
    CK(ctx, cudaSetDevice(ctx->device));
    TmpDev tmp;
    float *dI = tmp.upload(in, (size_t) inW[what] * n), *dO = tmp.alloc<float>((size_t) outW[what] * n);
    if (parity_mode) parity::launch_medium_probe(s->cfgParity, s->ds, medium, what, n, dI, seed, dO, ctx->stream);
    else fast::launch_medium_probe(s->cfgFast, s->ds, medium, what, n, dI, seed, dO, ctx->stream);
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(out, dO, (size_t) outW[what] * n * sizeof(float), cudaMemcpyDeviceToHost));
    return B2_OK;
}
// Texture probes (parity tests)
extern "C" int b2_texture_eval(b2_scene *s, int texture_id, uint64_t n, const float *uv, const float *partials, int parity_mode, float *out) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    if (texture_id < 0 || texture_id >= (int) s->textures.size()) return fail(ctx, B2_ERR_INVALID, "invalid texture id");
    if (!uv || !out) return fail(ctx, B2_ERR_INVALID, "b2_texture_eval: null argument");
    std::vector<float> in(6 * n, 0.0f);
    for (uint64_t i = 0; i < n; ++i) {
        in[6 * i] = uv[2 * i]; in[6 * i + 1] = uv[2 * i + 1];
        if (partials) for (int k = 0; k < 4; ++k) in[6 * i + 2 + k] = partials[4 * i + k];
    }
    CK(ctx, cudaSetDevice(ctx->device));
    TmpDev tmp;
    float *dI = tmp.upload(in.data(), 6 * n), *dO = tmp.alloc<float>(3 * n);
    if (parity_mode) parity::launch_texture_probe(s->cfgParity, s->ds, 0, texture_id, partials ? 1 : 0, 1.0f, n, dI, dO, ctx->stream);
    else fast::launch_texture_probe(s->cfgFast, s->ds, 0, texture_id, partials ? 1 : 0, 1.0f, n, dI, dO, ctx->stream);
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(out, dO, 3 * n * sizeof(float), cudaMemcpyDeviceToHost));
    return B2_OK;
}
// Probes of the committed environment map (tests): what 0 = Scene::evalEnvironment for n directions (in 3n -> out 3n), 1 = the same for sensor
// rays with differential directions (in 9n: d, rxD, ryD -> out 3n), 2 = Scene::pdfEmitterDirect of the map for n directions (in 3n -> out n)
extern "C" int b2_envmap_probe(b2_scene *s, int what, uint64_t n, const float *in, int parity_mode, float *out) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    if (!s->envmap) return fail(ctx, B2_ERR_INVALID, "b2_envmap_probe: the scene has no environment map");
    if (!in || !out || what < 0 || what > 2) return fail(ctx, B2_ERR_INVALID, "b2_envmap_probe: invalid argument");
    CK(ctx, cudaSetDevice(ctx->device));
    TmpDev tmp;
    const size_t nin = (what == 1 ? 9 : 3) * n, nout = (what == 2 ? 1 : 3) * n;
    float *dI = tmp.upload(in, nin), *dO = tmp.alloc<float>(nout);
    if (parity_mode) parity::launch_envmap_probe(s->cfgParity, s->ds, what, n, dI, dO, ctx->stream);
    else fast::launch_envmap_probe(s->cfgFast, s->ds, what, n, dI, dO, ctx->stream);
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(out, dO, nout * sizeof(float), cudaMemcpyDeviceToHost));
    return B2_OK;
}
extern "C" int b2_texture_partials(b2_scene *s, uint64_t n, const float *pos_hit, int spp, int parity_mode, float *out) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    if (!pos_hit || !out || spp <= 0) return fail(ctx, B2_ERR_INVALID, "b2_texture_partials: invalid argument");
    if (s->ds.nItems) return fail(ctx, B2_ERR_INVALID, "b2_texture_partials: instanced scenes are not supported by this probe");
    CK(ctx, cudaSetDevice(ctx->device));
    TmpDev tmp;
    float *dI = tmp.upload(pos_hit, 6 * n), *dO = tmp.alloc<float>(6 * n);
    const float diffScale = 1.0f / std::sqrt((float) spp);
    if (parity_mode) parity::launch_texture_probe(s->cfgParity, s->ds, 1, 0, 0, diffScale, n, dI, dO, ctx->stream);
    else fast::launch_texture_probe(s->cfgFast, s->ds, 1, 0, 0, diffScale, n, dI, dO, ctx->stream);
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(out, dO, 6 * n * sizeof(float), cudaMemcpyDeviceToHost));
    return B2_OK;
}
// One level of the MIP pyramid b2_scene_commit built (host data; RGB or luminance as given).  `out` may be NULL to query the size.
extern "C" int b2_texture_level(b2_scene *s, int texture_id, int level, int *levels, int *width, int *height, float *out) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    if (texture_id < 0 || texture_id >= (int) s->textures.size()) return fail(ctx, B2_ERR_INVALID, "invalid texture id");
    const b2host::MipPyramid &mp = s->textures[texture_id].mip;
    if (level < 0 || level >= (int) mp.level.size()) return fail(ctx, B2_ERR_INVALID, "invalid MIP level");
    if (levels) *levels = (int) mp.level.size();
    if (width) *width = mp.w[level];
    if (height) *height = mp.h[level];
    if (out) memcpy(out, mp.level[level].data(), mp.level[level].size() * sizeof(float));
    return B2_OK;
}
extern "C" int b2_camera_rays(b2_scene *s, uint64_t n, const float *pos, int parity_mode, float *rays) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    CK(ctx, cudaSetDevice(ctx->device));
    TmpDev tmp;
    float *dP = tmp.upload(pos, 2 * n), *dR = tmp.alloc<float>(8 * n);
    if (parity_mode) parity::launch_camera_rays(s->cfgParity, s->ds, n, dP, dR, ctx->stream);
    else fast::launch_camera_rays(s->cfgFast, s->ds, n, dP, dR, ctx->stream);
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(rays, dR, 8 * n * sizeof(float), cudaMemcpyDeviceToHost));
    return B2_OK;
}
extern "C" int b2_sampler_stream(b2_scene *s, int sampler, uint64_t seed, int spp, int px, int py, int sample_idx, int ndim, float *out) {
    NEED_COMMIT(s);
    b2_ctx *ctx = s->ctx;
    CK(ctx, cudaSetDevice(ctx->device));
    b2_render_params p;
    memset(&p, 0, sizeof(p));
    p.spp = spp; p.sampler = sampler; p.seed = seed; p.max_depth = -1; p.rr_depth = 5;
    DRender r;
    int rc = fillRender(s, &p, r);
    if (rc) return rc;
    TmpDev tmp;
    float *dO = tmp.alloc<float>(ndim);
    parity::launch_sampler_stream(s->ds, r, px, py, sample_idx, ndim, dO, ctx->stream);
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(out, dO, ndim * sizeof(float), cudaMemcpyDeviceToHost));
    return B2_OK;
}
extern "C" int b2_splat(b2_ctx *ctx, int W, int H, int rfilter, float param, uint64_t n, const float *pos, const float *val, float *film) {
    if (!ctx || !pos || !val || !film || W <= 0 || H <= 0) return fail(ctx, B2_ERR_INVALID, "b2_splat: invalid argument");
    CK(ctx, cudaSetDevice(ctx->device));
    DFilter f;
    int rc = makeFilter(ctx, rfilter, param, f);
    if (rc) return rc;
    TmpDev tmp;
    const size_t nPix = (size_t) W * H;
    float *dP = tmp.upload(pos, 2 * n), *dV = tmp.upload(val, 4 * n);
    float4 *dRGBA = tmp.alloc<float4>(nPix);
    float *dW = tmp.alloc<float>(nPix), *dOut = tmp.alloc<float>(5 * nPix);
    cudaMemsetAsync(dRGBA, 0, nPix * sizeof(float4), ctx->stream);
    cudaMemsetAsync(dW, 0, nPix * sizeof(float), ctx->stream);
    LaunchCfg cfg;
    cfg.numSMs = ctx->numSMs;
    parity::launch_splat(cfg, f, W, H, n, dP, dV, dRGBA, dW, ctx->stream);
    parity::launch_film_pack(cfg, dRGBA, dW, dOut, nPix, ctx->stream);
    CK(ctx, cudaStreamSynchronize(ctx->stream));
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpy(film, dOut, 5 * nPix * sizeof(float), cudaMemcpyDeviceToHost));
    return B2_OK;
}
