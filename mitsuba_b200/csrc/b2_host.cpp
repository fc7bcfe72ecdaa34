// C-ABI implementation (include/b2mts.h): scene description, the wavefront render loop, film handling and the component entry points.
// b2_scene_commit is in b2_commit.cpp.
#include "b2_host.h"

#include <dlfcn.h>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <mutex>
#include <string>
#include <vector>

namespace {
std::string g_lastError;
std::mutex g_errMutex;
}

int fail(b2_ctx *ctx, int code, const std::string &msg) {
    {
        std::lock_guard<std::mutex> g(g_errMutex);
        g_lastError = msg;
    }
    if (ctx) ctx->lastError = msg;
    return code;
}
extern "C" int b2_set_error_(b2_ctx *ctx, int code, const char *msg) { return fail(ctx, code, msg ? msg : ""); }

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
    const cudaStream_t st = ctx->stream;
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
            cudaMemcpyAsync(ctx->dNib, nib.data(), nib.size() * 4, cudaMemcpyHostToDevice, st) != cudaSuccess) {
            b2_context_destroy(ctx);
            return fail(nullptr, B2_ERR_CUDA, "b2_context_create: upload of the Sobol' nibble tables failed");
        }
    }
    if (cudaMalloc((void **) &ctx->dM32, m32.size() * 4) != cudaSuccess || cudaMalloc((void **) &ctx->dVdc, vdc.size() * 8) != cudaSuccess ||
        cudaMalloc((void **) &ctx->dInv, inv.size() * 8) != cudaSuccess ||
        cudaMemcpyAsync(ctx->dM32, m32.data(), m32.size() * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(ctx->dVdc, vdc.data(), vdc.size() * 8, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(ctx->dInv, inv.data(), inv.size() * 8, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) {
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
    s->accelBuild = ctx->accelBuild;
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

static bool validAccelBuild(int mode) { return mode == B2_ACCEL_BUILD_HOST || mode == B2_ACCEL_BUILD_DEVICE; }
extern "C" int b2_scene_set_accel_build(b2_scene *s, int mode) {
    if (!s) return fail(nullptr, B2_ERR_INVALID, "b2_scene_set_accel_build: null scene");
    if (!validAccelBuild(mode))
        return fail(s->ctx, B2_ERR_INVALID, "b2_scene_set_accel_build: unknown mode " + std::to_string(mode) + " (B2_ACCEL_BUILD_HOST = 0, B2_ACCEL_BUILD_DEVICE = 1)");
    if (s->committed) return fail(s->ctx, B2_ERR_INVALID, "b2_scene_set_accel_build: the scene is already committed; choose the builder before b2_scene_commit");
    s->accelBuild = mode;
    return B2_OK;
}
extern "C" int b2_context_set_accel_build(b2_ctx *ctx, int mode) {
    if (!ctx) return fail(nullptr, B2_ERR_INVALID, "b2_context_set_accel_build: null context");
    if (!validAccelBuild(mode))
        return fail(ctx, B2_ERR_INVALID, "b2_context_set_accel_build: unknown mode " + std::to_string(mode) + " (B2_ACCEL_BUILD_HOST = 0, B2_ACCEL_BUILD_DEVICE = 1)");
    ctx->accelBuild = mode;
    return B2_OK;
}

extern "C" int b2_scene_get_accel(b2_scene *s, int which, void *out, uint64_t *bytes) {
    if (!s || !bytes) return fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_scene_get_accel: null argument");
    if (!s->committed) return fail(s->ctx, B2_ERR_INVALID, "b2_scene_get_accel: scene not committed");
    const DScene &ds = s->ds;
    const void *src = nullptr;
    uint64_t size = 0;
    switch (which) {
    case B2_ACCEL_NODES: src = ds.nodes; size = (uint64_t) ds.nNodes * sizeof(BVHNode); break;
    case B2_ACCEL_NODES8: src = ds.nodes8; size = ds.nodes8 ? (uint64_t) ds.nNodes8 * sizeof(BVH8Node) : 0; break;
    case B2_ACCEL_LEAF_PRIMS: src = ds.leafPrim; size = (uint64_t) ds.nLeafTris * sizeof(uint32_t); break;
    default: return fail(s->ctx, B2_ERR_INVALID, "b2_scene_get_accel: unknown array " + std::to_string(which));
    }
    if (!out) { *bytes = size; return B2_OK; }
    if (*bytes < size) return fail(s->ctx, B2_ERR_INVALID, "b2_scene_get_accel: buffer too small");
    CK(s->ctx, cudaSetDevice(s->ctx->device));
    if (size) CK(s->ctx, cudaMemcpy(out, src, size, cudaMemcpyDeviceToHost));
    *bytes = size;
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
    if (p->integrator != B2_INTEGRATOR_PATH && p->integrator != B2_INTEGRATOR_VOLPATH && p->integrator != B2_INTEGRATOR_DIRECT)
        return fail(ctx, B2_ERR_INVALID, "unknown integrator");
    if (p->integrator == B2_INTEGRATOR_DIRECT) { // direct.cpp:93-108
        if (p->emitter_samples < 0 || p->bsdf_samples < 0) return fail(ctx, B2_ERR_INVALID, "direct: 'emitterSamples' and 'bsdfSamples' must not be negative");
        if (p->emitter_samples + p->bsdf_samples == 0) return fail(ctx, B2_ERR_INVALID, "direct: 'emitterSamples' + 'bsdfSamples' must be positive");
        // the index of an array entry, s * count + k, is a 32-bit sample index of the pixel (sobol.cpp:190)
        if ((uint64_t) p->spp * (uint64_t) std::max(p->emitter_samples, p->bsdf_samples) >= (1ull << 32))
            return fail(ctx, B2_ERR_INVALID, "direct: sampleCount x max(emitterSamples, bsdfSamples) must be below 2^32");
        if (p->flags & (32 | 64)) return fail(ctx, B2_ERR_INVALID, "direct: per-path diagnostics (flags bit5 / bit6) have no meaning without paths");
        r.emitterSamples = p->emitter_samples; r.bsdfSamples = p->bsdf_samples;
    }
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
    { // samples per tile visit: the largest divisor of the sample count that does not exceed `want` (0 = all samples at once).
      // A 5 x 5 gaussian splat wants the in-flight paths spread over many pixels (the L2 serialises atomics per address), a 1-pixel box
      // splat does not.
        const uint32_t nS = (uint32_t) (r.sampleHi - r.sampleLo);
        const uint32_t want = p->rfilter == B2_RFILTER_GAUSSIAN ? 8 : 0;
        r.roundSpp = nS;
        if (want > 0 && want < nS)
            for (uint32_t d = want; d >= 1; --d)
                if (nS % d == 0) { r.roundSpp = d; break; }
    }
    r.totalWork = (uint64_t) s->W * (uint64_t) s->H * (uint64_t) (r.sampleHi - r.sampleLo);
    // nibble tables of sobol::look_up for this m (sobolseq.h:104-133) and the nibble counts that cover the indices
    auto bitsOf = [](uint64_t v) { uint32_t b = 0; while (v) { ++b; v >>= 1; } return b; };
    // `direct` with sample arrays also looks up the pixel's points s * n + k below spp * n (sobol.cpp:190)
    uint64_t maxFrame = (uint64_t) r.sampleHi - 1;
    if (p->integrator == B2_INTEGRATOR_DIRECT && std::max(r.emitterSamples, r.bsdfSamples) > 1)
        maxFrame = (uint64_t) p->spp * (uint64_t) std::max(r.emitterSamples, r.bsdfSamples) - 1;
    const uint32_t frameBits = std::max(1u, bitsOf(maxFrame));
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
        if (cudaMemcpyAsync(s->dLookupNib.p, lut.data(), lut.size() * 8, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess)
            return fail(ctx, B2_ERR_CUDA, "upload of lookup tables failed");
        r.lookupNib = s->dLookupNib.p;
    }
    return B2_OK;
}

// Points the scene's DPool and `r` at a pool of Q empty slots and at a cleared progress ring.
static int ensurePool(b2_scene *s, uint32_t Q, bool vol, DRender &r) {
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
    CK(ctx, cudaMemsetAsync(R.pFlags.p, 0, (size_t) Q * sizeof(uint32_t), ctx->stream));
    if (!R.hRing) {
        CK(ctx, cudaHostAlloc((void **) &R.hRing, sizeof(unsigned long long) * 4 * B2_RING, cudaHostAllocMapped));
        CK(ctx, cudaHostGetDevicePointer((void **) &R.dRing, R.hRing, 0));
    }
    memset(R.hRing, 0, sizeof(unsigned long long) * 4 * B2_RING);
    r.ring = R.dRing;
    return B2_OK;
}

// The route of a `path` / `volpath` render: which kernels one iteration launches, and how many paths are in flight.
struct Route {
    bool volpath, sorted, resident;
    int shadeClass; // unsorted shading: the instance of the scene's one BSDF class, -1 for the generic one
    uint32_t Q;
};
static Route chooseRoute(const b2_scene *s, const b2_render_params *p, DRender &r) {
    Route w;
    w.volpath = p->integrator == B2_INTEGRATOR_VOLPATH;
    int nClasses = 0, onlyClass = -1;
    for (int c = 0; c < B2_NCLASS; ++c)
        if (s->classPresent[c]) { ++nClasses; onlyClass = c == B2_NCLASS - 1 ? -1 : c; }
    w.shadeClass = nClasses == 1 ? onlyClass : -1;
    // more than one class: k_extend bins the hits by BSDF class and every class gets its own shading launch over its queue -- the four
    // specialised instances, and the generic instance for the rest (null, twosided, dielectric, conductor, plastic); scenes with bitmap
    // textures or an environment map use the TEX instances of the same classes (launch_shade)
    w.sorted = nClasses > 1 && !(p->flags & 2);
    // a shared-memory resident scene shaded by one instance: k_bounce_flat runs each path to its end (or its vertex budget) and k_generate
    // drains the pool in slot order
    w.resident = !w.volpath && s->ds.rootCount && !w.sorted;
    r.drainSlots = w.resident ? 1 : 0;
    // 4M paths (~0.6 GB); also on the resident route, where Q only sets how much work one launch covers: 8 Mi and 16 Mi were slower
    // at the Cornell headline (DESIGN.md section 6)
    uint32_t Q = p->pool_size > 0 ? (uint32_t) p->pool_size : (1u << 22);
    Q = std::max<uint32_t>(Q, 1024u);
    Q = (uint32_t) std::min<uint64_t>(Q, std::max<uint64_t>(1024u, r.totalWork));
    w.Q = (Q + 255u) & ~255u;
    return w;
}

// The cleared diagnostic buffers of a `path` / `volpath` render: time stamps (flags bit2), pixel statistics (bit5), path traces (bit6)
static int diagnosticBuffers(b2_scene *s, const b2_render_params *p, DRender &r) {
    b2_ctx *ctx = s->ctx;
    RenderStore &R = *ctx->store;
    const cudaStream_t st = ctx->stream;
    const size_t nPix = (size_t) s->W * s->H;
    if (p->flags & 4) { // per-launch device time stamps (%globaltimer inside the kernels)
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
    return B2_OK;
}

// CUDA events around the stages of every iteration (flags bit3), reused from render to render: tick(stage) records the start of a stage,
// tick(-1) its end
struct StageEvents {
    b2_scene *s;
    bool on;
    std::vector<std::pair<int, size_t>> timed; // (stage, index of the start event)
    size_t used = 0;
    void tick(int stage) {
        if (!on) return;
        if (used == s->timingEvents.size()) { cudaEvent_t e; cudaEventCreate(&e); s->timingEvents.push_back(e); }
        cudaEventRecord(s->timingEvents[used], s->ctx->stream);
        if (stage >= 0) timed.emplace_back(stage, used);
        ++used;
    }
};

// Queues one iteration and returns its number of kernel launches.  One iteration = generate (+publish) -> extend -> shade (per material
// class) -> occluded; flat scenes shaded by one launch: generate (+publish) -> bounce
static int enqueueIteration(b2_scene *s, const Route &w, const DRender &r, const DFilter &filt, const Kernels &kn, StageEvents &ev) {
    const KernelSet &K = kn.set;
    const LaunchCfg &cfg = kn.cfg;
    const cudaStream_t st = s->ctx->stream;
    ev.tick(0); K.generate(cfg, s->ds, s->pool, r, filt, st); ev.tick(-1);
    if (w.volpath) { // volpath: every ray of an iteration is cast inline by k_volstep_lockstep
        ev.tick(2); K.volstep(cfg, s->ds, s->pool, r, st); ev.tick(-1);
        return 3;
    }
    if (w.resident) { // shared-memory resident scene, one shading instance: extend + shade + occluded in one launch
        ev.tick(2); K.bounce_flat(cfg, s->ds, s->pool, r, w.shadeClass, st); ev.tick(-1);
        return 3;
    }
    int launches = 0;
    ev.tick(1); K.extend(cfg, s->ds, s->pool, r, w.sorted, st); ev.tick(-1); ++launches;
    ev.tick(2);
    if (w.sorted) {
        for (int c = 0; c < B2_NCLASS; ++c)
            if (s->classPresent[c]) { K.shade(cfg, s->ds, s->pool, r, c, true, st); ++launches; }
    } else {
        K.shade(cfg, s->ds, s->pool, r, w.shadeClass, false, st);
        ++launches;
    }
    ev.tick(-1);
    ev.tick(3); K.occluded(cfg, s->ds, s->pool, r, st); ev.tick(-1); ++launches;
    return launches + 2;
}

// The state of one render between its set-up and its tear-down: the start and stop events, the captured graph and the counts the
// launch loop reports.  Its destructor leaves the stream idle and releases the events and the graph on every return path.
struct RenderRun {
    cudaStream_t st;
    cudaEvent_t start = nullptr, stop = nullptr;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    uint64_t iterations = 0, launches = 0;
    ~RenderRun() {
        cudaStreamSynchronize(st);
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
        if (start) cudaEventDestroy(start);
        if (stop) cudaEventDestroy(stop);
    }
};

// Runs the iterations of a `path` / `volpath` render until the progress k_publish writes into the mapped ring shows no path alive and
// every work item handed out; the cancel flag is read before each iteration.  The iterations replay one captured iteration (CTR_ITER,
// advanced by k_publish, numbers them on the device) or, with flags bit3, are queued one by one and timed by `ev`.
static int iterate(b2_scene *s, const Route &w, const DRender &r, const DFilter &filt, const Kernels &kn, StageEvents &ev, RenderRun &run) {
    b2_ctx *ctx = s->ctx;
    const cudaStream_t st = ctx->stream;
    const bool graph = !ev.on;
    auto enqueue = [&] { return enqueueIteration(s, w, r, filt, kn, ev); };
    int perIter = 0;
    if (graph) {
        if (w.volpath || s->ds.nTextures || s->ds.envmap) {
            // k_volstep_lockstep (and the textured k_shade) have a deep local-memory frame: their first launch may have to grow the context's
            // local-memory pool, which is not allowed inside a stream capture.  The first iteration therefore runs as plain launches.
            run.launches += enqueue();
            ++run.iterations;
        }
        CK(ctx, cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        perIter = enqueue();
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        cudaStreamIsCapturing(st, &cs);
        const cudaError_t le = cudaPeekAtLastError();
        if (cs != cudaStreamCaptureStatusActive || le != cudaSuccess) {
            cudaStreamEndCapture(st, &run.graph);
            cudaGetLastError();
            return fail(ctx, B2_ERR_CUDA, std::string("graph capture of the iteration failed: ") + cudaGetErrorString(le) +
                                          (w.volpath ? " (volpath), grid " + std::to_string(kn.cfg.gridVolLockstep) : std::string(" (path)")) + ", smem " + std::to_string(kn.cfg.traceSmem));
        }
        CK(ctx, cudaStreamEndCapture(st, &run.graph));
        CK(ctx, cudaGraphInstantiate(&run.exec, run.graph, 0));
    }
    volatile unsigned long long *ring = ctx->store->hRing;
    uint64_t &iter = run.iterations;
    uint64_t checked = 0;
    for (;;) {
        if (s->cancel.load()) return B2_ERR_CANCELLED;
        // consume published progress; never run more than B2_RING - 1 iterations ahead of the device
        for (;;) {
            while (checked < iter && ring[(checked % B2_RING) * 4] == checked + 1) {
                const unsigned long long active = ring[(checked % B2_RING) * 4 + 1], next = ring[(checked % B2_RING) * 4 + 2];
                ++checked;
                if (active == 0 && next >= r.totalWork) return B2_OK;
            }
            if (iter - checked < (uint64_t) B2_RING - 1) break;
            if (cudaStreamQuery(st) != cudaErrorNotReady && ring[(checked % B2_RING) * 4] != checked + 1) {
                cudaError_t e = cudaStreamSynchronize(st);
                if (ring[(checked % B2_RING) * 4] != checked + 1)
                    return fail(ctx, B2_ERR_CUDA, std::string("render loop: device made no progress: ") + cudaGetErrorString(e == cudaSuccess ? cudaGetLastError() : e));
            }
        }
        if (!graph) perIter = enqueue();
        else if (cudaGraphLaunch(run.exec, st) != cudaSuccess) return fail(ctx, B2_ERR_CUDA, "cudaGraphLaunch failed");
        run.launches += perIter;
        ++iter;
        if (iter > 100000000ull) return fail(ctx, B2_ERR_CUDA, "render loop did not terminate");
    }
}

// Adds the per-stage device times of a finished render to the zeroed b2_stats::ms_* and n_*: from the CUDA events around each stage
// (flags bit3), or from the %globaltimer stamps of the first B2_MAX_STAMPS iterations (`stamps`: flags bit2 in graph mode).
static int stageTimes(b2_scene *s, const StageEvents &ev, bool stamps) {
    b2_ctx *ctx = s->ctx;
    RenderStore &R = *ctx->store;
    b2_stats &t = s->stats;
    float *ms[4] = {&t.ms_generate, &t.ms_extend, &t.ms_shade, &t.ms_occluded};
    uint64_t *cnt[4] = {&t.n_generate, &t.n_extend, &t.n_shade, &t.n_occluded};
    for (auto &te : ev.timed) {
        float e = 0;
        cudaEventElapsedTime(&e, s->timingEvents[te.second], s->timingEvents[te.second + 1]);
        *ms[te.first] += e;
        ++*cnt[te.first];
    }
    if (!stamps) return B2_OK;
    const size_t nIt = (size_t) std::min<uint64_t>(t.iterations, B2_MAX_STAMPS);
    std::vector<unsigned long long> a(nIt * 4), b(nIt * 4);
    if (nIt) {
        CK(ctx, cudaMemcpy(a.data(), R.dStampStart.p, nIt * 4 * 8, cudaMemcpyDeviceToHost));
        CK(ctx, cudaMemcpy(b.data(), R.dStampEnd.p, nIt * 4 * 8, cudaMemcpyDeviceToHost));
    }
    double acc[4] = {0, 0, 0, 0};
    for (size_t i = 0; i < nIt; ++i)
        for (int k = 0; k < 4; ++k)
            if (b[i * 4 + k] > a[i * 4 + k] && a[i * 4 + k] != ~0ull) { acc[k] += (double) (b[i * 4 + k] - a[i * 4 + k]) * 1e-6; ++*cnt[k]; }
    for (int k = 0; k < 4; ++k) *ms[k] = (float) acc[k];
    return B2_OK;
}

// The call path of every render: clears the film accumulators (pointing `r` at them), the counters and the cancel flag; runs loop(run),
// the integrator's launches, between the start and stop events; packs the film into `film` (host or device) if the loop returned B2_OK;
// synchronises once, reads the counters back and fills the b2_stats fields every integrator shares.  Returns the loop's status.
template <typename Loop>
static int renderCall(b2_scene *s, const b2_render_params *p, float *film, DRender &r, const Kernels &kn, uint32_t poolSize, Loop &&loop) {
    b2_ctx *ctx = s->ctx;
    RenderStore &R = *ctx->store;
    const cudaStream_t st = ctx->stream;
    const size_t nPix = (size_t) s->W * s->H;
    CK(ctx, R.dFilmRGBA.alloc(nPix));
    CK(ctx, R.dFilmW.alloc(nPix));
    r.filmRGBA = R.dFilmRGBA.p; r.filmW = R.dFilmW.p;
    CK(ctx, cudaMemsetAsync(R.dFilmRGBA.p, 0, nPix * sizeof(float4), st));
    CK(ctx, cudaMemsetAsync(R.dFilmW.p, 0, nPix * sizeof(float), st));
    CK(ctx, cudaMemsetAsync(s->dCounters.p, 0, CTR_COUNT * sizeof(unsigned long long), st));
    s->cancel.store(0);
    RenderRun run{st};
    CK(ctx, cudaEventCreate(&run.start));
    CK(ctx, cudaEventCreate(&run.stop));
    CK(ctx, cudaEventRecord(run.start, st));
    const int status = loop(run);
    CK(ctx, cudaEventRecord(run.stop, st));
    if (status == B2_OK) {
        float *dOut = film;
        if (!p->film_on_device) {
            CK(ctx, R.dFilmOut.alloc(nPix * 5));
            dOut = R.dFilmOut.p;
        }
        kn.set.film_pack(kn.cfg, R.dFilmRGBA.p, R.dFilmW.p, dOut, nPix, st);
        if (!p->film_on_device) CK(ctx, cudaMemcpyAsync(film, dOut, nPix * 5 * sizeof(float), cudaMemcpyDeviceToHost, st));
    }
    CK(ctx, cudaStreamSynchronize(st));
    CK(ctx, cudaGetLastError());
    std::vector<unsigned long long> ctr(CTR_COUNT);
    CK(ctx, cudaMemcpy(ctr.data(), s->dCounters.p, CTR_COUNT * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    float ms = 0;
    cudaEventElapsedTime(&ms, run.start, run.stop);
    b2_stats &t = s->stats;
    t.ms_generate = t.ms_extend = t.ms_shade = t.ms_occluded = 0;
    t.n_generate = t.n_extend = t.n_shade = t.n_occluded = 0;
    t.pool_size = poolSize;
    t.unoccluded_shadow_rays = ctr[CTR_UNOCCLUDED];
    t.samples = ctr[CTR_SAMPLES]; t.rays = ctr[CTR_RAYS]; t.shadow_rays = ctr[CTR_SHADOWRAYS]; t.path_length_sum = ctr[CTR_PATHLEN];
    t.bad_samples = ctr[CTR_BAD]; t.dim_overflow = ctr[CTR_DIMOVF]; t.iterations = run.iterations; t.kernel_launches = run.launches + 1;
    t.ms_total = ms;
    return status;
}

// `direct`: k_direct over the work items in slices of whole samples of the film, so that b2_cancel is honoured between launches; no
// path pool, and every launch counts as an iteration.  k_direct never adds to CTR_PATHLEN, so path_length_sum stays 0.
static int directSlices(b2_scene *s, const DRender &r, const DFilter &filt, const Kernels &kn, RenderRun &run) {
    const cudaStream_t st = s->ctx->stream;
    // a slice: enough whole samples of the film for ~16M items (a few ms on the flat route), at least one sample; the cancel flag is
    // read before each launch
    const uint64_t perSample = (uint64_t) s->W * s->H, nS = (uint64_t) (r.sampleHi - r.sampleLo);
    const uint64_t slice = perSample * std::max<uint64_t>(1, std::min<uint64_t>(nS, (16ull << 20) / std::max<uint64_t>(1, perSample)));
    int status = B2_OK;
    for (uint64_t b = 0; b < r.totalWork; b += slice) {
        if (s->cancel.load()) { status = B2_ERR_CANCELLED; break; }
        if (run.launches >= 2) cudaStreamSynchronize(st); // from the third slice on, the host waits for the queued ones: a cancel waits for at most two slices, not for the render
        kn.set.direct(kn.cfg, s->ds, r, filt, s->dCounters.p, b, std::min(r.totalWork, b + slice), st);
        run.iterations = ++run.launches;
    }
    CK(s->ctx, cudaGetLastError());
    return status;
}

extern "C" int b2_render(b2_scene *s, const b2_render_params *p, float *film) {
    if (!s || !p || !film) return fail(s ? s->ctx : nullptr, B2_ERR_INVALID, "b2_render: null argument");
    b2_ctx *ctx = s->ctx;
    if (!s->committed) return fail(ctx, B2_ERR_INVALID, "b2_render: scene not committed");
    CK(ctx, cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> renderLock(ctx->store->renderMutex);
    DRender r;
    if (int rc = fillRender(s, p, r)) return rc;
    DFilter filt;
    if (int rc = makeFilter(ctx, p->rfilter, p->rfilter_param, filt)) return rc;
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
    const Kernels kn = kernelsFor(s, parityMode);
    if (p->integrator == B2_INTEGRATOR_DIRECT)
        return renderCall(s, p, film, r, kn, 0, [&](RenderRun &run) { return directSlices(s, r, filt, kn, run); });
    if (int rc = diagnosticBuffers(s, p, r)) return rc;
    const Route w = chooseRoute(s, p, r);
    if (int rc = ensurePool(s, w.Q, w.volpath, r)) return rc;
    const bool useEvents = (p->flags & 8) != 0; // no graph: plain launches bracketed by CUDA events (cross-check path)
    StageEvents ev{s, useEvents};
    const int status = renderCall(s, p, film, r, kn, w.Q, [&](RenderRun &run) { return iterate(s, w, r, filt, kn, ev, run); });
    if (status != B2_OK && status != B2_ERR_CANCELLED) return status; // the stats may still be those of the render before
    if (int rc = stageTimes(s, ev, (p->flags & 4) && !useEvents)) return rc;
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
#define NEED_COMMIT(s) if (!(s) || !(s)->committed) return fail((s) ? (s)->ctx : nullptr, B2_ERR_INVALID, "scene not committed")

// A host array of floats that a component call reads (In) or writes (Out).
struct In { const float *p; size_t n; };
struct Out { float *p; size_t n; };
// The call path of the component entry points: refuses a null array that is not empty, allocates a device buffer per array, queues the
// uploads, runs launch(d) with the device arrays (the inputs, then the outputs, each in the order given), checks the launch, queues the
// read-backs and synchronises once.  The buffers are freed on every return.
template <typename Launch>
static int componentCall(b2_ctx *ctx, const char *name, const std::vector<In> &in, const std::vector<Out> &out, Launch &&launch) {
    for (const In &a : in) if (!a.p && a.n) return fail(ctx, B2_ERR_INVALID, std::string(name) + ": null argument");
    for (const Out &a : out) if (!a.p && a.n) return fail(ctx, B2_ERR_INVALID, std::string(name) + ": null argument");
    CK(ctx, cudaSetDevice(ctx->device));
    const cudaStream_t st = ctx->stream;
    std::vector<DevBuf<float>> buf(in.size() + out.size());
    std::vector<float *> d(buf.size());
    for (size_t k = 0; k < buf.size(); ++k) {
        if (buf[k].alloc(std::max<size_t>(k < in.size() ? in[k].n : out[k - in.size()].n, 1)) != cudaSuccess)
            return fail(ctx, B2_ERR_CUDA, std::string(name) + ": device allocation failed");
        d[k] = buf[k].p;
    }
    for (size_t k = 0; k < in.size(); ++k)
        if (in[k].n) CK(ctx, cudaMemcpyAsync(d[k], in[k].p, in[k].n * sizeof(float), cudaMemcpyHostToDevice, st));
    launch(d.data());
    CK(ctx, cudaGetLastError());
    for (size_t k = 0; k < out.size(); ++k)
        if (out[k].n) CK(ctx, cudaMemcpyAsync(out[k].p, d[in.size() + k], out[k].n * sizeof(float), cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    return B2_OK;
}

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
    if (count) CK(ctx, cudaMemsetAsync(s->dCounters.p + CTR_NODEVIS, 0, 16, st));
    CK(ctx, cudaMemsetAsync(s->dCounters.p + CTR_TICKET_EXT, 0, 8, st));
    const Kernels kn = kernelsFor(s, parity_mode != 0);
    // the events bracket the kernel alone: ms_kernel is the `traversal` figure of bench.py
    if (int rc = componentCall(ctx, "b2_trace_device", {}, {}, [&](float *const *) {
            cudaEventRecord(ev.a, st);
            kn.set.trace(kn.cfg, s->ds, (const float4 *) d_rays, (float4 *) d_tuvp, n, shadow, count, s->dCounters.p, st);
            cudaEventRecord(ev.b, st);
        }))
        return rc;
    float ms = 0;
    cudaEventElapsedTime(&ms, ev.a, ev.b);
    if (ms_kernel) *ms_kernel = ms;
    if (count) {
        unsigned long long c[2];
        CK(ctx, cudaMemcpy(c, s->dCounters.p + CTR_NODEVIS, 16, cudaMemcpyDeviceToHost));
        s->stats.node_visits = c[0]; s->stats.prim_tests = c[1];
    }
    return B2_OK;
}
extern "C" int b2_trace(b2_scene *s, uint64_t n, const float *rays, int mode, int parity_mode, float *t, float *u, float *v, uint32_t *prim,
                        float *ms_kernel) {
    NEED_COMMIT(s);
    if (n > 0xFFFFFFFFull) return fail(s->ctx, B2_ERR_INVALID, "b2_trace: at most 2^32-1 rays per call");
    std::vector<float> h(4 * n);
    int rc = B2_OK;
    if (int e = componentCall(s->ctx, "b2_trace", {{rays, 8 * n}}, {{h.data(), 4 * n}},
                              [&](float *const *d) { rc = b2_trace_device(s, n, d[0], mode, parity_mode, d[1], ms_kernel); }))
        return e;
    if (rc) return rc;
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
    if (mat < 0 || mat >= (int) s->materials.size()) return fail(s->ctx, B2_ERR_INVALID, "invalid material id");
    const Kernels kn = kernelsFor(s, parity_mode != 0);
    return componentCall(s->ctx, "b2_bsdf_eval", {{wi, 3 * n}, {wo, 3 * n}}, {{out_rgb, 3 * n}, {out_pdf, n}},
                         [&](float *const *d) { kn.set.bsdf_eval(kn.cfg, s->ds, mat, n, d[0], d[1], d[2], d[3], s->ctx->stream); });
}
extern "C" int b2_bsdf_sample(b2_scene *s, int mat, uint64_t n, const float *wi, const float *samples, int parity_mode, float *out) {
    NEED_COMMIT(s);
    if (mat < 0 || mat >= (int) s->materials.size()) return fail(s->ctx, B2_ERR_INVALID, "invalid material id");
    const Kernels kn = kernelsFor(s, parity_mode != 0);
    return componentCall(s->ctx, "b2_bsdf_sample", {{wi, 3 * n}, {samples, 3 * n}}, {{out, 10 * n}},
                         [&](float *const *d) { kn.set.bsdf_sample(kn.cfg, s->ds, mat, n, d[0], d[1], d[2], s->ctx->stream); });
}
extern "C" int b2_sample_emitter_direct(b2_scene *s, uint64_t n, const float *ref, const float *samples, int parity_mode, float *out) {
    NEED_COMMIT(s);
    if (s->emitters.empty()) return fail(s->ctx, B2_ERR_INVALID, "scene has no emitters");
    const Kernels kn = kernelsFor(s, parity_mode != 0);
    if (int rc = componentCall(s->ctx, "b2_sample_emitter_direct", {{ref, 6 * n}, {samples, 2 * n}}, {{out, 12 * n}},
                               [&](float *const *d) { kn.set.emitter_direct(kn.cfg, s->ds, n, d[0], d[1], d[2], s->ctx->stream); }))
        return rc;
    // fold the visibility test (scene.cpp:838-843) into `visible` with the occlusion kernel
    std::vector<float> rays(8 * n);
    for (uint64_t i = 0; i < n; ++i) {
        float *r = &rays[8 * i];
        r[0] = ref[6 * i]; r[1] = ref[6 * i + 1]; r[2] = ref[6 * i + 2]; r[3] = 1e-4f;
        r[4] = out[12 * i]; r[5] = out[12 * i + 1]; r[6] = out[12 * i + 2]; r[7] = out[12 * i + 3] * (1 - 1e-3f);
    }
    std::vector<uint32_t> occ(n);
    if (int rc = b2_trace(s, n, rays.data(), 1, parity_mode, nullptr, nullptr, nullptr, occ.data(), nullptr)) return rc;
    for (uint64_t i = 0; i < n; ++i) {
        float *o = &out[12 * i];
        if (o[8] != 0 && occ[i]) { o[8] = 0; o[4] = 0; o[5] = o[6] = o[7] = 0; }
        else if (o[8] == 0) { o[4] = 0; }
    }
    return B2_OK;
}
// Medium component probe (parity tests): what = 0 evalTransmittance (in: n x 8 ray floats, out n x 3), 1 sampleDistance (out n x 12),
// 2 density lookup (in n x 3, out n), 3 phase sample (in n x 5: wi, two uniforms; out n x 5: wo, pdf, eval)
extern "C" int b2_medium_probe(b2_scene *s, int medium, int what, uint64_t n, const float *in, uint64_t seed, int parity_mode, float *out) {
    NEED_COMMIT(s);
    if (medium < 0 || medium >= (int) s->media.size()) return fail(s->ctx, B2_ERR_INVALID, "invalid medium id");
    if (what < 0 || what > 3 || !in || !out) return fail(s->ctx, B2_ERR_INVALID, "b2_medium_probe: invalid argument");
    static const int inW[4] = {8, 8, 3, 5}, outW[4] = {3, 12, 1, 5};
    const Kernels kn = kernelsFor(s, parity_mode != 0);
    return componentCall(s->ctx, "b2_medium_probe", {{in, inW[what] * n}}, {{out, outW[what] * n}},
                         [&](float *const *d) { kn.set.medium_probe(kn.cfg, s->ds, medium, what, n, d[0], seed, d[1], s->ctx->stream); });
}
// Texture probes (parity tests)
extern "C" int b2_texture_eval(b2_scene *s, int texture_id, uint64_t n, const float *uv, const float *partials, int parity_mode, float *out) {
    NEED_COMMIT(s);
    if (texture_id < 0 || texture_id >= (int) s->textures.size()) return fail(s->ctx, B2_ERR_INVALID, "invalid texture id");
    if (!uv || !out) return fail(s->ctx, B2_ERR_INVALID, "b2_texture_eval: null argument");
    std::vector<float> in(6 * n, 0.0f);
    for (uint64_t i = 0; i < n; ++i) {
        in[6 * i] = uv[2 * i]; in[6 * i + 1] = uv[2 * i + 1];
        if (partials) for (int k = 0; k < 4; ++k) in[6 * i + 2 + k] = partials[4 * i + k];
    }
    const Kernels kn = kernelsFor(s, parity_mode != 0);
    return componentCall(s->ctx, "b2_texture_eval", {{in.data(), 6 * n}}, {{out, 3 * n}}, [&](float *const *d) {
        kn.set.texture_probe(kn.cfg, s->ds, 0, texture_id, partials ? 1 : 0, 1.0f, n, d[0], d[1], s->ctx->stream);
    });
}
// Probes of the committed environment map (tests): what 0 = Scene::evalEnvironment for n directions (in 3n -> out 3n), 1 = the same for sensor
// rays with differential directions (in 9n: d, rxD, ryD -> out 3n), 2 = Scene::pdfEmitterDirect of the map for n directions (in 3n -> out n)
extern "C" int b2_envmap_probe(b2_scene *s, int what, uint64_t n, const float *in, int parity_mode, float *out) {
    NEED_COMMIT(s);
    if (!s->envmap) return fail(s->ctx, B2_ERR_INVALID, "b2_envmap_probe: the scene has no environment map");
    if (!in || !out || what < 0 || what > 2) return fail(s->ctx, B2_ERR_INVALID, "b2_envmap_probe: invalid argument");
    const Kernels kn = kernelsFor(s, parity_mode != 0);
    return componentCall(s->ctx, "b2_envmap_probe", {{in, (what == 1 ? 9 : 3) * n}}, {{out, (what == 2 ? 1 : 3) * n}},
                         [&](float *const *d) { kn.set.envmap_probe(kn.cfg, s->ds, what, n, d[0], d[1], s->ctx->stream); });
}
extern "C" int b2_texture_partials(b2_scene *s, uint64_t n, const float *pos_hit, int spp, int parity_mode, float *out) {
    NEED_COMMIT(s);
    if (!pos_hit || !out || spp <= 0) return fail(s->ctx, B2_ERR_INVALID, "b2_texture_partials: invalid argument");
    if (s->ds.nItems) return fail(s->ctx, B2_ERR_INVALID, "b2_texture_partials: instanced scenes are not supported by this probe");
    const float diffScale = 1.0f / std::sqrt((float) spp);
    const Kernels kn = kernelsFor(s, parity_mode != 0);
    return componentCall(s->ctx, "b2_texture_partials", {{pos_hit, 6 * n}}, {{out, 6 * n}},
                         [&](float *const *d) { kn.set.texture_probe(kn.cfg, s->ds, 1, 0, 0, diffScale, n, d[0], d[1], s->ctx->stream); });
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
    const Kernels kn = kernelsFor(s, parity_mode != 0);
    return componentCall(s->ctx, "b2_camera_rays", {{pos, 2 * n}}, {{rays, 8 * n}},
                         [&](float *const *d) { kn.set.camera_rays(kn.cfg, s->ds, n, d[0], d[1], s->ctx->stream); });
}
extern "C" int b2_sampler_stream(b2_scene *s, int sampler, uint64_t seed, int spp, int px, int py, int sample_idx, int ndim, float *out) {
    NEED_COMMIT(s);
    CK(s->ctx, cudaSetDevice(s->ctx->device));
    b2_render_params p;
    memset(&p, 0, sizeof(p));
    p.spp = spp; p.sampler = sampler; p.seed = seed; p.max_depth = -1; p.rr_depth = 5;
    DRender r;
    if (int rc = fillRender(s, &p, r)) return rc;
    return componentCall(s->ctx, "b2_sampler_stream", {}, {{out, (size_t) ndim}},
                         [&](float *const *d) { parity::kernels.sampler_stream(s->ds, r, px, py, sample_idx, ndim, d[0], s->ctx->stream); });
}
extern "C" int b2_splat(b2_ctx *ctx, int W, int H, int rfilter, float param, uint64_t n, const float *pos, const float *val, float *film) {
    if (!ctx || !pos || !val || !film || W <= 0 || H <= 0) return fail(ctx, B2_ERR_INVALID, "b2_splat: invalid argument");
    DFilter f;
    if (int rc = makeFilter(ctx, rfilter, param, f)) return rc;
    CK(ctx, cudaSetDevice(ctx->device));
    const size_t nPix = (size_t) W * H;
    DevBuf<float4> rgba;
    DevBuf<float> w;
    CK(ctx, rgba.alloc(nPix));
    CK(ctx, w.alloc(nPix));
    CK(ctx, cudaMemsetAsync(rgba.p, 0, nPix * sizeof(float4), ctx->stream));
    CK(ctx, cudaMemsetAsync(w.p, 0, nPix * sizeof(float), ctx->stream));
    LaunchCfg cfg;
    cfg.numSMs = ctx->numSMs;
    return componentCall(ctx, "b2_splat", {{pos, 2 * n}, {val, 4 * n}}, {{film, 5 * nPix}}, [&](float *const *d) {
        parity::kernels.splat(cfg, f, W, H, n, d[0], d[1], rgba.p, w.p, ctx->stream);
        parity::kernels.film_pack(cfg, rgba.p, w.p, d[2], nPix, ctx->stream);
    });
}
