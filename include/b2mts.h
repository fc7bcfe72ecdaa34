/* b2mts.h -- C-ABI of the H100 (sm_90a) wavefront path tracer that stands in for Mitsuba 0.6's
 * `path` integrator hot path.  Plain C: opaque handles, pointers and sizes; no C++ or torch types.
 *
 * Every entry point names the reference interface it replaces (paths relative to the Mitsuba 0.6
 * tree).  A Mitsuba-side `Integrator` plugin shim (INTEGRATION.md) marshals its Scene into these
 * calls from Integrator::render() (include/mitsuba/render/integrator.h:61-118), exactly like the
 * `vpl` integrator replaces block rendering wholesale (src/integrators/vpl/vpl.cpp:143-237).
 *
 * Conventions: every function returns 0 on success, non-zero on failure (b2_last_error() gives the
 * text; nothing throws across the boundary -- the reference's Log(EError) throws,
 * src/libcore/logger.cpp:100-147, the shim converts).  All input buffers are copied; the caller
 * keeps ownership.  Output buffers are caller-allocated.  There is NO CPU fallback: every compute
 * entry point fails with B2_ERR_NO_DEVICE when no CUDA device is usable.
 */
#ifndef B2MTS_H
#define B2MTS_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B2_OK 0
#define B2_ERR_INVALID 1
#define B2_ERR_NO_DEVICE 2
#define B2_ERR_CUDA 3
#define B2_ERR_IO 4
#define B2_ERR_CANCELLED 5

typedef struct b2_ctx b2_ctx;
typedef struct b2_scene b2_scene;

/* BSDF plugins on the path.  Field meaning = the reference constructors' properties after their
 * host-side preprocessing (IOR lookup, /extEta), see src/bsdfs/{diffuse,roughconductor,
 * roughdielectric,coating}.cpp and src/bsdfs/microfacet.h:99-148. */
enum { B2_BSDF_DIFFUSE = 0, B2_BSDF_ROUGHCONDUCTOR = 1, B2_BSDF_ROUGHDIELECTRIC = 2, B2_BSDF_COATING = 3,
       B2_BSDF_NULL = 4 /* index-matched boundary, src/bsdfs/null.cpp (what Shape::configure assigns to a BSDF-less medium transition, shape.cpp:64-68) */,
       B2_BSDF_TWOSIDED = 5, B2_BSDF_DIELECTRIC = 6, B2_BSDF_CONDUCTOR = 7, B2_BSDF_PLASTIC = 8 /* src/bsdfs/{twosided,dielectric,conductor,plastic}.cpp */ };
enum { B2_DISTR_BECKMANN = 0, B2_DISTR_GGX = 1, B2_DISTR_PHONG = 2 };
typedef struct b2_material_desc {
    int32_t type;            /* B2_BSDF_* */
    int32_t distr;           /* B2_DISTR_*            microfacet.h:48-57 */
    int32_t sample_visible;  /* microfacet.h:138 (must be 0 for phong, :145-148) */
    int32_t nested;          /* coating / twosided: material id of the nested BSDF (coating.cpp:190-199, twosided.cpp:186-197); else -1 */
    float alpha_u, alpha_v;  /* roughness before the 1e-4 clamp (microfacet.h:70-71) */
    float eta;               /* roughdielectric / coating: intIOR/extIOR */
    float thickness;         /* coating.cpp:126 */
    float reflectance[3];    /* diffuse: reflectance; others: specularReflectance */
    float transmittance[3];  /* roughdielectric / dielectric: specularTransmittance */
    float eta_c[3], k_c[3];  /* roughconductor / conductor eta, k divided by extEta (roughconductor.cpp:189-190, conductor.cpp:174-175) */
    float sigma_a[3];        /* coating.cpp:129-130 */
    int32_t nested2;         /* twosided: material id of the back-side BSDF (= nested when one child was given, twosided.cpp:89-90) */
    float diffuse_reflectance[3]; /* plastic.cpp:158-159 */
    float fdr_int, fdr_ext;  /* plastic.cpp:194-195: fresnelDiffuseReflectance(1/eta), (eta) */
    float spec_sampling_weight; /* plastic.cpp:199-202 */
    int32_t nonlinear;       /* plastic.cpp:161 */
    int32_t reflectance_texture; /* diffuse, roughconductor, conductor, plastic: 0 = the constant above; k > 0 = the bitmap texture with id k - 1
                                    (b2_scene_add_texture) is bound to `reflectance` of diffuse (diffuse.cpp:75-77,115,148), `specularReflectance`
                                    of roughconductor / conductor (roughconductor.cpp:285,369,415; conductor.cpp:221-256) or `diffuseReflectance` of plastic
                                    (plastic.cpp:158-159,271,304,415; spec_sampling_weight then takes the texture's average, :199-202) */
} b2_material_desc;

/* `bitmap` texture plugin (src/textures/bitmap.cpp; SURVEY.md 8f-4): the decoded image as linear float (what
 * Bitmap::convert(.., EFloat, gamma 1) hands to the MIP map, mipmap.h:225-229), 1 (luminance) or 3 (RGB) channels, row-major,
 * first row = top of the file.  The MIP pyramid (Lanczos-2, mipmap.h:155-303) is built by b2_scene_commit. */
enum { B2_TEX_NEAREST = 0, B2_TEX_BILINEAR = 1, B2_TEX_TRILINEAR = 2, B2_TEX_EWA = 3 };                     /* bitmap.cpp:213-230 */
enum { B2_WRAP_REPEAT = 0, B2_WRAP_CLAMP = 1, B2_WRAP_MIRROR = 2, B2_WRAP_ZERO = 3, B2_WRAP_ONE = 4 };        /* bitmap.cpp:324-338 */
typedef struct b2_texture_desc {
    int32_t width, height, channels;
    int32_t filter_type;       /* B2_TEX_*, plugin default ewa */
    int32_t wrap_u, wrap_v;    /* B2_WRAP_*, plugin default repeat */
    float max_anisotropy;      /* bitmap.cpp:232-235 (plugin default 20; ignored unless ewa) */
    float uoffset, voffset, uscale, vscale; /* texture.cpp:82-95 (plugin defaults 0, 0, 1, 1) */
    uint32_t reserved;
    const float *pixels;       /* width * height * channels float32; copied */
} b2_texture_desc;

/* Participating medium + phase function (SURVEY.md 8f-1): `homogeneous` (src/medium/homogeneous.cpp:156-222, strategies
 * balance / single / manual) or `heterogeneous` with method woodcock (src/medium/heterogeneous.cpp:182-260) over a float32
 * `gridvolume` density in [0,1] (src/volume/gridvolume.cpp) and a constant albedo (`constvolume`); phase `isotropic` or `hg`. */
enum { B2_MEDIUM_HOMOGENEOUS = 0, B2_MEDIUM_HETEROGENEOUS = 1 };
enum { B2_PHASE_ISOTROPIC = 0, B2_PHASE_HG = 1 };
typedef struct b2_medium_desc {
    int32_t type;               /* B2_MEDIUM_* */
    int32_t phase;              /* B2_PHASE_* */
    float g;                    /* hg.cpp:49 */
    float sigma_a[3], sigma_s[3]; /* homogeneous (medium.cpp:30-36) */
    int32_t strategy;           /* homogeneous.cpp:186-222: 0 balance, 1 single, 2 manual */
    float sampling_density;     /* single: sigma_t[channel]; manual: `samplingDensity` */
    float medium_sampling_weight; /* homogeneous.cpp:160-183, after its max(., 0.5) clamp */
    float scale;                /* heterogeneous.cpp:185 */
    float albedo[3];            /* heterogeneous: constant `albedo` volume */
    int32_t res[3];             /* grid resolution x, y, z */
    float world_to_grid[12];    /* rows of m_worldToGrid, gridvolume.cpp:186-193 */
    float aabb_min[3], aabb_max[3]; /* world box of the transformed data box, gridvolume.cpp:197-199 */
    const float *density;       /* res[0]*res[1]*res[2] float32, x fastest; copied */
} b2_medium_desc;

/* Integrator + Sampler + Film/ReconstructionFilter properties that parameterise one render:
 * MonteCarloIntegrator (src/librender/integrator.cpp:190-225), SobolSampler / IndependentSampler
 * (src/samplers/sobol.cpp:86-102, independent.cpp:52-58), rfilters (src/rfilters/{box,gaussian}.cpp). */
enum { B2_SAMPLER_SOBOL = 0, B2_SAMPLER_INDEPENDENT = 2 };
enum { B2_RFILTER_BOX = 0, B2_RFILTER_GAUSSIAN = 1 };
enum { B2_INTEGRATOR_PATH = 0 /* src/integrators/path/path.cpp */, B2_INTEGRATOR_VOLPATH = 1 /* src/integrators/path/volpath.cpp */ };
typedef struct b2_render_params {
    int32_t spp;             /* sampleCount */
    int32_t sampler;         /* B2_SAMPLER_* (independent = counter-based stream, see DESIGN.md) */
    uint64_t seed;           /* sobol: `scramble`; independent: stream seed */
    int32_t max_depth;       /* -1 = unbounded */
    int32_t rr_depth;        /* 5 */
    int32_t strict_normals, hide_emitters;
    int32_t rfilter;         /* B2_RFILTER_* */
    float rfilter_param;     /* box: radius (0.5); gaussian: stddev (0.5) */
    int32_t sample_lo, sample_hi; /* this call renders sample indices [lo,hi) of every pixel; hi<=0 -> spp.
                                     Shards the work across GPUs (replaces BlockedImageProcess work units,
                                     src/librender/imageproc.cpp:43-78) */
    int32_t parity_mode;     /* 1: kernels compiled with -fmad=false (tight float parity); 0: throughput kernels (FMA contraction, fast math),
                                except where flags bit8 explains */
    int32_t pool_size;       /* in-flight paths (0 = default) */
    int32_t film_on_device;  /* 1: `film` of b2_render is a device pointer on the context's device */
    int32_t flags;           /* bit1: force unsorted shading (default: material-sorted when > 1 BSDF class);
                                bit2: per-launch device time stamps (fills b2_stats.ms_*); bit3: plain launches + CUDA events
                                instead of the CUDA graph; bit4: fuse the ray casts into generate/shade for tiny scenes (experiment, slower);
                                bit5: collect per-pixel path diagnostics (b2_get_pixel_stats); bit6: per-sample event traces (b2_get_path_traces);
                                bit8: force the throughput kernels (parity_mode 0 renders `path` scenes that contain a transmissive BSDF with the
                                IEEE kernels: such scenes amplify ulp-level differences chaotically, DESIGN.md "parity") */
    int32_t integrator;      /* B2_INTEGRATOR_* (<integrator type="path"|"volpath">) */
    int32_t reserved;        /* must be 0 */
} b2_render_params;

/* Counters with the meaning of the reference's statistics (path.cpp:24,290-291; skdtree.cpp:46-47) plus
 * per-stage device times of the last b2_render. */
typedef struct b2_stats {
    uint64_t samples, rays, shadow_rays, path_length_sum, bad_samples, dim_overflow;
    uint64_t node_visits, prim_tests;       /* only counted when built with B2_COUNT_TRAVERSAL */
    uint64_t iterations, kernel_launches;
    float ms_total, ms_generate, ms_extend, ms_shade, ms_occluded, ms_film;
    uint64_t n_triangles, n_bvh_nodes;
    uint64_t n_generate, n_extend, n_shade, n_occluded; /* launches behind the ms_* sums (flags bit2) */
    uint64_t bytes_uploaded;                /* host->device bytes of the last b2_scene_commit */
    uint64_t pool_size;                     /* in-flight paths of the last b2_render */
    uint64_t unoccluded_shadow_rays;        /* shadow rays that reached the emitter (their contribution was added) */
    uint64_t bvh_node_bytes;                /* size of one node of the tree the ray queries walk (80: 8-wide compressed, 64: binary) */
} b2_stats;

/* ---- lifetime -------------------------------------------------------------------------------- */
int b2_context_create(int device, b2_ctx **out);          /* one context per GPU / per rank */
void b2_context_destroy(b2_ctx *);
const char *b2_last_error(b2_ctx *);                       /* NULL ctx -> last global error */
int b2_scene_create(b2_ctx *, b2_scene **out);            /* replaces Scene (src/librender/scene.cpp) for the path */
void b2_scene_destroy(b2_scene *);

/* ---- scene description (what the shim reads through Scene::getMeshes/getEmitters/getSensor,
 *      include/mitsuba/render/scene.h:992-1094, trimesh.h:122-153) ------------------------------- */
/* PerspectiveCameraImpl::configure (src/sensors/perspective.cpp:126-179): camera-to-world matrix (row
 * major), x field of view in degrees, clip planes, film size.  m_sampleToCamera is derived inside. */
int b2_scene_set_camera(b2_scene *, const float to_world[16], float xfov_deg, float near_clip, float far_clip,
                        int width, int height);
/* Film crop window (src/librender/film.cpp:36-47: cropOffsetX/Y, cropWidth/Height; "Invalid crop window specification!" when it
 * leaves the film).  Call after b2_scene_set_camera.  As in the reference the crop window becomes the film every later call sees
 * (Film::getCropSize): b2_scene_film_size, sample positions, the Sobol' resolution and the b2_render output are crop_width x
 * crop_height; the sensor's sampleToCamera takes the relative size / offset (src/sensors/perspective.cpp:133-153). */
int b2_scene_set_crop(b2_scene *, int crop_offset_x, int crop_offset_y, int crop_width, int crop_height);
/* ThinLens (src/sensors/thinlens.cpp:132-142,327-350): aperture radius and focus distance of the camera set before; 0 = pinhole.
 * The aperture sample takes Sobol' dimensions 2 and 3 (integrator.cpp:173-174). */
int b2_scene_set_thinlens(b2_scene *, float aperture_radius, float focus_distance);
int b2_scene_get_sample_to_camera(b2_scene *, float out[16]);
int b2_scene_film_size(b2_scene *, int *width, int *height);   /* Film::getSize (include/mitsuba/render/film.h) */
/* BSDF plugin instance -> id (>=0) or -1 */
int b2_scene_add_material(b2_scene *, const b2_material_desc *);
/* AreaLight (src/emitters/area.cpp:64-70): radiance, samplingWeight -> id (>=0) or -1 */
int b2_scene_add_area_emitter(b2_scene *, const float radiance[3], float sampling_weight);
/* ConstantBackgroundEmitter (src/emitters/constant.cpp:47-52): radiance, samplingWeight -> emitter id (>=0) or -1.  At most one
 * environment emitter per scene (scene.cpp:510-514).  In the emitter-selection CDF it precedes the shapes' area emitters whatever the
 * call order, as in Scene::m_emitters (Scene::addChild appends it at once, scene.cpp:510-516; area emitters join in Scene::initialize,
 * scene.cpp:322-335): b2_scene_commit applies that order. */
int b2_scene_add_constant_emitter(b2_scene *, const float radiance[3], float sampling_weight);
/* EnvironmentMap (src/emitters/envmap.cpp:106-181): a latitude-longitude radiance map around the scene -> emitter id (>=0) or -1.
 * `pixels` is the decoded image (what Bitmap::convert(ERGB, EFloat) hands to the MIP map, envmap.cpp:172-175): width x height x 3 linear
 * floats, row-major, top row first; decoding image files is the caller's side of the boundary.  scale = the plugin's `scale`;
 * to_world / to_local = the plugin's toWorld and its inverse as row-major 4x4 (both NULL: identity); sampling_weight = `samplingWeight`.
 * b2_scene_commit builds what the plugin builds when it is loaded and configured: the half-precision MIP pyramid (2-lobe Lanczos, repeat /
 * clamp boundaries, no upper clamp) and the marginal / conditional CDF tables over luminance x sin(theta) (envmap.cpp:260-329).  The
 * kernels then implement evalEnvironment (:380-410, EWA-filtered with the sensor ray's differentials for directly visible background),
 * sampleDirect / pdfDirect (:516-560) and fillDirectSamplingRecord (:359-374).  Shares the one-environment-emitter rule and the
 * emitter order of b2_scene_add_constant_emitter.  Errors as the plugin raises them: a black map, a non-finite pixel, a side > 65535. */
int b2_scene_add_envmap_emitter(b2_scene *, int width, int height, const float *pixels, float scale, const float *to_world, const float *to_local,
                                float sampling_weight);
/* TriMesh after configure(): positions, optional normals / texcoords (NULL = none -> face normals,
 * skdtree.h:383-399), triangles, material and emitter ids (-1 = no emitter).  An emitter id may be
 * attached to exactly one mesh (area.cpp:185-199).  Returns mesh id or -1. */
int b2_scene_add_mesh(b2_scene *, const float *P, const float *N, const float *UV, uint32_t n_vertices,
                      const uint32_t *idx, uint32_t n_triangles, int material_id, int emitter_id);
/* Medium plugin instance -> id (>=0) or -1; <ref name="interior"/"exterior"> of a shape (shape.cpp:160-176; -1 = none).
 * A mesh whose material is B2_BSDF_NULL is an index-matched boundary. */
int b2_scene_add_medium(b2_scene *, const b2_medium_desc *);
/* Texture plugin instance -> id (>=0) or -1; bind it with b2_material_desc::reflectance_texture = id + 1 (materials added afterwards).
 * `path` only. */
int b2_scene_add_texture(b2_scene *, const b2_texture_desc *);
int b2_scene_set_mesh_media(b2_scene *, int mesh_id, int interior_medium, int exterior_medium);
/* Instancing (src/shapes/{shapegroup,instance}.cpp): meshes assigned to a shapegroup live in its object space and are only
 * visible through instances; `to_world` / `to_object` are the affine instance transform and its inverse (row major).
 * Emitters cannot be instanced (shapegroup.cpp:115-116); `path` only. */
int b2_scene_add_shapegroup(b2_scene *);                                   /* -> group id */
int b2_scene_set_mesh_group(b2_scene *, int mesh_id, int group_id);
int b2_scene_add_instance(b2_scene *, int group_id, const float to_world[16], const float to_object[16]);
/* Scene::initialize (src/librender/scene.cpp:322-384): TriAccel precompute (skdtree.cpp:74-109),
 * acceleration structure build (BVH; replaces GenericKDTree::buildInternal, gkdtree.h:958-1263),
 * emitter / triangle-area CDFs (scene.cpp:375-380, trimesh.cpp:388-403), upload to HBM. */
int b2_scene_commit(b2_scene *);

/* ---- the hot path: SamplingIntegrator::render + renderBlock + MIPathTracer::Li
 *      (src/librender/integrator.cpp:95-188, src/integrators/path/path.cpp:119-294) ------------- */
/* film: H*W*5 floats (R,G,B,alpha,weight) = the HDRFilm storage format ESpectrumAlphaWeight
 * (src/films/hdrfilm.cpp:351-356), overwritten.  Host pointer unless params->film_on_device. */
int b2_render(b2_scene *, const b2_render_params *, float *film);
/* Integrator::cancel (integrator.h:90-93): callable from another thread */
int b2_cancel(b2_scene *);
/* Film::develop normalisation (src/libcore/fmtconv.cpp:979-990): rgb = spec * (w != 0 ? 1/w : w). host buffers */
int b2_film_develop(const float *film, int width, int height, float *rgb);
int b2_get_stats(b2_scene *, b2_stats *);
/* Per-pixel path diagnostics of the last b2_render with flags bit5: out[y * W + x] = (sum of squared path lengths << 32) | sum of
 * path lengths over the pixel's samples (the per-pixel form of the reference's "average path length" statistic, path.cpp:24,290).
 * Comparing two builds word by word gives the fraction of pixels in which a path changed length (SURVEY.md 8d). */
int b2_get_pixel_stats(b2_scene *, uint64_t *out);
/* Per-sample event traces of the last b2_render with flags bit6 (diagnostics; sobol sampler): out[(y * W + x) * n_samples + s], one event
 * byte per bounce (material hit, shadow ray emitted, how the vertex ended, reflected / transmitted lobe), see b2_host.cpp. */
int b2_get_path_traces(b2_scene *, uint64_t n_words, uint64_t *out);

/* ---- component entry points (the reference exposes the same pieces through its Python bindings
 *      and test plugins: ShapeKDTree::rayIntersect src/libpython/render.cpp:352-369, BSDF
 *      sample/eval/pdf src/tests/test_chisquare.cpp:94-200, kdbench src/utils/kdbench.cpp) ------- */
/* rays: n x 8 floats (o.xyz, mint, d.xyz, maxt); mode 0 closest hit -> t,u,v,prim (prim = 0xFFFFFFFF on miss,
 * t = +inf); mode 1 occlusion -> prim = 0/1.  Host buffers.  ShapeKDTree::rayIntersect, skdtree.cpp:112-226. */
int b2_trace(b2_scene *, uint64_t n, const float *rays, int mode, int parity_mode, float *t, float *u, float *v,
             uint32_t *prim, float *ms_kernel);
/* Same, all buffers resident on the device (traversal benchmark) */
int b2_trace_device(b2_scene *, uint64_t n, const float *d_rays, int mode, int parity_mode, float *d_tuvp, float *ms_kernel);
/* BSDF::eval + pdf for local-frame (wi, wo) pairs: out_rgb n x 3, out_pdf n */
int b2_bsdf_eval(b2_scene *, int material_id, uint64_t n, const float *wi, const float *wo, int parity_mode,
                 float *out_rgb, float *out_pdf);
/* BSDF::sample(bRec, pdf, sample): samples n x 3 (2-D sample + the extra 1-D a rough dielectric draws);
 * out n x 10: wo(3) weight(3) pdf sampledType eta pad */
int b2_bsdf_sample(b2_scene *, int material_id, uint64_t n, const float *wi, const float *samples, int parity_mode, float *out);
/* Scene::sampleEmitterDirect without the visibility test folded into `visible`:
 * ref n x 6 (ref, refN), samples n x 2 -> out n x 12: d(3) dist pdf value(3) visible p(3) */
int b2_sample_emitter_direct(b2_scene *, uint64_t n, const float *ref, const float *samples, int parity_mode, float *out);
/* Medium components: what = 0 Medium::evalTransmittance (in n x 8 rays (o, mint, d, maxt) -> out n x 3), 1 Medium::sampleDistance
 * (-> n x 12: ok t sigmaS(3) transmittance(3) pdfSuccess pdfFailure - -), 2 GridDataSource::lookupFloat (in n x 3 -> n),
 * 3 PhaseFunction::sample + eval (in n x 5: wi, two uniforms -> n x 5: wo pdf eval); random numbers: counter stream `seed` */
int b2_medium_probe(b2_scene *, int medium_id, int what, uint64_t n, const float *in, uint64_t seed, int parity_mode, float *out);
/* Texture components: Texture2D::eval (texture.cpp:124-133) of n look-ups, uv n x 2, partials n x 4 (dudx dudy dvdx dvdy; NULL = the
 * unfiltered look-up of a ray without differentials) -> out n x 3 */
int b2_texture_eval(b2_scene *, int texture_id, uint64_t n, const float *uv, const float *partials, int parity_mode, float *out);
/* uv and uv partials of camera-ray hits (sampleRayDifferential + scaleDifferential(1/sqrt(spp)) + Intersection::computePartials):
 * pos_hit n x 6 = film position (2), then t, u, v, prim as b2_trace returns them -> out n x 6: u v dudx dudy dvdx dvdy */
int b2_texture_partials(b2_scene *, uint64_t n, const float *pos_hit, int spp, int parity_mode, float *out);
/* Host-only (no device): decode an image file the way b2_load_xml does for `bitmap` textures and `envmap` emitters -- OpenEXR scan-line
 * files (NONE / RLE / ZIPS / ZIP; HALF / FLOAT / UINT; R,G,B or a luminance channel), PNG (non-interlaced), Radiance RGBE (.hdr), PFM, 8-bit binary PPM -- into
 * linear floats, row-major, top row first (what Bitmap::convert(.., EFloat32, gamma 1) hands to the MIP map).  gamma 0 = the file's own
 * (EXR / RGBE / PFM linear, PPM sRGB, PNG sRGB or its gAMA), -1 = sRGB, > 0 = that exponent (bitmap.cpp:251-252).  out NULL: size query.  0 or -1 + message. */
int b2_load_image(const char *path, float gamma, int *width, int *height, int *channels, float *out, char *err, int err_len);
/* Host-only: (wavelength nm, value) samples in increasing wavelength -> ITU-R BT.709 linear RGB, what the scene file's <spectrum filename="x.spd">
 * and <spectrum value="l0:v0, l1:v1, ..."> become (scenehandler.cpp:557-611: InterpolatedSpectrum, zeroExtend, fromContinuousSpectrum against the
 * CIE 1931 observer, clampNegative).  The integrals are evaluated exactly; the reference's adaptive quadrature agrees to 1e-4.  0 or -1 + message. */
int b2_spectrum_to_rgb(const float *wavelengths, const float *values, int n, int zero_extend, float rgb[3], char *err, int err_len);
/* Probes of the committed environment map: what 0 = Scene::evalEnvironment for n world directions (in n x 3 -> out n x 3); 1 = the same
 * for sensor rays with differentials (in n x 9: d, rxDirection, ryDirection -> out n x 3); 2 = Scene::pdfEmitterDirect of the map for n
 * directions, solid-angle measure including the emitter-selection probability (in n x 3 -> out n) */
int b2_envmap_probe(b2_scene *, int what, uint64_t n, const float *in, int parity_mode, float *out);
/* One level of the MIP pyramid built at commit (TMIPMap constructor, mipmap.h:155-303); out may be NULL to query the size */
int b2_texture_level(b2_scene *, int texture_id, int level, int *levels, int *width, int *height, float *out);
/* The same without a scene or a device: host-side pyramid construction for the given description */
int b2_mipmap_level(const b2_texture_desc *, int level, int *levels, int *width, int *height, float *out);
/* The first ndim sampler outputs of (pixel, sample) as renderBlock + Li draw them */
int b2_sampler_stream(b2_scene *, int sampler, uint64_t seed, int spp, int px, int py, int sample_idx, int ndim, float *out);
/* primary rays (PerspectiveCameraImpl::sampleRayDifferential, perspective.cpp:271-298): pos n x 2 -> rays n x 8 */
int b2_camera_rays(b2_scene *, uint64_t n, const float *pos, int parity_mode, float *rays);
/* ImageBlock::put (imageblock.h:124-204) for n samples: pos n x 2, val n x 4 (rgb, alpha) -> film H*W*5 */
int b2_splat(b2_ctx *, int width, int height, int rfilter, float rfilter_param, uint64_t n, const float *pos,
             const float *val, float *film);
/* TriAccel records (n_triangles x 12 words) as uploaded, in prim order */
int b2_get_triaccel(b2_scene *, float *out);

/* ---- scene files: the SceneHandler subset (src/librender/scenehandler.cpp:70-106) --------------- */
/* defines: "key=value" strings ($key substitution, src/mitsuba/mitsuba.cpp:154).  Fills *params from the
 * <integrator>/<sampler>/<film>/<rfilter> elements. */
int b2_load_xml(b2_ctx *, const char *path, const char *const *defines, int n_defines, b2_scene **out,
                b2_render_params *params);

const char *b2_version(void);
int b2_device_count(void);

#ifdef __cplusplus
}
#endif
#endif
