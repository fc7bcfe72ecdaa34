/* b200path -- the Mitsuba 0.6 side of the drop-in: an `Integrator` plugin that hands the scene to libb2mts.so through the C-ABI of
 * include/b2mts.h and returns the film.  `<integrator type="b200path"/>` selects it through the reference's ordinary plugin route
 * (dlopen + CreateInstance(const Properties&): include/mitsuba/core/cobject.h:99-107, src/libcore/plugin.cpp:71-96); it replaces
 * SamplingIntegrator::render + renderBlock + MIPathTracer::Li wholesale (src/librender/integrator.cpp:95-188,
 * src/integrators/path/path.cpp:119-294), as `vpl` replaces block rendering (src/integrators/vpl/vpl.cpp:143-237).
 *
 * This file only marshals -- it contains no rendering logic -- and uses nothing but the reference's public object API:
 *   Scene::getMeshes / getShapes / getEmitters / getSensor / getFilm / getSampler (include/mitsuba/render/scene.h:899-1096),
 *   TriMesh buffers (trimesh.h:122-153), Shape::getBSDF / getEmitter (shape.h), ConfigurableObject::getProperties (cobject.h:77:
 *   every object keeps the Properties it was created from, incl. the plugin name), PerspectiveCamera / ProjectiveCamera accessors
 *   (sensor.h:403-499), Film::getSize / getCropSize / getCropOffset / getReconstructionFilter (film.h:40-98), Film::setBitmap.
 *
 * What the 0.6 object API does NOT expose are the children a plugin received through addChild (coating / twosided nested BSDFs, a
 * medium's volume and phase function, a BSDF's texture): they are private members.  This shim therefore covers BSDFs whose parameters
 * are values (all nine plugins of the path, without nesting or bitmap textures) and reports the others with the reference's own
 * wording; the two ways a maintainer can lift that are listed in INTEGRATION.md (HWResource dependency walk through
 * BSDF::createShader / Shader::putDependencies, or the plugin's serialize() stream).
 *
 * It is not part of libb2mts.so.  The test infrastructure compiles it against the reference's headers and links it with the reference's
 * own translation units (the checker's Makefile, target _ref/libb200shim.so); tests/test_gpu_shim.py then renders reference Scene objects
 * through it on the GPU and compares with the reference's own films. */
#include <mitsuba/render/scene.h>
#include <mitsuba/render/renderjob.h>
#include <mitsuba/render/renderqueue.h>
#include <mitsuba/core/bitmap.h>
#include <map>
#include <b2mts.h>

MTS_NAMESPACE_BEGIN

static void rgbOf(const Spectrum &s, float out[3]) { /* SPECTRUM_SAMPLES == 3: the coefficients are linear RGB (spectrum.h) */
    Float r, g, b;
    s.toLinearRGB(r, g, b);
    out[0] = (float) r; out[1] = (float) g; out[2] = (float) b;
}

/* src/bsdfs/ior.h lookupIOR: the named materials a dielectric plugin accepts for intIOR / extIOR */
static float iorOf(const Properties &p, const std::string &name, const char *defaultName) {
    static const struct { const char *n; float v; } table[] = {
        {"vacuum", 1.0f}, {"helium", 1.00004f}, {"hydrogen", 1.00013f}, {"air", 1.00028f}, {"carbon dioxide", 1.00045f}, {"water", 1.3330f},
        {"acetone", 1.36f}, {"ethanol", 1.361f}, {"carbon tetrachloride", 1.461f}, {"glycerol", 1.4729f}, {"benzene", 1.501f},
        {"silicone oil", 1.52045f}, {"bromine", 1.661f}, {"water ice", 1.31f}, {"fused quartz", 1.458f}, {"pyrex", 1.470f},
        {"acrylic glass", 1.49f}, {"polypropylene", 1.49f}, {"bk7", 1.5046f}, {"sodium chloride", 1.544f}, {"amber", 1.55f},
        {"pet", 1.575f}, {"diamond", 2.419f}};
    std::string v = defaultName;
    if (p.hasProperty(name)) {
        if (p.getType(name) == Properties::EFloat) return (float) p.getFloat(name);
        v = p.getString(name);
    }
    for (size_t i = 0; i < sizeof(table) / sizeof(table[0]); ++i)
        if (v == table[i].n) return table[i].v;
    SLog(EError, "Unable to find an IOR value for \"%s\"!", v.c_str());
    return 0;
}

class B200PathTracer : public Integrator {
public:
    B200PathTracer(const Properties &props) : Integrator(props), m_handle(NULL) {
        /* same property names and defaults as MonteCarloIntegrator, src/librender/integrator.cpp:190-225 */
        m_rrDepth = props.getInteger("rrDepth", 5);
        m_maxDepth = props.getInteger("maxDepth", -1);
        m_strictNormals = props.getBoolean("strictNormals", false);
        m_hideEmitters = props.getBoolean("hideEmitters", false);
        m_device = props.getInteger("device", 0);
        m_parity = props.getBoolean("parity", false);
        /* acceleration-structure builder of b2_scene_commit: "host" (multi-threaded CPU build) or "device" (the same tree built on the GPU) */
        const std::string accelBuild = props.getString("accelBuild", "host");
        if (accelBuild == "host") m_accelBuild = B2_ACCEL_BUILD_HOST;
        else if (accelBuild == "device") m_accelBuild = B2_ACCEL_BUILD_DEVICE;
        else Log(EError, "'accelBuild' must be \"host\" or \"device\", not \"%s\"", accelBuild.c_str());
        if (m_rrDepth <= 0) Log(EError, "'rrDepth' must be set to a value greater than zero!");
        if (m_maxDepth <= 0 && m_maxDepth != -1) Log(EError, "'maxDepth' must be set to -1 (infinite) or a value greater than zero!");
    }
    B200PathTracer(Stream *stream, InstanceManager *manager) : Integrator(stream, manager), m_handle(NULL) {
        m_rrDepth = stream->readInt(); m_maxDepth = stream->readInt();
        m_strictNormals = stream->readBool(); m_hideEmitters = stream->readBool();
        m_device = stream->readInt(); m_parity = stream->readBool();
        m_accelBuild = stream->readInt();
    }
    void serialize(Stream *stream, InstanceManager *manager) const {
        Integrator::serialize(stream, manager);
        stream->writeInt(m_rrDepth); stream->writeInt(m_maxDepth);
        stream->writeBool(m_strictNormals); stream->writeBool(m_hideEmitters);
        stream->writeInt(m_device); stream->writeBool(m_parity);
        stream->writeInt(m_accelBuild);
    }

    /* BSDF plugin -> b2_material_desc from its construction Properties: the same host-side preprocessing the plugin constructors do
       (src/bsdfs/{diffuse,roughconductor,roughdielectric,conductor,dielectric,plastic}.cpp; microfacet.h:99-148) */
    int addBSDF(b2_scene *sc, const BSDF *bsdf, std::map<const BSDF *, int> &seen) {
        if (seen.count(bsdf)) return seen[bsdf];
        const Properties &p = bsdf->getProperties();
        const std::string type = p.getPluginName();
        b2_material_desc d;
        memset(&d, 0, sizeof(d));
        d.nested = -1; d.nested2 = -1; d.eta = 1.0f; d.thickness = 1.0f;
        for (int k = 0; k < 3; ++k) { d.reflectance[k] = 1.0f; d.transmittance[k] = 1.0f; }
        auto spec = [&](const char *name, float dflt, float out[3]) { rgbOf(p.getSpectrum(name, Spectrum(dflt)), out); };
        auto microfacet = [&]() { /* microfacet.h:99-148 */
            std::string distr = p.getString("distribution", "beckmann");
            for (size_t i = 0; i < distr.size(); ++i) distr[i] = (char) tolower(distr[i]);
            d.distr = distr == "beckmann" ? B2_DISTR_BECKMANN : distr == "ggx" ? B2_DISTR_GGX : distr == "phong" ? B2_DISTR_PHONG : -1;
            if (distr == "as") { d.distr = B2_DISTR_PHONG; } /* Ashikhmin-Shirley = anisotropic Phong (microfacet.h:113-115) */
            if (d.distr < 0) Log(EError, "Specified an invalid distribution \"%s\", must be \"beckmann\", \"ggx\", or \"phong\"/\"as\"!", distr.c_str());
            const Float alpha = p.getFloat("alpha", 0.1f);
            /* the plugins read the roughness as a texture value averaged over the spectrum: (a + a + a) * (1/3) in float */
            auto avg = [](Float a) { return (float) ((a + a + a) * (1.0f / 3.0f)); };
            d.alpha_u = avg(p.getFloat("alphaU", alpha)); d.alpha_v = avg(p.getFloat("alphaV", alpha));
            d.sample_visible = p.getBoolean("sampleVisible", true) ? 1 : 0;
        };
        if (type == "diffuse") {
            d.type = B2_BSDF_DIFFUSE;
            rgbOf(p.getSpectrum(p.hasProperty("reflectance") ? "reflectance" : "diffuseReflectance", Spectrum(0.5f)), d.reflectance);
        } else if (type == "roughconductor" || type == "conductor") {
            d.type = type == "conductor" ? B2_BSDF_CONDUCTOR : B2_BSDF_ROUGHCONDUCTOR;
            if (type == "roughconductor") microfacet();
            spec("specularReflectance", 1.0f, d.reflectance);
            if (p.hasProperty("material") && p.getString("material") != "none")
                Log(EError, "b200path: measured conductor data (material=\"%s\") must be given as eta / k spectra", p.getString("material").c_str());
            const float ext = iorOf(p, "extEta", "air");
            float eta[3], k[3];
            rgbOf(p.getSpectrum("eta", Spectrum(0.0f)), eta); rgbOf(p.getSpectrum("k", Spectrum(1.0f)), k);
            const float rcp = 1.0f / ext; /* Spectrum / Float multiplies by the reciprocal (spectrum.h) */
            for (int c = 0; c < 3; ++c) { d.eta_c[c] = eta[c] * rcp; d.k_c[c] = k[c] * rcp; }
        } else if (type == "roughdielectric" || type == "dielectric") {
            d.type = type == "dielectric" ? B2_BSDF_DIELECTRIC : B2_BSDF_ROUGHDIELECTRIC;
            if (type == "roughdielectric") microfacet();
            const float intIOR = iorOf(p, "intIOR", "bk7"), extIOR = iorOf(p, "extIOR", "air");
            if (intIOR < 0 || extIOR < 0 || intIOR == extIOR) Log(EError, "The interior and exterior indices of refraction must be positive and differ!");
            d.eta = intIOR / extIOR;
            spec("specularReflectance", 1.0f, d.reflectance); spec("specularTransmittance", 1.0f, d.transmittance);
        } else if (type == "plastic") {
            d.type = B2_BSDF_PLASTIC;
            const float intIOR = iorOf(p, "intIOR", "polypropylene"), extIOR = iorOf(p, "extIOR", "air");
            if (intIOR < 0 || extIOR < 0) Log(EError, "The interior and exterior indices of refraction must be positive!");
            d.eta = intIOR / extIOR;
            spec("specularReflectance", 1.0f, d.reflectance); spec("diffuseReflectance", 0.5f, d.diffuse_reflectance);
            d.nonlinear = p.getBoolean("nonlinear", false) ? 1 : 0;
            /* plastic.cpp:186-202 (configure): the diffuse Fresnel reflectances and the sampling weight */
            d.fdr_int = (float) fresnelDiffuseReflectance(1 / d.eta, false); d.fdr_ext = (float) fresnelDiffuseReflectance(d.eta, false);
            const Float dAvg = p.getSpectrum("diffuseReflectance", Spectrum(0.5f)).getLuminance(), sAvg = p.getSpectrum("specularReflectance", Spectrum(1.0f)).getLuminance();
            d.spec_sampling_weight = (float) (sAvg / (dAvg + sAvg));
        } else if (type == "coating" || type == "twosided" || type == "roughcoating" || type == "mask" || type == "mixturebsdf" || type == "blendbsdf" || type == "bumpmap") {
            Log(EError, "b200path: BSDF \"%s\" wraps another BSDF, which Mitsuba 0.6 keeps in a private member (INTEGRATION.md 1.2)", type.c_str());
        } else if (type == "null") {
            d.type = B2_BSDF_NULL;
        } else {
            Log(EError, "b200path: unsupported BSDF plugin \"%s\"", type.c_str());
        }
        const int id = b2_scene_add_material(sc, &d);
        if (id < 0) Log(EError, "%s", b2_last_error(NULL));
        return seen[bsdf] = id;
    }

    /* Integrator::render is pure virtual (include/mitsuba/render/integrator.h:86-88); it runs on the RenderJob thread
       (src/librender/renderjob.cpp:87-121).  No ImageBlocks, no Scheduler work units: the GPU renders the whole (crop of the) film. */
    bool render(Scene *scene, RenderQueue *queue, const RenderJob *job, int, int, int) {
        b2_ctx *ctx = NULL;
        b2_scene *sc = NULL;
        if (b2_context_create(m_device, &ctx)) Log(EError, "%s", b2_last_error(NULL)); /* Log(EError) throws */
        if (b2_scene_create(ctx, &sc)) Log(EError, "%s", b2_last_error(ctx));
        if (b2_scene_set_accel_build(sc, m_accelBuild)) Log(EError, "%s", b2_last_error(ctx));
        m_handle = sc;
        /* ---- sensor + film: src/sensors/{perspective,thinlens}.cpp, film.cpp:36-47 ---- */
        const Sensor *sensor = scene->getSensor();
        const std::string sensorType = sensor->getProperties().getPluginName();
        if (sensorType != "perspective" && sensorType != "thinlens") Log(EError, "b200path: unsupported sensor \"%s\"", sensorType.c_str());
        const PerspectiveCamera *cam = static_cast<const PerspectiveCamera *>(sensor);
        const Film *film = scene->getFilm();
        const Transform camToWorld = cam->getWorldTransform((Float) 0); /* (returned by value: keep it alive while the matrix is read) */
        const Matrix4x4 &m = camToWorld.getMatrix();
        float toWorld[16];
        for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) toWorld[4 * i + j] = (float) m.m[i][j];
        const Vector2i full = film->getSize(), crop = film->getCropSize();
        const Point2i cropOffset = film->getCropOffset();
        if (b2_scene_set_camera(sc, toWorld, (float) cam->getXFov(), (float) cam->getNearClip(), (float) cam->getFarClip(), full.x, full.y)) Log(EError, "%s", b2_last_error(ctx));
        if ((crop.x != full.x || crop.y != full.y) && b2_scene_set_crop(sc, cropOffset.x, cropOffset.y, crop.x, crop.y)) Log(EError, "%s", b2_last_error(ctx));
        if (sensorType == "thinlens") {
            const Properties &sp = sensor->getProperties();
            Float aperture = sp.getFloat("apertureRadius");
            if (aperture == 0) aperture = Epsilon; /* thinlens.cpp:134-138 */
            if (b2_scene_set_thinlens(sc, (float) aperture, (float) cam->getFocusDistance())) Log(EError, "%s", b2_last_error(ctx));
        }
        /* ---- scene-level emitters (Scene::m_emitters holds them before the shapes' area lights: scene.cpp:510-516) ---- */
        const ref_vector<Emitter> &emitters = scene->getEmitters();
        for (size_t i = 0; i < emitters.size(); ++i) {
            const Emitter *e = emitters[i].get();
            if (e->getShape() != NULL && !e->isEnvironmentEmitter()) continue; /* area lights are marshalled with their mesh */
            const Properties &ep = e->getProperties();
            if (ep.getPluginName() == "envmap") { /* EnvironmentMap: src/emitters/envmap.cpp */
                /* the image as the plugin holds it: level 0 of its half-precision pyramid (Emitter::getBitmap -> TMIPMap::toBitmap,
                   envmap.cpp:632-634, mipmap.h:486-497).  b2_scene_commit rebuilds the coarser levels from it (from the rounded, not the
                   original float image: only the EWA look-up of directly visible background reads them) and the sampling tables */
                ref<Bitmap> bm = e->getBitmap(Vector2i(0));
                if (bm == NULL || bm->getPixelFormat() != Bitmap::ERGB || bm->getComponentFormat() != Bitmap::EFloat16)
                    Log(EError, "b200path: the environment map is not an RGB half-precision image (spectral builds are not supported)");
                const Vector2i size = bm->getSize();
                const half *src = (const half *) bm->getData();
                std::vector<float> px((size_t) size.x * size.y * 3);
                for (size_t k = 0; k < px.size(); ++k) px[k] = (float) src[k];
                const Transform envToWorld = e->getWorldTransform()->eval(0);
                float a[16], b[16];
                for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) {
                    a[4 * r + c] = (float) envToWorld.getMatrix().m[r][c]; b[4 * r + c] = (float) envToWorld.getInverseMatrix().m[r][c];
                }
                if (b2_scene_add_envmap_emitter(sc, size.x, size.y, px.data(), (float) ep.getFloat("scale", 1.0f), a, b, (float) ep.getFloat("samplingWeight", 1.0f)) < 0)
                    Log(EError, "%s", b2_last_error(ctx));
                continue;
            }
            if (ep.getPluginName() != "constant") Log(EError, "b200path: unsupported emitter \"%s\" (supported: area, constant, envmap)", ep.getPluginName().c_str());
            float rad[3];
            rgbOf(ep.getSpectrum("radiance", Spectrum(1.0f)), rad);
            if (b2_scene_add_constant_emitter(sc, rad, (float) ep.getFloat("samplingWeight", 1.0f)) < 0) Log(EError, "%s", b2_last_error(ctx));
        }
        /* ---- shapes: Scene::getMeshes (scene.h:1080) holds the TriMeshes after configure() ---- */
        std::map<const BSDF *, int> bsdfId;
        const std::vector<TriMesh *> &meshes = scene->getMeshes();
        if (meshes.size() != scene->getShapes().size())
            Log(EError, "b200path: the scene holds shapes that are not triangle meshes (shapegroup / instance / analytic shapes need the scene-file route, b2_load_xml)");
        for (size_t i = 0; i < meshes.size(); ++i) {
            const TriMesh *mesh = meshes[i];
            if (mesh->getInteriorMedium() || mesh->getExteriorMedium()) Log(EError, "b200path: participating media need the scene-file route (a medium's volume and phase function are private children)");
            const int mat = addBSDF(sc, mesh->getBSDF(), bsdfId);
            int em = -1;
            if (mesh->isEmitter()) { /* AreaLight: src/emitters/area.cpp:64-70 */
                const Properties &ep = mesh->getEmitter()->getProperties();
                if (ep.getPluginName() != "area") Log(EError, "b200path: unsupported shape emitter \"%s\"", ep.getPluginName().c_str());
                float rad[3];
                rgbOf(ep.getSpectrum("radiance", Spectrum(1.0f)), rad);
                em = b2_scene_add_area_emitter(sc, rad, (float) ep.getFloat("samplingWeight", 1.0f));
                if (em < 0) Log(EError, "%s", b2_last_error(ctx));
            }
            /* trimesh.h:122-153: positions / normals / texcoords / Triangle{uint32_t idx[3]} are contiguous arrays (SINGLE_PRECISION) */
            if (b2_scene_add_mesh(sc, (const float *) mesh->getVertexPositions(), (const float *) mesh->getVertexNormals(), (const float *) mesh->getVertexTexcoords(),
                                  (uint32_t) mesh->getVertexCount(), (const uint32_t *) mesh->getTriangles(), (uint32_t) mesh->getTriangleCount(), mat, em) < 0)
                Log(EError, "%s", b2_last_error(ctx));
        }
        if (b2_scene_commit(sc)) Log(EError, "%s", b2_last_error(ctx));
        /* ---- sampler + reconstruction filter ---- */
        b2_render_params rp;
        memset(&rp, 0, sizeof(rp));
        const Sampler *sampler = scene->getSampler();
        const Properties &sp = sampler->getProperties();
        rp.spp = (int) sampler->getSampleCount();
        if (sp.getPluginName() == "sobol") { rp.sampler = B2_SAMPLER_SOBOL; rp.seed = (uint64_t) sp.getInteger("scramble", 0); }
        else if (sp.getPluginName() == "independent") { rp.sampler = B2_SAMPLER_INDEPENDENT; rp.seed = (uint64_t) sp.getInteger("seed", 0); }
        else Log(EError, "b200path: unsupported sampler \"%s\" (hot path: sobol, independent)", sp.getPluginName().c_str());
        rp.max_depth = m_maxDepth; rp.rr_depth = m_rrDepth; rp.strict_normals = m_strictNormals; rp.hide_emitters = m_hideEmitters;
        const Properties &fp = film->getReconstructionFilter()->getProperties();
        if (fp.getPluginName() == "box") { rp.rfilter = B2_RFILTER_BOX; rp.rfilter_param = (float) fp.getFloat("radius", 0.5f); }
        else if (fp.getPluginName() == "gaussian") { rp.rfilter = B2_RFILTER_GAUSSIAN; rp.rfilter_param = (float) fp.getFloat("stddev", 0.5f); }
        else Log(EError, "b200path: unsupported reconstruction filter \"%s\" (supported: box, gaussian)", fp.getPluginName().c_str());
        rp.parity_mode = m_parity ? 1 : 0;
        rp.integrator = B2_INTEGRATOR_PATH;
        /* ---- hot path ---- */
        std::vector<float> storage((size_t) crop.x * crop.y * 5); /* (R,G,B,alpha,weight) = ESpectrumAlphaWeight, hdrfilm.cpp:351-356 */
        const int rc = b2_render(sc, &rp, &storage[0]);
        if (rc == B2_ERR_CANCELLED) { m_handle = NULL; b2_scene_destroy(sc); b2_context_destroy(ctx); return false; } /* integrator.cpp:128 */
        if (rc) Log(EError, "%s", b2_last_error(ctx));
        /* hand the film back: Film::setBitmap (film.h:49-64; HDRFilm::setBitmap hdrfilm.cpp:395-397) */
        ref<Bitmap> bitmap = new Bitmap(Bitmap::ESpectrumAlphaWeight, Bitmap::EFloat32, crop);
        memcpy(bitmap->getFloat32Data(), &storage[0], storage.size() * sizeof(float));
        scene->getFilm()->setBitmap(bitmap);
        if (queue) queue->signalRefresh(job);
        m_handle = NULL;
        b2_scene_destroy(sc);
        b2_context_destroy(ctx);
        return true;
    }

    void cancel() { if (m_handle) b2_cancel((b2_scene *) m_handle); } /* integrator.h:90-93, called from another thread */

    std::string toString() const { return "B200PathTracer[]"; }
    MTS_DECLARE_CLASS()
private:
    int m_rrDepth, m_maxDepth, m_device;
    bool m_strictNormals, m_hideEmitters, m_parity;
    int m_accelBuild;
    void *m_handle;
};

MTS_IMPLEMENT_CLASS_S(B200PathTracer, false, Integrator)
MTS_EXPORT_PLUGIN(B200PathTracer, "GPU wavefront path tracer (libb2mts)");
MTS_NAMESPACE_END
