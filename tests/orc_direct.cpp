/* TEST INFRASTRUCTURE ONLY: the oracle of the `direct` integrator.  MIDirectIntegrator::Li (src/integrators/direct/direct.cpp:146-305)
 * restated line by line on the oracle's scene (oracle/mts_oracle.cpp, compiled into the same library: tests/direct_pins.py builds
 * both), with the sample arrays of tests/orc_direct_sampler.h.  Same floating-point rules as the oracle (IEEE, no contraction). */
#include "mts_oracle.cpp"
#include "orc_direct_sampler.h"

namespace {

/* rRec.depth is 1 and the query is not adaptive, so the reduction of :202-208 never applies.  Counts above 1 read the sampler's 2-D
   arrays (configureSampler :138-144: the emitter's array first); a count of 0 or 1 draws one regular 2-D sample.  The emitter sample
   is drawn before the ESmooth test (:210-214). */
template <class S>
Spectrum LiDirect(const Scene &sc, const Ray &r, S *sampler, uint32_t nDirect, uint32_t nBSDF, const OrcRenderParams &rp, float &alpha, OrcStats &st,
                  const RayDiff *sensorDiff) {
    BsdfSet bs{sc.bsdfs.data(), (int) sc.bsdfs.size()};
    Intersection its;
    const Ray ray(r);
    RayDiff rayDiff;
    if (sensorDiff) rayDiff = *sensorDiff;
    Spectrum Li(0.0f);
    sc.rayIntersect(ray, its, st);
    alpha = its.isValid() ? 1.0f : 0.0f;
    if (!its.isValid()) { /* :158-165 */
        if (!rp.hideEmitters && sc.envEmitter >= 0) return sc.evalEnvironment(ray, &rayDiff);
        return Spectrum(0.0f);
    }
    const Mesh &mesh = sc.meshes[its.mesh];
    const int bsdf = mesh.bsdf;
    if (mesh.emitter >= 0 && !rp.hideEmitters) Li += sc.emitterEval(mesh.emitter, its, -ray.d); /* :168-169 */
    if (bs.usesRayDifferentials(bsdf)) Scene::computePartials(its, ray, rayDiff); /* its.getBSDF(ray), :175 */
    if (rp.strictNormals && dot(ray.d, its.geoFrame.n) * Frame::cosTheta(its.wi) >= 0) return Li; /* :177-189 */
    /* configure(), :128-136 */
    const float sum = (float) (nDirect + nBSDF);
    const float weightBSDF = 1 / (float) nBSDF, weightLum = 1 / (float) nDirect;
    const float fracBSDF = nBSDF / sum, fracLum = nDirect / sum;
    const uint32_t bsdfArray = nDirect > 1 ? 1 : 0, bsdfOffset = nDirect > 1 ? nDirect : 0;
    const uint32_t btype = bs.type(bsdf);
    /* ---- emitter sampling, :197-243 ---- */
    float sx = 0, sy = 0;
    if (nDirect <= 1) sampler->next2D(sx, sy);
    DRec dRec;
    dRec.ref = its.p; dRec.refN = V3(0.0f);
    if ((btype & (ETransmission | EBackSide)) == 0) dRec.refN = its.shFrame.n;
    if (btype & ESmooth) {
        for (uint32_t i = 0; i < nDirect && !sc.emitters.empty(); ++i) {
            if (nDirect > 1) sampler->arrayEntry(0, 0, nDirect, i, sx, sy);
            Spectrum value = sc.sampleEmitterDirect(dRec, sx, sy, st);
            if (value.isZero()) continue;
            BRec bRec; bRec.wi = its.wi; bRec.wo = its.shFrame.toLocal(dRec.d); bRec.sampler = sampler; bRec.its = &its.tex;
            const Spectrum bsdfVal = bs.eval(bsdf, bRec);
            if (!bsdfVal.isZero() && (!rp.strictNormals || dot(its.geoFrame.n, dRec.d) * Frame::cosTheta(bRec.wo) > 0)) {
                const float bsdfPdf = bs.pdf(bsdf, bRec); /* every emitter here is EOnSurface (area, constant, envmap) */
                const float weight = Scene::miWeight(dRec.pdf * fracLum, bsdfPdf * fracBSDF) * weightLum;
                Li += value * bsdfVal * weight;
            }
        }
    }
    /* ---- BSDF sampling, :245-302 ---- */
    if (nBSDF <= 1) sampler->next2D(sx, sy);
    for (uint32_t i = 0; i < nBSDF; ++i) {
        if (nBSDF > 1) sampler->arrayEntry(bsdfArray, bsdfOffset, nBSDF, i, sx, sy);
        float bsdfPdf;
        BRec bRec; bRec.wi = its.wi; bRec.sampler = sampler; bRec.its = &its.tex;
        const Spectrum bsdfVal = bs.sample(bsdf, bRec, bsdfPdf, sx, sy);
        if (bsdfVal.isZero()) continue;
        const V3 wo = its.shFrame.toWorld(bRec.wo);
        const float woDotGeoN = dot(its.geoFrame.n, wo);
        if (rp.strictNormals && woDotGeoN * Frame::cosTheta(bRec.wo) <= 0) continue;
        const Ray bsdfRay(its.p, wo);
        Intersection bsdfIts;
        Spectrum value;
        if (sc.rayIntersect(bsdfRay, bsdfIts, st)) {
            const Mesh &m2 = sc.meshes[bsdfIts.mesh];
            if (m2.emitter < 0) continue;
            value = sc.emitterEval(m2.emitter, bsdfIts, -bsdfRay.d);
            /* dRec.setQuery(bsdfRay, bsdfIts): records.inl:171-179 */
            dRec.p = bsdfIts.p; dRec.n = bsdfIts.shFrame.n; dRec.solidAngle = true; dRec.emitter = m2.emitter;
            dRec.d = bsdfRay.d; dRec.dist = bsdfIts.t;
        } else {
            if (sc.envEmitter < 0 || (rp.hideEmitters && bRec.sampledType == ENull)) continue;
            value = sc.evalEnvironment(bsdfRay); /* RayDifferential(bsdfRay): no differentials */
            /* fillDirectSamplingRecord (constant.cpp:246-262, envmap.cpp:358-374) */
            float nearT, farT;
            if (!sc.bsphereIntersect(bsdfRay.o, bsdfRay.d, nearT, farT) || nearT > 0 || farT < 0) continue;
            dRec.p = bsdfRay(farT); dRec.n = normalize(sc.bsCenter - dRec.p); dRec.solidAngle = true; dRec.emitter = sc.envEmitter;
            dRec.d = bsdfRay.d; dRec.dist = farT;
        }
        const float lumPdf = (!(bRec.sampledType & EDelta)) ? sc.pdfEmitterDirect(dRec) : 0;
        const float weight = Scene::miWeight(bsdfPdf * fracBSDF, lumPdf * fracLum) * weightBSDF;
        Li += value * bsdfVal * weight;
    }
    return Li;
}

/* SamplingIntegrator::renderBlock (integrator.cpp:140-188) as the oracle's render_impl does it, with `direct` and its samplers */
template <class S>
void renderDirect(Scene *sc, const OrcRenderParams *rp, uint32_t nE, uint32_t nB, float *film, OrcStats *stats, float *perSample) {
    const int W = sc->W, H = sc->H;
    RFilter filter(rp->rfilter, rp->rfilterParam);
    const int bs = rp->blockSize > 0 ? rp->blockSize : 32;
    const int nbx = (W + bs - 1) / bs, nby = (H + bs - 1) / bs, nBlocks = nbx * nby;
    const int lo = rp->sampleLo, hi = rp->sampleHi > 0 ? rp->sampleHi : rp->spp;
    int nThreads = rp->threads > 0 ? rp->threads : (int) std::thread::hardware_concurrency();
    if (nThreads < 1) nThreads = 1;
    std::vector<std::unique_ptr<ImageBlock>> blocks(nBlocks);
    std::atomic<int> next(0);
    std::vector<OrcStats> tstats(nThreads);
    const bool useDiff = !sc->textures.empty() || !sc->envmaps.empty();
    const float diffScaleFactor = 1.0f / std::sqrt((float) rp->spp); /* integrator.cpp:144-145 */
    /* configureSampler, direct.cpp:138-144: one 2-D array per count above 1 */
    const uint32_t nArrays = (nE > 1 ? 1u : 0u) + (nB > 1 ? 1u : 0u), arrayEntries = (nE > 1 ? nE : 0u) + (nB > 1 ? nB : 0u);
    auto worker = [&](int tid) {
        OrcStats st{};
        std::unique_ptr<S> sampler;
        if constexpr (std::is_same<S, SobolArraySampler>::value) {
            sampler.reset(new S(&sc->sobol, rp->seed, W, H));
            sampler->arrayEnd = 5 + 2 * nArrays;
        } else {
            sampler.reset(new S(W, (uint32_t) rp->spp, rp->seed));
            sampler->arrayEnd = 5 + 2 * arrayEntries;
        }
        for (;;) {
            int b = next.fetch_add(1);
            if (b >= nBlocks) break;
            int bx = b % nbx, by = b / nbx;
            int ox = bx * bs, oy = by * bs, sx = std::min(bs, W - ox), sy = std::min(bs, H - oy);
            std::unique_ptr<ImageBlock> blk(new ImageBlock(ox, oy, sx, sy, &filter));
            for (int y = oy; y < oy + sy; ++y)
                for (int x = ox; x < ox + sx; ++x) {
                    sampler->generate(x, y);
                    for (int j = 0; j < lo; ++j) sampler->advance();
                    for (int j = lo; j < hi; ++j) {
                        float ax, ay; sampler->next2D(ax, ay);
                        float spx = (float) x + ax, spy = (float) y + ay;
                        float apx = 0.5f, apy = 0.5f;
                        if (sc->apertureRadius > 0) sampler->next2D(apx, apy); /* integrator.cpp:173-174 */
                        RayDiff rd;
                        Ray ray = sc->sampleRay(spx, spy, apx, apy, useDiff ? &rd : nullptr, diffScaleFactor);
                        float alpha;
                        Spectrum spec = LiDirect(*sc, ray, sampler.get(), nE, nB, *rp, alpha, st, useDiff ? &rd : nullptr);
                        if (!blk->put(spx, spy, spec, alpha)) ++st.badSamples;
                        if (perSample) {
                            float *o = perSample + (((size_t) y * W + x) * (size_t) (hi - lo) + (size_t) (j - lo)) * 4;
                            o[0] = spec.x; o[1] = spec.y; o[2] = spec.z; o[3] = alpha;
                        }
                        ++st.samples;
                        sampler->advance();
                    }
                }
            blocks[b] = std::move(blk);
        }
        tstats[tid] = st;
    };
    std::vector<std::thread> th;
    for (int t = 1; t < nThreads; ++t) th.emplace_back(worker, t);
    worker(0);
    for (auto &t : th) t.join();
    memset(film, 0, (size_t) W * H * 5 * sizeof(float)); /* merged in block order, as render_impl */
    for (int b = 0; b < nBlocks; ++b) {
        ImageBlock &blk = *blocks[b];
        for (int y = 0; y < blk.bh(); ++y) {
            int fy = blk.oy - blk.border + y;
            if (fy < 0 || fy >= H) continue;
            for (int x = 0; x < blk.bw(); ++x) {
                int fx = blk.ox - blk.border + x;
                if (fx < 0 || fx >= W) continue;
                const float *src = blk.data.data() + ((size_t) y * blk.bw() + x) * 5;
                float *dst = film + ((size_t) fy * W + fx) * 5;
                for (int k = 0; k < 5; ++k) dst[k] += src[k];
            }
        }
    }
    if (stats) {
        OrcStats tot{};
        for (auto &s : tstats) {
            tot.samples += s.samples; tot.rays += s.rays; tot.shadowRays += s.shadowRays;
            tot.nodeVisits += s.nodeVisits; tot.primTests += s.primTests; tot.badSamples += s.badSamples;
        }
        *stats = tot;
    }
}

} // namespace

extern "C" {
/* rp->sampler: 0 Sobol', 2 counter stream (the reference's SFMT `independent` has no array definition here) */
int orcd_render(void *s, const OrcRenderParams *rp, int emitterSamples, int bsdfSamples, float *film, OrcStats *stats, float *perSample) {
    if (emitterSamples < 0 || bsdfSamples < 0 || emitterSamples + bsdfSamples == 0) return -1;
    if (rp->sampler == 0) renderDirect<SobolArraySampler>((Scene *) s, rp, (uint32_t) emitterSamples, (uint32_t) bsdfSamples, film, stats, perSample);
    else if (rp->sampler == 2) renderDirect<CounterArraySampler>((Scene *) s, rp, (uint32_t) emitterSamples, (uint32_t) bsdfSamples, film, stats, perSample);
    else return -1;
    return 0;
}
}
