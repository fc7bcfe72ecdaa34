/* TEST INFRASTRUCTURE ONLY: the reference's own `direct` integrator (src/integrators/direct/direct.cpp) inside the renderer that
 * oracle/path_ref_shim.cpp assembles from the reference's sources.  tests/direct_pins.py compiles this file, direct.cpp and the objects
 * of oracle/_build/pathref (all but that harness's own object, which this file includes) into one library that writes
 * tests/golden/path_ref_direct.npz; it runs only where the reference tree is present. */
#include "path_ref_shim.cpp"
#include "orc_direct_sampler.h"

extern "C" void *CreateInstance_direct(const Properties &props);

/* this repository's counter stream (CounterSamplerPlugin) with the 2-D sample arrays `direct` requests (Sampler::request2DArray), filled
 * for every sample of the pixel from tests/orc_direct_sampler.h and handed out by the reference's own Sampler::next2DArray */
class CounterArraySamplerPlugin : public Sampler {
public:
    CounterArraySamplerPlugin(int W, size_t spp, uint64_t seed) : Sampler(Properties()), m_impl(W, (uint32_t) spp, seed) { m_sampleCount = spp; }
    void generate(const Point2i &pos) {
        uint32_t entries = 0, offset = 0;
        for (size_t n : m_req2D) entries += (uint32_t) n;
        m_impl.arrayEnd = 5 + 2 * entries;
        m_impl.generate(pos.x, pos.y);
        for (size_t s = 0; s < m_sampleCount; ++s, m_impl.advance()) {
            offset = 0;
            for (size_t r = 0; r < m_req2D.size(); ++r) {
                const size_t n = m_req2D[r];
                for (size_t k = 0; k < n; ++k) {
                    float a, b;
                    m_impl.arrayEntry((uint32_t) r, offset, (uint32_t) n, (uint32_t) k, a, b);
                    m_sampleArrays2D[r][s * n + k] = Point2(a, b);
                }
                offset += (uint32_t) n;
            }
        }
        m_impl.generate(pos.x, pos.y);
        m_sampleIndex = 0;
        m_dimension1DArray = m_dimension2DArray = 0;
    }
    void advance() { m_impl.advance(); ++m_sampleIndex; m_dimension1DArray = m_dimension2DArray = 0; }
    Float next1D() { return m_impl.next1D(); }
    Point2 next2D() { float a, b; m_impl.next2D(a, b); return Point2(a, b); }
    ref<Sampler> clone() { return this; }
    void setSampleIndex(size_t) {}
    std::string toString() const { return "CounterArraySampler"; }
    const Class *getClass() const { return Sampler::m_theClass; }
private:
    orc::CounterArraySampler m_impl;
};

extern "C" {
/* After pathref_setup4 (which configured the scene with `path`): render with `direct` instead.  samplerKind 2 replaces the counter
 * sampler by the one with arrays (W: the crop width, as pathref_setup4 keys the stream).  configureSampler is called once here: it is
 * where `direct` requests its arrays (Scene::configure has already run it for `path`, which requests none). */
void pathref_use_direct(void *h, int samplerKind, int W, int spp, uint64_t seed, int emitterSamples, int bsdfSamples, int strictNormals,
                        int hideEmitters) {
    PathRef *p = (PathRef *) h;
    if (samplerKind == 2) {
        p->sampler = new CounterArraySamplerPlugin(W, (size_t) spp, seed);
        p->sampler->configure();
    }
    Properties ip("direct");
    ip.setInteger("emitterSamples", emitterSamples); ip.setInteger("bsdfSamples", bsdfSamples);
    ip.setBoolean("strictNormals", strictNormals != 0); ip.setBoolean("hideEmitters", hideEmitters != 0);
    p->integrator = (Integrator *) CreateInstance_direct(ip);
    p->integrator->configure();
    p->integrator->configureSampler(p->scene, p->sampler);
}
}
