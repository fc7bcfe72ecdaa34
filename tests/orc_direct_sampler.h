/* TEST INFRASTRUCTURE ONLY.  The 2-D sample arrays of the `direct` integrator on top of the oracle's samplers (oracle/orc_sampler.h), shared
 * by the oracle of `direct` (tests/orc_direct.cpp) and the reference harness that serves the counter stream to the reference's
 * MIDirectIntegrator (tests/direct_ref_shim.cpp).
 *
 * Sobol' (src/samplers/sobol.cpp:171-196, 218-247): array r occupies dimensions 5 + 2r and 6 + 2r; entry k of pixel sample s is the point
 * look_up(m, s * n + k, px, py) of the pixel's sequence (sampler.cpp:86); regular draws skip [5, arrayEnd), arrayEnd = 5 + 2 * #arrays.
 * Counter stream (this repository's definition, DESIGN.md section 8f): entry k of array r of sample s is the stream of (pixel, s) at
 * dimensions 5 + 2 (sum_{q<r} n_q + k) and + 1; regular draws skip [5, arrayEnd), arrayEnd = 5 + 2 sum n, with the Sobol' sampler's
 * two tests -- only when there are arrays, so that the stream of `path` / `volpath` is unchanged. */
#pragma once
#include "orc_sampler.h"

namespace orc {

struct SobolArraySampler : SobolSampler {
    uint32_t arrayEnd = 5;
    using SobolSampler::SobolSampler;
    float next1D() override {
        if (dimension >= 5 && dimension < arrayEnd) dimension = arrayEnd; /* sobol.cpp:220-221 */
        return SobolSampler::next1D();
    }
    void next2D(float &a, float &b) override {
        if (dimension + 1 >= 5 && dimension < arrayEnd) dimension = arrayEnd; /* sobol.cpp:234-235 */
        SobolSampler::next2D(a, b);
    }
    /* entry k of array r (n entries per sample) of the current pixel sample */
    void arrayEntry(uint32_t r, uint32_t /* offset */, uint32_t n, uint32_t k, float &a, float &b) const {
        const uint32_t j = (uint32_t) (sampleIndex * n + k);
        const uint64_t idx = logResolution > 1 ? sobolLookUp(*T, logResolution, j, (uint32_t) px, (uint32_t) py, scramble) : j;
        a = sobolSample(*T, idx, 5 + 2 * r, (uint32_t) scramble);
        b = sobolSample(*T, idx, 6 + 2 * r, (uint32_t) scramble);
    }
};

struct CounterArraySampler : CounterSampler {
    uint32_t arrayEnd = 5;
    using CounterSampler::CounterSampler;
    /* word d of the current sample's stream (CounterSampler::next1D without advancing) */
    float word(uint32_t d) const {
        const uint64_t r = sampleTEA(key, (d >> 1) ^ seedHi, 8);
        const uint32_t w = (d & 1u) ? (uint32_t) (r >> 32) : (uint32_t) r;
        union { uint32_t u; float f; } x;
        x.u = (w >> 9) | 0x3f800000UL;
        return x.f - 1.0f;
    }
    float next1D() override {
        if (arrayEnd > 5 && dim >= 5 && dim < arrayEnd) dim = arrayEnd;
        return CounterSampler::next1D();
    }
    void next2D(float &a, float &b) override {
        if (arrayEnd > 5 && dim + 1 >= 5 && dim < arrayEnd) dim = arrayEnd;
        a = CounterSampler::next1D();
        b = CounterSampler::next1D();
    }
    /* entry k of the array whose first entry sits at `offset` entries into the reserved range */
    void arrayEntry(uint32_t /* r */, uint32_t offset, uint32_t /* n */, uint32_t k, float &a, float &b) const {
        a = word(5 + 2 * (offset + k));
        b = word(6 + 2 * (offset + k));
    }
};

} // namespace orc
