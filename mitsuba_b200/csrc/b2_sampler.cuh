// Sampler state in registers: Sobol' (src/samplers/sobol.cpp:204-252 + sobolseq.h:45-133) and the
// counter-based `independent` stream (TEA, include/mitsuba/core/qmc.h:146-156).
#pragma once
#include "b2_math.cuh"
#include "b2_types.h"

namespace b2 {

B2_HD uint64_t sampleTEA(uint32_t v0, uint32_t v1, int rounds = 4) {
    uint32_t sum = 0;
    for (int i = 0; i < rounds; ++i) {
        sum += 0x9e3779b9u;
        v0 += ((v1 << 4) + 0xA341316Cu) ^ (v1 + sum) ^ ((v1 >> 5) + 0xC8013EA4u);
        v1 += ((v0 << 4) + 0xAD90777Du) ^ (v0 + sum) ^ ((v0 >> 5) + 0x7E95761Eu);
    }
    return ((uint64_t) v1 << 32) + v0;
}

// sobolseq.h:45-60: XOR of the matrix columns selected by the set bits of `index`.  XOR is
// associative, so visiting only the set bits (ffs) gives the identical word.
B2_DEV float sobolSample(const uint32_t *__restrict__ m32, uint64_t index, uint32_t dimension, uint32_t scramble) {
    uint32_t result = scramble;
    const uint32_t *col = m32 + dimension * 52u;
    uint32_t lo = (uint32_t) index, hi = (uint32_t) (index >> 32);
    while (lo) {
        int b = __ffs(lo) - 1;
        result ^= __ldg(col + b);
        lo &= lo - 1;
    }
    while (hi) {
        int b = __ffs(hi) - 1;
        result ^= __ldg(col + 32 + b);
        hi &= hi - 1;
    }
    return fminf(result * (1.0f / 4294967296.0f), B2_ONE_MINUS_EPS);
}

// Same word through nibble-sliced tables: nib[dim][p][v] = XOR of columns 4p..4p+3 of `dim` selected by the bits of v.
// XOR is associative/commutative, so the result is bit-identical to the column loop; 8 independent loads cover a
// 32-bit index (no data-dependent trip count, no divergence), `extra` more nibbles cover longer indices.
B2_DEV float sobolSampleNib(const uint32_t *__restrict__ nib, uint64_t index, uint32_t dimension, uint32_t scramble, uint32_t nNib) {
    const uint32_t *t = nib + dimension * (13u * 16u);
    const uint32_t lo = (uint32_t) index;
    uint32_t r0 = __ldg(t + 0 * 16 + (lo & 15u)), r1 = __ldg(t + 1 * 16 + ((lo >> 4) & 15u)), r2 = __ldg(t + 2 * 16 + ((lo >> 8) & 15u)),
             r3 = __ldg(t + 3 * 16 + ((lo >> 12) & 15u)), r4 = __ldg(t + 4 * 16 + ((lo >> 16) & 15u)), r5 = __ldg(t + 5 * 16 + ((lo >> 20) & 15u)),
             r6 = __ldg(t + 6 * 16 + ((lo >> 24) & 15u)), r7 = __ldg(t + 7 * 16 + (lo >> 28));
    uint32_t result = scramble ^ r0 ^ r1 ^ r2 ^ r3 ^ r4 ^ r5 ^ r6 ^ r7;
    if (nNib > 8u) { // uniform across the launch
        uint32_t hi = (uint32_t) (index >> 32);
        for (uint32_t p = 8; p < nNib; ++p, hi >>= 4) result ^= __ldg(t + p * 16 + (hi & 15u));
    }
    return fminf(result * (1.0f / 4294967296.0f), B2_ONE_MINUS_EPS);
}

// sobolseq.h:104-133 look_up through nibble tables built on the host for this render's m (see DRender::lookupNib)
B2_DEV uint64_t sobolLookUpNib(const uint64_t *__restrict__ lut, uint32_t m, uint32_t frame, uint32_t px, uint32_t py, uint64_t scramble,
                               uint32_t frameNib, uint32_t bNib) {
    const uint32_t m2 = m << 1;
    uint64_t index = (uint64_t) frame << m2;
    uint64_t delta = 0;
    for (uint32_t p = 0; p < frameNib; ++p) delta ^= __ldg(lut + p * 16 + ((frame >> (4 * p)) & 15u));
    scramble = (scramble & 0xFFFFFFFFull) >> (32 - m);
    uint64_t b = (((uint64_t) (px ^ scramble) << m) | (py ^ scramble)) ^ delta;
    const uint64_t *inv = lut + 13 * 16;
    for (uint32_t p = 0; p < bNib; ++p) index ^= __ldg(inv + p * 16 + (uint32_t) ((b >> (4 * p)) & 15ull));
    return index;
}

// sobolseq.h:104-133 look_up (SINGLE_PRECISION scramble branch)
B2_DEV uint64_t sobolLookUp(const uint64_t *__restrict__ vdc, const uint64_t *__restrict__ inv, uint32_t m, uint32_t frame,
                            uint32_t px, uint32_t py, uint64_t scramble) {
    const uint32_t m2 = m << 1;
    uint64_t index = (uint64_t) frame << m2;
    uint64_t delta = 0;
    const uint64_t *vrow = vdc + (m - 1) * 52u;
    while (frame) {
        int c = __ffs(frame) - 1;
        delta ^= __ldg(vrow + c);
        frame &= frame - 1;
    }
    scramble = (scramble & 0xFFFFFFFFull) >> (32 - m);
    uint64_t b = (((uint64_t) (px ^ scramble) << m) | (py ^ scramble)) ^ delta;
    const uint64_t *irow = inv + (m - 1) * 52u;
    while (b) {
        int c = __ffsll((long long) b) - 1;
        index ^= __ldg(irow + c);
        b &= b - 1;
    }
    return index;
}

// The per-path sampler: 12 bytes of state (u64 index/key, u32 dimension), lives in registers inside
// a kernel and in DPool::smp / meta between kernels.
struct PathSampler {
    uint64_t index;      // sobol: m_sobolSampleIndex; independent: stream key
    uint32_t dim;
    int kind;            // 0 sobol, 2 counter
    uint32_t scramble32; // sobol scramble (low 32 bits) / seed hi for the counter stream
    const uint32_t *m32;   // nibble-sliced tables (DScene::sobolNib)
    uint32_t nNib;
    bool overflow;
    float replayA, replayB; // kind 4 (component tests): next1D alternates A, B

    B2_DEV float next1D() {
        if (kind == 3) return __uint_as_float(scramble32); // replay (component tests)
        if (kind == 4) return (dim++ & 1u) ? replayB : replayA;
        if (kind == 0) {
            if (dim >= 1024u) { overflow = true; dim = 1023u; } // sobol.cpp:223-225 raises an error here
            return sobolSampleNib(m32, index, dim++, scramble32, nNib);
        } else {
            // one 8-round TEA block (4 rounds leave consecutive keys correlated) serves two dimensions: 2k -> low word, 2k+1 -> high word
            const uint32_t d = dim++;
            const uint64_t r = sampleTEA((uint32_t) index, (d >> 1) ^ scramble32, 8);
            const uint32_t w = (d & 1u) ? (uint32_t) (r >> 32) : (uint32_t) r;
            uint32_t u = (w >> 9) | 0x3f800000u; // random.cpp:630-640
            return __uint_as_float(u) - 1.0f;
        }
    }
    B2_DEV void next2D(float &a, float &b) {
        // sobol.cpp:231-232: with no sample arrays requested m_arrayStartDim == m_arrayEndDim == 5, and a 2-D request at dimension 4
        // ("dim + 1 >= start && dim < end") jumps to dimension 5 -- Sobol' dimension 4 is never used by consecutive next2D() calls
        if (kind == 0 && dim == 4u) dim = 5u;
        if (kind == 0 && dim + 1 >= 1024u) { overflow = true; dim = 1022u; }
        a = next1D();
        b = next1D();
    }
};

// The sampler of the `direct` integrator: the regular dimensions of a PathSampler that skip the range [5, arrayEnd) its 2-D sample
// arrays occupy (sobol.cpp:218-238), and the array entries themselves.  Its own type, so that PathSampler and the kernels that use it
// are compiled as before.  arrayEnd = 5 + 2 * (number of arrays) for Sobol' (with no array the range is empty and only next2D's jump
// from dimension 4 to 5 remains, as in PathSampler); the counter stream skips only when there are arrays, and its arrays fill the
// range entry by entry (DESIGN.md "direct").
struct ArraySampler {
    PathSampler p;
    uint32_t arrayEnd;
    bool skip;
    B2_DEV float next1D() {
        if (skip && p.dim >= 5u && p.dim < arrayEnd) p.dim = arrayEnd; // sobol.cpp:220-221
        return p.next1D();
    }
    B2_DEV void next2D(float &a, float &b) {
        if (skip && p.dim + 1u >= 5u && p.dim < arrayEnd) p.dim = arrayEnd; // sobol.cpp:234-235
        if (p.kind == 0 && p.dim + 1 >= 1024u) { p.overflow = true; p.dim = 1022u; }
        a = p.next1D();
        b = p.next1D();
    }
};

// word d of the counter stream of key (see PathSampler::next1D)
B2_DEV float counterAt(uint32_t key, uint32_t seedHi, uint32_t d) {
    const uint64_t r = sampleTEA(key, (d >> 1) ^ seedHi, 8);
    const uint32_t w = (d & 1u) ? (uint32_t) (r >> 32) : (uint32_t) r;
    return __uint_as_float((w >> 9) | 0x3f800000u) - 1.0f;
}

} // namespace b2
