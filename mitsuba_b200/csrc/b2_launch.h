// Host-callable launchers of the wavefront kernels.  The kernel translation unit is compiled twice
// (b2::parity with -fmad=false, b2::fast with FMA contraction); each build exports its launchers as one KernelSet.
#pragma once
#include "b2_types.h"

#define B2_TRACE_BLOCK 256
#define B2_SHADE_BLOCK 128

namespace b2 {

struct LaunchCfg {
    int numSMs = 0;
    size_t traceSmem = 0;
    int gridExtend = 0, gridExtendSort = 0, gridOccluded = 0, gridTrace = 0, gridGenerate = 0, gridVolLockstep = 0;
    int gridGenerateSlots = 0; // k_generate<SLOTS = true>: the slot-order drain of k_bounce_flat's route
    int gridShade[5] = {0, 0, 0, 0, 0};
    int gridShadeTex = 0; // k_shade<-1, TEX = true> (textured scenes)
    int gridShadeTexCls[4] = {0, 0, 0, 0}; // k_shade<c, TEX = true>: class-sorted dispatch of textured / environment-mapped scenes
    // flat-leaf variants (shared-memory resident scenes): k_extend_flat / k_occluded_flat (class-sorted), k_bounce_flat[TEX][class]
    size_t flatSmem = 0;
    int gridExtendFlatSort = 0, gridOccludedFlat = 0;
    int gridBounceFlat[2][5] = {{0, 0, 0, 0, 0}, {0, 0, 0, 0, 0}};
    // k_direct[TEX][walk]: walk 0 flat leaf, 1 binary BVH, 2 instances; its shared memory for the scene's walk
    size_t directSmem = 0;
    int gridDirect[2][3] = {{0, 0, 0}, {0, 0, 0}};
};

struct KernelSet {
    void (*init)(LaunchCfg &cfg, const DScene &sc, int numSMs);
    void (*generate)(const LaunchCfg &, const DScene &, const DPool &, const DRender &, const DFilter &, cudaStream_t);
    void (*extend)(const LaunchCfg &, const DScene &, const DPool &, const DRender &, bool sort, cudaStream_t);
    void (*shade)(const LaunchCfg &, const DScene &, const DPool &, const DRender &, int cls, bool queued, cudaStream_t);
    void (*occluded)(const LaunchCfg &, const DScene &, const DPool &, const DRender &, cudaStream_t);
    // flat scenes shaded by one launch: extend + shade + occluded in one kernel, cls as for shade (unqueued)
    void (*bounce_flat)(const LaunchCfg &, const DScene &, const DPool &, const DRender &, int cls, cudaStream_t);
    void (*volstep)(const LaunchCfg &, const DScene &, const DPool &, const DRender &, cudaStream_t);
    void (*medium_probe)(const LaunchCfg &, const DScene &, int medium, int what, uint64_t n, const float *in, uint64_t seed, float *out,
                         cudaStream_t);
    void (*film_pack)(const LaunchCfg &, const float4 *rgba, const float *w, float *out, size_t n, cudaStream_t);
    void (*trace)(const LaunchCfg &, const DScene &, const float4 *rays, float4 *out, uint64_t n, bool shadow, bool count,
                  unsigned long long *counters, cudaStream_t);
    void (*bsdf_eval)(const LaunchCfg &, const DScene &, int mat, uint64_t n, const float *wi, const float *wo, float *rgb, float *pdf,
                      cudaStream_t);
    void (*bsdf_sample)(const LaunchCfg &, const DScene &, int mat, uint64_t n, const float *wi, const float *samples, float *out,
                        cudaStream_t);
    void (*emitter_direct)(const LaunchCfg &, const DScene &, uint64_t n, const float *ref, const float *samples, float *out, cudaStream_t);
    void (*camera_rays)(const LaunchCfg &, const DScene &, uint64_t n, const float *pos, float *rays, cudaStream_t);
    void (*texture_probe)(const LaunchCfg &, const DScene &, int what, int tex, int hasPartials, float diffScale, uint64_t n, const float *in,
                          float *out, cudaStream_t);
    void (*envmap_probe)(const LaunchCfg &, const DScene &, int what, uint64_t n, const float *in, float *out, cudaStream_t);
    void (*sampler_stream)(const DScene &, const DRender &, int px, int py, int sampleIdx, int ndim, float *out, cudaStream_t);
    void (*splat)(const LaunchCfg &, const DFilter &, int W, int H, uint64_t n, const float *pos, const float *val, float4 *rgba, float *wgt,
                  cudaStream_t);
    // `direct`: work items [begin, end) of the render (camera ray to splat in one thread each); counters: CTR_* of the scene
    void (*direct)(const LaunchCfg &, const DScene &, const DRender &, const DFilter &, unsigned long long *counters, uint64_t begin, uint64_t end,
                   cudaStream_t);
};

namespace parity { extern const KernelSet kernels; }
namespace fast { extern const KernelSet kernels; }

} // namespace b2
