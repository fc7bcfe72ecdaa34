// Device-side BVH build (bvh_device.cu): the same trees buildBVH makes, built in HBM.
#pragma once
#include <stdint.h>
#include <string>
#include <vector>
#include <cuda_runtime.h>
#include "bvh_builder.h"

namespace b2 {

// Node arrays stay on the device (cudaMalloc'd, owned by the caller afterwards); only the leaf order comes back.
struct DeviceBVHResult {
    BVHNode *nodes = nullptr;
    size_t nNodes = 0;
    BVH8Node *nodes8 = nullptr; // only with `wide`
    size_t nNodes8 = 0;
    std::vector<uint32_t> leafPrims;
    int32_t rootRef = -1;
    int depth = 0, depth8 = 0;
    float ms = 0; // CUDA-event time from the box upload to the leaf-order readback
    DeviceBVHResult() = default;
    DeviceBVHResult(const DeviceBVHResult &) = delete;
    DeviceBVHResult &operator=(const DeviceBVHResult &) = delete;
    ~DeviceBVHResult() { if (nodes) cudaFree(nodes); if (nodes8) cudaFree(nodes8); }
};

// Same inputs and outputs as buildBVH: BVHNode[] / BVH8Node[] byte-identical to it, leafPrims identical as a sequence except below a
// node where the host builder took its object-median fallback (there: the same set in every binary leaf).  Returns a message on
// failure (empty on success).  `out` must be freshly constructed.
std::string buildBVHDevice(const std::vector<PrimBox> &boxes, const std::vector<uint32_t> &ids, int maxLeaf, int maxDepth, bool wide,
                           cudaStream_t st, DeviceBVHResult &out);

// dst[i] = src[i] with inner references moved by nodeBase and leaf starts by leafBase (a tree appended to merged arrays)
cudaError_t appendTreeDevice(BVHNode *dst, const BVHNode *src, size_t n, uint32_t nodeBase, uint32_t leafBase, cudaStream_t st);

} // namespace b2
