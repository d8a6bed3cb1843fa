// Device helpers shared by the marker graph vertices (markergraph.cu) and edges (markergraph_edges.cu): Uint40 loads and
// stores, the reverse complement of a marker, and the segmented rank sorts of distinct uint64 keys. The oriented read of a
// marker is rowOf (primitives.cuh).
#pragma once

#include "context.cuh"

#include <algorithm>

namespace shb {
namespace {

constexpr uint64_t kInvalid40 = (1ull << 40) - 1;     // MarkerGraph::invalidCompressedVertexId (Uint40 of the uint64 max)
constexpr uint32_t kMgThreads = 256;
constexpr uint32_t kWarpSortMax = 32;                 // sets up to this size are sorted in registers by one warp
constexpr uint32_t kBlockSortMax = 4096;              // up to this size in shared memory by one block; larger by radixSort

// Sets of up to 32 markers: one warp each, rank sort in registers. Larger sets are listed for the next kernels.
__global__ void __launch_bounds__(kMgThreads) warpSortKernel(uint64_t* keys, const uint64_t* __restrict__ setOffset, const uint64_t* __restrict__ setSize,
                                                             uint64_t setCount, uint64_t* bigSets, unsigned long long* bigCount)
{
    const uint64_t k = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(k >= setCount) return;
    const uint64_t n = setSize[k], off = setOffset[k];
    if(n > kWarpSortMax) {
        if(lane == 0) bigSets[atomicAdd(bigCount, 1ull)] = k;
        return;
    }
    const uint64_t v = lane < n ? keys[off + lane] : ~0ull;
    uint32_t rank = 0;
    for(uint32_t j = 0; j < kWarpSortMax; j++) {
        const uint64_t u = __shfl_sync(0xffffffffu, v, j);
        rank += (u < v) ? 1u : 0u;                       // keys of one set are distinct
    }
    if(lane < n) keys[off + rank] = v;
}

// One block per listed set of up to kBlockSortMax markers: rank sort in shared memory.
__global__ void __launch_bounds__(kMgThreads) blockSortKernel(uint64_t* keys, const uint64_t* __restrict__ setOffset, const uint64_t* __restrict__ setSize,
                                                              const uint64_t* __restrict__ sets)
{
    __shared__ uint64_t s[kBlockSortMax];
    const uint64_t k = sets[blockIdx.x];
    const uint32_t n = uint32_t(setSize[k]);
    uint64_t* seg = keys + setOffset[k];
    for(uint32_t j = threadIdx.x; j < n; j += blockDim.x) s[j] = seg[j];
    __syncthreads();
    for(uint32_t j = threadIdx.x; j < n; j += blockDim.x) {
        const uint64_t v = s[j];
        uint32_t rank = 0;
        for(uint32_t t = 0; t < n; t++) rank += s[t] < v ? 1u : 0u;
        seg[rank] = v;
    }
}

__device__ __forceinline__ void store40(uint8_t* p, uint64_t v)
{
#pragma unroll
    for(int b = 0; b < 5; b++) p[b] = uint8_t(v >> (8 * b));
}
__device__ __forceinline__ uint64_t load40(const uint8_t* p)
{
    uint64_t v = 0;
#pragma unroll
    for(int b = 0; b < 5; b++) v |= uint64_t(p[b]) << (8 * b);
    return v;
}

__device__ __forceinline__ uint64_t reverseComplementMarker(const uint64_t* __restrict__ toc, uint32_t rows, uint64_t m)
{
    const uint32_t lo = rowOf(toc, 0u, rows, m);
    const uint64_t ordinal = m - toc[lo], size = toc[lo + 1] - toc[lo];
    return toc[lo ^ 1u] + (size - 1 - ordinal);
}

unsigned gridFor(uint64_t n, uint32_t threads = kMgThreads)
{
    return unsigned(std::min<uint64_t>((n + threads - 1) / threads, 132ull * 16));
}

} // namespace
} // namespace shb
