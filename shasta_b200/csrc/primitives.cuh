// Hand-written device-wide primitives used by the LowHash and alignment pipelines:
// exclusive scan, stream compaction helpers, (radix_sort.cuh) the LSD radix sort, row starts and the row search that
// inverts them, and the k-mer id reverse complement.
// All are plain sm_90a CUDA (warp shuffles / match_any / shared-memory atomics); no CUB/Thrust.
#pragma once

#include "common.cuh"

namespace shb {

constexpr int kScanThreads = 256;
constexpr int kScanItemsPerThread = 16;
constexpr int kScanTile = kScanThreads * kScanItemsPerThread;     // 4096

// ---------------------------------------------------------------------------------------------
// Block-wide exclusive scan of one value per thread (256 threads). Returns the exclusive prefix;
// `total` receives the block total. `smem` must hold 8 T values. Ends with a __syncthreads so the
// scratch can be reused immediately.
template<class T> __device__ __forceinline__ T blockExclusiveScan256(T v, T& total, T* smem)
{
    const unsigned lane = threadIdx.x & 31u;
    const unsigned warp = threadIdx.x >> 5;
    T inc = v;
#pragma unroll
    for(int d = 1; d < 32; d <<= 1) {
        T t = __shfl_up_sync(0xffffffffu, inc, d);
        if(lane >= (unsigned)d) inc += t;
    }
    if(lane == 31) smem[warp] = inc;
    __syncthreads();
    T warpOffset = 0;
    T tot = 0;
#pragma unroll
    for(int w = 0; w < kScanThreads / 32; w++) {
        T s = smem[w];
        if((unsigned)w < warp) warpOffset += s;
        tot += s;
    }
    __syncthreads();
    total = tot;
    return warpOffset + inc - v;
}

template<class T> __global__ void __launch_bounds__(kScanThreads)
scanReduceKernel(const T* __restrict__ in, T* __restrict__ blockSums, uint64_t n)
{
    __shared__ T smem[kScanThreads / 32];
    const uint64_t base = uint64_t(blockIdx.x) * kScanTile;
    T sum = 0;
#pragma unroll
    for(int i = 0; i < kScanItemsPerThread; i++) {
        const uint64_t idx = base + uint64_t(i) * kScanThreads + threadIdx.x;
        if(idx < n) sum += in[idx];
    }
    T total;
    blockExclusiveScan256<T>(sum, total, smem);
    if(threadIdx.x == 0) blockSums[blockIdx.x] = total;
}

// out[i] = blockOffsets[block] + exclusive prefix within the block tile. in and out may alias.
// If totalOut != nullptr (single-block top level) it receives the grand total.
template<class T> __global__ void __launch_bounds__(kScanThreads)
scanDownsweepKernel(const T* in, T* out, const T* __restrict__ blockOffsets, uint64_t n, T* totalOut)
{
    __shared__ T smem[kScanThreads / 32];
    const uint64_t base = uint64_t(blockIdx.x) * kScanTile;
    T running = blockOffsets ? blockOffsets[blockIdx.x] : T(0);
#pragma unroll 1
    for(int i = 0; i < kScanItemsPerThread; i++) {
        const uint64_t idx = base + uint64_t(i) * kScanThreads + threadIdx.x;
        const T v = (idx < n) ? in[idx] : T(0);
        T total;
        const T ex = blockExclusiveScan256<T>(v, total, smem);
        if(idx < n) out[idx] = running + ex;
        running += total;
    }
    if(totalOut && threadIdx.x == 0) *totalOut = running;
}

// Workspace elements (of T) needed by exclusiveScan for n items.
inline uint64_t scanWorkspaceElements(uint64_t n)
{
    uint64_t total = 0;
    while(n > kScanTile) {
        n = (n + kScanTile - 1) / kScanTile;
        total += n;
    }
    return total + 1;
}

// Exclusive scan of n items. in/out may alias. totalOut (device pointer, may be null) receives the
// sum of all items. workspace must hold scanWorkspaceElements(n) items.
template<class T> void exclusiveScan(const T* in, T* out, uint64_t n, T* totalOut, T* workspace, cudaStream_t stream)
{
    if(n == 0) {
        if(totalOut) SHB_CUDA(cudaMemsetAsync(totalOut, 0, sizeof(T), stream));
        return;
    }
    if(n <= kScanTile) {
        SHB_LAUNCH((scanDownsweepKernel<T>), 1, kScanThreads, 0, stream, in, out, (const T*)nullptr, n, totalOut);
        return;
    }
    const uint64_t blocks = (n + kScanTile - 1) / kScanTile;
    T* sums = workspace;
    SHB_LAUNCH((scanReduceKernel<T>), (unsigned)blocks, kScanThreads, 0, stream, in, sums, n);
    exclusiveScan<T>(sums, sums, blocks, totalOut, workspace + blocks, stream);
    SHB_LAUNCH((scanDownsweepKernel<T>), (unsigned)blocks, kScanThreads, 0, stream, in, out, (const T*)sums, n, (T*)nullptr);
}

} // namespace shb

#include "radix_sort.cuh"      // radixSort<HAS_VALUES>, SortWorkspace

namespace shb {

// counts[digit] += 1 for every key (warp-aggregated atomics; the input is sorted by digit so runs are long).
static __global__ void digitCountKernel(const uint64_t* __restrict__ keys, uint32_t n, int shift, uint32_t digitMask,
                                        unsigned long long* __restrict__ counts)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i < n;
    const uint32_t d = active ? (uint32_t(keys[i] >> shift) & digitMask) : 0xffffffffu;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if(active && (__ffs(peers) - 1) == int(threadIdx.x & 31u)) atomicAdd(&counts[d], (unsigned long long)__popc(peers));
}

// ---------------------------------------------------------------------------------------------
// Run detection on a sorted key array: flags[i] = 1 where (keys[i] >> shift) differs from its
// predecessor (or i == 0).
static __global__ void headFlagsKernel(const uint64_t* __restrict__ keys, uint32_t n, int shift, uint32_t* __restrict__ flags)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n) return;
    flags[i] = (i == 0 || (keys[i] >> shift) != (keys[i-1] >> shift)) ? 1u : 0u;
}

// Given flags and their exclusive scan (segIndex), write segStart[segIndex[i]] = i for heads and
// segStart[numSegments] = n (thread n-1 does the latter).
static __global__ void segmentStartsKernel(const uint32_t* __restrict__ flags, const uint32_t* __restrict__ segIndexExclusive,
                                    uint32_t n, uint32_t* __restrict__ segStart)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n) return;
    if(flags[i]) segStart[segIndexExclusive[i]] = i;
    if(i == n - 1) segStart[segIndexExclusive[i] + flags[i]] = n;
}

// Row starts of a table sorted by row (bits 32-63 of the keys): toc[row] = the first of `entries` keys whose row is >= row,
// for row = 0 ... rows.
template<class T> __global__ void rowStartsKernel(const uint64_t* __restrict__ sortedKeys, uint32_t entries, uint32_t rows, T* __restrict__ toc)
{
    const uint32_t row = blockIdx.x * blockDim.x + threadIdx.x;
    if(row > rows) return;
    uint32_t lo = 0, hi = entries;
    while(lo < hi) { const uint32_t mid = lo + ((hi - lo) >> 1); if(uint32_t(sortedKeys[mid] >> 32) < row) lo = mid + 1; else hi = mid; }
    toc[row] = T(lo);
}

// The inverse of rowStartsKernel: the last row r in [lo, hi) with toc[r] <= p, for a non-decreasing toc with toc[lo] <= p.
// For the marker toc this is the oriented read of marker position p (shasta::findMarkerId); empty rows are skipped.
template<class T, class P> __device__ __forceinline__ uint32_t rowOf(const T* toc, uint32_t lo, uint32_t hi, P p)
{
    while(hi - lo > 1) { const uint32_t mid = lo + ((hi - lo) >> 1); if(toc[mid] <= p) lo = mid; else hi = mid; }
    return lo;
}

// The reverse complement of a k-mer id (k <= 16). Bit-plane reverse complement: complement = invert both planes, reverse =
// bit-reverse each k-bit plane (src/ShortBaseSequence.hpp:109-118, src/Base.hpp:139-143).
__device__ __forceinline__ uint32_t reverseComplementKmer(uint32_t kmer, uint32_t k)
{
    const uint32_t mask = (k == 16) ? 0xffffu : ((1u << k) - 1u);
    const uint32_t lsb = ~kmer & mask;
    const uint32_t msb = ~(kmer >> k) & mask;
    return ((__brev(msb) >> (32 - k)) << k) | (__brev(lsb) >> (32 - k));
}

// out[i] = in[i] widened to 64 bits, for i < n. N, the index type, is uint32_t or uint64_t.
template<class N> __global__ void widenKernel(const uint32_t* __restrict__ in, N n, unsigned long long* __restrict__ out)
{
    const N i = N(blockIdx.x) * blockDim.x + threadIdx.x;
    if(i < n) out[i] = in[i];
}

} // namespace shb
