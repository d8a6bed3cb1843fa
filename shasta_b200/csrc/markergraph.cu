// Assembler::createMarkerGraphVertices (src/AssemblerMarkerGraph.cpp:38-518, threads :522-770) and
// findMarkerGraphReverseComplementVertices (:1134-1230) on the GPU.
//   * union: every read-graph edge pair that passes the filters has its compressed alignment decoded by one warp (all lanes
//     parse the same bytes, lane j keeps the j-th streak of each group of 32) and the aligned marker pairs of the group are
//     spread over the lanes; each pair unites (m0, m1) and (rc(m0), rc(m1)) in a union-find over all M markers;
//   * the union-find is lock-free and min-linking: a root is hooked under the smaller root with atomicCAS, finds halve the
//     path. Every non-root's parent is smaller than itself, so the root of a set is its smallest marker and the partition
//     and the roots do not depend on the schedule (the reference's concurrent union by rank, src/dset64-gccAtomic.hpp:145-176,
//     gives schedule-dependent representatives);
//   * the parent array is then reused for everything per marker: root, then FLAG|size at the roots, then FLAG|kept-set id;
//   * kept sets (minCoverage <= size <= maxCoverage) and good sets (not bad) are numbered by scans in root order, so the
//     vertices come out in increasing order of their smallest marker; each kept set's markers are scattered, sorted as
//     (oriented read, ordinal) keys, which is marker-id order, and checked for the two "bad" conditions.
#include "compressed_alignment.cuh"
#include "context.cuh"
#include "hostpool.cuh"
#include "markergraph_kernels.cuh"

#include <algorithm>
#include <chrono>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

namespace shb {
namespace {

constexpr uint64_t kRootFlag = 1ull << 63;           // parent slot of a root after the compression pass
constexpr uint64_t kValueMask = kRootFlag - 1;
constexpr uint64_t kNoSet = ~0ull;                    // root slot of a set that is not kept
constexpr uint32_t kTile = kScanTile;                 // markers per block of the kept-set numbering (4096)

struct MgPair {                 // one read-graph edge pair that passes the filters
    uint64_t byteBegin;         // its compressed alignment in the batch's byte buffer
    uint32_t byteCount;
    uint32_t o0, o1;            // orientedReadIds of the first edge of the pair
    uint32_t pairIndex;         // edge pair index in the read graph (its first edge is 2 * pairIndex)
};

// ---- union-find ---------------------------------------------------------------------------------------------------
// Loads and stores go through L2 (.cg): other SMs hook roots and halve paths concurrently. A stale parent is still an
// ancestor, so every read value is safe to follow.
__device__ __forceinline__ uint64_t findRoot(uint64_t* P, uint64_t x)
{
    uint64_t p = __ldcg(P + x);
    while(p != x) {
        const uint64_t gp = __ldcg(P + p);
        if(gp == p) return p;
        __stcg(P + x, gp);                      // path halving: x is not a root, so no hook can target this slot
        x = gp;
        p = __ldcg(P + x);
    }
    return x;
}

__device__ __forceinline__ void unite(uint64_t* P, uint64_t a, uint64_t b)
{
    for(;;) {
        a = findRoot(P, a);
        b = findRoot(P, b);
        if(a == b) return;
        if(a < b) { const uint64_t t = a; a = b; b = t; }
        const uint64_t old = atomicCAS(reinterpret_cast<unsigned long long*>(P + a), a, b);   // hook the larger root
        if(old == a) return;
        a = old;                                // hooked by someone else meanwhile: continue from its new parent
    }
}

__global__ void initParentKernel(uint64_t* P, uint64_t M)
{
    for(uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < M; i += uint64_t(gridDim.x) * blockDim.x) P[i] = i;
}

// One warp per edge pair (createMarkerGraphVerticesThreadFunction1, :537-606).
__global__ void __launch_bounds__(kMgThreads) uniteKernel(const MgPair* __restrict__ pairs, uint32_t n, const uint8_t* __restrict__ bytes,
                                                          const uint64_t* __restrict__ toc, const uint32_t* __restrict__ kmerIds,
                                                          uint64_t* P, unsigned long long* errKmer,
                                                          unsigned long long* errFormat, unsigned long long* alignedCount)
{
    // The warp's pair, compared in 64 bits (n * 32 threads may pass 2^32); below n it fits 32 bits.
    const uint64_t warp64 = uint64_t(blockIdx.x) * (kMgThreads / 32) + (threadIdx.x >> 5);
    const uint32_t lane = threadIdx.x & 31u;
    __shared__ uint32_t streaks[3][kMgThreads];
    uint32_t* sEnd = streaks[0] + (threadIdx.x & ~31u);
    uint32_t* s0 = streaks[1] + (threadIdx.x & ~31u);
    uint32_t* s1 = streaks[2] + (threadIdx.x & ~31u);
    if(warp64 >= n) return;                             // the whole warp
    const MgPair q = pairs[uint32_t(warp64)];
    const uint64_t b0 = toc[q.o0], n0 = toc[q.o0 + 1] - b0, r0 = toc[q.o0 ^ 1u];
    const uint64_t b1 = toc[q.o1], n1 = toc[q.o1 + 1] - b1, r1 = toc[q.o1 ^ 1u];
    const uint8_t* s = bytes + q.byteBegin;
    const uint64_t end = q.byteCount;
    uint64_t pos = 0, total = 0;
    uint32_t ord0 = 0, ord1 = 0;
    bool malformed = false;
    while(pos < end && !malformed) {                    // uniform: every lane parses the same bytes
        uint32_t my0 = 0, my1 = 0, myLen = 0;
        for(uint32_t k = 0; k < 32 && pos < end; k++) {
            int32_t skip0, skip1; uint32_t len;
            if(!decodeStreak(s, pos, end, skip0, skip1, len)) { malformed = true; break; }
            ord0 += uint32_t(skip0); ord1 += uint32_t(skip1);
            if(lane == k) { my0 = ord0; my1 = ord1; myLen = len; }
            ord0 += len - 1; ord1 += len - 1;
        }
        // An ordinal outside its oriented read would address another read's markers: the call fails, nothing is united.
        if(myLen && (uint64_t(my0) + myLen > n0 || uint64_t(my1) + myLen > n1)) { malformed = true; myLen = 0; }
        malformed = __any_sync(0xffffffffu, malformed);
        if(malformed) break;
        uint32_t inc = myLen;
#pragma unroll
        for(int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d); if(lane >= uint32_t(d)) inc += t; }
        const uint32_t T = __shfl_sync(0xffffffffu, inc, 31);
        total += T;
        // The group's streaks go to shared memory, so that the lanes run their unions without warp-wide operations.
        sEnd[lane] = inc; s0[lane] = my0; s1[lane] = my1;
        __syncwarp();
        // Flat index g: aligned pair g >> 1; bit 0 selects (m0, m1) or findReverseComplement of both (one unite site: two
        // inlined unions spill).
        for(uint32_t g = lane; g < 2 * T; g += 32) {
            const uint32_t f = g >> 1;
            uint32_t lo = 0;                            // the streak that holds f: the first with sEnd > f
#pragma unroll
            for(uint32_t step = 16; step; step >>= 1) if(sEnd[lo + step - 1] <= f) lo += step;
            const uint32_t i = f - (lo ? sEnd[lo - 1] : 0u);
            const uint32_t a0 = s0[lo] + i, a1 = s1[lo] + i;
            const uint64_t m0 = b0 + a0, m1 = b1 + a1;
            if(__ldg(kmerIds + m0) != __ldg(kmerIds + m1)) { atomicMin(errKmer, 2ull * q.pairIndex); continue; }
            const bool rc = g & 1u;
            unite(P, rc ? r0 + (n0 - 1 - a0) : m0, rc ? r1 + (n1 - 1 - a1) : m1);
        }
        __syncwarp();
    }
    if(lane == 0) {
        if(malformed) atomicMin(errFormat, 2ull * q.pairIndex);
        atomicAdd(alignedCount, (unsigned long long)total);
    }
}

// ---- sets, sizes, histogram ---------------------------------------------------------------------------------------
// Every slot gets its root. The walk does not halve: a halving store could land after the slot's own thread wrote the
// root and leave an inner node there. Each slot is written once, by its own thread, with its root.
__global__ void compressKernel(uint64_t* P, uint64_t M)
{
    for(uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < M; i += uint64_t(gridDim.x) * blockDim.x) {
        uint64_t r = __ldcg(P + i);
        if(r == i) continue;
        for(uint64_t q = __ldcg(P + r); q != r; q = __ldcg(P + r)) r = q;
        __stcg(P + i, r);
    }
}

__global__ void flagRootsKernel(uint64_t* P, uint64_t M)
{
    for(uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < M; i += uint64_t(gridDim.x) * blockDim.x)
        if(P[i] == i) P[i] = kRootFlag;
}

// Set sizes into the roots' slots (FLAG | size), and the largest size.
__global__ void countKernel(uint64_t* P, uint64_t M)
{
    for(uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < M; i += uint64_t(gridDim.x) * blockDim.x) {
        const uint64_t x = P[i];                        // non-root slots are not written by this kernel
        atomicAdd(reinterpret_cast<unsigned long long*>(P + ((x & kRootFlag) ? i : x)), 1ull);
    }
}

constexpr uint32_t kSmemBins = 1024;
__global__ void __launch_bounds__(kMgThreads) histogramKernel(const uint64_t* __restrict__ P, uint64_t M, unsigned long long* hist,
                                                              unsigned long long* maxSize)
{
    __shared__ unsigned long long bins[kSmemBins];
    for(uint32_t b = threadIdx.x; b < kSmemBins; b += blockDim.x) bins[b] = 0;
    __syncthreads();
    unsigned long long mx = 0;
    for(uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < M; i += uint64_t(gridDim.x) * blockDim.x) {
        const uint64_t x = P[i];
        if(!(x & kRootFlag)) continue;
        const uint64_t size = x & kValueMask;
        mx = max(mx, (unsigned long long)size);
        if(hist) {
            if(size < kSmemBins) atomicAdd(&bins[size], 1ull);
            else atomicAdd(hist + size, 1ull);
        }
    }
    if(!hist) {
        for(int d = 16; d; d >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
        if((threadIdx.x & 31u) == 0) atomicMax(maxSize, mx);
        return;
    }
    __syncthreads();
    for(uint32_t b = threadIdx.x; b < kSmemBins; b += blockDim.x) if(bins[b]) atomicAdd(hist + b, bins[b]);
}

// ---- first renumbering (:266-303): kept sets by a two-level scan over the roots ---------------------------------------
__device__ __forceinline__ bool keptRoot(uint64_t x, uint64_t minCoverage, uint64_t maxCoverage)
{
    if(!(x & kRootFlag)) return false;
    const uint64_t size = x & kValueMask;
    return size >= minCoverage && size <= maxCoverage;
}

__global__ void __launch_bounds__(kScanThreads) keptTileCountKernel(const uint64_t* __restrict__ P, uint64_t M, uint64_t minCoverage,
                                                                   uint64_t maxCoverage, uint64_t* __restrict__ tileCounts)
{
    __shared__ uint64_t smem[kScanThreads / 32];
    const uint64_t base = uint64_t(blockIdx.x) * kTile;
    uint64_t c = 0;
    for(uint32_t j = threadIdx.x; j < kTile; j += kScanThreads) {
        const uint64_t i = base + j;
        if(i < M && keptRoot(P[i], minCoverage, maxCoverage)) c++;
    }
    uint64_t total;
    blockExclusiveScan256<uint64_t>(c, total, smem);
    if(threadIdx.x == 0) tileCounts[blockIdx.x] = total;
}

// Root slots become FLAG | kept-set id, or kNoSet; setSize[k] = the size.
__global__ void __launch_bounds__(kScanThreads) keptTileWriteKernel(uint64_t* P, uint64_t M, uint64_t minCoverage, uint64_t maxCoverage,
                                                                   const uint64_t* __restrict__ tileOffsets, uint64_t* __restrict__ setSize)
{
    __shared__ uint64_t smem[kScanThreads / 32];
    const uint64_t base = uint64_t(blockIdx.x) * kTile;
    uint64_t running = tileOffsets[blockIdx.x];
    for(uint32_t j = 0; j < kTile; j += kScanThreads) {
        const uint64_t i = base + j + threadIdx.x;
        const uint64_t x = i < M ? P[i] : 0;
        const bool kept = i < M && keptRoot(x, minCoverage, maxCoverage);
        uint64_t total;
        const uint64_t ex = blockExclusiveScan256<uint64_t>(kept ? 1ull : 0ull, total, smem);
        if(kept) { setSize[running + ex] = x & kValueMask; P[i] = kRootFlag | (running + ex); }
        else if(i < M && (x & kRootFlag)) P[i] = kNoSet;
        running += total;
    }
}

// Non-root slots take their root's value (the root slots are not written here).
__global__ void relabelKernel(uint64_t* P, uint64_t M)
{
    for(uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < M; i += uint64_t(gridDim.x) * blockDim.x) {
        const uint64_t x = P[i];
        if(!(x & kRootFlag)) P[i] = P[x];
    }
}

// ---- gathering (:324-345) -----------------------------------------------------------------------------------------
// One warp per oriented read: every kept marker goes to its set's segment as the key (orientedReadId << 32 | ordinal),
// whose order is marker-id order. The position inside the segment comes from an atomic: the segments are sorted next.
__global__ void __launch_bounds__(kMgThreads) scatterKernel(const uint64_t* __restrict__ P, const uint64_t* __restrict__ toc, uint32_t rows,
                                                            const uint64_t* __restrict__ setOffset, uint32_t* cursor, uint64_t* __restrict__ keys)
{
    const uint64_t o = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(o >= rows) return;
    const uint64_t b = toc[o], e = toc[o + 1];
    for(uint64_t i = b + lane; i < e; i += 32) {
        const uint64_t x = P[i];
        if(x == kNoSet) continue;
        const uint64_t k = x & kValueMask;
        const uint32_t slot = atomicAdd(cursor + k, 1u);
        keys[setOffset[k] + slot] = (uint64_t(o) << 32) | uint32_t(i - b);
    }
}

// ---- bad sets (:697-745) ------------------------------------------------------------------------------------------
// One warp per kept set (its keys sorted). Markers of one read are contiguous in marker-id order (both strands, 2r and
// 2r+1), so "two consecutive markers on the same read" is "two consecutive keys with the same readId".
__global__ void __launch_bounds__(kMgThreads) badSetKernel(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ setOffset,
                                                           const uint64_t* __restrict__ setSize, uint64_t setCount, uint64_t minCoveragePerStrand,
                                                           bool allowDuplicateMarkers, uint64_t* __restrict__ good, uint64_t* __restrict__ goodSize)
{
    const uint64_t k = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(k >= setCount) return;
    const uint64_t n = setSize[k], off = setOffset[k];
    bool bad;
    if(n == 1) {
        bad = 1 < minCoveragePerStrand;                  // the reference's singleton rule, kept as it is
    } else {
        uint64_t c1 = 0;
        bool dup = false;
        uint32_t carry = 0xffffffffu;                    // read of the last key of the previous group of 32
        for(uint64_t j0 = 0; j0 < n; j0 += 32) {
            const uint64_t j = j0 + lane;
            const uint32_t o = j < n ? uint32_t(keys[off + j] >> 32) : 0xffffffffu;
            const uint32_t read = o >> 1;
            uint32_t prev = __shfl_up_sync(0xffffffffu, read, 1);
            if(lane == 0) prev = carry;
            if(j < n && read == prev) dup = true;
            c1 += __popc(__ballot_sync(0xffffffffu, j < n && (o & 1u)));
            carry = __shfl_sync(0xffffffffu, read, 31);
        }
        dup = __any_sync(0xffffffffu, dup);
        bad = (!allowDuplicateMarkers && dup) || (n - c1) < minCoveragePerStrand || c1 < minCoveragePerStrand;
    }
    if(lane == 0) { good[k] = bad ? 0 : 1; goodSize[k] = bad ? 0 : n; }
}

// ---- output ----------------------------------------------------------------------------------------------------------
// One warp per kept set: good sets write their marker ids at goodOffset[k] and their toc entry at vertexId[k].
__global__ void __launch_bounds__(kMgThreads) vertexDataKernel(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ setOffset,
                                                               const uint64_t* __restrict__ setSize, uint64_t setCount,
                                                               const uint64_t* __restrict__ goodFlag, const uint64_t* __restrict__ vertexId,
                                                               const uint64_t* __restrict__ goodOffset, const uint64_t* __restrict__ toc,
                                                               uint64_t* __restrict__ data, uint64_t* __restrict__ vtoc)
{
    const uint64_t k = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(k >= setCount || !goodFlag[k]) return;
    const uint64_t n = setSize[k], off = setOffset[k], out = goodOffset[k];
    for(uint64_t j = lane; j < n; j += 32) {
        const uint64_t key = keys[off + j];
        data[out + j] = toc[key >> 32] + (key & 0xffffffffu);
    }
    if(lane == 0) vtoc[vertexId[k]] = out;
}

__global__ void vertexTableKernel(const uint64_t* __restrict__ P, uint64_t begin, uint64_t n, const uint64_t* __restrict__ goodFlag,
                                  const uint64_t* __restrict__ vertexId, uint8_t* __restrict__ out)
{
    for(uint64_t j = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; j < n; j += uint64_t(gridDim.x) * blockDim.x) {
        const uint64_t x = P[begin + j];
        uint64_t v = kInvalid40;
        if(x != kNoSet) {
            const uint64_t k = x & kValueMask;
            if(goodFlag[k]) v = vertexId[k];
        }
        store40(out + 5 * j, v);
    }
}

__global__ void toc40Kernel(const uint64_t* __restrict__ in, uint64_t n, uint8_t* __restrict__ out)
{
    for(uint64_t j = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; j < n; j += uint64_t(gridDim.x) * blockDim.x) store40(out + 5 * j, in[j]);
}

// ---- reverse complement vertices (:1177-1230) -------------------------------------------------------------------------
__global__ void rcVertexKernel(const uint8_t* __restrict__ table, const uint64_t* __restrict__ vtoc, const uint64_t* __restrict__ data,
                               uint64_t V, const uint64_t* __restrict__ toc, uint32_t rows, uint64_t M, uint64_t* __restrict__ rc,
                               unsigned long long* errMarker, unsigned long long* errVertex)
{
    for(uint64_t v = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; v < V; v += uint64_t(gridDim.x) * blockDim.x) {
        uint64_t r = kInvalid40;
        for(uint64_t j = vtoc[v]; j < vtoc[v + 1]; j++) {
            const uint64_t m = data[j];
            if(m >= M) { atomicMin(errMarker, (unsigned long long)v); break; }
            const uint64_t t = load40(table + 5 * reverseComplementMarker(toc, rows, m));
            if(j == vtoc[v]) r = t;
            if(t == kInvalid40 || t >= V || t != r) { atomicMin(errVertex, (unsigned long long)v); break; }
        }
        rc[v] = r;
    }
}

__global__ void rcInvolutionKernel(const uint64_t* __restrict__ rc, uint64_t V, unsigned long long* errVertex)
{
    for(uint64_t v = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; v < V; v += uint64_t(gridDim.x) * blockDim.x) {
        const uint64_t r = rc[v];
        if(r >= V || rc[r] != v) atomicMin(errVertex, (unsigned long long)v);
    }
}

} // namespace

// PeakFinder::findPeaks + findXCutoff (src/PeakFinder.cpp:23-198). Returns true where the reference throws
// PeakFinderException (observed = its observedPercentArea); otherwise *cutoff is the value it returns. An empty histogram
// (no markers) is undefined in the reference (findPeaks reads peaks[0] of an empty vector); here it counts as a throw with
// observed area 0.
bool peakFinderCutoff(const uint64_t* y, uint64_t n, double minAreaFraction, uint64_t startIndex, uint64_t* cutoff, double* observed)
{
    *observed = 0;
    if(n == 0) return true;
    struct Peak { uint64_t start, stop, left, right; bool isMerged; uint64_t persistence; };
    std::vector<int64_t> peakIndex(n, -1);
    std::vector<uint64_t> indexes(n);
    std::iota(indexes.begin(), indexes.end(), 0);
    // A total order (equal y: lower x first), so any sort gives the reference's sequence.
    std::sort(indexes.begin(), indexes.end(), [&](uint64_t a, uint64_t b) { return y[a] == y[b] ? a < b : y[a] > y[b]; });
    std::vector<Peak> peaks;
    for(const uint64_t i : indexes) {
        const bool hasLeftPeak = i > 0 && peakIndex[i - 1] >= 0;
        const bool hasRightPeak = i < n - 1 && peakIndex[i + 1] >= 0;
        if(!hasLeftPeak && !hasRightPeak) {
            peaks.push_back(Peak{i, 0, i, i, false, 0});
            peakIndex[i] = int64_t(peaks.size() - 1);
        } else if(hasLeftPeak && !hasRightPeak) {
            peaks[size_t(peakIndex[i - 1])].right = i;
            peakIndex[i] = peakIndex[i - 1];
        } else if(!hasLeftPeak && hasRightPeak) {
            peaks[size_t(peakIndex[i + 1])].left = i;
            peakIndex[i] = peakIndex[i + 1];
        } else {
            Peak& leftPeak = peaks[size_t(peakIndex[i - 1])];
            Peak& rightPeak = peaks[size_t(peakIndex[i + 1])];
            if(y[rightPeak.start] > y[leftPeak.start]) {
                rightPeak.left = leftPeak.left;
                peakIndex[i] = peakIndex[i + 1];
                leftPeak.right = i;
                peakIndex[leftPeak.left] = peakIndex[i + 1];
                peakIndex[leftPeak.right] = peakIndex[i + 1];
                leftPeak.stop = i;
                leftPeak.isMerged = true;
                leftPeak.persistence = y[rightPeak.start] - y[i];      // sic: the surviving peak's height (:104)
            } else {
                leftPeak.right = rightPeak.right;
                peakIndex[i] = peakIndex[i - 1];
                rightPeak.left = i;
                peakIndex[rightPeak.right] = peakIndex[i - 1];
                peakIndex[rightPeak.left] = peakIndex[i - 1];
                rightPeak.stop = i;
                rightPeak.isMerged = true;
                rightPeak.persistence = y[rightPeak.start] - y[i];
            }
        }
    }
    peaks[0].persistence = y[peaks[0].start];
    if(peaks.size() < 2) return true;
    // Starts are distinct: a total order again.
    std::sort(peaks.begin(), peaks.end(), [](const Peak& a, const Peak& b) {
        return a.persistence == b.persistence ? a.start < b.start : a.persistence > b.persistence; });
    uint64_t leftBound, rightBound;
    if(peaks[1].start < peaks[0].start) { leftBound = peaks[1].right; rightBound = peaks[0].right; }
    else { leftBound = peaks[1].left; rightBound = peaks[1].right; }
    auto area = [&](uint64_t xMin, uint64_t xMax) { uint64_t t = 0; for(uint64_t i = xMin; i <= xMax; i++) t += y[i]; return t; };
    const uint64_t totalArea = area(startIndex, n - 1);
    const uint64_t peakArea = area(leftBound, rightBound);
    const double areaFraction = double(peakArea) / double(totalArea);
    if(areaFraction > minAreaFraction) { *cutoff = leftBound; return false; }
    *observed = areaFraction;
    return true;
}

void createMarkerGraphVertices(shb_context* c, const shb_marker_graph_params& p, const uint32_t* edges, uint64_t edgeCount,
                               const uint64_t* ctoc, const uint8_t* cdata, uint64_t alignmentCount, const uint8_t* readFlags,
                               uint8_t** vertexTableOut, uint8_t** verticesTocOut, uint64_t** verticesDataOut, uint64_t** histogramOut,
                               shb_marker_graph_result* result)
{
    SHB_CUDA(cudaSetDevice(c->device));
    requireWholeAssembly(c, "createMarkerGraphVertices");
    const auto t0 = std::chrono::steady_clock::now();
    const uint64_t launches0 = g_launchCount;
    cudaStream_t st = c->stream;
    const uint64_t M = c->localMarkerCount, R = c->readCountTotal;
    const uint32_t rows = uint32_t(2 * R);
    const std::vector<uint64_t>& toc = c->tocHost;
    SHB_REQUIRE(R < (1ull << 31), SHB_ERR_INVALID, "Too many reads.");
    // 2^34 markers need 128 GiB for the parent array alone; the bound keeps every per-set launch within 2^31 blocks.
    SHB_REQUIRE(M < (1ull << 34), SHB_ERR_INVALID, "More than 2^34 markers.");
    SHB_REQUIRE(edgeCount % 2 == 0, SHB_ERR_INVALID, "The read graph has an odd number of edges.");
    SHB_REQUIRE(edgeCount < (1ull << 33), SHB_ERR_INVALID, "More than 2^33 read graph edges.");

    // Edge pairs (:544-586), in edge order, checked on the host as the reference asserts them.
    shb_marker_graph_result res{};
    res.markerCount = M;
    std::vector<MgPair> pairs;
    for(uint64_t i = 0; i < edgeCount; i += 2) {
        const uint32_t* e = edges + 4 * i;
        const uint32_t* f = edges + 4 * (i + 1);
        SHB_REQUIRE((f[0] ^ 1u) == e[0] && (f[1] ^ 1u) == e[1], SHB_ERR_INVALID,
                    "Read graph edge " + std::to_string(i + 1) + " is not the reverse complement of edge " + std::to_string(i) + ".");
        if(e[3] >> 30) { res.edgePairsSkipped++; continue; }          // crossesStrands (bit 62), hasInconsistentAlignment (bit 63)
        SHB_REQUIRE(e[0] < e[1], SHB_ERR_INVALID, "Read graph edge " + std::to_string(i) + ": orientedReadIds[0] >= orientedReadIds[1].");
        SHB_REQUIRE(e[1] < rows, SHB_ERR_INVALID, "Read graph edge " + std::to_string(i) + " refers to a read that does not exist.");
        if((readFlags[e[0] >> 1] | readFlags[e[1] >> 1]) & 2u) { res.edgePairsSkipped++; continue; }  // isChimeric
        const uint64_t a = uint64_t(e[2]) | (uint64_t(e[3] & 0x3fffffffu) << 32);
        SHB_REQUIRE(a < alignmentCount, SHB_ERR_INVALID, "Read graph edge " + std::to_string(i) + ": alignmentId out of range.");
        SHB_REQUIRE(ctoc[a] <= ctoc[a + 1] && ctoc[a + 1] - ctoc[a] < (1ull << 32), SHB_ERR_INVALID, "Invalid compressed alignment toc.");
        for(const uint32_t o : {e[0], e[1]})
            SHB_REQUIRE(toc[o + 1] - toc[o] == toc[(o ^ 1u) + 1] - toc[o ^ 1u], SHB_ERR_INVALID,
                        "The two strands of a read have different marker counts.");
        pairs.push_back(MgPair{ctoc[a], uint32_t(ctoc[a + 1] - ctoc[a]), e[0], e[1], uint32_t(i / 2)});
    }
    res.edgePairsUsed = pairs.size();

    Footprint fp;
    DeviceBuffer<uint64_t> P;
    fp.add(P, M + 1);
    EventTimer timer;
    timer.start(st);
    if(M) SHB_LAUNCH(initParentKernel, gridFor(M), kMgThreads, 0, st, P.get(), M);

    // Union, in batches of edge pairs (SHB_MARKERGRAPH_PAIR_BATCH, SHB_MARKERGRAPH_BATCH_BYTES: test hooks).
    unsigned long long* scal = c->scalar(kSlotMarkerGraphVertices);    // errKmer, errFormat, alignedCount, maxSize, scan total, bigCount
    const unsigned long long init[6] = {~0ull, ~0ull, 0, 0, 0, 0};
    SHB_CUDA(cudaMemcpyAsync(scal, init, sizeof(init), cudaMemcpyHostToDevice, st));
    {
        const uint64_t pairLimit = envCount("SHB_MARKERGRAPH_PAIR_BATCH", 1u << 22);
        const uint64_t byteBudget = envCount("SHB_MARKERGRAPH_BATCH_BYTES", 1u << 30);
        DeviceBuffer<uint8_t> dBytes;
        DeviceBuffer<MgPair> dPairs;
        std::vector<uint8_t> gather;
        std::vector<MgPair> batch;
        for(uint64_t begin = 0; begin < pairs.size(); ) {
            uint64_t end = begin, bytes = 0, lo = ~0ull, hi = 0;
            while(end < pairs.size() && end - begin < pairLimit && (end == begin || bytes + pairs[end].byteCount <= byteBudget)) {
                bytes += pairs[end].byteCount;
                lo = std::min(lo, pairs[end].byteBegin); hi = std::max(hi, pairs[end].byteBegin + pairs[end].byteCount);
                end++;
            }
            batch.assign(pairs.begin() + begin, pairs.begin() + end);
            const uint8_t* src;
            uint64_t uploadBytes;
            if(hi - lo <= std::max(bytes, byteBudget)) {     // dense (alignment order): upload the span as it lies
                for(MgPair& q : batch) q.byteBegin -= lo;
                src = cdata + lo; uploadBytes = hi - lo;
            } else {                                         // scattered: gather the batch's alignments
                gather.resize(bytes);
                uint64_t w = 0;
                for(MgPair& q : batch) { memcpy(gather.data() + w, cdata + q.byteBegin, q.byteCount); q.byteBegin = w; w += q.byteCount; }
                src = gather.data(); uploadBytes = bytes;
            }
            fp.add(dBytes, uploadBytes + 16); fp.add(dPairs, batch.size());     // slack: decodeStreak reads whole words
            SHB_CUDA(cudaMemcpyAsync(dBytes.get(), src, uploadBytes, cudaMemcpyHostToDevice, st));
            SHB_CUDA(cudaMemcpyAsync(dPairs.get(), batch.data(), batch.size() * sizeof(MgPair), cudaMemcpyHostToDevice, st));
            SHB_LAUNCH(uniteKernel, ceilDiv(batch.size() * 32, kMgThreads), kMgThreads, 0, st, dPairs.get(), uint32_t(batch.size()),
                       dBytes.get(), (const uint64_t*)c->toc.get(), c->kmerIds, P.get(), scal, scal + 1, scal + 2);
            SHB_CUDA(cudaStreamSynchronize(st));            // the host buffers are reused by the next batch
            begin = end;
        }
        fp.drop(dBytes); fp.drop(dPairs);
    }
    // Read on the call's stream, after its last union kernel and after the reset of the counters (even without any pair).
    unsigned long long s5[3];
    SHB_CUDA(cudaMemcpyAsync(s5, scal, sizeof(s5), cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaStreamSynchronize(st));
    SHB_REQUIRE(s5[1] == ~0ull, SHB_ERR_INVALID, "The compressed alignment of read graph edge " + std::to_string(s5[1]) +
                " is malformed or has an ordinal outside its oriented read.");
    SHB_REQUIRE(s5[0] == ~0ull, SHB_ERR_INVALID, "Read graph edge " + std::to_string(s5[0]) +
                ": aligned markers have different k-mer ids.");
    res.alignedMarkerPairs = s5[2];

    // Sets and their sizes (:128-231).
    if(M) {
        SHB_LAUNCH(compressKernel, gridFor(M), kMgThreads, 0, st, P.get(), M);
        SHB_LAUNCH(flagRootsKernel, gridFor(M), kMgThreads, 0, st, P.get(), M);
        SHB_LAUNCH(countKernel, gridFor(M), kMgThreads, 0, st, P.get(), M);
        SHB_LAUNCH(histogramKernel, gridFor(M), kMgThreads, 0, st, (const uint64_t*)P.get(), M, (unsigned long long*)nullptr, scal + 3);
    }
    const uint64_t maxSize = readBack(scal + 3, st);
    const uint64_t histSize = M ? maxSize + 1 : 0;
    HostResult histBlock(allocHostResult(8 * histSize + 8));
    SHB_REQUIRE(histBlock.p, SHB_ERR_OOM, "Out of host memory for the histogram.");
    uint64_t* hist = static_cast<uint64_t*>(histBlock.p);
    if(M) {
        DeviceBuffer<unsigned long long> dHist;
        fp.add(dHist, histSize);
        SHB_CUDA(cudaMemsetAsync(dHist.get(), 0, 8 * histSize, st));
        SHB_LAUNCH(histogramKernel, gridFor(M), kMgThreads, 0, st, (const uint64_t*)P.get(), M, dHist.get(), scal + 3);
        SHB_CUDA(cudaMemcpyAsync(hist, dHist.get(), 8 * histSize, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        fp.drop(dHist);
    }
    for(uint64_t s = 0; s < histSize; s++) res.disjointSetCount += hist[s];

    // minCoverage (:233-254).
    uint64_t minCoverage = p.minCoverage;
    if(minCoverage == 0) {
        uint64_t cutoff = 0;
        double observed = 0;
        if(peakFinderCutoff(hist, histSize, p.peakFinderMinAreaFraction, p.peakFinderAreaStartIndex, &cutoff, &observed)) {
            minCoverage = 5;
            res.peakFinderFailed = 1;
            res.peakFinderObservedAreaFraction = observed;
        } else {
            minCoverage = cutoff;
        }
    }
    res.minCoverageUsed = minCoverage;
    // A kept set's markers are counted into a 32-bit cursor when they are gathered, and its sort takes fewer than 2^32 keys.
    for(uint64_t s = std::max<uint64_t>(minCoverage, 1ull << 32); s < histSize && s <= p.maxCoverage; s++)
        SHB_REQUIRE(hist[s] == 0, SHB_ERR_INVALID, "A disjoint set of 2^32 or more markers would be kept (maxCoverage allows it).");

    // Kept sets, numbered in root order (:266-303).
    const uint64_t tiles = (M + kTile - 1) / kTile;
    DeviceBuffer<uint64_t> tileOffsets, scanWs, setSize, setOffset;
    uint64_t* total = reinterpret_cast<uint64_t*>(scal + 4);
    uint64_t keptSets = 0;
    if(M) {
        fp.add(tileOffsets, tiles + 1); fp.add(scanWs, scanWorkspaceElements(tiles) + 1);
        SHB_LAUNCH(keptTileCountKernel, unsigned(tiles), kScanThreads, 0, st, (const uint64_t*)P.get(), M, minCoverage, p.maxCoverage, tileOffsets.get());
        exclusiveScan<uint64_t>(tileOffsets.get(), tileOffsets.get(), tiles, total, scanWs.get(), st);
        keptSets = readBack(total, st);
        fp.add(setSize, keptSets + 1);
        SHB_LAUNCH(keptTileWriteKernel, unsigned(tiles), kScanThreads, 0, st, P.get(), M, minCoverage, p.maxCoverage,
                   (const uint64_t*)tileOffsets.get(), setSize.get());
        SHB_LAUNCH(relabelKernel, gridFor(M), kMgThreads, 0, st, P.get(), M);
        fp.drop(tileOffsets);
    }
    res.keptDisjointSetCount = keptSets;

    // Markers of each kept set, sorted (:324-345).
    uint64_t keptMarkers = 0;
    DeviceBuffer<uint64_t> keys, good, goodSize, bigSets, sortTmp;
    DeviceBuffer<uint32_t> cursor;
    if(keptSets) {
        fp.add(setOffset, keptSets + 1); fp.add(scanWs, scanWorkspaceElements(keptSets) + 1);
        exclusiveScan<uint64_t>(setSize.get(), setOffset.get(), keptSets, total, scanWs.get(), st);
        keptMarkers = readBack(total, st);
        fp.add(cursor, keptSets);
        SHB_CUDA(cudaMemsetAsync(cursor.get(), 0, 4 * keptSets, st));
        fp.add(keys, keptMarkers + 1);
        SHB_LAUNCH(scatterKernel, ceilDiv(uint64_t(rows) * 32, kMgThreads), kMgThreads, 0, st, (const uint64_t*)P.get(),
                   (const uint64_t*)c->toc.get(), rows, (const uint64_t*)setOffset.get(), cursor.get(), keys.get());
        fp.drop(cursor);
        fp.add(bigSets, keptSets);
        SHB_LAUNCH(warpSortKernel, ceilDiv(keptSets * 32, kMgThreads), kMgThreads, 0, st, keys.get(), (const uint64_t*)setOffset.get(),
                   (const uint64_t*)setSize.get(), keptSets, bigSets.get(), scal + 5);
        const uint64_t bigCount = readBack(scal + 5, st);
        if(bigCount) {
            // The listed sets in a fixed order (the list's order comes from atomics), split by size.
            std::vector<uint64_t> big(bigCount), sizes(keptSets), offsets(keptSets);
            SHB_CUDA(cudaMemcpyAsync(big.data(), bigSets.get(), 8 * bigCount, cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaMemcpyAsync(sizes.data(), setSize.get(), 8 * keptSets, cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaMemcpyAsync(offsets.data(), setOffset.get(), 8 * keptSets, cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaStreamSynchronize(st));
            std::vector<uint64_t> medium;
            // The radix sort's workspace belongs to the context; what it grows by here counts towards this call's peak.
            auto sortWsBytes = [&] { return 8 * (c->sortWs.hist.capacity() + c->sortWs.status.capacity()); };
            const uint64_t sortWs0 = sortWsBytes();
            for(const uint64_t k : big) {
                if(sizes[k] <= kBlockSortMax) { medium.push_back(k); continue; }
                fp.add(sortTmp, sizes[k]);                   // sizes[k] < 2^32: checked on the histogram
                const int ranges[2][2] = {{0, 32}, {32, 64}};
                if(radixSort<false>(keys.get() + offsets[k], sortTmp.get(), nullptr, nullptr, sizes[k], ranges, 2, c->sortWs, st))
                    SHB_CUDA(cudaMemcpyAsync(keys.get() + offsets[k], sortTmp.get(), 8 * sizes[k], cudaMemcpyDeviceToDevice, st));
                fp.peak = std::max(fp.peak, fp.live + (sortWsBytes() - sortWs0));
            }
            if(!medium.empty()) {
                SHB_CUDA(cudaMemcpyAsync(bigSets.get(), medium.data(), 8 * medium.size(), cudaMemcpyHostToDevice, st));
                SHB_LAUNCH(blockSortKernel, unsigned(medium.size()), kMgThreads, 0, st, keys.get(), (const uint64_t*)setOffset.get(),
                           (const uint64_t*)setSize.get(), (const uint64_t*)bigSets.get());
            }
            SHB_CUDA(cudaStreamSynchronize(st));
            fp.drop(sortTmp);
        }
        fp.drop(bigSets);

        // Bad sets (:371-410), then the second renumbering.
        fp.add(good, keptSets + 1); fp.add(goodSize, keptSets + 1);
        SHB_LAUNCH(badSetKernel, ceilDiv(keptSets * 32, kMgThreads), kMgThreads, 0, st, (const uint64_t*)keys.get(),
                   (const uint64_t*)setOffset.get(), (const uint64_t*)setSize.get(), keptSets, p.minCoveragePerStrand,
                   p.allowDuplicateMarkers != 0, good.get(), goodSize.get());
    }

    // Vertices (:423-464): ids and offsets by scans over the kept sets, in place.
    uint64_t V = 0, vertexMarkers = 0;
    DeviceBuffer<uint64_t> vertexId, data, vtoc;
    if(keptSets) {
        fp.add(vertexId, keptSets + 1);
        exclusiveScan<uint64_t>(good.get(), vertexId.get(), keptSets, total, scanWs.get(), st);
        SHB_CUDA(cudaMemcpyAsync(&V, total, 8, cudaMemcpyDeviceToHost, st));
        exclusiveScan<uint64_t>(goodSize.get(), goodSize.get(), keptSets, total, scanWs.get(), st);
        SHB_CUDA(cudaMemcpyAsync(&vertexMarkers, total, 8, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        fp.add(data, vertexMarkers + 1); fp.add(vtoc, V + 1);
        SHB_LAUNCH(vertexDataKernel, ceilDiv(keptSets * 32, kMgThreads), kMgThreads, 0, st, (const uint64_t*)keys.get(),
                   (const uint64_t*)setOffset.get(), (const uint64_t*)setSize.get(), keptSets, (const uint64_t*)good.get(),
                   (const uint64_t*)vertexId.get(), (const uint64_t*)goodSize.get(), (const uint64_t*)c->toc.get(), data.get(), vtoc.get());
        SHB_CUDA(cudaMemcpyAsync(vtoc.get() + V, &vertexMarkers, 8, cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        fp.drop(keys); fp.drop(goodSize); fp.drop(setOffset); fp.drop(setSize); fp.drop(scanWs);
    }
    res.vertexCount = V;
    res.badDisjointSetCount = keptSets - V;

    // Host outputs: MarkerGraphVertexTable (Uint40 per marker), MarkerGraphVertices toc (Uint40) and data (uint64).
    HostResult tableBlock(allocHostResult(5 * M + 8)), toc5Block(allocHostResult(5 * (V + 1) + 8)),
               vdataBlock(allocHostResult(8 * vertexMarkers + 8));
    SHB_REQUIRE(tableBlock.p && toc5Block.p && vdataBlock.p, SHB_ERR_OOM, "Out of host memory for the marker graph vertices.");
    uint8_t* table = static_cast<uint8_t*>(tableBlock.p);
    uint8_t* toc5 = static_cast<uint8_t*>(toc5Block.p);
    DeviceBuffer<uint8_t> stage;
    if(V) {
        fp.add(stage, 5 * (V + 1));
        SHB_LAUNCH(toc40Kernel, gridFor(V + 1), kMgThreads, 0, st, (const uint64_t*)vtoc.get(), V + 1, stage.get());
        SHB_CUDA(cudaMemcpyAsync(toc5, stage.get(), 5 * (V + 1), cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaMemcpyAsync(vdataBlock.p, data.get(), 8 * vertexMarkers, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
    } else {
        memset(toc5, 0, 5);
    }
    fp.drop(vtoc); fp.drop(data);
    if(M) {
        // In chunks of SHB_MARKERGRAPH_TABLE_CHUNK markers (test hook).
        const uint64_t chunk = std::min<uint64_t>(M, envCount("SHB_MARKERGRAPH_TABLE_CHUNK", 1u << 28));
        fp.add(stage, 5 * chunk);
        if(!keptSets) { fp.add(good, 1); fp.add(vertexId, 1); }
        for(uint64_t b = 0; b < M; b += chunk) {
            const uint64_t n = std::min(chunk, M - b);
            SHB_LAUNCH(vertexTableKernel, gridFor(n), kMgThreads, 0, st, (const uint64_t*)P.get(), b, n, (const uint64_t*)good.get(),
                       (const uint64_t*)vertexId.get(), stage.get());
            SHB_CUDA(cudaMemcpyAsync(table + 5 * b, stage.get(), 5 * n, cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaStreamSynchronize(st));
        }
    }
    timer.stop(st);
    SHB_CUDA(cudaEventSynchronize(timer.stopEvent));
    const float ms = timer.elapsedMs();

    *vertexTableOut = static_cast<uint8_t*>(tableBlock.take()); *verticesTocOut = static_cast<uint8_t*>(toc5Block.take());
    *verticesDataOut = static_cast<uint64_t*>(vdataBlock.take()); *histogramOut = static_cast<uint64_t*>(histBlock.take());
    if(result) {
        res.histogramSize = histSize;
        res.peakDeviceBytes = fp.peak;
        res.deviceMs = ms;
        res.totalMs = msSince(t0);
        res.kernelLaunches = g_launchCount - launches0;
        *result = res;
    }
}

void findMarkerGraphReverseComplementVertices(shb_context* c, const uint8_t* table5, const uint8_t* toc5, const uint64_t* vdata,
                                              uint64_t V, uint64_t** rcOut)
{
    SHB_CUDA(cudaSetDevice(c->device));
    requireWholeAssembly(c, "findMarkerGraphReverseComplementVertices");
    cudaStream_t st = c->stream;
    const uint64_t M = c->localMarkerCount;
    const uint32_t rows = uint32_t(2 * c->readCountTotal);
    std::vector<uint64_t> vtoc(V + 1);
    for(uint64_t v = 0; v <= V; v++) {
        uint64_t x = 0;
        for(int b = 0; b < 5; b++) x |= uint64_t(toc5[5 * v + b]) << (8 * b);
        vtoc[v] = x;
        SHB_REQUIRE(v == 0 ? x == 0 : x > vtoc[v - 1], SHB_ERR_INVALID,
                    "The marker graph vertices toc is not increasing (a vertex without markers).");
    }
    const uint64_t n = vtoc[V];
    for(uint64_t o = 0; o < rows; o += 2)
        SHB_REQUIRE(c->tocHost[o + 1] - c->tocHost[o] == c->tocHost[o + 2] - c->tocHost[o + 1], SHB_ERR_INVALID,
                    "The two strands of a read have different marker counts.");
    HostResult out(allocHostResult(8 * V + 8));
    SHB_REQUIRE(out.p, SHB_ERR_OOM, "Out of host memory for the reverse complement vertices.");
    if(V) {
        DeviceBuffer<uint8_t> dTable;
        DeviceBuffer<uint64_t> dToc, dData, dRc;
        dTable.reserve(5 * M + 8); dToc.reserve(V + 1); dData.reserve(n); dRc.reserve(V);
        SHB_CUDA(cudaMemcpyAsync(dTable.get(), table5, 5 * M, cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(dToc.get(), vtoc.data(), 8 * (V + 1), cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(dData.get(), vdata, 8 * n, cudaMemcpyHostToDevice, st));
        unsigned long long* err = c->scalar(kSlotMarkerGraphRcErrors);
        const unsigned long long init[2] = {~0ull, ~0ull};
        SHB_CUDA(cudaMemcpyAsync(err, init, sizeof(init), cudaMemcpyHostToDevice, st));
        SHB_LAUNCH(rcVertexKernel, gridFor(V), kMgThreads, 0, st, (const uint8_t*)dTable.get(), (const uint64_t*)dToc.get(),
                   (const uint64_t*)dData.get(), V, (const uint64_t*)c->toc.get(), rows, M, dRc.get(), err, err + 1);
        unsigned long long e[2];
        SHB_CUDA(cudaMemcpyAsync(e, err, sizeof(e), cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        SHB_REQUIRE(e[0] == ~0ull, SHB_ERR_INVALID, "Marker graph vertex " + std::to_string(e[0]) + " has a marker id out of range.");
        SHB_REQUIRE(e[1] == ~0ull, SHB_ERR_INVALID, "The reverse complemented markers of marker graph vertex " + std::to_string(e[1]) +
                    " are not all on one vertex.");
        SHB_LAUNCH(rcInvolutionKernel, gridFor(V), kMgThreads, 0, st, (const uint64_t*)dRc.get(), V, err + 1);
        SHB_CUDA(cudaMemcpyAsync(e, err, sizeof(e), cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaMemcpyAsync(out.p, dRc.get(), 8 * V, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        SHB_REQUIRE(e[1] == ~0ull, SHB_ERR_INVALID, "The reverse complement of the reverse complement of marker graph vertex " +
                    std::to_string(e[1]) + " is not the vertex itself.");
    }
    *rcOut = static_cast<uint64_t*>(out.take());
}

} // namespace shb
