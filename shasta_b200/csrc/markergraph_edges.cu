// Assembler::createMarkerGraphEdges (src/AssemblerMarkerGraph.cpp:2028-2085, worker :2116-2180, children :1025-1080),
// createMarkerGraphEdgesBySourceAndTarget (:2089-2112, :2192-2213) and findMarkerGraphReverseComplementEdges (:1244-1389)
// on the GPU. The output is the reference's run with one thread:
//   * every marker of a vertex gets its successor: the next marker of its oriented read that is on a vertex. One warp per
//     source vertex, one lane per marker, walks up to kShortWalk markers; longer gaps go to a list that one warp per marker
//     scans 32 markers at a time, so a read with vertices only at its two ends does not serialise a warp;
//   * each vertex's markers are sorted stably by successor vertex with the segmented sorters of the vertex stage (registers up
//     to 32, one block in shared memory up to 4096, radixSort above). The markers of a vertex are in increasing marker id,
//     which is (orientedReadId, ordinal0) order, so each run of one target holds its MarkerIntervals in sorted order, and the
//     runs come out in increasing target: edges are numbered in increasing (source, target);
//   * source vertices are processed in chunks under a byte budget; each chunk's edges, intervals and edgesBySource row
//     (the vertex's edge range, reversed) go to the host before the next chunk;
//   * edgesByTarget: the counts per target are scanned into its toc, then the edges are sorted by target in chunks of edge
//     ids (radixSort, stable) and every edge takes the slot toc[t+1]-1-rank, so each row is in decreasing edge id.
#include "context.cuh"
#include "hostpool.cuh"
#include "markergraph_kernels.cuh"

#include "../../include/shb_marker_graph_edges.h"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace shb {
namespace {

constexpr uint32_t kShortWalk = 16;                   // markers a lane walks before its marker goes to the long-walk list
constexpr uint32_t kSmallKeyBits = 12;                // segments up to kBlockSortMax: key = target << 12 | position
constexpr uint32_t kEdgeBytes = 14;                   // sizeof(MarkerGraph::Edge)

struct Interval { uint32_t o, a0, a1; };              // MarkerInterval: orientedReadId, ordinals[2]

__device__ __forceinline__ bool ivLess(const Interval& x, const Interval& y)
{
    return x.o != y.o ? x.o < y.o : x.a0 != y.a0 ? x.a0 < y.a0 : x.a1 < y.a1;
}
__device__ __forceinline__ bool ivEqual(const Interval& x, const Interval& y) { return x.o == y.o && x.a0 == y.a0 && x.a1 == y.a1; }
__device__ __forceinline__ Interval loadIv(const uint32_t* p, uint64_t k) { return Interval{p[3 * k], p[3 * k + 1], p[3 * k + 2]}; }

// ---- successors (:1032-1051) -----------------------------------------------------------------------------------------
// One warp per source vertex of the chunk. targets[i] receives the successor's vertex (kInvalid40: none), iv[i] the interval.
__global__ void __launch_bounds__(kMgThreads) successorKernel(const uint64_t* __restrict__ markers, const uint64_t* __restrict__ segOff,
                                                              uint64_t segCount, const uint8_t* __restrict__ table, uint64_t M, uint64_t V,
                                                              const uint64_t* __restrict__ toc, uint32_t rows, uint64_t* __restrict__ targets,
                                                              uint32_t* __restrict__ iv, uint64_t* __restrict__ longList,
                                                              unsigned long long* scal)
{
    const uint64_t s = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(s >= segCount) return;
    const uint64_t b = segOff[s], e = segOff[s + 1];
    for(uint64_t i = b + lane; i < e; i += 32) {
        const uint64_t m0 = markers[i];
        if(m0 >= M) { atomicMin(scal + 0, (unsigned long long)i); targets[i] = kInvalid40; continue; }
        if(i > b && markers[i - 1] >= m0) atomicMin(scal + 1, (unsigned long long)i);
        const uint32_t o = rowOf(toc, 0u, rows, m0);
        const uint64_t first = toc[o], end = toc[o + 1];
        uint64_t t = kInvalid40, m = m0 + 1;
        for(uint32_t k = 0; k < kShortWalk && m < end; k++, m++) {
            t = load40(table + 5 * m);
            if(t != kInvalid40) break;
        }
        iv[3 * i] = o; iv[3 * i + 1] = uint32_t(m0 - first);
        if(t != kInvalid40) {
            if(t >= V) atomicMin(scal + 2, (unsigned long long)m);
            iv[3 * i + 2] = uint32_t(m - first);
        } else if(m < end) {
            longList[atomicAdd(scal + 3, 1ull)] = i;
        }
        targets[i] = t;
    }
}

// One warp per listed marker: the rest of its walk, 32 markers per step.
__global__ void __launch_bounds__(kMgThreads) longWalkKernel(const uint64_t* __restrict__ longList, uint64_t n, const uint64_t* __restrict__ markers,
                                                             const uint8_t* __restrict__ table, uint64_t V, const uint64_t* __restrict__ toc,
                                                             uint64_t* __restrict__ targets, uint32_t* __restrict__ iv, unsigned long long* scal)
{
    const uint64_t w = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(w >= n) return;
    const uint64_t i = longList[w];
    const uint32_t o = iv[3 * i];
    const uint64_t first = toc[o], end = toc[o + 1];
    for(uint64_t m = markers[i] + 1 + kShortWalk; m < end; m += 32) {
        const uint64_t t = m + lane < end ? load40(table + 5 * (m + lane)) : kInvalid40;
        const uint32_t hit = __ballot_sync(0xffffffffu, t != kInvalid40);
        if(hit) {
            const uint32_t l = __ffs(hit) - 1;
            if(lane == l) {
                if(t >= V) atomicMin(scal + 2, (unsigned long long)(m + l));
                targets[i] = t;
                iv[3 * i + 2] = uint32_t(m + l - first);
            }
            return;
        }
    }
}

// Sort keys: target << 12 | position for segments of up to kBlockSortMax markers (distinct, as the rank sorts need);
// target alone, with the position as the value, for larger segments (radixSort is stable).
__global__ void __launch_bounds__(kMgThreads) keyKernel(const uint64_t* __restrict__ targets, const uint64_t* __restrict__ segOff, uint64_t segCount,
                                                        uint64_t* __restrict__ keys, uint32_t* __restrict__ vals)
{
    const uint64_t s = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(s >= segCount) return;
    const uint64_t b = segOff[s], n = segOff[s + 1] - b;
    for(uint64_t j = lane; j < n; j += 32) {
        const uint64_t t = targets[b + j];
        keys[b + j] = n <= kBlockSortMax ? (t << kSmallKeyBits) | j : t;
        vals[b + j] = uint32_t(j);
    }
}

// Back to (target, position) in sorted order, and the counts per vertex: intervals (markers with a successor, a prefix of the
// sorted segment since kInvalid40 sorts last) and edges (runs of one target).
__global__ void __launch_bounds__(kMgThreads) groupKernel(uint64_t* __restrict__ keys, uint32_t* __restrict__ vals, const uint64_t* __restrict__ segOff,
                                                          uint64_t segCount, uint64_t* __restrict__ intervalCount, uint64_t* __restrict__ edgeCount)
{
    const uint64_t s = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(s >= segCount) return;
    const uint64_t b = segOff[s], n = segOff[s + 1] - b;
    uint64_t carry = kInvalid40, intervals = 0, edges = 0;
    for(uint64_t j0 = 0; j0 < n; j0 += 32) {
        const uint64_t j = j0 + lane;
        uint64_t t = kInvalid40;
        if(j < n) {
            const uint64_t k = keys[b + j];
            t = n <= kBlockSortMax ? k >> kSmallKeyBits : k;
            if(n <= kBlockSortMax) vals[b + j] = uint32_t(k & ((1u << kSmallKeyBits) - 1));
            keys[b + j] = t;
        }
        uint64_t prev = __shfl_up_sync(0xffffffffu, t, 1);
        if(lane == 0) prev = carry;
        const bool valid = j < n && t != kInvalid40;
        intervals += __popc(__ballot_sync(0xffffffffu, valid));
        edges += __popc(__ballot_sync(0xffffffffu, valid && (j == 0 || t != prev)));
        carry = __shfl_sync(0xffffffffu, t, 31);
    }
    if(lane == 0) { intervalCount[s] = intervals; edgeCount[s] = edges; }
}

// One warp per source vertex: the edges (coverage later), their interval toc, the intervals and the edgesBySource entries.
__global__ void __launch_bounds__(kMgThreads) writeKernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                                          const uint64_t* __restrict__ segOff, uint64_t segCount, uint64_t firstVertex,
                                                          const uint32_t* __restrict__ iv, const uint64_t* __restrict__ intervalOff,
                                                          const uint64_t* __restrict__ edgeOff, const uint64_t* __restrict__ edgeCount,
                                                          uint64_t edgeBase, uint64_t intervalBase, uint8_t* __restrict__ edgesOut,
                                                          uint64_t* __restrict__ itocOut, uint32_t* __restrict__ ivOut,
                                                          uint8_t* __restrict__ bySourceOut, unsigned long long* __restrict__ targetCount)
{
    const uint64_t s = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(s >= segCount) return;
    const uint64_t b = segOff[s], n = segOff[s + 1] - b;
    const uint64_t rowBegin = edgeBase + edgeOff[s], rowEnd = rowBegin + edgeCount[s];
    uint64_t carry = kInvalid40, heads = 0;
    for(uint64_t j0 = 0; j0 < n; j0 += 32) {
        const uint64_t j = j0 + lane;
        const uint64_t t = j < n ? keys[b + j] : kInvalid40;
        uint64_t prev = __shfl_up_sync(0xffffffffu, t, 1);
        if(lane == 0) prev = carry;
        const bool valid = t != kInvalid40;
        const bool head = valid && (j == 0 || t != prev);
        const uint32_t ballot = __ballot_sync(0xffffffffu, head);
        if(valid) {
            const uint64_t p = intervalOff[s] + j;                         // chunk-local interval index
            const uint64_t src = b + vals[b + j];
            ivOut[3 * p] = iv[3 * src]; ivOut[3 * p + 1] = iv[3 * src + 1]; ivOut[3 * p + 2] = iv[3 * src + 2];
            if(head) {
                const uint64_t e = edgeOff[s] + heads + __popc(ballot & ((1u << lane) - 1u));    // chunk-local edge id
                uint8_t* r = edgesOut + uint64_t(kEdgeBytes) * e;
                store40(r, firstVertex + s);
                store40(r + 5, t);
#pragma unroll
                for(int k = 10; k < 14; k++) r[k] = 0;
                itocOut[e] = intervalBase + p;
                store40(bySourceOut + 5 * e, rowBegin + rowEnd - 1 - (edgeBase + e));
                atomicAdd(targetCount + t, 1ull);
            }
        }
        heads += __popc(ballot);
        carry = __shfl_sync(0xffffffffu, t, 31);
    }
}

// coverage = min(intervals, 255) (:2155-2160); itoc[edges] holds the chunk's interval end.
__global__ void coverageKernel(const uint64_t* __restrict__ itoc, uint64_t edges, uint8_t* __restrict__ edgesOut, unsigned long long* saturated)
{
    for(uint64_t e = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; e < edges; e += uint64_t(gridDim.x) * blockDim.x) {
        const uint64_t c = itoc[e + 1] - itoc[e];
        edgesOut[uint64_t(kEdgeBytes) * e + 10] = uint8_t(c < 256 ? c : 255);
        if(c >= 256) atomicAdd(saturated, 1ull);
    }
}

// ---- edgesByTarget (:2192-2213) --------------------------------------------------------------------------------------
__global__ void targetKeyKernel(const uint8_t* __restrict__ records, uint64_t n, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals)
{
    for(uint64_t e = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; e < n; e += uint64_t(gridDim.x) * blockDim.x) {
        keys[e] = load40(records + uint64_t(kEdgeBytes) * e + 5);
        vals[e] = uint32_t(e);
    }
}

__device__ __forceinline__ uint64_t lowerBound(const uint64_t* __restrict__ a, uint64_t n, uint64_t x)
{
    uint64_t lo = 0, hi = n;
    while(lo < hi) { const uint64_t mid = lo + ((hi - lo) >> 1); if(a[mid] < x) lo = mid + 1; else hi = mid; }
    return lo;
}

// Sorted by target, stable: an edge's rank among the chunk's edges of its target is its distance to the run's start; the
// earlier chunks' edges of that target come before it (seen).
__global__ void targetPlaceKernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint64_t n, uint64_t firstEdge,
                                  const uint64_t* __restrict__ toc, const uint64_t* __restrict__ seen, uint8_t* __restrict__ data)
{
    for(uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < n; i += uint64_t(gridDim.x) * blockDim.x) {
        const uint64_t t = keys[i];
        const uint64_t rank = seen[t] + (i - lowerBound(keys, n, t));
        store40(data + 5 * (toc[t + 1] - 1 - rank), firstEdge + vals[i]);
    }
}

__global__ void targetSeenKernel(const uint64_t* __restrict__ keys, uint64_t n, uint64_t* __restrict__ seen)
{
    for(uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < n; i += uint64_t(gridDim.x) * blockDim.x) {
        const uint64_t t = keys[i];
        if(i == 0 || keys[i - 1] != t) seen[t] += lowerBound(keys, n, t + 1) - i;
    }
}

// ---- reverse complement edges (:1283-1389) ---------------------------------------------------------------------------
// Per edge: bit 0 = its intervals are non-decreasing, bit 1 = strictly increasing. An interval on an oriented read that
// does not exist is refused.
__global__ void __launch_bounds__(kMgThreads) orderKernel(const uint64_t* __restrict__ itoc, const uint32_t* __restrict__ iv, uint64_t E,
                                                          uint32_t rows, uint8_t* __restrict__ order, unsigned long long* errInput)
{
    const uint64_t e = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(e >= E) return;
    const uint64_t b = itoc[e], n = itoc[e + 1] - b;
    bool nondecreasing = true, increasing = true, bad = false;
    for(uint64_t j = lane; j < n; j += 32) {
        const Interval x = loadIv(iv, b + j);
        if(x.o >= rows) bad = true;
        if(j) {
            const Interval p = loadIv(iv, b + j - 1);
            if(ivLess(x, p)) nondecreasing = false;
            if(!ivLess(p, x)) increasing = false;
        }
    }
    nondecreasing = __all_sync(0xffffffffu, nondecreasing);
    increasing = __all_sync(0xffffffffu, increasing);
    if(__any_sync(0xffffffffu, bad) && lane == 0) atomicMin(errInput, (unsigned long long)e);
    if(lane == 0) order[e] = uint8_t((nondecreasing ? 1u : 0u) | (increasing ? 2u : 0u));
}

__device__ __forceinline__ Interval reverseComplementInterval(const Interval& x, const uint64_t* __restrict__ toc)
{
    const uint32_t mc = uint32_t(toc[x.o + 1] - toc[x.o]);
    return Interval{x.o ^ 1u, mc - 1 - x.a1, mc - 1 - x.a0};
}

// Is sort(reverse complement of c's intervals) == e's intervals? Warp-uniform result.
__device__ bool intervalsMatch(const uint32_t* __restrict__ iv, const uint64_t* __restrict__ itoc, const uint8_t* __restrict__ order,
                               const uint64_t* __restrict__ toc, uint64_t e, uint64_t c, uint32_t lane)
{
    const uint64_t be = itoc[e], n = itoc[e + 1] - be, bc = itoc[c];
    if(itoc[c + 1] - bc != n) return false;
    if(!(order[e] & 1u)) return n == 0;                // a sorted sequence never equals unsorted intervals
    bool ok = true;
    if((order[e] & 2u) && (order[c] & 2u)) {
        // Both strictly increasing: the reverse complements are distinct, so they sort to e's intervals when each is one of them.
        for(uint64_t j = lane; j < n && ok; j += 32) {
            const Interval x = reverseComplementInterval(loadIv(iv, bc + j), toc);
            uint64_t lo = 0, hi = n;
            while(lo < hi) { const uint64_t mid = lo + ((hi - lo) >> 1); if(ivLess(loadIv(iv, be + mid), x)) lo = mid + 1; else hi = mid; }
            ok = lo < n && ivEqual(loadIv(iv, be + lo), x);
        }
    } else {
        // General case (repeated intervals): x occupies positions [less, less + equal) of the sorted sequence.
        for(uint64_t j = lane; j < n && ok; j += 32) {
            const Interval x = reverseComplementInterval(loadIv(iv, bc + j), toc);
            uint64_t less = 0, equal = 0;
            for(uint64_t k = 0; k < n; k++) {
                const Interval y = reverseComplementInterval(loadIv(iv, bc + k), toc);
                less += ivLess(y, x) ? 1 : 0;
                equal += ivEqual(y, x) ? 1 : 0;
            }
            ok = ivEqual(loadIv(iv, be + less), x) && ivEqual(loadIv(iv, be + less + equal - 1), x);
        }
    }
    return __all_sync(0xffffffffu, ok);
}

// One warp per edge: edgesBySource[rc(v1)] in stored order, the first candidate with target rc(v0) and matching intervals.
__global__ void __launch_bounds__(kMgThreads) rcEdgeKernel(const uint8_t* __restrict__ edges, uint64_t first, uint64_t count, uint64_t E,
                                                           const uint64_t* __restrict__ rcVertex, uint64_t V, const uint64_t* __restrict__ itoc,
                                                           const uint32_t* __restrict__ iv, const uint8_t* __restrict__ order,
                                                           const uint64_t* __restrict__ stoc, const uint8_t* __restrict__ sdata,
                                                           const uint64_t* __restrict__ toc, uint64_t* __restrict__ rcEdge,
                                                           unsigned long long* scal)
{
    const uint64_t w = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if(w >= count) return;
    const uint64_t e = first + w;
    const uint64_t v0 = load40(edges + uint64_t(kEdgeBytes) * e), v1 = load40(edges + uint64_t(kEdgeBytes) * e + 5);
    if(v0 >= V || v1 >= V) { if(lane == 0) atomicMin(scal + 0, (unsigned long long)e); return; }
    const uint64_t v0Rc = rcVertex[v0], v1Rc = rcVertex[v1];
    for(uint64_t k = stoc[v1Rc]; k < stoc[v1Rc + 1]; k++) {
        const uint64_t c = load40(sdata + 5 * k);
        if(c >= E) { if(lane == 0) atomicMin(scal + 0, (unsigned long long)e); return; }
        if(load40(edges + uint64_t(kEdgeBytes) * c) != v1Rc) { if(lane == 0) atomicMin(scal + 1, (unsigned long long)e); return; }
        if(load40(edges + uint64_t(kEdgeBytes) * c + 5) != v0Rc) continue;
        if(intervalsMatch(iv, itoc, order, toc, e, c, lane)) {
            if(lane == 0) rcEdge[e] = c;
            return;
        }
    }
    if(lane == 0) atomicMin(scal + 2, (unsigned long long)e);
}

__global__ void rcRcKernel(const uint64_t* __restrict__ rcEdge, uint64_t E, unsigned long long* errRcRc)
{
    for(uint64_t e = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; e < E; e += uint64_t(gridDim.x) * blockDim.x)
        if(rcEdge[rcEdge[e]] != e) atomicMin(errRcRc, (unsigned long long)e);
}

uint64_t load40Host(const uint8_t* p)
{
    uint64_t x = 0;
    for(int b = 0; b < 5; b++) x |= uint64_t(p[b]) << (8 * b);
    return x;
}

} // namespace

void createMarkerGraphEdges(shb_context* c, const uint8_t* table5, uint64_t tableCount, const uint8_t* toc5, const uint64_t* vdata,
                            uint64_t V, uint8_t** edgesOut, uint64_t** itocOut, uint8_t** idataOut, uint64_t** stocOut,
                            uint8_t** sdataOut, uint64_t** ttocOut, uint8_t** tdataOut, shb_marker_graph_edges_result* result)
{
    SHB_CUDA(cudaSetDevice(c->device));
    requireWholeAssembly(c, "createMarkerGraphEdges");
    const auto t0 = std::chrono::steady_clock::now();
    const uint64_t launches0 = g_launchCount;
    cudaStream_t st = c->stream;
    const uint64_t M = c->localMarkerCount;
    const uint32_t rows = uint32_t(2 * c->readCountTotal);
    SHB_REQUIRE(tableCount == M, SHB_ERR_INVALID, "The marker graph vertex table has " + std::to_string(tableCount) + " entries for " +
                std::to_string(M) + " markers.");
    SHB_REQUIRE(V < kInvalid40, SHB_ERR_INVALID, "Too many marker graph vertices.");
    std::vector<uint64_t> vtoc(V + 1);
    for(uint64_t v = 0; v <= V; v++) {
        vtoc[v] = load40Host(toc5 + 5 * v);
        SHB_REQUIRE(v == 0 ? vtoc[v] == 0 : vtoc[v] >= vtoc[v - 1], SHB_ERR_INVALID,
                    "The marker graph vertices toc does not start at 0 or decreases at vertex " + std::to_string(v) + ".");
    }
    const uint64_t N = vtoc[V];                                       // vertex markers: at most one interval each
    for(uint64_t v = 0; v < V; v++)
        SHB_REQUIRE(vtoc[v + 1] - vtoc[v] < (1ull << 32), SHB_ERR_INVALID, "A marker graph vertex has 2^32 or more markers.");

    // Host results, sized for one interval and one edge per vertex marker. They are plain malloc blocks, not the library's
    // recycled page-locked ones: the pages past the real counts are never touched, so they take no memory (shb_free frees
    // any block the pool does not hold).
    HostResult edgesBlock(malloc(kEdgeBytes * N + 8)), itocBlock(malloc(8 * (N + 1) + 8)), idataBlock(malloc(12 * N + 8)),
               stocBlock(malloc(8 * (V + 1) + 8)), sdataBlock(malloc(5 * N + 8)), ttocBlock(malloc(8 * (V + 1) + 8)),
               tdataBlock(malloc(5 * N + 8));
    SHB_REQUIRE(edgesBlock.p && itocBlock.p && idataBlock.p && stocBlock.p && sdataBlock.p && ttocBlock.p && tdataBlock.p, SHB_ERR_OOM,
                "Out of host memory for the marker graph edges.");
    uint8_t* hEdges = static_cast<uint8_t*>(edgesBlock.p);
    uint64_t* hItoc = static_cast<uint64_t*>(itocBlock.p);
    uint8_t* hIdata = static_cast<uint8_t*>(idataBlock.p);
    uint64_t* hStoc = static_cast<uint64_t*>(stocBlock.p);
    uint8_t* hSdata = static_cast<uint8_t*>(sdataBlock.p);
    uint64_t* hTtoc = static_cast<uint64_t*>(ttocBlock.p);
    uint8_t* hTdata = static_cast<uint8_t*>(tdataBlock.p);

    Footprint fp;
    EventTimer timer;
    timer.start(st);
    unsigned long long* scal = c->scalar(kSlotMarkerGraphEdges);
    const unsigned long long init[8] = {~0ull, ~0ull, ~0ull, 0, 0, 0, 0, 0};
    SHB_CUDA(cudaMemcpyAsync(scal, init, sizeof(init), cudaMemcpyHostToDevice, st));
    DeviceBuffer<uint8_t> dTable;
    DeviceBuffer<unsigned long long> dTargetCount;
    fp.add(dTable, 5 * M + 8); fp.add(dTargetCount, V + 1);
    SHB_CUDA(cudaMemcpyAsync(dTable.get(), table5, 5 * M, cudaMemcpyHostToDevice, st));
    SHB_CUDA(cudaMemsetAsync(dTargetCount.get(), 0, 8 * (V + 1), st));
    auto sortWsBytes = [&] { return 8 * (c->sortWs.hist.capacity() + c->sortWs.status.capacity()); };
    const uint64_t sortWs0 = sortWsBytes();

    // Chunks of source vertices under SHB_MARKERGRAPH_EDGES_BUDGET_MB (test hook): about 80 device bytes per vertex marker.
    const uint64_t budget = uint64_t(envCount("SHB_MARKERGRAPH_EDGES_BUDGET_MB", 16384)) << 20;
    const uint64_t chunkItems = std::max<uint64_t>(budget / 80, 1);
    uint64_t E = 0, I = 0;
    {
        DeviceBuffer<uint64_t> markers, segOff, targets, keys, keysTmp, intervalCount, edgeCount, intervalOff, edgeOff, longList, bigSets,
                               scanWs, itoc;
        DeviceBuffer<uint32_t> iv, vals, valsTmp, ivOut;
        DeviceBuffer<uint8_t> edgesOut, bySourceOut;
        std::vector<uint64_t> segOffHost, edgeOffHost;
        for(uint64_t vb = 0; vb < V; ) {
            uint64_t ve = vb + 1;
            while(ve < V && vtoc[ve + 1] - vtoc[vb] <= chunkItems) ve++;
            const uint64_t S = ve - vb, db = vtoc[vb], n = vtoc[ve] - db;
            segOffHost.resize(S + 1);
            for(uint64_t s = 0; s <= S; s++) segOffHost[s] = vtoc[vb + s] - db;
            fp.add(markers, n + 1); fp.add(segOff, S + 1); fp.add(targets, n + 1); fp.add(iv, 3 * n + 3); fp.add(longList, n + 1);
            SHB_CUDA(cudaMemcpyAsync(markers.get(), vdata + db, 8 * n, cudaMemcpyHostToDevice, st));
            SHB_CUDA(cudaMemcpyAsync(segOff.get(), segOffHost.data(), 8 * (S + 1), cudaMemcpyHostToDevice, st));
            SHB_CUDA(cudaMemsetAsync(scal + 3, 0, 8 * 2, st));
            SHB_LAUNCH(successorKernel, ceilDiv(S * 32, kMgThreads), kMgThreads, 0, st, (const uint64_t*)markers.get(), (const uint64_t*)segOff.get(),
                       S, (const uint8_t*)dTable.get(), M, V, (const uint64_t*)c->toc.get(), rows, targets.get(), iv.get(), longList.get(), scal);
            const uint64_t longCount = readBack(scal + 3, st);
            if(longCount)
                SHB_LAUNCH(longWalkKernel, ceilDiv(longCount * 32, kMgThreads), kMgThreads, 0, st, (const uint64_t*)longList.get(), longCount,
                           (const uint64_t*)markers.get(), (const uint8_t*)dTable.get(), V, (const uint64_t*)c->toc.get(), targets.get(),
                           iv.get(), scal);
            unsigned long long err[3];
            SHB_CUDA(cudaMemcpyAsync(err, scal, sizeof(err), cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaStreamSynchronize(st));
            if(err[0] != ~0ull) {
                const uint64_t v = uint64_t(std::upper_bound(vtoc.begin(), vtoc.end(), db + err[0]) - vtoc.begin()) - 1;
                SHB_REQUIRE(false, SHB_ERR_INVALID, "Marker graph vertex " + std::to_string(v) + " has a marker id out of range.");
            }
            if(err[1] != ~0ull) {
                const uint64_t v = uint64_t(std::upper_bound(vtoc.begin(), vtoc.end(), db + err[1]) - vtoc.begin()) - 1;
                SHB_REQUIRE(false, SHB_ERR_INVALID, "The markers of marker graph vertex " + std::to_string(v) + " are not in increasing order.");
            }
            SHB_REQUIRE(err[2] == ~0ull, SHB_ERR_INVALID, "The marker graph vertex table gives marker " + std::to_string(err[2]) +
                        " a vertex id >= the vertex count.");
            fp.drop(longList); fp.drop(markers);

            // Each vertex's markers, sorted stably by successor.
            fp.add(keys, n + 1); fp.add(vals, n + 1); fp.add(bigSets, S + 1); fp.add(intervalCount, S + 1); fp.add(edgeCount, S + 1);
            SHB_LAUNCH(keyKernel, ceilDiv(S * 32, kMgThreads), kMgThreads, 0, st, (const uint64_t*)targets.get(), (const uint64_t*)segOff.get(), S,
                       keys.get(), vals.get());
            fp.drop(targets);
            // The sorters take a size per segment; intervalCount holds the sizes until groupKernel writes the counts.
            std::vector<uint64_t> sizes(S);
            for(uint64_t s = 0; s < S; s++) sizes[s] = segOffHost[s + 1] - segOffHost[s];
            SHB_CUDA(cudaMemcpyAsync(intervalCount.get(), sizes.data(), 8 * S, cudaMemcpyHostToDevice, st));
            SHB_LAUNCH(warpSortKernel, ceilDiv(S * 32, kMgThreads), kMgThreads, 0, st, keys.get(), (const uint64_t*)segOff.get(),
                       (const uint64_t*)intervalCount.get(), S, bigSets.get(), scal + 4);
            const uint64_t bigCount = readBack(scal + 4, st);
            if(bigCount) {
                std::vector<uint64_t> big(bigCount), medium;
                SHB_CUDA(cudaMemcpyAsync(big.data(), bigSets.get(), 8 * bigCount, cudaMemcpyDeviceToHost, st));
                SHB_CUDA(cudaStreamSynchronize(st));
                std::sort(big.begin(), big.end());                     // the list's order comes from atomics
                for(const uint64_t s : big) {
                    if(sizes[s] <= kBlockSortMax) { medium.push_back(s); continue; }
                    fp.add(keysTmp, sizes[s]); fp.add(valsTmp, sizes[s]);
                    const int ranges[1][2] = {{0, 40}};
                    const uint64_t off = segOffHost[s];
                    if(radixSort<true>(keys.get() + off, keysTmp.get(), vals.get() + off, valsTmp.get(), sizes[s], ranges, 1, c->sortWs, st)) {
                        SHB_CUDA(cudaMemcpyAsync(keys.get() + off, keysTmp.get(), 8 * sizes[s], cudaMemcpyDeviceToDevice, st));
                        SHB_CUDA(cudaMemcpyAsync(vals.get() + off, valsTmp.get(), 4 * sizes[s], cudaMemcpyDeviceToDevice, st));
                    }
                    fp.peak = std::max(fp.peak, fp.live + (sortWsBytes() - sortWs0));
                }
                if(!medium.empty()) {
                    SHB_CUDA(cudaMemcpyAsync(bigSets.get(), medium.data(), 8 * medium.size(), cudaMemcpyHostToDevice, st));
                    SHB_LAUNCH(blockSortKernel, unsigned(medium.size()), kMgThreads, 0, st, keys.get(), (const uint64_t*)segOff.get(),
                               (const uint64_t*)intervalCount.get(), (const uint64_t*)bigSets.get());
                }
                SHB_CUDA(cudaStreamSynchronize(st));
                fp.drop(keysTmp); fp.drop(valsTmp);
            }
            fp.drop(bigSets);
            SHB_LAUNCH(groupKernel, ceilDiv(S * 32, kMgThreads), kMgThreads, 0, st, keys.get(), vals.get(), (const uint64_t*)segOff.get(), S,
                       intervalCount.get(), edgeCount.get());

            // Edge ids and interval offsets by scans over the chunk's vertices.
            fp.add(intervalOff, S + 1); fp.add(edgeOff, S + 1); fp.add(scanWs, scanWorkspaceElements(S) + 1);
            uint64_t* totals = reinterpret_cast<uint64_t*>(scal + 6);
            exclusiveScan<uint64_t>(intervalCount.get(), intervalOff.get(), S, totals + 1, scanWs.get(), st);
            exclusiveScan<uint64_t>(edgeCount.get(), edgeOff.get(), S, totals, scanWs.get(), st);
            uint64_t tot[2];
            SHB_CUDA(cudaMemcpyAsync(tot, totals, sizeof(tot), cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaStreamSynchronize(st));
            const uint64_t ce = tot[0], ci = tot[1];
            fp.add(edgesOut, kEdgeBytes * ce + 8); fp.add(itoc, ce + 1); fp.add(ivOut, 3 * ci + 3); fp.add(bySourceOut, 5 * ce + 8);
            SHB_LAUNCH(writeKernel, ceilDiv(S * 32, kMgThreads), kMgThreads, 0, st, (const uint64_t*)keys.get(), (const uint32_t*)vals.get(),
                       (const uint64_t*)segOff.get(), S, vb, (const uint32_t*)iv.get(), (const uint64_t*)intervalOff.get(),
                       (const uint64_t*)edgeOff.get(), (const uint64_t*)edgeCount.get(), E, I, edgesOut.get(), itoc.get(), ivOut.get(),
                       bySourceOut.get(), dTargetCount.get());
            const uint64_t intervalEnd = I + ci;
            SHB_CUDA(cudaMemcpyAsync(itoc.get() + ce, &intervalEnd, 8, cudaMemcpyHostToDevice, st));
            if(ce) SHB_LAUNCH(coverageKernel, gridFor(ce), kMgThreads, 0, st, (const uint64_t*)itoc.get(), ce, edgesOut.get(), scal + 5);

            // The chunk's results to the host.
            edgeOffHost.resize(S);
            SHB_CUDA(cudaMemcpyAsync(edgeOffHost.data(), edgeOff.get(), 8 * S, cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaMemcpyAsync(hEdges + kEdgeBytes * E, edgesOut.get(), kEdgeBytes * ce, cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaMemcpyAsync(hItoc + E, itoc.get(), 8 * ce, cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaMemcpyAsync(hIdata + 12 * I, ivOut.get(), 12 * ci, cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaMemcpyAsync(hSdata + 5 * E, bySourceOut.get(), 5 * ce, cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaStreamSynchronize(st));
            for(uint64_t s = 0; s < S; s++) hStoc[vb + s] = E + edgeOffHost[s];
            fp.drop(keys); fp.drop(vals); fp.drop(iv); fp.drop(segOff); fp.drop(intervalCount); fp.drop(edgeCount); fp.drop(intervalOff);
            fp.drop(edgeOff); fp.drop(scanWs); fp.drop(edgesOut); fp.drop(itoc); fp.drop(ivOut); fp.drop(bySourceOut);
            E += ce; I += ci;
            vb = ve;
        }
    }
    fp.drop(dTable);
    hItoc[E] = I;
    hStoc[V] = E;

    // edgesByTarget: toc by a scan of the counts, rows filled in chunks of edge ids.
    {
        DeviceBuffer<uint64_t> ttoc, seen, scanWs, keys, keysTmp;
        DeviceBuffer<uint32_t> vals, valsTmp;
        DeviceBuffer<uint8_t> records, tdata;
        fp.add(ttoc, V + 2); fp.add(scanWs, scanWorkspaceElements(V + 1) + 1);
        exclusiveScan<uint64_t>(reinterpret_cast<const uint64_t*>(dTargetCount.get()), ttoc.get(), V + 1, (uint64_t*)nullptr, scanWs.get(), st);
        fp.drop(scanWs); fp.drop(dTargetCount);
        SHB_CUDA(cudaMemcpyAsync(hTtoc, ttoc.get(), 8 * (V + 1), cudaMemcpyDeviceToHost, st));
        if(E) {
            fp.add(seen, V + 1); fp.add(tdata, 5 * E + 8);
            SHB_CUDA(cudaMemsetAsync(seen.get(), 0, 8 * (V + 1), st));
            const uint64_t chunk = std::min<uint64_t>(std::max<uint64_t>(budget / 40, 1), (1ull << 32) - 1);
            const int ranges[1][2] = {{0, int(bitsFor(V ? V - 1 : 0))}};
            for(uint64_t e0 = 0; e0 < E; e0 += chunk) {
                const uint64_t n = std::min(chunk, E - e0);
                fp.add(records, kEdgeBytes * n); fp.add(keys, n); fp.add(keysTmp, n); fp.add(vals, n); fp.add(valsTmp, n);
                SHB_CUDA(cudaMemcpyAsync(records.get(), hEdges + kEdgeBytes * e0, kEdgeBytes * n, cudaMemcpyHostToDevice, st));
                SHB_LAUNCH(targetKeyKernel, gridFor(n), kMgThreads, 0, st, (const uint8_t*)records.get(), n, keys.get(), vals.get());
                const bool inB = radixSort<true>(keys.get(), keysTmp.get(), vals.get(), valsTmp.get(), n, ranges, 1, c->sortWs, st);
                fp.peak = std::max(fp.peak, fp.live + (sortWsBytes() - sortWs0));
                const uint64_t* k = inB ? keysTmp.get() : keys.get();
                const uint32_t* v = inB ? valsTmp.get() : vals.get();
                SHB_LAUNCH(targetPlaceKernel, gridFor(n), kMgThreads, 0, st, k, v, n, e0, (const uint64_t*)ttoc.get(), (const uint64_t*)seen.get(),
                           tdata.get());
                SHB_LAUNCH(targetSeenKernel, gridFor(n), kMgThreads, 0, st, k, n, seen.get());
                SHB_CUDA(cudaStreamSynchronize(st));                   // the staging of the next chunk reuses the buffers
            }
            SHB_CUDA(cudaMemcpyAsync(hTdata, tdata.get(), 5 * E, cudaMemcpyDeviceToHost, st));
        }
    }
    const uint64_t saturated = readBack(reinterpret_cast<const uint64_t*>(scal + 5), st);
    timer.stop(st);
    SHB_CUDA(cudaEventSynchronize(timer.stopEvent));
    const float ms = timer.elapsedMs();

    *edgesOut = static_cast<uint8_t*>(edgesBlock.take()); *itocOut = static_cast<uint64_t*>(itocBlock.take());
    *idataOut = static_cast<uint8_t*>(idataBlock.take()); *stocOut = static_cast<uint64_t*>(stocBlock.take());
    *sdataOut = static_cast<uint8_t*>(sdataBlock.take()); *ttocOut = static_cast<uint64_t*>(ttocBlock.take());
    *tdataOut = static_cast<uint8_t*>(tdataBlock.take());
    if(result) {
        result->vertexCount = V;
        result->edgeCount = E;
        result->markerIntervalCount = I;
        result->saturatedEdgeCount = saturated;
        result->peakDeviceBytes = fp.peak;
        result->kernelLaunches = g_launchCount - launches0;
        result->deviceMs = ms;
        result->totalMs = msSince(t0);
    }
}

void findMarkerGraphReverseComplementEdges(shb_context* c, const uint64_t* rcVertex, uint64_t V, const uint8_t* edges, uint64_t E,
                                           const uint64_t* itoc, const uint8_t* idata, const uint64_t* stoc, const uint8_t* sdata,
                                           uint64_t** rcOut, shb_marker_graph_edges_result* result)
{
    SHB_CUDA(cudaSetDevice(c->device));
    requireWholeAssembly(c, "findMarkerGraphReverseComplementEdges");
    const auto t0 = std::chrono::steady_clock::now();
    const uint64_t launches0 = g_launchCount;
    cudaStream_t st = c->stream;
    const uint32_t rows = uint32_t(2 * c->readCountTotal);
    for(uint64_t v = 0; v < V; v++)
        SHB_REQUIRE(rcVertex[v] < V, SHB_ERR_INVALID, "The reverse complement of marker graph vertex " + std::to_string(v) + " is out of range.");
    SHB_REQUIRE(itoc[0] == 0 && stoc[0] == 0, SHB_ERR_INVALID, "A marker graph edge toc does not start at 0.");
    for(uint64_t e = 0; e < E; e++)
        SHB_REQUIRE(itoc[e + 1] >= itoc[e], SHB_ERR_INVALID, "The marker interval toc decreases at edge " + std::to_string(e) + ".");
    for(uint64_t v = 0; v < V; v++)
        SHB_REQUIRE(stoc[v + 1] >= stoc[v], SHB_ERR_INVALID, "The edgesBySource toc decreases at vertex " + std::to_string(v) + ".");
    const uint64_t I = itoc[E], S = stoc[V];
    uint64_t saturated = 0;
    for(uint64_t e = 0; e < E; e++) saturated += edges[uint64_t(kEdgeBytes) * e + 10] == 255;

    HostResult out(allocHostResult(8 * E + 8));
    SHB_REQUIRE(out.p, SHB_ERR_OOM, "Out of host memory for the reverse complement edges.");
    Footprint fp;
    EventTimer timer;
    timer.start(st);
    if(E) {
        DeviceBuffer<uint8_t> dEdges, dSdata, dOrder;
        DeviceBuffer<uint64_t> dItoc, dStoc, dRcVertex, dRc;
        DeviceBuffer<uint32_t> dIv;
        fp.add(dEdges, kEdgeBytes * E + 8); fp.add(dSdata, 5 * S + 8); fp.add(dOrder, E); fp.add(dItoc, E + 1); fp.add(dStoc, V + 1);
        fp.add(dRcVertex, V + 1); fp.add(dRc, E); fp.add(dIv, 3 * I + 3);
        SHB_CUDA(cudaMemcpyAsync(dEdges.get(), edges, kEdgeBytes * E, cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(dSdata.get(), sdata, 5 * S, cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(dItoc.get(), itoc, 8 * (E + 1), cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(dStoc.get(), stoc, 8 * (V + 1), cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(dRcVertex.get(), rcVertex, 8 * V, cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(dIv.get(), idata, 12 * I, cudaMemcpyHostToDevice, st));
        unsigned long long* err = c->scalar(kSlotMarkerGraphRcEdges);
        const unsigned long long init[4] = {~0ull, ~0ull, ~0ull, ~0ull};
        SHB_CUDA(cudaMemcpyAsync(err, init, sizeof(init), cudaMemcpyHostToDevice, st));
        SHB_LAUNCH(orderKernel, ceilDiv(E * 32, kMgThreads), kMgThreads, 0, st, (const uint64_t*)dItoc.get(), (const uint32_t*)dIv.get(), E, rows,
                   dOrder.get(), err);
        const uint64_t badInterval = readBack(reinterpret_cast<const uint64_t*>(err), st);
        SHB_REQUIRE(badInterval == ~0ull, SHB_ERR_INVALID, "Marker graph edge " + std::to_string(badInterval) +
                    " has a marker interval on an oriented read that does not exist.");
        // In launches of SHB_MARKERGRAPH_EDGES_RC_CHUNK edges (test hook).
        const uint64_t chunk = envCount("SHB_MARKERGRAPH_EDGES_RC_CHUNK", 1u << 24);
        for(uint64_t e0 = 0; e0 < E; e0 += chunk) {
            const uint64_t n = std::min(chunk, E - e0);
            SHB_LAUNCH(rcEdgeKernel, ceilDiv(n * 32, kMgThreads), kMgThreads, 0, st, (const uint8_t*)dEdges.get(), e0, n, E,
                       (const uint64_t*)dRcVertex.get(), V, (const uint64_t*)dItoc.get(), (const uint32_t*)dIv.get(),
                       (const uint8_t*)dOrder.get(), (const uint64_t*)dStoc.get(), (const uint8_t*)dSdata.get(), (const uint64_t*)c->toc.get(),
                       dRc.get(), err);
        }
        unsigned long long e[4];
        SHB_CUDA(cudaMemcpyAsync(e, err, sizeof(e), cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        const uint64_t firstBad = std::min(e[0], std::min(e[1], e[2]));
        if(firstBad != ~0ull) {
            const uint64_t v0 = load40Host(edges + kEdgeBytes * firstBad), v1 = load40Host(edges + kEdgeBytes * firstBad + 5);
            SHB_REQUIRE(e[0] != firstBad, SHB_ERR_INVALID, "Marker graph edge " + std::to_string(firstBad) +
                        " refers to a vertex, an edge or an oriented read that does not exist.");
            SHB_REQUIRE(e[1] != firstBad, SHB_ERR_INVALID, "Assertion failed: edgeRc.source == v1Rc (edgesBySource[" +
                        std::to_string(rcVertex[v1]) + "] lists an edge of another source, looking for the reverse complement of edge " +
                        std::to_string(firstBad) + ").");
            SHB_REQUIRE(false, SHB_ERR_INVALID, "Unable to locate reverse complement of marker graph edge " + std::to_string(firstBad) + " " +
                        std::to_string(v0) + "->" + std::to_string(v1));
        }
        SHB_LAUNCH(rcRcKernel, gridFor(E), kMgThreads, 0, st, (const uint64_t*)dRc.get(), E, err + 3);
        SHB_CUDA(cudaMemcpyAsync(out.p, dRc.get(), 8 * E, cudaMemcpyDeviceToHost, st));
        const uint64_t bad = readBack(reinterpret_cast<const uint64_t*>(err + 3), st);
        if(bad != ~0ull) {
            const uint64_t* rc = static_cast<const uint64_t*>(out.p);
            SHB_REQUIRE(false, SHB_ERR_INVALID, "Reverse complement edge check failed at edge " + std::to_string(bad) + ": " +
                        std::to_string(rc[bad]) + " " + std::to_string(rc[rc[bad]]));
        }
    }
    timer.stop(st);
    SHB_CUDA(cudaEventSynchronize(timer.stopEvent));
    const float ms = timer.elapsedMs();
    *rcOut = static_cast<uint64_t*>(out.take());
    if(result) {
        result->vertexCount = V;
        result->edgeCount = E;
        result->markerIntervalCount = I;
        result->saturatedEdgeCount = saturated;
        result->peakDeviceBytes = fp.peak;
        result->kernelLaunches = g_launchCount - launches0;
        result->deviceMs = ms;
        result->totalMs = msSince(t0);
    }
}

} // namespace shb
