// Assembler::createReadGraph, ReadGraph.creationMethod 0 (src/AssemblerReadGraph.cpp:35-175) on the GPU: the first consumer
// of AlignmentData after the hot path (SURVEY.md section 8, row f4).
//   * per read, the best maxAlignmentCount alignments by (markerCount, alignmentId), both descending — the set
//     std::nth_element with std::greater<pair<markerCount, alignmentId>> leaves in front (:59-74; the set does not depend on
//     nth_element's internal order). One (readId, markerCount, alignmentId) item per alignment and side, generated in
//     DESCENDING alignmentId order and stably sorted by (readId ascending, markerCount descending): an item's rank inside
//     its read is its distance from the read's first item;
//   * an alignment is kept when it is among the best of EITHER of its reads (:77-85); kept alignments get
//     AlignmentInfo::isInReadGraph (:103) and two edges each, in alignmentId order (:110-140). A kept alignment whose edge
//     or reverse-complement edge is not ordered (readIds[0] > readIds[1], or a read aligned to itself) is refused, where
//     the reference stops on SHASTA_ASSERT (:134, :140);
//   * ReadGraphConnectivity: for every oriented read the indices of its edges in DECREASING order (:147-159): the
//     reference stores the edges in increasing order and MemoryMapped::VectorOfVectors::store fills each row from its end
//     (src/MemoryMappedVectorOfVectors.hpp:384-387).
// Assembler::createReadGraph2, ReadGraph.creationMethod 2 (src/AssemblerReadGraph2.cpp:182-248; what Nanopore-May2022.conf and
// Nanopore-UL-May2022.conf select): the same selection over the alignments that pass five thresholds, which are read off
// histograms of the alignments' quality indicators at given percentiles (setReadGraph2Criteria, :99-179). The histograms are
// filled in alignment order on the host (Histogram2 with dynamic bounds is order dependent, see DynamicHistogram below).
#include "context.cuh"
#include "hostpool.cuh"

#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace shb {
namespace {

constexpr uint32_t kAlignmentWords = 16;            // 64-byte AlignmentData
constexpr uint32_t kMarkerCountWord = 9;            // readIds[2], isSameStrand, AlignmentInfo: data[2] (6 words), markerCount

constexpr uint32_t kNoRead = 0x7fffffffu;           // items of alignments that fail the creation-method-2 criteria sort behind every read

__global__ void readGraphItemsKernel(const uint32_t* __restrict__ records, const uint8_t* __restrict__ eligible, uint32_t n,
                                     uint64_t* __restrict__ keys, uint32_t* __restrict__ vals)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if(j >= 2 * n) return;
    const uint32_t a = n - 1u - (j >> 1);               // alignment ids in descending order
    const uint32_t readId = (eligible && !eligible[a]) ? kNoRead : records[uint64_t(kAlignmentWords) * a + (j & 1u)];
    const uint32_t markerCount = records[uint64_t(kAlignmentWords) * a + kMarkerCountWord];
    keys[j] = (uint64_t(readId) << 32) | (0xffffffffu - markerCount);
    vals[j] = a;
}

__global__ void readGraphKeepKernel(const uint64_t* __restrict__ sortedKeys, const uint32_t* __restrict__ sortedVals, uint32_t items,
                                    uint32_t maxAlignmentCount, uint32_t* __restrict__ keep)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= items) return;
    const uint64_t readKey = sortedKeys[i] & 0xffffffff00000000ull;
    if(uint32_t(readKey >> 32) == kNoRead) return;
    uint32_t lo = 0, hi = i;                            // first item of this read
    while(lo < hi) { const uint32_t mid = lo + ((hi - lo) >> 1); if(sortedKeys[mid] < readKey) lo = mid + 1; else hi = mid; }
    if(i - lo < maxAlignmentCount) keep[sortedVals[i]] = 1u;
}

// 16-byte ReadGraphEdge (src/ReadGraph.hpp:37-57): orientedReadIds[2], alignmentId:62 | crossesStrands:1 | hasInconsistentAlignment:1.
// The (row, edge) entries are written in DECREASING edge order, so the stable sort on the row alone leaves every row in
// decreasing edge order, the reference's. That costs nothing beyond the index arithmetic; sorting on (row, ~edge) instead
// would add radix passes over the edge bits. The two entries of one edge have different rows (the edge is ordered), so
// their relative order does not matter.
__global__ void readGraphEdgesKernel(const uint32_t* __restrict__ records, uint32_t n, const uint32_t* __restrict__ keep,
                                     const uint32_t* __restrict__ keepIndex, uint32_t entries, uint32_t* __restrict__ edges,
                                     uint64_t* __restrict__ rowKeys, uint32_t* __restrict__ rowVals)
{
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if(a >= n || !keep[a]) return;
    const uint32_t r0 = records[uint64_t(kAlignmentWords) * a], r1 = records[uint64_t(kAlignmentWords) * a + 1];
    const bool same = (records[uint64_t(kAlignmentWords) * a + 2] & 0xffu) != 0;
    const uint32_t o0 = 2u * r0, o1 = 2u * r1 + (same ? 0u : 1u);
    const uint32_t e = 2u * keepIndex[a];
#pragma unroll
    for(uint32_t k = 0; k < 2; k++) {                   // the edge and its reverse complement
        uint32_t* w = edges + 4ull * (e + k);
        w[0] = o0 ^ k; w[1] = o1 ^ k; w[2] = a; w[3] = 0u;      // alignmentId < 2^32: the flags in the top two bits stay 0
        const uint64_t slot = uint64_t(entries) - 2u * (e + k + 1u);     // edge e + k from the back
        rowKeys[slot] = uint64_t(o0 ^ k) << 32;      rowVals[slot] = e + k;
        rowKeys[slot + 1] = uint64_t(o1 ^ k) << 32;  rowVals[slot + 1] = e + k;
    }
}

__global__ void readGraphTocKernel(const uint64_t* __restrict__ sortedKeys, uint32_t entries, uint32_t rows, uint32_t* __restrict__ toc)
{
    const uint32_t row = blockIdx.x * blockDim.x + threadIdx.x;
    if(row > rows) return;
    uint32_t lo = 0, hi = entries;                      // first entry whose row is >= this row
    while(lo < hi) { const uint32_t mid = lo + ((hi - lo) >> 1); if(uint32_t(sortedKeys[mid] >> 32) < row) lo = mid + 1; else hi = mid; }
    toc[row] = lo;
}

struct HostBlocks {         // frees what was not handed to the caller (error paths)
    void* p[4] = {nullptr, nullptr, nullptr, nullptr};
    ~HostBlocks() { for(void* q : p) if(q) HostPool::instance().release(q); }
    void disarm() { for(void*& q : p) q = nullptr; }
};

// shasta::Histogram2 (src/Histogram.cpp:14-140) as createReadGraph2 uses it: dynamicBounds = true. update() grows the
// histogram to `index` bins when index > size and then increments bin `index` — which, for index >= the size before the call,
// lies one past the end: the reference's write lands outside the deque and the sample is never seen by getSum() /
// thresholdByCumulativeProportion(). So a sample is counted iff its index is below max(initial bins, every earlier index):
// the content depends on the order of the updates, and this class reproduces it for the reference's (alignment id) order.
class DynamicHistogram {
public:
    DynamicHistogram(double start, double stop, uint64_t binCount) : start(start), binSize((stop - start) / double(binCount)), bins(binCount, 0) {}
    void update(double x)
    {
        const int64_t index = int64_t(std::floor((x - start) / binSize));
        if(index < 0) return;                                   // not reachable for the five indicators (all >= 0)
        if(uint64_t(index) > bins.size()) bins.resize(uint64_t(index), 0);
        if(uint64_t(index) < bins.size()) bins[uint64_t(index)]++;
    }
    double thresholdByCumulativeProportion(double fraction) const
    {
        uint64_t total = 0;
        for(uint64_t v : bins) total += v;
        double cumulativeSum = 0;
        uint64_t i;
        for(i = 0; i < bins.size(); i++) {
            cumulativeSum += double(bins[i]);
            if(double(cumulativeSum) / double(total) >= fraction) break;
        }
        return start + binSize * double(i) + binSize / 2;
    }
private:
    double start, binSize;
    std::vector<uint64_t> bins;
};

struct AlignmentIndicators { double minAlignedFraction; uint32_t markerCount, maxDrift, maxSkip, trim; };

// AlignmentInfo accessors (src/Alignment.hpp:103-121, 252-284) on the 13 info words of a 64-byte record.
AlignmentIndicators indicators(const uint32_t* rec)
{
    const uint32_t* d0 = rec + 3; const uint32_t* d1 = rec + 6;         // Data: markerCount, firstOrdinal, lastOrdinal
    AlignmentIndicators r;
    r.markerCount = rec[9]; r.maxSkip = rec[13]; r.maxDrift = rec[14];
    const double f0 = double(r.markerCount) / double(d0[2] + 1 - d0[1]), f1 = double(r.markerCount) / double(d1[2] + 1 - d1[1]);
    r.minAlignedFraction = std::min(f0, f1);
    const uint32_t leftTrim = std::min(d0[1], d1[1]), rightTrim = std::min(d0[0] - 1 - d0[2], d1[0] - 1 - d1[2]);
    r.trim = std::max(leftTrim, rightTrim);
    return r;
}

} // namespace

// setReadGraph2Criteria (src/AssemblerReadGraph2.cpp:99-179) + passesReadGraph2Criteria (:69-96): thresholds, and which
// alignments pass them. percentiles = markerCount, alignedFraction, maxSkip, maxDrift, maxTrim (the member's argument order).
void readGraph2Criteria(const uint32_t* rec, uint64_t n, const double* percentiles, shb_read_graph2_criteria& out, std::vector<uint8_t>& eligible)
{
    DynamicHistogram alignedFraction(0, 1, 100), markerCount(0, 3000, 300), maxDrift(0, 100, 100), maxSkip(0, 100, 100), maxTrim(0, 100, 100);
    for(uint64_t i = 0; i < n; i++) {
        const AlignmentIndicators a = indicators(rec + kAlignmentWords * i);
        alignedFraction.update(a.minAlignedFraction);
        markerCount.update(a.markerCount);
        maxDrift.update(a.maxDrift);
        maxSkip.update(a.maxSkip);
        maxTrim.update(a.trim);
    }
    out.minAlignedFraction = alignedFraction.thresholdByCumulativeProportion(percentiles[1]);
    out.minAlignedMarkerCount = uint64_t(std::round(markerCount.thresholdByCumulativeProportion(percentiles[0])));
    out.maxDrift = uint64_t(std::round(maxDrift.thresholdByCumulativeProportion(1 - percentiles[3])));
    out.maxSkip = uint64_t(std::round(maxSkip.thresholdByCumulativeProportion(1 - percentiles[2])));
    out.maxTrim = uint64_t(std::round(maxTrim.thresholdByCumulativeProportion(1 - percentiles[4])));
    eligible.resize(n);
    for(uint64_t i = 0; i < n; i++) {
        const AlignmentIndicators a = indicators(rec + kAlignmentWords * i);
        eligible[i] = !(a.minAlignedFraction < out.minAlignedFraction) && !(a.markerCount < out.minAlignedMarkerCount) &&
                      !(a.maxDrift > out.maxDrift) && !(a.maxSkip > out.maxSkip) && !(a.trim > out.maxTrim);
    }
}

void createReadGraph(shb_context* c, void* alignmentData, uint64_t n, uint64_t readCount, uint32_t maxAlignmentCount,
                     const uint8_t* eligibleHost,
                     uint8_t** keepOut, void** edgesOut, uint64_t* edgeCountOut, uint32_t** connectivityTocOut, uint32_t** connectivityDataOut)
{
    SHB_REQUIRE(4 * n < (1ull << 32), SHB_ERR_INVALID, "Too many alignments for one read graph (limit 2^30-1).");
    SHB_REQUIRE(readCount < (1ull << 31), SHB_ERR_INVALID, "Too many reads.");
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    uint32_t* rec = static_cast<uint32_t*>(alignmentData);
    const uint32_t rows = uint32_t(2 * readCount);
    HostBlocks hb;
    uint8_t* keepHost = (uint8_t*)(hb.p[0] = allocHostResult(n + 1));
    uint32_t* toc = (uint32_t*)(hb.p[1] = allocHostResult(4ull * (uint64_t(rows) + 1)));
    SHB_REQUIRE(keepHost && toc, SHB_ERR_OOM, "Out of host memory for the read graph.");
    for(uint64_t i = 0; i < n; i++) {
        SHB_REQUIRE(rec[kAlignmentWords * i] < readCount && rec[kAlignmentWords * i + 1] < readCount, SHB_ERR_INVALID,
                    "One of the alignments refers to a read that does not exist.");
    }
    DeviceBuffer<uint32_t> dRec, valsA, valsB, keep, keepIndex, scanWs, dToc, dEdges;
    DeviceBuffer<uint8_t> dEligible;
    DeviceBuffer<uint64_t> keysA, keysB;
    const uint32_t items = uint32_t(2 * n);
    uint32_t edgeCount = 0;
    if(n) {
        dRec.reserve(uint64_t(kAlignmentWords) * n); keysA.reserve(2ull * items + 4); keysB.reserve(2ull * items + 4);
        valsA.reserve(2ull * items + 4); valsB.reserve(2ull * items + 4);
        keep.reserve(n); keepIndex.reserve(n); scanWs.reserve(scanWorkspaceElements(n));
        SHB_CUDA(cudaMemcpyAsync(dRec.get(), rec, 4ull * kAlignmentWords * n, cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemsetAsync(keep.get(), 0, 4ull * n, st));
        if(maxAlignmentCount) {
            if(eligibleHost) {
                dEligible.reserve(n);
                SHB_CUDA(cudaMemcpyAsync(dEligible.get(), eligibleHost, n, cudaMemcpyHostToDevice, st));
            }
            SHB_LAUNCH(readGraphItemsKernel, ceilDiv(items, 256), 256, 0, st, (const uint32_t*)dRec.get(),
                       (const uint8_t*)(eligibleHost ? dEligible.get() : nullptr), uint32_t(n), keysA.get(), valsA.get());
            const int ranges[2][2] = {{0, 32}, {32, 63}};          // read id (or the "no read" mark) in 31 bits
            const bool inB = radixSort<true>(keysA.get(), keysB.get(), valsA.get(), valsB.get(), items, ranges, 2, c->sortWs, st);
            SHB_LAUNCH(readGraphKeepKernel, ceilDiv(items, 256), 256, 0, st, (const uint64_t*)(inB ? keysB.get() : keysA.get()),
                       (const uint32_t*)(inB ? valsB.get() : valsA.get()), items, maxAlignmentCount, keep.get());
        }
        uint32_t* totalDev = reinterpret_cast<uint32_t*>(c->scalars.get() + 32);
        exclusiveScan<uint32_t>(keep.get(), keepIndex.get(), n, totalDev, scanWs.get(), st);
        uint32_t kept = 0;
        SHB_CUDA(cudaMemcpyAsync(&kept, totalDev, sizeof(kept), cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        edgeCount = 2u * kept;
    }
    uint32_t* edges = (uint32_t*)(hb.p[2] = allocHostResult(16ull * edgeCount + 16));
    uint32_t* data = (uint32_t*)(hb.p[3] = allocHostResult(4ull * (2ull * edgeCount) + 4));
    SHB_REQUIRE(edges && data, SHB_ERR_OOM, "Out of host memory for the read graph.");
    if(edgeCount == 0) {
        memset(toc, 0, 4ull * (uint64_t(rows) + 1));
        memset(keepHost, 0, n);
    } else {
        const uint32_t entries = 2u * edgeCount;
        dEdges.reserve(4ull * edgeCount); dToc.reserve(uint64_t(rows) + 1);
        // the item buffers are free again: reuse them for the (row, edge) entries
        SHB_LAUNCH(readGraphEdgesKernel, ceilDiv(n, 256), 256, 0, st, (const uint32_t*)dRec.get(), uint32_t(n), (const uint32_t*)keep.get(),
                   (const uint32_t*)keepIndex.get(), entries, dEdges.get(), keysA.get(), valsA.get());
        uint32_t rowBits = 1;
        while((1ull << rowBits) < uint64_t(rows)) rowBits++;
        const int ranges[1][2] = {{32, 32 + int(rowBits)}};
        const bool inB = radixSort<true>(keysA.get(), keysB.get(), valsA.get(), valsB.get(), entries, ranges, 1, c->sortWs, st);
        SHB_LAUNCH(readGraphTocKernel, ceilDiv(uint64_t(rows) + 1, 256), 256, 0, st, (const uint64_t*)(inB ? keysB.get() : keysA.get()),
                   entries, rows, dToc.get());
        SHB_CUDA(cudaMemcpyAsync(toc, dToc.get(), 4ull * (uint64_t(rows) + 1), cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaMemcpyAsync(data, inB ? valsB.get() : valsA.get(), 4ull * entries, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaMemcpyAsync(edges, dEdges.get(), 16ull * edgeCount, cudaMemcpyDeviceToHost, st));
        // keep flags as bytes: narrow on the host (n words)
        std::vector<uint32_t> keepWords(n);
        SHB_CUDA(cudaMemcpyAsync(keepWords.data(), keep.get(), 4ull * n, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        for(uint64_t i = 0; i < n; i++) keepHost[i] = uint8_t(keepWords[i]);
    }
    // src/AssemblerReadGraph.cpp:134,140: SHASTA_ASSERT(edge.orientedReadIds[0] < edge.orientedReadIds[1]) for every kept
    // alignment, on the edge and on its reverse complement. Checked before isInReadGraph is written, so a refused call leaves
    // the records as they were.
    for(uint64_t i = 0; i < n; i++) {
        if(!keepHost[i]) continue;
        const uint32_t* r = rec + kAlignmentWords * i;
        const uint32_t o0 = 2u * r[0], o1 = 2u * r[1] + ((r[2] & 0xffu) ? 0u : 1u);
        SHB_REQUIRE(o0 < o1 && (o0 ^ 1u) < (o1 ^ 1u), SHB_ERR_INVALID,
                    "Alignment " + std::to_string(i) + " (reads " + std::to_string(r[0]) + " and " + std::to_string(r[1]) +
                    ((r[2] & 0xffu) ? ", same strand" : ", opposite strands") +
                    ") is kept for the read graph but its oriented reads are not in increasing order.");
    }
    // AlignmentInfo::isInReadGraph (src/Alignment.hpp:194: bit 0 of the flag byte after maxDrift), src/AssemblerReadGraph.cpp:103.
    for(uint64_t i = 0; i < n; i++) {
        uint32_t& w = rec[kAlignmentWords * i + 15];
        w = (w & ~1u) | uint32_t(keepHost[i] & 1u);
    }
    *keepOut = keepHost; *edgesOut = edges; *edgeCountOut = edgeCount; *connectivityTocOut = toc; *connectivityDataOut = data;
    hb.disarm();
}

} // namespace shb
