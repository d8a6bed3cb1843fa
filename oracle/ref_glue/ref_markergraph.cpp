// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
// extern "C" access to Assembler::createMarkerGraphVertices (src/AssemblerMarkerGraph.cpp:38-518, threads :522-770) and
// findMarkerGraphReverseComplementVertices (:1134-1230), built by oracle/Makefile into
// oracle/_ref/libshasta_ref_markergraph.so. Assembler cannot be linked here, so this glue follows the members' control flow
// over the reference's own components, compiled unmodified from where they lie:
//   DisjointSets          src/dset64-gccAtomic.hpp   (concurrent union-find, used by threadCount threads as in :124-152)
//   shasta::decompress    src/compressAlignment.cpp
//   shasta::PeakFinder    src/PeakFinder.cpp
//   MemoryMapped::Vector  src/MemoryMappedVector.hpp (to open the Uint40 files the facade writes)
// The MemoryMapped containers of the member are plain vectors here. The vertex numbering is the reference's: sets in
// increasing order of their DisjointSets representative, which depends on the thread schedule when threadCount > 1.
#include "compressAlignment.hpp"
#include "dset64-gccAtomic.hpp"
#include "MemoryMappedVector.hpp"
#include "PeakFinder.hpp"
#include "Uint.hpp"

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <thread>
#include <vector>

using namespace shasta;

namespace {
constexpr uint64_t kInvalidVertex = std::numeric_limits<uint64_t>::max();     // MarkerGraph::invalidVertexId
constexpr uint64_t kInvalid40 = (1ull << 40) - 1;                            // invalidCompressedVertexId as Uint40

struct Markers {
    const uint64_t* toc; uint64_t rows;
    uint64_t size(uint64_t o) const { return toc[o + 1] - toc[o]; }
    uint64_t orientedReadOf(uint64_t m) const        // shasta::findMarkerId (src/Marker.cpp)
    {
        return uint64_t(std::upper_bound(toc, toc + rows + 1, m) - toc) - 1;
    }
    uint64_t reverseComplement(uint64_t m) const     // src/AssemblerMarkers.cpp:140-153
    {
        const uint64_t o = orientedReadOf(m), ordinal = m - toc[o];
        return toc[o ^ 1] + (size(o) - 1 - ordinal);
    }
};

template<class F> void runThreads(uint64_t n, uint64_t threads, F f)      // getNextBatch over batches of 10000
{
    std::atomic<uint64_t> next(0);
    auto body = [&] { for(;;) { const uint64_t b = next.fetch_add(10000); if(b >= n) return; f(b, std::min(n, b + 10000)); } };
    if(threads <= 1) { body(); return; }
    std::vector<std::thread> t;
    for(uint64_t i = 0; i < threads; i++) t.emplace_back(body);
    for(auto& x : t) x.join();
}
}

extern "C" {

// Status: 0 ok, 1 a reference assertion or exception (message on stderr).
// params: minCoverage, maxCoverage, minCoveragePerStrand, allowDuplicateMarkers, peakFinderAreaStartIndex, threadCount.
// counts[12]: minCoverageUsed, peakFinderFailed, (unused), (unused), (unused), disjointSets, kept, bad, V, histogramSize,
//             total vertex markers, observedPercentArea (bits of a double). Outputs malloc'ed, ref_free_markergraph.
int ref_create_marker_graph_vertices(const uint64_t* toc, uint64_t R, const uint32_t* kmerIds, const uint32_t* edges, uint64_t edgeCount,
                                     const uint64_t* ctoc, const uint8_t* cdata, uint64_t alignmentCount, const uint8_t* readFlags,
                                     const uint64_t* params, double peakFinderMinAreaFraction,
                                     uint64_t** tableOut, uint64_t** vtocOut, uint64_t** vdataOut, uint64_t** histOut, uint64_t* counts)
{
    try {
        const Markers markers{toc, 2 * R};
        const uint64_t M = toc[2 * R];
        uint64_t minCoverage = params[0];
        const uint64_t maxCoverage = params[1], minCoveragePerStrand = params[2];
        const bool allowDuplicateMarkers = params[3] != 0;
        const uint64_t threads = params[5] ? params[5] : 1;
        std::memset(counts, 0, 12 * 8);
        // :99-115
        std::vector<DisjointSets::Aint> table(M + 1);
        DisjointSets dsets(table.data(), M);
        // :119-124, :537-606
        SHASTA_ASSERT(edgeCount % 2 == 0);
        runThreads(edgeCount / 2, threads, [&](uint64_t b, uint64_t e) {
            Alignment alignment;
            for(uint64_t pair = b; pair < e; pair++) {
                const uint64_t i = 2 * pair;
                const uint32_t* edge = edges + 4 * i;
                const uint32_t* next = edges + 4 * (i + 1);
                SHASTA_ASSERT((next[0] ^ 1u) == edge[0] && (next[1] ^ 1u) == edge[1]);
                if(edge[3] >> 30) continue;                                 // crossesStrands, hasInconsistentAlignment
                SHASTA_ASSERT(edge[0] < edge[1]);
                if((readFlags[edge[0] >> 1] | readFlags[edge[1] >> 1]) & 2u) continue;     // isChimeric
                const uint64_t alignmentId = uint64_t(edge[2]) | (uint64_t(edge[3] & 0x3fffffffu) << 32);
                SHASTA_ASSERT(alignmentId < alignmentCount);
                const span<const char> compressed(reinterpret_cast<const char*>(cdata + ctoc[alignmentId]),
                                                  reinterpret_cast<const char*>(cdata + ctoc[alignmentId + 1]));
                shasta::decompress(compressed, alignment);
                for(const auto& p : alignment.ordinals) {
                    const uint64_t m0 = toc[edge[0]] + p[0], m1 = toc[edge[1]] + p[1];
                    SHASTA_ASSERT(kmerIds[m0] == kmerIds[m1]);
                    dsets.unite(m0, m1);
                    dsets.unite(markers.reverseComplement(m0), markers.reverseComplement(m1));
                }
            }
        });
        // :131-166
        uint64_t pass = 1;
        do {
            dsets.parentUpdated = 0;
            runThreads(M, threads, [&](uint64_t b, uint64_t e) { for(uint64_t i = b; i < e; i++) dsets.find(i, true); });
            pass++;
        } while(dsets.parentUpdated > 0 && pass <= 10);
        SHASTA_ASSERT(pass <= 10);
        std::vector<uint64_t> disjointSetTable(M);
        for(uint64_t i = 0; i < M; i++) { SHASTA_ASSERT(dsets.parent(i) == dsets.find(i)); disjointSetTable[i] = dsets.parent(i); }
        // :186-231
        std::vector<uint64_t> workArea(M, 0);
        for(uint64_t i = 0; i < M; i++) workArea[disjointSetTable[i]]++;
        std::vector<uint64_t> histogram;
        for(uint64_t i = 0; i < M; i++) {
            const uint64_t markerCount = workArea[i];
            if(markerCount == 0) continue;
            if(markerCount >= histogram.size()) histogram.resize(markerCount + 1, 0);
            ++histogram[markerCount];
            counts[5]++;
        }
        // :233-254
        if(minCoverage == 0) {
            try {
                PeakFinder p;
                p.findPeaks(histogram);
                minCoverage = p.findXCutoff(histogram, peakFinderMinAreaFraction, params[4]);
            } catch(PeakFinderException& e) {
                minCoverage = 5;
                counts[1] = 1;
                const double observed = e.observedPercentArea;
                std::memcpy(&counts[11], &observed, 8);
            }
        }
        counts[0] = minCoverage;
        // :266-305
        uint64_t newDisjointSetId = 0;
        for(uint64_t i = 0; i < M; i++) {
            auto& w = workArea[i];
            if(w < minCoverage || w > maxCoverage) w = kInvalidVertex; else w = newDisjointSetId++;
        }
        const uint64_t disjointSetCount = newDisjointSetId;
        for(uint64_t i = 0; i < M; i++) disjointSetTable[i] = workArea[disjointSetTable[i]];
        // :324-345
        std::vector<std::vector<uint64_t>> disjointSetMarkers(disjointSetCount);
        for(uint64_t i = 0; i < M; i++) if(disjointSetTable[i] != kInvalidVertex) disjointSetMarkers[disjointSetTable[i]].push_back(i);
        for(auto& v : disjointSetMarkers) std::sort(v.begin(), v.end());
        // :377-389, :697-745
        std::vector<bool> isBad(disjointSetCount, false);
        for(uint64_t d = 0; d < disjointSetCount; d++) {
            const auto& m = disjointSetMarkers[d];
            const size_t markerCount = m.size();
            SHASTA_ASSERT(markerCount > 0);
            if(markerCount == 1) { if(1 < minCoveragePerStrand) isBad[d] = true; continue; }
            uint64_t countByStrand[2] = {0, 0};
            for(size_t j = 0; j < markerCount; j++) {
                const uint64_t o = markers.orientedReadOf(m[j]);
                ++countByStrand[o & 1];
                if(!allowDuplicateMarkers && j > 0 && (markers.orientedReadOf(m[j - 1]) >> 1) == (o >> 1)) { isBad[d] = true; break; }
            }
            if(!isBad[d]) isBad[d] = countByStrand[0] < minCoveragePerStrand || countByStrand[1] < minCoveragePerStrand;
        }
        const uint64_t bad = std::count(isBad.begin(), isBad.end(), true);
        // :393-464
        std::vector<uint64_t> renumber(disjointSetCount);
        newDisjointSetId = 0;
        for(uint64_t d = 0; d < disjointSetCount; d++) renumber[d] = isBad[d] ? kInvalidVertex : newDisjointSetId++;
        SHASTA_ASSERT(newDisjointSetId + bad == disjointSetCount);
        uint64_t* vt = (uint64_t*)malloc(8 * (M + 1));
        for(uint64_t i = 0; i < M; i++) {
            const uint64_t old = disjointSetTable[i];
            vt[i] = (old == kInvalidVertex) ? kInvalid40 : (renumber[old] & kInvalid40);       // Uint40 of invalidVertexId
        }
        const uint64_t V = newDisjointSetId;
        uint64_t vm = 0;
        for(uint64_t d = 0; d < disjointSetCount; d++) if(!isBad[d]) vm += disjointSetMarkers[d].size();
        uint64_t* vtoc = (uint64_t*)malloc(8 * (V + 1));
        uint64_t* vdata = (uint64_t*)malloc(8 * (vm + 1));
        vtoc[0] = 0;
        for(uint64_t d = 0, v = 0; d < disjointSetCount; d++) {
            if(isBad[d]) continue;
            std::memcpy(vdata + vtoc[v], disjointSetMarkers[d].data(), 8 * disjointSetMarkers[d].size());
            vtoc[v + 1] = vtoc[v] + disjointSetMarkers[d].size();
            v++;
        }
        uint64_t* hist = (uint64_t*)malloc(8 * (histogram.size() + 1));
        if(!histogram.empty()) std::memcpy(hist, histogram.data(), 8 * histogram.size());
        counts[6] = disjointSetCount; counts[7] = bad; counts[8] = V; counts[9] = histogram.size(); counts[10] = vm;
        *tableOut = vt; *vtocOut = vtoc; *vdataOut = vdata; *histOut = hist;
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_create_marker_graph_vertices: %s\n", e.what());
        return 1;
    }
}

// :1177-1230. Returns 0, or 1 on a reference assertion.
int ref_find_rc_vertices(const uint64_t* toc, uint64_t R, const uint64_t* table, const uint64_t* vtoc, const uint64_t* vdata, uint64_t V,
                         uint64_t* rc)
{
    try {
        const Markers markers{toc, 2 * R};
        for(uint64_t v = 0; v < V; v++) {
            SHASTA_ASSERT(vtoc[v + 1] > vtoc[v]);
            const uint64_t r = table[markers.reverseComplement(vdata[vtoc[v]])];
            SHASTA_ASSERT(r != kInvalid40);
            for(uint64_t j = vtoc[v]; j < vtoc[v + 1]; j++) SHASTA_ASSERT(table[markers.reverseComplement(vdata[j])] == r);
            rc[v] = r;
        }
        for(uint64_t v = 0; v < V; v++) SHASTA_ASSERT(rc[rc[v]] == v);
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_find_rc_vertices: %s\n", e.what());
        return 1;
    }
}

// PeakFinder::findPeaks + findXCutoff. Returns 1 when they throw PeakFinderException (*observed = observedPercentArea).
int ref_peak_finder_cutoff(const uint64_t* y, uint64_t n, double minAreaFraction, uint64_t startIndex, uint64_t* cutoff, double* observed)
{
    const std::vector<uint64_t> h(y, y + n);
    *observed = 0;
    try {
        PeakFinder p;
        p.findPeaks(h);
        *cutoff = p.findXCutoff(h, minAreaFraction, startIndex);
        return 0;
    } catch(PeakFinderException& e) {
        *observed = e.observedPercentArea;
        return 1;
    }
}

// Object count of a MemoryMapped::Vector<Uint40> file (Data/MarkerGraphVertexTable, MarkerGraphVertices.toc) as the
// reference's own accessExistingReadOnly sees it, and its values. Returns nonzero on failure.
int ref_open_vector40(const char* path, uint64_t* count, uint64_t** values)
{
    try {
        MemoryMapped::Vector<Uint40> v;
        v.accessExistingReadOnly(path);
        *count = v.size();
        uint64_t* out = (uint64_t*)malloc(8 * (v.size() + 1));
        for(uint64_t i = 0; i < v.size(); i++) out[i] = uint64_t(v[i]);
        *values = out;
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_open_vector40: %s\n", e.what());
        return 1;
    }
}

void ref_free_markergraph(void* p) { free(p); }

} // extern "C"
