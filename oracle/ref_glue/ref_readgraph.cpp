// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
// extern "C" access to the read graph stage of the reference and to the tables it reads, linked into
// oracle/_ref/libshasta_ref.so:
//   Assembler::computeAlignmentTable            src/AssemblerAlign.cpp:509-571
//   AlignmentCandidates::computeCandidateTable  src/AssemblerAlignmentCandidates.cpp:388-448
//   Assembler::createReadGraph                  src/AssemblerReadGraph.cpp:35-103 (ReadGraph.creationMethod 0)
//   Assembler::createReadGraph2                 src/AssemblerReadGraph2.cpp:69-248 (ReadGraph.creationMethod 2)
//   createReadGraphUsingSelectedAlignments      src/AssemblerReadGraph.cpp:108-160
// Assembler cannot be linked here, so this glue follows the members' control flow over the reference's own objects, compiled
// from where they lie: anonymous MemoryMapped::VectorOfVectors and MemoryMapped::Vector (the row fill, including the order in
// which store() fills a row, is theirs), AlignmentData / AlignmentInfo, OrientedReadId, OrientedReadPair::getOther,
// ReadGraphEdge, Histogram2 and std::nth_element. Used to pin oracle/readgraph_oracle.c, oracle/align_oracle.c's tables and
// the device; nothing here is product code.
#include "Alignment.hpp"
#include "Histogram.hpp"
#include "ReadGraph.hpp"
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <functional>
#include <stdexcept>
#include <vector>
using namespace shasta;

namespace {
constexpr size_t kPageSize = 4096;
static_assert(sizeof(AlignmentData) == 64, "AlignmentData is 16 words");
static_assert(sizeof(OrientedReadPair) == 12, "OrientedReadPair is 3 words");
static_assert(sizeof(ReadGraphEdge) == 16, "ReadGraphEdge is 4 words");

// computeAlignmentTable / computeCandidateTable: the same control flow over AlignmentData or OrientedReadPair records.
template<class Item, class Int> void computePairTable(const Item* items, uint64_t n, ReadId readCount,
                                                      MemoryMapped::VectorOfVectors<Int, Int>& table)
{
    table.createNew("", kPageSize);
    table.beginPass1(ReadId(2 * readCount));
    for(uint64_t i = 0; i < n; i++) {
        const OrientedReadPair& pair = items[i];
        OrientedReadId orientedReadId0(pair.readIds[0], 0);
        OrientedReadId orientedReadId1(pair.readIds[1], pair.isSameStrand ? 0 : 1);
        table.incrementCount(orientedReadId0.getValue());
        table.incrementCount(orientedReadId1.getValue());
        orientedReadId0.flipStrand();
        orientedReadId1.flipStrand();
        table.incrementCount(orientedReadId0.getValue());
        table.incrementCount(orientedReadId1.getValue());
    }
    table.beginPass2();
    for(Int i = 0; i < n; i++) {
        const OrientedReadPair& pair = items[i];
        OrientedReadId orientedReadId0(pair.readIds[0], 0);
        OrientedReadId orientedReadId1(pair.readIds[1], pair.isSameStrand ? 0 : 1);
        table.store(orientedReadId0.getValue(), i);
        table.store(orientedReadId1.getValue(), i);
        orientedReadId0.flipStrand();
        orientedReadId1.flipStrand();
        table.store(orientedReadId0.getValue(), i);
        table.store(orientedReadId1.getValue(), i);
    }
    table.endPass2();
    // Sort each section by (other OrientedReadId, index): pair<OrientedReadId, uint32_t> in both members.
    std::vector<std::pair<OrientedReadId, uint32_t>> v;
    for(ReadId readId0 = 0; readId0 < readCount; readId0++) {
        for(Strand strand0 = 0; strand0 < 2; strand0++) {
            const OrientedReadId orientedReadId0(readId0, strand0);
            const auto section = table[orientedReadId0.getValue()];
            v.clear();
            for(const Int index : section) v.push_back(std::make_pair(items[index].getOther(orientedReadId0), uint32_t(index)));
            std::sort(v.begin(), v.end());
            for(size_t i = 0; i < v.size(); i++) section[i] = v[i].second;
        }
    }
}

template<class Int, class Out> void copyTable(const MemoryMapped::VectorOfVectors<Int, Int>& table, Out* toc, Out* data)
{
    toc[0] = 0;
    for(uint64_t r = 0; r < table.size(); r++) {
        toc[r + 1] = Out(toc[r] + table.size(r));
        for(uint64_t j = 0; j < table.size(r); j++) data[toc[r] + j] = Out(table.begin(r)[j]);
    }
}

// Assembler::assemblerInfo's actual* members (src/Assembler.hpp:154-158), set by setReadGraph2Criteria.
struct Criteria { double minAlignedFraction; uint64_t minAlignedMarkerCount, maxDrift, maxSkip, maxTrim; };

// setReadGraph2Criteria, src/AssemblerReadGraph2.cpp:94-179 (without its csv files).
Criteria setReadGraph2Criteria(const std::vector<AlignmentData>& alignmentData, double markerCountPercentile,
                               double alignedFractionPercentile, double maxSkipPercentile, double maxDriftPercentile,
                               double maxTrimPercentile)
{
    Histogram2 alignedFractionHistogram(0, 1, 100, false, false, true);
    Histogram2 markerCountHistogram(0, 3000, 300, false, false, true);
    Histogram2 maxDriftHistogram(0, 100, 100, false, false, true);
    Histogram2 maxSkipHistogram(0, 100, 100, false, false, true);
    Histogram2 maxTrimHistogram(0, 100, 100, false, false, true);
    for(size_t i = 0; i < alignmentData.size(); i++) {
        const auto info = alignmentData[i].info;
        const auto trims = info.computeTrim();
        const auto trim = std::max(trims.first, trims.second);
        alignedFractionHistogram.update(info.minAlignedFraction());
        markerCountHistogram.update(info.markerCount);
        maxDriftHistogram.update(info.maxDrift);
        maxSkipHistogram.update(info.maxSkip);
        maxTrimHistogram.update(trim);
    }
    Criteria c;
    c.minAlignedFraction = alignedFractionHistogram.thresholdByCumulativeProportion(alignedFractionPercentile);
    c.minAlignedMarkerCount = uint64_t(std::round(markerCountHistogram.thresholdByCumulativeProportion(markerCountPercentile)));
    c.maxDrift = uint64_t(std::round(maxDriftHistogram.thresholdByCumulativeProportion(1 - maxDriftPercentile)));
    c.maxSkip = uint64_t(std::round(maxSkipHistogram.thresholdByCumulativeProportion(1 - maxSkipPercentile)));
    c.maxTrim = uint64_t(std::round(maxTrimHistogram.thresholdByCumulativeProportion(1 - maxTrimPercentile)));
    return c;
}

// passesReadGraph2Criteria, src/AssemblerReadGraph2.cpp:69-91.
bool passesReadGraph2Criteria(const AlignmentInfo& info, const Criteria& c)
{
    const auto trims = info.computeTrim();
    const auto trim = std::max(trims.first, trims.second);
    if(info.minAlignedFraction() < c.minAlignedFraction) return false;
    if(info.markerCount < c.minAlignedMarkerCount) return false;
    if(info.maxDrift > c.maxDrift) return false;
    if(info.maxSkip > c.maxSkip) return false;
    if(trim > c.maxTrim) return false;
    return true;
}

// createReadGraph (criteria == nullptr) or the selection of createReadGraph2, then createReadGraphUsingSelectedAlignments.
// Each read's alignments come from the alignment table built above, as in the members.
void createReadGraph(std::vector<AlignmentData>& alignmentData, ReadId readCount, uint32_t maxAlignmentCount, const Criteria* criteria,
                     std::vector<bool>& keepAlignment, MemoryMapped::Vector<ReadGraphEdge>& edges,
                     MemoryMapped::VectorOfVectors<uint32_t, uint32_t>& connectivity)
{
    MemoryMapped::VectorOfVectors<uint32_t, uint32_t> alignmentTable;
    computePairTable(alignmentData.data(), alignmentData.size(), readCount, alignmentTable);
    keepAlignment.assign(alignmentData.size(), false);
    std::vector<std::pair<uint32_t, uint32_t>> readAlignments;
    for(ReadId readId = 0; readId < readCount; readId++) {
        readAlignments.clear();
        for(const uint32_t alignmentId : alignmentTable[OrientedReadId(readId, 0).getValue()]) {
            const AlignmentInfo& info = alignmentData[alignmentId].info;
            if(criteria && !passesReadGraph2Criteria(info, *criteria)) continue;
            readAlignments.push_back(std::make_pair(info.markerCount, alignmentId));
        }
        if(readAlignments.size() > maxAlignmentCount) {
            std::nth_element(readAlignments.begin(), readAlignments.begin() + maxAlignmentCount, readAlignments.end(),
                             std::greater<std::pair<uint32_t, uint32_t>>());
            readAlignments.resize(maxAlignmentCount);
        }
        for(const auto& p : readAlignments) keepAlignment[p.second] = true;
    }
    // createReadGraphUsingSelectedAlignments
    edges.createNew("", kPageSize);
    for(size_t alignmentId = 0; alignmentId < alignmentData.size(); alignmentId++) {
        const bool keepThisAlignment = keepAlignment[alignmentId];
        AlignmentData& alignment = alignmentData[alignmentId];
        alignment.info.isInReadGraph = uint8_t(keepThisAlignment);
        if(not keepThisAlignment) continue;
        ReadGraphEdge edge;
        edge.alignmentId = alignmentId & 0x3fff'ffff'ffff'ffff;
        edge.crossesStrands = 0;
        edge.hasInconsistentAlignment = 0;
        edge.orientedReadIds[0] = OrientedReadId(alignment.readIds[0], 0);
        edge.orientedReadIds[1] = OrientedReadId(alignment.readIds[1], alignment.isSameStrand ? 0 : 1);
        SHASTA_ASSERT(edge.orientedReadIds[0] < edge.orientedReadIds[1]);
        edges.push_back(edge);
        edge.orientedReadIds[0].flipStrand();
        edge.orientedReadIds[1].flipStrand();
        SHASTA_ASSERT(edge.orientedReadIds[0] < edge.orientedReadIds[1]);
        edges.push_back(edge);
    }
    connectivity.createNew("", kPageSize);
    connectivity.beginPass1(2 * readCount);
    for(const ReadGraphEdge& edge : edges) {
        connectivity.incrementCount(edge.orientedReadIds[0].getValue());
        connectivity.incrementCount(edge.orientedReadIds[1].getValue());
    }
    connectivity.beginPass2();
    for(size_t i = 0; i < edges.size(); i++) {
        const ReadGraphEdge& edge = edges[i];
        connectivity.store(edge.orientedReadIds[0].getValue(), uint32_t(i));
        connectivity.store(edge.orientedReadIds[1].getValue(), uint32_t(i));
    }
    connectivity.endPass2();
}

// records uint32[n][16] in/out (isInReadGraph), keep uint8[n], edges uint32[2n][4], connToc uint32[2R+1], connData uint32[4n].
int readGraphEntry(const char* what, uint32_t* records, uint64_t n, uint64_t readCount, uint32_t maxAlignmentCount,
                   const double* percentiles, void* criteriaOut, uint8_t* keep, uint32_t* edgesOut, uint64_t* edgeCount,
                   uint32_t* connToc, uint32_t* connData)
{
    try {
        std::vector<AlignmentData> alignmentData(n);
        if(n) std::memcpy(static_cast<void*>(alignmentData.data()), records, 64 * n);
        Criteria criteria;
        if(percentiles) {
            criteria = setReadGraph2Criteria(alignmentData, percentiles[0], percentiles[1], percentiles[2], percentiles[3], percentiles[4]);
            std::memcpy(criteriaOut, &criteria, sizeof(criteria));
        }
        std::vector<bool> keepAlignment;
        MemoryMapped::Vector<ReadGraphEdge> edges;
        MemoryMapped::VectorOfVectors<uint32_t, uint32_t> connectivity;
        createReadGraph(alignmentData, ReadId(readCount), maxAlignmentCount, percentiles ? &criteria : nullptr, keepAlignment, edges,
                        connectivity);
        if(n) std::memcpy(records, static_cast<const void*>(alignmentData.data()), 64 * n);
        for(uint64_t i = 0; i < n; i++) keep[i] = keepAlignment[i] ? 1 : 0;
        *edgeCount = edges.size();
        if(edges.size()) std::memcpy(edgesOut, static_cast<const void*>(edges.begin()), 16 * edges.size());
        copyTable(connectivity, connToc, connData);
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "%s: %s\n", what, e.what());
        return 1;
    }
}
}

extern "C" {

double ref_histogram2_threshold(const double* x, uint64_t n, double start, double stop, uint64_t binCount, double fraction)
{
    Histogram2 h(start, stop, binCount, false, false, true);
    for(uint64_t i = 0; i < n; i++) h.update(x[i]);
    return h.thresholdByCumulativeProportion(fraction);
}

// out: minAlignedFraction, markerCount, maxDrift, maxSkip, max(leftTrim, rightTrim) of a 64-byte AlignmentData record's info
void ref_alignment_indicators(const uint32_t* record16, double* out5)
{
    static_assert(sizeof(AlignmentInfo) == 52, "AlignmentInfo is 13 words");
    AlignmentInfo info;
    std::memcpy(&info, record16 + 3, sizeof(info));
    const auto trims = info.computeTrim();
    out5[0] = info.minAlignedFraction();
    out5[1] = double(info.markerCount);
    out5[2] = double(info.maxDrift);
    out5[3] = double(info.maxSkip);
    out5[4] = double(std::max(trims.first, trims.second));
}

// Status: 0 ok, 1 a reference assertion or exception (message on stderr). toc uint32[2R+1], data uint32[4n].
int ref_compute_alignment_table(const uint32_t* records, uint64_t n, uint64_t readCount, uint32_t* toc, uint32_t* data)
{
    try {
        std::vector<AlignmentData> alignmentData(n);
        if(n) std::memcpy(static_cast<void*>(alignmentData.data()), records, 64 * n);
        MemoryMapped::VectorOfVectors<uint32_t, uint32_t> table;
        computePairTable(alignmentData.data(), n, ReadId(readCount), table);
        copyTable(table, toc, data);
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_compute_alignment_table: %s\n", e.what());
        return 1;
    }
}

// candidates: 12-byte OrientedReadPair records. toc uint64[2R+1], data uint64[4n].
int ref_compute_candidate_table(const uint32_t* candidates, uint64_t n, uint64_t readCount, uint64_t* toc, uint64_t* data)
{
    try {
        std::vector<OrientedReadPair> pairs(n);
        if(n) std::memcpy(static_cast<void*>(pairs.data()), candidates, 12 * n);
        MemoryMapped::VectorOfVectors<uint64_t, uint64_t> table;
        computePairTable(pairs.data(), n, ReadId(readCount), table);
        copyTable(table, toc, data);
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_compute_candidate_table: %s\n", e.what());
        return 1;
    }
}

int ref_create_read_graph(uint32_t* records, uint64_t n, uint64_t readCount, uint32_t maxAlignmentCount, uint8_t* keep,
                          uint32_t* edges, uint64_t* edgeCount, uint32_t* connToc, uint32_t* connData)
{
    return readGraphEntry("ref_create_read_graph", records, n, readCount, maxAlignmentCount, nullptr, nullptr, keep, edges, edgeCount,
                          connToc, connData);
}

// percentiles: markerCount, alignedFraction, maxSkip, maxDrift, maxTrim (the member's argument order). criteria: double
// minAlignedFraction, then uint64 minAlignedMarkerCount, maxDrift, maxSkip, maxTrim.
int ref_create_read_graph2(uint32_t* records, uint64_t n, uint64_t readCount, uint32_t maxAlignmentCount, const double* percentiles,
                           void* criteria, uint8_t* keep, uint32_t* edges, uint64_t* edgeCount, uint32_t* connToc, uint32_t* connData)
{
    return readGraphEntry("ref_create_read_graph2", records, n, readCount, maxAlignmentCount, percentiles, criteria, keep, edges, edgeCount,
                          connToc, connData);
}

} // extern "C"
