// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
// extern "C" access to Assembler::flagCrossStrandReadGraphEdges1 (src/AssemblerReadGraph.cpp:775-1041) and
// Assembler::flagChimericReads (:355-583), built by oracle/readgraph_flags.mk into oracle/_ref/libshasta_ref_readgraph_flags.so.
// Assembler cannot be linked here, so this glue follows the members' control flow over the reference's own objects,
// compiled unmodified from where they lie:
//   ReadGraph, ReadGraphEdge, ReadGraph::computeShortPath   src/ReadGraph.{hpp,cpp}
//   OrderPairsBySecondOnly, OrderPairsBySecondOnlyGreater   src/orderPairs.hpp (with std::sort, as the member)
//   MemoryMapped::Vector / VectorOfVectors (anonymous), AlignmentData, OrientedReadId, ReadFlags
//   boost::disjoint_sets                                    the shim in oracle/ref_glue/shims (boost is absent)
// The batches of 10000 reads over threadCount threads are the members' (setupLoadBalancing / getNextBatch).
#include "Alignment.hpp"
#include "orderPairs.hpp"
#include "ReadFlags.hpp"
#include "ReadGraph.hpp"
#include <boost/pending/disjoint_sets.hpp>

#include <algorithm>
#include <array>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <map>
#include <queue>
#include <stdexcept>
#include <thread>
#include <vector>

using namespace shasta;

namespace {
constexpr size_t kPageSize = 4096;

template<class F> void runThreads(uint64_t n, uint64_t threads, F f)
{
    std::atomic<uint64_t> next(0);
    auto body = [&] { for(;;) { const uint64_t b = next.fetch_add(10000); if(b >= n) return; f(b, std::min(n, b + 10000)); } };
    if(threads <= 1) { body(); return; }
    std::vector<std::thread> t;
    for(uint64_t i = 0; i < threads; i++) t.emplace_back(body);
    for(auto& x : t) x.join();
}

// The read graph as the member sees it: the edges, and each connectivity row in the caller's order (store() fills a row
// from its end, so each row is stored back to front).
void load(ReadGraph& g, const ReadGraphEdge* edges, uint64_t edgeCount, const uint32_t* toc, const uint32_t* data, uint64_t rows)
{
    g.edges.createNew("", kPageSize);
    for(uint64_t e = 0; e < edgeCount; e++) g.edges.push_back(edges[e]);
    g.connectivity.createNew("", kPageSize);
    g.connectivity.beginPass1(rows);
    for(uint64_t v = 0; v < rows; v++) for(uint32_t p = toc[v]; p < toc[v + 1]; p++) g.connectivity.incrementCount(v);
    g.connectivity.beginPass2();
    for(uint64_t v = 0; v < rows; v++) for(uint32_t p = toc[v + 1]; p-- > toc[v];) g.connectivity.store(v, data[p]);
    g.connectivity.endPass2();
}
}

extern "C" {

// Opens a Data/ReadGraphEdges file with the reference's MemoryMapped::Vector<ReadGraphEdge> and copies up to `capacity`
// records to out; *count receives the number of records. Status 0 ok, 1 the reference could not open it.
int ref_open_read_graph_edges(const char* path, void* out, uint64_t capacity, uint64_t* count)
{
    try {
        MemoryMapped::Vector<ReadGraphEdge> v;
        v.accessExistingReadOnly(path);
        *count = v.size();
        std::memcpy(out, v.begin(), 16 * std::min<uint64_t>(capacity, v.size()));
        return 0;
    } catch(const std::exception& e) {
        std::fprintf(stderr, "ref_open_read_graph_edges: %s\n", e.what());
        return 1;
    }
}

// Status 0 ok, 1 a reference assertion or exception (message on stderr). counts[3]: the printed near-strand-jump count,
// the strand jump regions, the edges flagged. edges (16-byte ReadGraphEdge) and alignmentData are rewritten in place.
int ref_flag_cross_strand_read_graph_edges1(int64_t maxDistance, void* edgesIo, uint64_t edgeCount, const uint32_t* toc,
                                            const uint32_t* data, uint64_t readCount, void* alignmentDataIo, uint64_t threadCount,
                                            uint64_t* counts)
{
    try {
        ReadGraphEdge* edgesOut = static_cast<ReadGraphEdge*>(edgesIo);
        AlignmentData* alignmentData = static_cast<AlignmentData*>(alignmentDataIo);
        const size_t orientedReadCount = 2 * readCount;
        ReadGraph readGraph;
        load(readGraph, edgesOut, edgeCount, toc, data, orientedReadCount);
        std::memset(counts, 0, 3 * 8);
        for(size_t e = 0; e < edgeCount; e++) readGraph.edges[e].crossesStrands = 0;
        if(maxDistance == 0) {
            std::memcpy(edgesOut, readGraph.edges.begin(), 16 * edgeCount);
            return 0;
        }
        // :809-813 (vector<bool> written by several threads as in the member; one thread by default)
        std::vector<bool> isNearStrandJump(orientedReadCount, false);
        std::vector<uint8_t> nearRead(readCount, 0);
        runThreads(readCount, threadCount, [&](uint64_t begin, uint64_t end) {
            std::vector<uint32_t> distance(orientedReadCount, ReadGraph::infiniteDistance), parentEdges(orientedReadCount), path;
            std::vector<OrientedReadId> reached;
            for(ReadId readId = ReadId(begin); readId != ReadId(end); readId++) {
                readGraph.computeShortPath(OrientedReadId(readId, 0), OrientedReadId(readId, 1), size_t(maxDistance), path, distance,
                                           reached, parentEdges);
                if(!path.empty()) nearRead[readId] = 1;
            }
        });
        for(ReadId r = 0; r < readCount; r++) if(nearRead[r]) isNearStrandJump[2 * r] = isNearStrandJump[2 * r + 1] = true;
        for(ReadId readId = 0; readId < readCount; readId++) if(isNearStrandJump[readId]) counts[0]++;
        // :830-863
        std::vector<ReadId> rank(orientedReadCount), parent(orientedReadCount);
        boost::disjoint_sets<ReadId*, ReadId*> disjointSets(rank.data(), parent.data());
        for(ReadId v = 0; v < orientedReadCount; v++) disjointSets.make_set(v);
        for(const ReadGraphEdge& edge : readGraph.edges) {
            const auto v0 = edge.orientedReadIds[0].getValue(), v1 = edge.orientedReadIds[1].getValue();
            if(isNearStrandJump[v0] && isNearStrandJump[v1]) disjointSets.union_set(v0, v1);
        }
        std::vector<std::vector<OrientedReadId>> componentVertices(orientedReadCount);
        for(ReadId readId = 0; readId < readCount; readId++) {
            for(Strand strand = 0; strand < 2; strand++) {
                const OrientedReadId o(readId, strand);
                if(isNearStrandJump[o.getValue()]) componentVertices[disjointSets.find_set(o.getValue())].push_back(o);
            }
        }
        // :870-1010
        for(ReadId componentId = 0; componentId != orientedReadCount; componentId++) {
            const std::vector<OrientedReadId>& vertices = componentVertices[componentId];
            const size_t vertexCount = vertices.size();
            if(vertexCount < 2) continue;
            counts[1]++;
            SHASTA_ASSERT((vertexCount % 2) == 0);
            for(size_t i = 0; i < vertexCount; i += 2) {
                SHASTA_ASSERT(vertices[i].getReadId() == vertices[i + 1].getReadId());
                SHASTA_ASSERT(vertices[i].getStrand() == 0);
                SHASTA_ASSERT(vertices[i + 1].getStrand() == 1);
            }
            std::map<OrientedReadId, uint32_t> vertexMap;
            for(uint32_t i = 0; i < vertexCount; i++) vertexMap.insert(std::make_pair(vertices[i], i));
            std::vector<std::pair<uint32_t, uint64_t>> edgeIds;
            for(const OrientedReadId o0 : vertices) {
                for(const uint32_t edgeId : readGraph.connectivity[o0.getValue()]) {
                    const ReadGraphEdge& edge = readGraph.edges[edgeId];
                    const OrientedReadId o1 = edge.getOther(o0);
                    if(vertexMap.find(o1) == vertexMap.end()) continue;
                    if(edge.orientedReadIds[0] == o0) edgeIds.push_back(std::make_pair(edgeId, uint64_t(edge.alignmentId)));
                }
            }
            SHASTA_ASSERT((edgeIds.size() % 2) == 0);
            std::sort(edgeIds.begin(), edgeIds.end(), OrderPairsBySecondOnly<uint32_t, uint64_t>());
            for(size_t i = 0; i < edgeIds.size(); i += 2) SHASTA_ASSERT(edgeIds[i].second == edgeIds[i + 1].second);
            std::vector<std::pair<std::array<uint32_t, 2>, uint32_t>> edgePairs;
            for(size_t i = 0; i < edgeIds.size(); i += 2) {
                const uint64_t alignmentId = edgeIds[i].second;
                const std::array<uint32_t, 2> edgePair = {edgeIds[i].first, edgeIds[i + 1].first};
                edgePairs.push_back(std::make_pair(edgePair, uint32_t(alignmentData[alignmentId].info.markerCount)));
            }
            std::sort(edgePairs.begin(), edgePairs.end(), OrderPairsBySecondOnlyGreater<std::array<uint32_t, 2>, uint32_t>());
            std::vector<ReadId> rrank(vertexCount), rparent(vertexCount);
            boost::disjoint_sets<ReadId*, ReadId*> regionSets(rrank.data(), rparent.data());
            for(size_t i = 0; i < vertexCount; i++) regionSets.make_set(ReadId(i));
            for(const auto& p : edgePairs) {
                for(const uint32_t edgeId : p.first) {
                    ReadGraphEdge& edge = readGraph.edges[edgeId];
                    OrientedReadId o0rc = edge.orientedReadIds[0], o1rc = edge.orientedReadIds[1];
                    o0rc.flipStrand();
                    o1rc.flipStrand();
                    const uint32_t c0 = regionSets.find_set(vertexMap[edge.orientedReadIds[0]]);
                    const uint32_t c1 = regionSets.find_set(vertexMap[edge.orientedReadIds[1]]);
                    const uint32_t c0rc = regionSets.find_set(vertexMap[o0rc]);
                    const uint32_t c1rc = regionSets.find_set(vertexMap[o1rc]);
                    SHASTA_ASSERT(c0 != c0rc);
                    SHASTA_ASSERT(c1 != c1rc);
                    if(c0 == c1rc || c1 == c0rc) {
                        edge.crossesStrands = 1;
                        alignmentData[edge.alignmentId].info.isInReadGraph = 0;
                    } else {
                        regionSets.union_set(vertexMap[edge.orientedReadIds[0]], vertexMap[edge.orientedReadIds[1]]);
                        regionSets.union_set(vertexMap[o0rc], vertexMap[o1rc]);
                    }
                }
            }
        }
        for(size_t e = 0; e < edgeCount; e++) counts[2] += readGraph.edges[e].crossesStrands;
        std::memcpy(edgesOut, readGraph.edges.begin(), 16 * edgeCount);
        return 0;
    } catch(const std::exception& e) {
        std::fprintf(stderr, "ref_flag_cross_strand_read_graph_edges1: %s\n", e.what());
        return 1;
    }
}

// Status as above. readFlags (R bytes) and alignmentData are rewritten in place; *chimericCount receives the count printed.
int ref_flag_chimeric_reads(uint64_t maxDistance, const void* edgesIn, uint64_t edgeCount, const uint32_t* toc, const uint32_t* data,
                            uint64_t readCount, uint8_t* readFlagsIo, void* alignmentDataIo, uint64_t alignmentCount,
                            uint64_t threadCount, uint64_t* chimericCount)
{
    try {
        ReadFlags* flags = reinterpret_cast<ReadFlags*>(readFlagsIo);
        AlignmentData* alignmentData = static_cast<AlignmentData*>(alignmentDataIo);
        *chimericCount = 0;
        ReadGraph readGraph;
        load(readGraph, static_cast<const ReadGraphEdge*>(edgesIn), edgeCount, toc, data, 2 * readCount);
        const size_t orientedReadCount = readGraph.connectivity.size();
        SHASTA_ASSERT((orientedReadCount % 2) == 0);
        if(maxDistance == 0) {
            for(ReadId r = 0; r < readCount; r++) flags[r].isChimeric = 0;
            return 0;
        }
        SHASTA_ASSERT(maxDistance < 255);
        // Assembler::computeAlignmentTable (src/AssemblerAlign.cpp:505-540): every alignment under both strands of both reads.
        std::vector<std::vector<uint32_t>> alignmentTable(orientedReadCount);
        for(uint32_t i = 0; i < alignmentCount; i++) {
            const AlignmentData& ad = alignmentData[i];
            OrientedReadId o0(ad.readIds[0], 0), o1(ad.readIds[1], ad.isSameStrand ? 0 : 1);
            SHASTA_ASSERT(o0.getValue() < orientedReadCount && o1.getValue() < orientedReadCount);
            alignmentTable[o0.getValue()].push_back(i);
            alignmentTable[o1.getValue()].push_back(i);
            o0.flipStrand();
            o1.flipStrand();
            alignmentTable[o0.getValue()].push_back(i);
            alignmentTable[o1.getValue()].push_back(i);
        }
        // :401-553
        runThreads(readCount, threadCount, [&](uint64_t begin, uint64_t end) {
            std::vector<uint32_t> vertexTable(orientedReadCount, std::numeric_limits<uint32_t>::max());
            const uint32_t notReached = std::numeric_limits<uint32_t>::max();
            std::vector<std::pair<OrientedReadId, uint32_t>> localVertices;
            std::queue<OrientedReadId> q;
            std::vector<uint32_t> rank, parent;
            for(ReadId startReadId = ReadId(begin); startReadId != ReadId(end); startReadId++) {
                flags[startReadId].isChimeric = 0;
                const OrientedReadId start(startReadId, 0);
                uint32_t localVertexId = 0;
                q.push(start);
                localVertices.push_back(std::make_pair(start, 0));
                vertexTable[start.getValue()] = localVertexId++;
                while(!q.empty()) {
                    const OrientedReadId v0 = q.front();
                    q.pop();
                    const uint32_t distance1 = localVertices[vertexTable[v0.getValue()]].second + 1;
                    for(const uint32_t edgeId : readGraph.connectivity[v0.getValue()]) {
                        const ReadGraphEdge& edge = readGraph.edges[edgeId];
                        if(edge.crossesStrands) continue;
                        const OrientedReadId v1 = edge.getOther(v0);
                        if(vertexTable[v1.getValue()] != notReached) continue;
                        localVertices.push_back(std::make_pair(v1, distance1));
                        vertexTable[v1.getValue()] = localVertexId++;
                        if(distance1 < maxDistance) q.push(v1);
                    }
                }
                const ReadId n = ReadId(localVertices.size());
                rank.resize(n);
                parent.resize(n);
                boost::disjoint_sets<ReadId*, ReadId*> disjointSets(rank.data(), parent.data());
                for(ReadId i = 0; i < n; i++) disjointSets.make_set(i);
                for(const auto& p : localVertices) {
                    const OrientedReadId v0 = p.first;
                    if(v0.getReadId() == startReadId) continue;
                    const uint32_t u0 = vertexTable[v0.getValue()];
                    for(const uint32_t edgeId : readGraph.connectivity[v0.getValue()]) {
                        const ReadGraphEdge& edge = readGraph.edges[edgeId];
                        if(edge.crossesStrands) continue;
                        const OrientedReadId v1 = edge.getOther(v0);
                        if(v1.getReadId() == startReadId) continue;
                        const uint32_t u1 = vertexTable[v1.getValue()];
                        if(u1 != notReached) disjointSets.union_set(u0, u1);
                    }
                }
                uint32_t component = std::numeric_limits<uint32_t>::max();
                for(const auto& p : localVertices) {
                    if(p.second != maxDistance || p.first.getReadId() == startReadId) continue;
                    const uint32_t c = disjointSets.find_set(vertexTable[p.first.getValue()]);
                    if(component == std::numeric_limits<uint32_t>::max()) {
                        component = c;
                    } else if(c != component) {
                        flags[startReadId].isChimeric = 1;
                        for(const uint32_t a : alignmentTable[start.getValue()]) alignmentData[a].info.isInReadGraph = 0;
                        break;
                    }
                }
                for(const auto& p : localVertices) vertexTable[p.first.getValue()] = notReached;
                localVertices.clear();
            }
        });
        for(ReadId r = 0; r < readCount; r++) *chimericCount += flags[r].isChimeric;
        return 0;
    } catch(const std::exception& e) {
        std::fprintf(stderr, "ref_flag_chimeric_reads: %s\n", e.what());
        return 1;
    }
}

}
