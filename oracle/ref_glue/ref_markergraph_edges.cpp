// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
// extern "C" access to Assembler::createMarkerGraphEdges (src/AssemblerMarkerGraph.cpp:2028-2085, worker :2116-2180,
// children :1025-1080), createMarkerGraphEdgesBySourceAndTarget (:2089-2112, :2192-2213) and
// findMarkerGraphReverseComplementEdges (:1244-1389), built by oracle/Makefile into
// oracle/_ref/libshasta_ref_markergraph_edges.so. Assembler cannot be linked here, so this glue follows the members' control
// flow over the reference's own objects, compiled unmodified from where they lie:
//   shasta::MarkerGraph           src/MarkerGraph.cpp (its Edge, vertices, vertexTable, edges, edgeMarkerIntervals,
//                                 edgesBySource / edgesByTarget, reverseComplementVertex, reverseComplementEdge)
//   MultithreadedObject           src/MultithreadedObject.cpp (runThreads, setupLoadBalancing, getNextBatch)
//   MemoryMapped::VectorOfVectors incrementCountMultithreaded / storeMultithreaded from real threads
//   shasta::findMarkerId          src/findMarkerId.hpp, over a Markers VectorOfVectors<CompressedMarker, uint64_t>
//   MarkerInterval                src/MarkerInterval.hpp
// Every container is anonymous (MemoryMapped with an empty name). With threadCount > 1 the edge numbering and the row order
// depend on the thread schedule, as in the reference.
#include "Coverage.hpp"
#include "findMarkerId.hpp"
#include "MarkerGraph.hpp"
#include "MarkerInterval.hpp"
#include "MultithreadedObject.tpp"
#include "SHASTA_ASSERT.hpp"

#include <cstdlib>
#include <cstring>
#include <iostream>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

// timestamp.cpp needs boost date_time; nothing here prints a timestamp.
namespace shasta { std::ostream& timestamp(std::ostream& s) { return s; } }

using namespace shasta;

namespace {
constexpr uint64_t kPage = 4096;

class EdgesRun : public MultithreadedObject<EdgesRun> {
public:
    EdgesRun() : MultithreadedObject<EdgesRun>(*this) {}
    MemoryMapped::VectorOfVectors<CompressedMarker, uint64_t> markers;
    MarkerGraph markerGraph;

    // :2028-2085
    std::vector<std::shared_ptr<MemoryMapped::Vector<MarkerGraph::Edge>>> threadEdges;
    std::vector<std::shared_ptr<MemoryMapped::VectorOfVectors<MarkerInterval, uint64_t>>> threadEdgeMarkerIntervals;
    void createMarkerGraphEdges(size_t threadCount)
    {
        threadEdges.resize(threadCount);
        threadEdgeMarkerIntervals.resize(threadCount);
        setupLoadBalancing(markerGraph.vertexCount(), 100);
        runThreads(&EdgesRun::threadFunction0, threadCount);
        markerGraph.edges.createNew("", kPage);
        markerGraph.edgeMarkerIntervals.createNew("", kPage);
        for(size_t threadId = 0; threadId < threadCount; threadId++) {
            auto& thisThreadEdges = *threadEdges[threadId];
            auto& thisThreadEdgeMarkerIntervals = *threadEdgeMarkerIntervals[threadId];
            SHASTA_ASSERT(thisThreadEdges.size() == thisThreadEdgeMarkerIntervals.size());
            for(size_t i = 0; i < thisThreadEdges.size(); i++) {
                markerGraph.edges.push_back(thisThreadEdges[i]);
                markerGraph.edgeMarkerIntervals.appendVector();
                for(auto edgeMarkerInterval : thisThreadEdgeMarkerIntervals[i]) markerGraph.edgeMarkerIntervals.append(edgeMarkerInterval);
            }
            thisThreadEdges.remove();
            thisThreadEdgeMarkerIntervals.remove();
        }
        SHASTA_ASSERT(markerGraph.edges.size() == markerGraph.edgeMarkerIntervals.size());
        // :2089-2112
        markerGraph.edgesBySource.createNew("", kPage);
        markerGraph.edgesByTarget.createNew("", kPage);
        markerGraph.edgesBySource.beginPass1(markerGraph.vertexCount());
        markerGraph.edgesByTarget.beginPass1(markerGraph.vertexCount());
        setupLoadBalancing(markerGraph.edges.size(), 100000);
        runThreads(&EdgesRun::threadFunction1, threadCount);
        markerGraph.edgesBySource.beginPass2();
        markerGraph.edgesByTarget.beginPass2();
        setupLoadBalancing(markerGraph.edges.size(), 100000);
        runThreads(&EdgesRun::threadFunction2, threadCount);
        markerGraph.edgesBySource.endPass2();
        markerGraph.edgesByTarget.endPass2();
    }

    // :1025-1066 (getGlobalMarkerGraphVertexChildren)
    void children(MarkerGraph::VertexId vertexId, std::vector<std::pair<MarkerGraph::VertexId, std::vector<MarkerInterval>>>& children,
                  std::vector<std::pair<MarkerGraph::VertexId, MarkerInterval>>& workArea)
    {
        children.clear();
        workArea.clear();
        for(const MarkerId markerId : markerGraph.getVertexMarkerIds(vertexId)) {
            MarkerInterval info;
            tie(info.orientedReadId, info.ordinals[0]) = findMarkerId(markerId, markers);
            const auto markerCount = markers.size(info.orientedReadId.getValue());
            for(info.ordinals[1] = info.ordinals[0] + 1; info.ordinals[1] < markerCount; ++info.ordinals[1]) {
                const MarkerId childMarkerId = markers.begin(info.orientedReadId.getValue()) - markers.begin() + info.ordinals[1];
                const MarkerGraph::VertexId childVertexId = markerGraph.vertexTable[childMarkerId];
                if(childVertexId != MarkerGraph::invalidCompressedVertexId) {
                    workArea.push_back(std::make_pair(childVertexId, info));
                    break;
                }
            }
        }
        sort(workArea.begin(), workArea.end());
        for(auto streakBegin = workArea.begin(); streakBegin != workArea.end();) {
            auto streakEnd = streakBegin + 1;
            for(; streakEnd != workArea.end() && streakEnd->first == streakBegin->first; streakEnd++) {}
            children.resize(children.size() + 1);
            children.back().first = streakBegin->first;
            for(auto it = streakBegin; it != streakEnd; it++) children.back().second.push_back(it->second);
            streakBegin = streakEnd;
        }
    }

    // :2116-2180
    void threadFunction0(size_t threadId)
    {
        auto edgesPointer = std::make_shared<MemoryMapped::Vector<MarkerGraph::Edge>>();
        threadEdges[threadId] = edgesPointer;
        edgesPointer->createNew("", kPage);
        auto intervalsPointer = std::make_shared<MemoryMapped::VectorOfVectors<MarkerInterval, uint64_t>>();
        threadEdgeMarkerIntervals[threadId] = intervalsPointer;
        intervalsPointer->createNew("", kPage);
        std::vector<std::pair<MarkerGraph::VertexId, std::vector<MarkerInterval>>> childrenList;
        std::vector<std::pair<MarkerGraph::VertexId, MarkerInterval>> workArea;
        MarkerGraph::Edge edge;
        uint64_t begin, end;
        while(getNextBatch(begin, end)) {
            for(MarkerGraph::VertexId vertex0 = begin; vertex0 != end; ++vertex0) {
                edge.source = vertex0;
                children(vertex0, childrenList, workArea);
                for(const auto& p : childrenList) {
                    edge.target = p.first;
                    const size_t coverage = p.second.size();
                    edge.coverage = coverage < 256 ? uint8_t(coverage) : 255;
                    edgesPointer->push_back(edge);
                    intervalsPointer->appendVector();
                    for(const MarkerInterval markerInterval : p.second) intervalsPointer->append(markerInterval);
                }
            }
        }
    }

    // :2192-2213
    void threadFunction1(size_t) { threadFunction12(1); }
    void threadFunction2(size_t) { threadFunction12(2); }
    void threadFunction12(size_t pass)
    {
        uint64_t begin, end;
        while(getNextBatch(begin, end)) {
            for(uint64_t i = begin; i != end; ++i) {
                const auto& edge = markerGraph.edges[i];
                if(pass == 1) {
                    markerGraph.edgesBySource.incrementCountMultithreaded(edge.source);
                    markerGraph.edgesByTarget.incrementCountMultithreaded(edge.target);
                } else {
                    markerGraph.edgesBySource.storeMultithreaded(edge.source, Uint40(i));
                    markerGraph.edgesByTarget.storeMultithreaded(edge.target, Uint40(i));
                }
            }
        }
    }

    // :1244-1389, without the debug CSV files written before the throws.
    void findMarkerGraphReverseComplementEdges(size_t threadCount)
    {
        markerGraph.reverseComplementEdge.createNew("", kPage);
        markerGraph.reverseComplementEdge.resize(markerGraph.edges.size());
        setupLoadBalancing(markerGraph.edges.size(), 10000);
        runThreads(&EdgesRun::rcThreadFunction1, threadCount);
        setupLoadBalancing(markerGraph.edges.size(), 10000);
        runThreads(&EdgesRun::rcThreadFunction2, threadCount);
    }
    std::string firstMessage;
    std::mutex messageMutex;
    void fail(const std::string& m)
    {
        std::lock_guard<std::mutex> lock(messageMutex);
        if(firstMessage.empty()) firstMessage = m;
    }
    void rcThreadFunction1(size_t)
    {
        using VertexId = MarkerGraph::VertexId;
        using EdgeId = MarkerGraph::EdgeId;
        vector<MarkerInterval> resortedMarkers;
        uint64_t begin, end;
        try {
            while(getNextBatch(begin, end)) {
                for(EdgeId edgeId = begin; edgeId != end; edgeId++) {
                    const MarkerGraph::Edge& edge = markerGraph.edges[edgeId];
                    const VertexId v0 = edge.source;
                    const VertexId v1 = edge.target;
                    const VertexId v0Rc = markerGraph.reverseComplementVertex[v0];
                    const VertexId v1Rc = markerGraph.reverseComplementVertex[v1];
                    const span<MarkerInterval> markerIntervals = markerGraph.edgeMarkerIntervals[edgeId];
                    const span<Uint40> v1rcOutEdges = markerGraph.edgesBySource[v1Rc];
                    bool found = false;
                    for(const Uint40 edgeIdRc : v1rcOutEdges) {
                        const MarkerGraph::Edge& edgeRc = markerGraph.edges[edgeIdRc];
                        SHASTA_ASSERT(edgeRc.source == v1Rc);
                        if(edgeRc.target != v0Rc) continue;
                        resortedMarkers.clear();
                        const span<MarkerInterval> markerIntervalsRc = markerGraph.edgeMarkerIntervals[edgeIdRc];
                        for(MarkerInterval markerInterval : markerIntervalsRc) {
                            const uint32_t markerCount = uint32_t(markers.size(markerInterval.orientedReadId.getValue()));
                            markerInterval.orientedReadId.flipStrand();
                            markerInterval.ordinals[0] = markerCount - 1 - markerInterval.ordinals[0];
                            markerInterval.ordinals[1] = markerCount - 1 - markerInterval.ordinals[1];
                            swap(markerInterval.ordinals[0], markerInterval.ordinals[1]);
                            resortedMarkers.push_back(markerInterval);
                        }
                        sort(resortedMarkers.begin(), resortedMarkers.end());
                        const span<MarkerInterval> resortedMarkersSpan(resortedMarkers.data(), resortedMarkers.data() + resortedMarkers.size());
                        if(resortedMarkersSpan == markerIntervals) {
                            markerGraph.reverseComplementEdge[edgeId] = edgeIdRc;
                            found = true;
                            break;
                        }
                    }
                    if(not found) throw std::runtime_error("Unable to locate reverse complement of marker graph edge " +
                                                           std::to_string(edgeId) + " " + std::to_string(v0) + "->" + std::to_string(v1));
                }
            }
        } catch(const std::exception& e) {
            fail(e.what());                 // the reference's thread stops here too; its runThreads then throws
        }
    }
    void rcThreadFunction2(size_t)
    {
        using EdgeId = MarkerGraph::EdgeId;
        uint64_t begin, end;
        if(!firstMessage.empty()) return;
        while(getNextBatch(begin, end)) {
            for(EdgeId edgeId = begin; edgeId != end; edgeId++) {
                const EdgeId r = markerGraph.reverseComplementEdge[edgeId];
                if(markerGraph.reverseComplementEdge[r] != edgeId) {
                    fail("Reverse complement edge check failed at edge " + std::to_string(edgeId) + ": " + std::to_string(r) + " " +
                         std::to_string(markerGraph.reverseComplementEdge[r]));
                    return;
                }
            }
        }
    }

    void setMarkers(const uint64_t* toc, uint64_t R)
    {
        markers.createNew("", kPage);
        for(uint64_t o = 0; o < 2 * R; o++) markers.appendVector(toc[o + 1] - toc[o]);
    }
    void setVertices(const uint64_t* table, uint64_t M, const uint64_t* vtoc, const uint64_t* vdata, uint64_t V)
    {
        markerGraph.vertexTable.createNew("", kPage);
        markerGraph.vertexTable.resize(M);
        for(uint64_t i = 0; i < M; i++) markerGraph.vertexTable[i] = table[i];
        markerGraph.constructVertices();
        markerGraph.vertices().createNew("", kPage);
        for(uint64_t v = 0; v < V; v++) markerGraph.vertices().appendVector(vdata + vtoc[v], vdata + vtoc[v + 1]);
    }
};

template<class T> T* copyOut(const T* p, uint64_t n)
{
    T* out = static_cast<T*>(malloc(sizeof(T) * n + 16));
    if(n) std::memcpy(out, p, sizeof(T) * n);
    return out;
}

uint64_t* rowsOut(const MemoryMapped::VectorOfVectors<Uint40, uint64_t>& t, uint64_t** tocOut)
{
    const uint64_t rows = t.size();
    uint64_t* toc = static_cast<uint64_t*>(malloc(8 * (rows + 1)));
    uint64_t* data = static_cast<uint64_t*>(malloc(8 * t.totalSize() + 8));
    toc[0] = 0;
    for(uint64_t r = 0, k = 0; r < rows; r++) {
        for(const Uint40 x : t[r]) data[k++] = uint64_t(x);
        toc[r + 1] = toc[r] + t.size(r);
    }
    *tocOut = toc;
    return data;
}
}

extern "C" {

// Status 0, or 1 on a reference assertion or exception (message on stderr). Outputs malloc'ed (ref_free_markergraph_edges):
// edges uint8[14E] (the reference's Edge bytes), itoc uint64[E+1], idata uint32[3I], stoc/ttoc uint64[V+1],
// sdata/tdata uint64[E]; counts[2] = E, I.
int ref_create_marker_graph_edges(const uint64_t* toc, uint64_t R, const uint64_t* table, const uint64_t* vtoc, const uint64_t* vdata,
                                  uint64_t V, uint64_t threads, uint8_t** edgesOut, uint64_t** itocOut, uint32_t** idataOut,
                                  uint64_t** stocOut, uint64_t** sdataOut, uint64_t** ttocOut, uint64_t** tdataOut, uint64_t* counts)
{
    try {
        EdgesRun run;
        run.setMarkers(toc, R);
        run.setVertices(table, toc[2 * R], vtoc, vdata, V);
        run.createMarkerGraphEdges(threads ? threads : std::thread::hardware_concurrency());
        const auto& mg = run.markerGraph;
        const uint64_t E = mg.edges.size(), I = mg.edgeMarkerIntervals.totalSize();
        static_assert(sizeof(MarkerGraph::Edge) == 14, "MarkerGraph::Edge is 14 bytes");
        static_assert(sizeof(MarkerInterval) == 12, "MarkerInterval is 12 bytes");
        *edgesOut = copyOut(reinterpret_cast<const uint8_t*>(mg.edges.begin()), 14 * E);
        uint64_t* itoc = static_cast<uint64_t*>(malloc(8 * (E + 1)));
        itoc[0] = 0;
        for(uint64_t e = 0; e < E; e++) itoc[e + 1] = itoc[e] + mg.edgeMarkerIntervals.size(e);
        *itocOut = itoc;
        *idataOut = copyOut(reinterpret_cast<const uint32_t*>(mg.edgeMarkerIntervals.begin()), 3 * I);
        *sdataOut = rowsOut(mg.edgesBySource, stocOut);
        *tdataOut = rowsOut(mg.edgesByTarget, ttocOut);
        counts[0] = E; counts[1] = I;
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_create_marker_graph_edges: %s\n", e.what());
        return 1;
    }
}

// Status 0, or 1 with the reference's message in msg (the first thrown by any thread).
int ref_find_rc_edges(const uint64_t* toc, uint64_t R, const uint64_t* rcVertex, uint64_t V, const uint8_t* edges, uint64_t E,
                      const uint64_t* itoc, const uint32_t* idata, const uint64_t* stoc, const uint64_t* sdata, uint64_t threads,
                      uint64_t* rc, char* msg, uint64_t msgCapacity)
{
    try {
        EdgesRun run;
        run.setMarkers(toc, R);
        auto& mg = run.markerGraph;
        mg.reverseComplementVertex.createNew("", kPage);
        mg.reverseComplementVertex.resize(V);
        for(uint64_t v = 0; v < V; v++) mg.reverseComplementVertex[v] = rcVertex[v];
        mg.edges.createNew("", kPage);
        mg.edges.resize(E);
        if(E) std::memcpy(reinterpret_cast<uint8_t*>(mg.edges.begin()), edges, 14 * E);
        mg.edgeMarkerIntervals.createNew("", kPage);
        for(uint64_t e = 0; e < E; e++) {
            mg.edgeMarkerIntervals.appendVector();
            for(uint64_t k = itoc[e]; k < itoc[e + 1]; k++) {
                MarkerInterval x;
                std::memcpy(&x, idata + 3 * k, 12);
                mg.edgeMarkerIntervals.append(x);
            }
        }
        mg.edgesBySource.createNew("", kPage);
        for(uint64_t v = 0; v < V; v++) {
            mg.edgesBySource.appendVector();
            for(uint64_t k = stoc[v]; k < stoc[v + 1]; k++) mg.edgesBySource.append(Uint40(sdata[k]));
        }
        run.findMarkerGraphReverseComplementEdges(threads ? threads : std::thread::hardware_concurrency());
        if(!run.firstMessage.empty()) {
            snprintf(msg, msgCapacity, "%s", run.firstMessage.c_str());
            return 1;
        }
        for(uint64_t e = 0; e < E; e++) rc[e] = mg.reverseComplementEdge[e];
        return 0;
    } catch(const std::exception& e) {
        snprintf(msg, msgCapacity, "%s", e.what());
        return 1;
    }
}

// The five edge file sets as the reference's own MemoryMapped code opens them (Data/GlobalMarkerGraphEdges, ...); the
// name arguments are full paths without the .toc / .data suffixes. counts[4] = E, I, rows of edgesBySource, rows of
// edgesByTarget. rc may be NULL (no reverse complement file).
int ref_open_marker_graph_edges(const char* edgesPath, const char* intervalsName, const char* bySourceName, const char* byTargetName,
                                const char* rcPath, uint8_t** edgesOut, uint64_t** itocOut, uint32_t** idataOut, uint64_t** stocOut,
                                uint64_t** sdataOut, uint64_t** ttocOut, uint64_t** tdataOut, uint64_t** rcOut, uint64_t* counts)
{
    try {
        MemoryMapped::Vector<MarkerGraph::Edge> edges;
        edges.accessExistingReadOnly(edgesPath);
        MemoryMapped::VectorOfVectors<MarkerInterval, uint64_t> intervals;
        intervals.accessExistingReadOnly(intervalsName);
        MemoryMapped::VectorOfVectors<Uint40, uint64_t> bySource, byTarget;
        bySource.accessExistingReadOnly(bySourceName);
        byTarget.accessExistingReadOnly(byTargetName);
        const uint64_t E = edges.size();
        *edgesOut = copyOut(reinterpret_cast<const uint8_t*>(edges.begin()), 14 * E);
        uint64_t* itoc = static_cast<uint64_t*>(malloc(8 * (intervals.size() + 1)));
        itoc[0] = 0;
        for(uint64_t e = 0; e < intervals.size(); e++) itoc[e + 1] = itoc[e] + intervals.size(e);
        *itocOut = itoc;
        *idataOut = copyOut(reinterpret_cast<const uint32_t*>(intervals.begin()), 3 * intervals.totalSize());
        *sdataOut = rowsOut(bySource, stocOut);
        *tdataOut = rowsOut(byTarget, ttocOut);
        counts[0] = E; counts[1] = intervals.totalSize(); counts[2] = bySource.size(); counts[3] = byTarget.size();
        if(rcPath) {
            MemoryMapped::Vector<uint64_t> rc;
            rc.accessExistingReadOnly(rcPath);
            SHASTA_ASSERT(rc.size() == E);
            *rcOut = copyOut(rc.begin(), E);
        }
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_open_marker_graph_edges: %s\n", e.what());
        return 1;
    }
}

void ref_free_markergraph_edges(void* p) { free(p); }

} // extern "C"
