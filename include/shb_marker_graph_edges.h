/* createMarkerGraphEdges and findMarkerGraphReverseComplementEdges (src/AssemblerMarkerGraph.cpp:1025-1080, :1244-1389,
 * :2028-2213) on the GPU. Part of the C ABI of include/shasta_b200.h, which includes this header. */
#ifndef SHB_MARKER_GRAPH_EDGES_H
#define SHB_MARKER_GRAPH_EDGES_H

#include "shasta_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
    uint64_t vertexCount, edgeCount;
    uint64_t markerIntervalCount;           // intervals over all edges (the sum of the uncapped coverages)
    uint64_t saturatedEdgeCount;            // edges whose coverage was capped at 255
    uint64_t peakDeviceBytes;               // high-water mark of the device memory this call allocated (its own buffers and
                                            // the growth of the context's radix-sort workspace)
    uint64_t kernelLaunches;
    double deviceMs, totalMs;               // device time line from the first to the last kernel; wall time of the call
} shb_marker_graph_edges_result;

/* Replaces Assembler::createMarkerGraphEdges (:2028-2085, children :1025-1080) and createMarkerGraphEdgesBySourceAndTarget
 * (:2089-2213) on the markers held by ctx (every read: a context that holds a read range returns SHB_ERR_STATE), for
 * vertices in any numbering (the reference's own files included). The output is the reference's run with one thread:
 * edges in increasing (source, target) order, each edge's MarkerIntervals sorted, every edgesBySource / edgesByTarget row
 * in decreasing edge id.
 *   vertexTable  : Uint40[M] (Data/MarkerGraphVertexTable payload, 2^40-1 = no vertex).
 *   verticesToc  : Uint40[vertexCount+1]; verticesData: uint64[toc[vertexCount]], each vertex's markers in increasing
 *                  marker id (Data/MarkerGraphVertices.{toc,data}).
 *   edges        : receives edgeCount 14-byte MarkerGraph::Edge records (Data/GlobalMarkerGraphEdges payload): Uint40 source,
 *                  Uint40 target, coverage (min(intervals, 255)), then three zero bytes (every flag cleared).
 *   intervalsToc : receives uint64[edgeCount+1]; intervalsData: 12-byte MarkerInterval records {uint32 orientedReadId,
 *                  uint32 ordinals[2]} (Data/GlobalMarkerGraphEdgeMarkerIntervals.{toc,data}).
 *   bySourceToc / bySourceData, byTargetToc / byTargetData: receive uint64[vertexCount+1] and Uint40[edgeCount]
 *                  (Data/GlobalMarkerGraphEdgesBySource.{toc,data}, ...ByTarget.{toc,data}).
 * Free the seven arrays with shb_free. Returns SHB_ERR_INVALID, with the outputs untouched, for a vertex table of another size
 * than the markers, a toc that does not start at 0 or decreases, a marker id >= M, a vertex id >= vertexCount in the vertex
 * table, or a vertex whose markers are not in increasing order. */
shb_status shb_create_marker_graph_edges(shb_context* ctx, const uint8_t* vertexTable, uint64_t vertexTableCount,
                                         const uint8_t* verticesToc, const uint64_t* verticesData, uint64_t vertexCount,
                                         uint8_t** edges, uint64_t** intervalsToc, uint8_t** intervalsData,
                                         uint64_t** bySourceToc, uint8_t** bySourceData, uint64_t** byTargetToc,
                                         uint8_t** byTargetData, shb_marker_graph_edges_result* result);

/* Replaces Assembler::findMarkerGraphReverseComplementEdges (:1244-1389) for edges in any numbering, parallel edges
 * included: for edge e = v0->v1 the first edge of edgesBySource[rc(v1)], in stored order, with target rc(v0) whose
 * reverse-complemented and sorted intervals equal e's. rcEdge receives uint64[edgeCount], free with shb_free.
 * Returns SHB_ERR_INVALID, with the reference's message where it has one, when an edge has no reverse complement, when
 * rc(rc(e)) != e, when an edgesBySource row lists an edge of another source, and for out-of-range vertex, edge or oriented
 * read ids in the inputs. The result's vertexCount, edgeCount, markerIntervalCount, peakDeviceBytes, kernelLaunches,
 * deviceMs and totalMs are filled; saturatedEdgeCount counts the input edges of coverage 255. */
shb_status shb_find_marker_graph_reverse_complement_edges(shb_context* ctx, const uint64_t* rcVertex, uint64_t vertexCount,
                                                          const uint8_t* edges, uint64_t edgeCount, const uint64_t* intervalsToc,
                                                          const uint8_t* intervalsData, const uint64_t* bySourceToc,
                                                          const uint8_t* bySourceData, uint64_t** rcEdge,
                                                          shb_marker_graph_edges_result* result);

#ifdef __cplusplus
}
#endif
#endif
