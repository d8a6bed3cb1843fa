/* TEST INFRASTRUCTURE. Sequential plain-C restatement of Assembler::createMarkerGraphEdges
 * (src/AssemblerMarkerGraph.cpp:2028-2085, worker :2116-2180, children :1025-1080), createMarkerGraphEdgesBySourceAndTarget
 * (:2089-2112, :2192-2213) and findMarkerGraphReverseComplementEdges (:1244-1389), as the reference runs them with one thread.
 * Markers are given as the Markers toc (2R+1 entries); the vertex table and the vertices toc as uint64. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MGE_INVALID40 ((1ull << 40) - 1)

typedef struct { uint64_t child; uint32_t o, a0, a1; } mge_item;      /* pair<VertexId, MarkerInterval> of workArea */

static int byChild(const void* pa, const void* pb)                     /* :1054 sort(workArea): pair order */
{
    const mge_item* a = (const mge_item*)pa; const mge_item* b = (const mge_item*)pb;
    if(a->child != b->child) return a->child < b->child ? -1 : 1;
    if(a->o != b->o) return a->o < b->o ? -1 : 1;
    if(a->a0 != b->a0) return a->a0 < b->a0 ? -1 : 1;
    if(a->a1 != b->a1) return a->a1 < b->a1 ? -1 : 1;
    return 0;
}

static uint64_t orientedReadOf(const uint64_t* toc, uint64_t rows, uint64_t m)     /* findMarkerId: last row with toc[row] <= m */
{
    uint64_t lo = 0, hi = rows;
    while(hi - lo > 1) { const uint64_t mid = lo + (hi - lo) / 2; if(toc[mid] <= m) lo = mid; else hi = mid; }
    return lo;
}

static void put40(uint8_t* p, uint64_t v) { for(int b = 0; b < 5; b++) p[b] = (uint8_t)(v >> (8 * b)); }
static uint64_t get40(const uint8_t* p) { uint64_t v = 0; for(int b = 0; b < 5; b++) v |= (uint64_t)p[b] << (8 * b); return v; }

/* Status: 0 ok; 1 a marker id >= M; 2 a vertex id >= V in the vertex table (the reference's edgesByTarget would be indexed
 * out of range). Outputs (malloc'ed, free with orc_free): edges uint8[14E] (bytes 11-13 zero), itoc uint64[E+1],
 * idata uint32[3I], stoc/ttoc uint64[V+1], sdata/tdata uint64[E]. counts[3]: E, I, edges with coverage capped at 255. */
int orc_create_marker_graph_edges(const uint64_t* toc, uint64_t R, const uint64_t* table, const uint64_t* vtoc, const uint64_t* vdata,
                                  uint64_t V, uint8_t** edgesOut, uint64_t** itocOut, uint32_t** idataOut, uint64_t** stocOut,
                                  uint64_t** sdataOut, uint64_t** ttocOut, uint64_t** tdataOut, uint64_t* counts)
{
    const uint64_t rows = 2 * R, M = toc[rows], N = vtoc[V];
    uint8_t* edges = malloc(14 * N + 14);
    uint64_t* itoc = malloc(8 * (N + 1));
    uint32_t* idata = malloc(12 * N + 12);
    mge_item* work = malloc(sizeof(mge_item) * (N + 1));
    uint64_t E = 0, I = 0, saturated = 0;
    itoc[0] = 0;
    for(uint64_t v0 = 0; v0 < V; v0++) {                                   /* :2143-2173, one thread: vertices in order */
        uint64_t w = 0;
        for(uint64_t j = vtoc[v0]; j < vtoc[v0 + 1]; j++) {                /* getGlobalMarkerGraphVertexChildren :1032-1051 */
            const uint64_t m = vdata[j];
            if(m >= M) { free(edges); free(itoc); free(idata); free(work); return 1; }
            const uint64_t o = orientedReadOf(toc, rows, m);
            const uint64_t markerCount = toc[o + 1] - toc[o];
            for(uint64_t a1 = m - toc[o] + 1; a1 < markerCount; a1++) {
                const uint64_t child = table[toc[o] + a1];
                if(child != MGE_INVALID40) {
                    if(child >= V) { free(edges); free(itoc); free(idata); free(work); return 2; }
                    mge_item it = {child, (uint32_t)o, (uint32_t)(m - toc[o]), (uint32_t)a1};
                    work[w++] = it;
                    break;
                }
            }
        }
        qsort(work, w, sizeof(mge_item), byChild);
        for(uint64_t b = 0; b < w; ) {                                     /* :1058-1074 streaks, :2150-2171 one edge each */
            uint64_t e = b + 1;
            while(e < w && work[e].child == work[b].child) e++;
            uint8_t* r = edges + 14 * E;
            put40(r, v0); put40(r + 5, work[b].child);
            r[10] = (uint8_t)(e - b < 256 ? e - b : 255);
            if(e - b >= 256) saturated++;
            r[11] = r[12] = r[13] = 0;
            for(uint64_t k = b; k < e; k++) { idata[3 * I] = work[k].o; idata[3 * I + 1] = work[k].a0; idata[3 * I + 2] = work[k].a1; I++; }
            E++;
            itoc[E] = I;
            b = e;
        }
    }
    free(work);
    /* :2089-2112 with one thread: pass 1 counts, pass 2 stores edges in increasing id, each row filled from its end
     * (MemoryMappedVectorOfVectors.hpp:384-392). */
    uint64_t* stoc = calloc(V + 1, 8);
    uint64_t* ttoc = calloc(V + 1, 8);
    uint64_t* sdata = malloc(8 * E + 8);
    uint64_t* tdata = malloc(8 * E + 8);
    for(uint64_t e = 0; e < E; e++) { stoc[get40(edges + 14 * e)]++; ttoc[get40(edges + 14 * e + 5)]++; }
    for(uint64_t v = 0, s = 0, t = 0; v <= V; v++) {                       /* toc[v] = end of row v, then filled downwards */
        if(v < V) { s += stoc[v]; t += ttoc[v]; }
        stoc[v] = s; ttoc[v] = t;
    }
    for(uint64_t e = 0; e < E; e++) {
        sdata[--stoc[get40(edges + 14 * e)]] = e;
        tdata[--ttoc[get40(edges + 14 * e + 5)]] = e;
    }
    stoc[V] = ttoc[V] = E;
    *edgesOut = edges; *itocOut = itoc; *idataOut = idata; *stocOut = stoc; *sdataOut = sdata; *ttocOut = ttoc; *tdataOut = tdata;
    counts[0] = E; counts[1] = I; counts[2] = saturated;
    return 0;
}

static int byInterval(const void* pa, const void* pb)                   /* MarkerInterval::operator< */
{
    const uint32_t* a = (const uint32_t*)pa; const uint32_t* b = (const uint32_t*)pb;
    for(int k = 0; k < 3; k++) if(a[k] != b[k]) return a[k] < b[k] ? -1 : 1;
    return 0;
}

/* :1283-1389 with one thread. Status: 0 ok; 1 "Unable to locate reverse complement" (info = edge, v0, v1); 2 "Reverse
 * complement edge check failed" (info = edge, rc, rc of rc); 3 the assertion edgeRc.source == v1Rc (info = edge). */
int orc_find_rc_edges(const uint64_t* toc, uint64_t R, const uint64_t* rcVertex, uint64_t V, const uint8_t* edges, uint64_t E,
                      const uint64_t* itoc, const uint32_t* idata, const uint64_t* stoc, const uint64_t* sdata, uint64_t* rc, uint64_t* info)
{
    (void)R; (void)V;
    uint64_t maxCoverage = 0;
    for(uint64_t e = 0; e < E; e++) if(itoc[e + 1] - itoc[e] > maxCoverage) maxCoverage = itoc[e + 1] - itoc[e];
    uint32_t* resorted = malloc(12 * maxCoverage + 12);
    for(uint64_t e = 0; e < E; e++) {
        const uint64_t v0 = get40(edges + 14 * e), v1 = get40(edges + 14 * e + 5);
        const uint64_t v0Rc = rcVertex[v0], v1Rc = rcVertex[v1];
        const uint64_t n = itoc[e + 1] - itoc[e];
        int found = 0;
        for(uint64_t k = stoc[v1Rc]; k < stoc[v1Rc + 1] && !found; k++) {
            const uint64_t c = sdata[k];
            if(get40(edges + 14 * c) != v1Rc) { info[0] = e; free(resorted); return 3; }
            if(get40(edges + 14 * c + 5) != v0Rc) continue;
            const uint64_t m = itoc[c + 1] - itoc[c];
            for(uint64_t j = 0; j < m; j++) {
                const uint32_t* x = idata + 3 * (itoc[c] + j);
                const uint32_t markerCount = (uint32_t)(toc[x[0] + 1] - toc[x[0]]);
                resorted[3 * j] = x[0] ^ 1u;
                resorted[3 * j + 1] = markerCount - 1 - x[2];
                resorted[3 * j + 2] = markerCount - 1 - x[1];
            }
            qsort(resorted, m, 12, byInterval);
            if(m == n && (n == 0 || memcmp(resorted, idata + 3 * itoc[e], 12 * n) == 0)) { rc[e] = c; found = 1; }
        }
        if(!found) { info[0] = e; info[1] = v0; info[2] = v1; free(resorted); return 1; }
    }
    free(resorted);
    for(uint64_t e = 0; e < E; e++)
        if(rc[rc[e]] != e) { info[0] = e; info[1] = rc[e]; info[2] = rc[rc[e]]; return 2; }
    return 0;
}
