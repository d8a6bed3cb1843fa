/* TEST INFRASTRUCTURE (oracle): CPU restatement of Assembler::flagPalindromicReads (src/AssemblerAlign.cpp:652-770) with
 * alignment method 0 (shasta::align, src/AlignmentGraph.cpp:14-136). Only tests/ may call it.
 *
 * The reference's result depends on tie-breaks among equal keys and equal distances, so this file restates the libstdc++
 * algorithms the reference runs, step for step (GCC's bits/stl_algo.h and bits/stl_heap.h are their specification):
 *   std::sort       introsort, median-of-three pivot moved to the first element, heapsort once the depth limit
 *                   2 * floor(log2 n) is used up, then an insertion sort whose first 16 elements are guarded;
 *   push_heap/pop_heap of std::priority_queue.
 * Parity: equal to the reference build (oracle/_ref, ref_palindromic.cpp) read for read, path for path
 * (tests/test_oracle_palindromic.py). */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { uint32_t kmerId, ordinal; } PalMarker;            /* MarkerWithOrdinal, src/Marker.hpp:95-116 */
typedef struct { uint32_t o0, o1; } PalVertex;                      /* AlignmentGraphVertex, src/AlignmentGraph.hpp:85-112 */
typedef struct { uint32_t a, b; uint64_t w; } PalEdge;              /* CompactUndirectedGraph EdgeInfo (:333-345) */
typedef struct { uint64_t d; uint64_t v; } PalHeapItem;             /* pair<uint64_t, vertex_descriptor> */

typedef struct {
    uint64_t heapsortFallbacks;     /* introsort ranges that hit the depth limit, over all sorts */
    uint64_t vertices, edges, heapPushes;
    uint64_t exactReads;            /* reads that got the graph and the path */
} orc_palindromic_counters;

static int floorLog2(uint64_t n) { int r = 0; while(n >>= 1) r++; return r; }     /* std::__lg */

/* std::sort (bits/stl_algo.h: __sort, __introsort_loop, __unguarded_partition_pivot, __move_median_to_first,
 * __unguarded_partition, __partial_sort = __heap_select + __sort_heap, __final_insertion_sort, __insertion_sort,
 * __unguarded_linear_insert) and the heap primitives (bits/stl_heap.h: __adjust_heap, __push_heap, __make_heap). */
#define DEFINE_STD_SORT(NAME, T, LESS)                                                                                 \
static void NAME##_push_heap(T* f, ptrdiff_t hole, ptrdiff_t top, T value)                                             \
{                                                                                                                      \
    ptrdiff_t parent = (hole - 1) / 2;                                                                                 \
    while(hole > top && LESS(f[parent], value)) { f[hole] = f[parent]; hole = parent; parent = (hole - 1) / 2; }       \
    f[hole] = value;                                                                                                   \
}                                                                                                                      \
static void NAME##_adjust_heap(T* f, ptrdiff_t hole, ptrdiff_t len, T value)                                           \
{                                                                                                                      \
    const ptrdiff_t top = hole;                                                                                        \
    ptrdiff_t child = hole;                                                                                            \
    while(child < (len - 1) / 2) {                                                                                     \
        child = 2 * (child + 1);                                                                                       \
        if(LESS(f[child], f[child - 1])) child--;                                                                      \
        f[hole] = f[child]; hole = child;                                                                              \
    }                                                                                                                  \
    if((len & 1) == 0 && child == (len - 2) / 2) { child = 2 * (child + 1); f[hole] = f[child - 1]; hole = child - 1; } \
    NAME##_push_heap(f, hole, top, value);                                                                             \
}                                                                                                                      \
static void NAME##_heapsort(T* f, ptrdiff_t len)                                                                       \
{                                                                                                                      \
    if(len >= 2) {                                                  /* __make_heap */                                  \
        for(ptrdiff_t parent = (len - 2) / 2; ; parent--) {                                                            \
            NAME##_adjust_heap(f, parent, len, f[parent]);                                                             \
            if(parent == 0) break;                                                                                     \
        }                                                                                                              \
    }                                                                                                                  \
    while(len > 1) {                                                /* __sort_heap: __pop_heap(first, last, last) */   \
        len--;                                                                                                         \
        const T value = f[len]; f[len] = f[0];                                                                         \
        NAME##_adjust_heap(f, 0, len, value);                                                                          \
    }                                                                                                                  \
}                                                                                                                      \
static void NAME##_swap(T* a, T* b) { const T t = *a; *a = *b; *b = t; }                                               \
static void NAME##_introsort(T* f, T* l, int depth, uint64_t* fallbacks)                                               \
{                                                                                                                      \
    while(l - f > 16) {                                                                                                \
        if(depth == 0) { NAME##_heapsort(f, l - f); (*fallbacks)++; return; }                                          \
        --depth;                                                                                                       \
        T* a = f + 1; T* b = f + (l - f) / 2; T* c = l - 1;         /* __move_median_to_first(f, f+1, mid, l-1) */     \
        if(LESS(*a, *b)) {                                                                                             \
            if(LESS(*b, *c)) NAME##_swap(f, b); else if(LESS(*a, *c)) NAME##_swap(f, c); else NAME##_swap(f, a);       \
        } else if(LESS(*a, *c)) NAME##_swap(f, a);                                                                     \
        else if(LESS(*b, *c)) NAME##_swap(f, c);                                                                       \
        else NAME##_swap(f, b);                                                                                        \
        T* lo = f + 1; T* hi = l;                                   /* __unguarded_partition(f+1, l, f) */             \
        for(;;) {                                                                                                      \
            while(LESS(*lo, *f)) ++lo;                                                                                 \
            --hi;                                                                                                      \
            while(LESS(*f, *hi)) --hi;                                                                                 \
            if(!(lo < hi)) break;                                                                                      \
            NAME##_swap(lo, hi); ++lo;                                                                                 \
        }                                                                                                              \
        NAME##_introsort(lo, l, depth, fallbacks);                                                                     \
        l = lo;                                                                                                        \
    }                                                                                                                  \
}                                                                                                                      \
static void NAME##_linear_insert(T* last)                                                                              \
{                                                                                                                      \
    const T value = *last;                                                                                             \
    T* next = last - 1;                                                                                                \
    while(LESS(value, *next)) { *last = *next; last = next; --next; }                                                  \
    *last = value;                                                                                                     \
}                                                                                                                      \
static void NAME##_insertion_sort(T* f, T* l)                                                                          \
{                                                                                                                      \
    if(f == l) return;                                                                                                 \
    for(T* i = f + 1; i != l; ++i) {                                                                                   \
        if(LESS(*i, *f)) { const T value = *i; memmove(f + 1, f, (size_t)(i - f) * sizeof(T)); *f = value; }           \
        else NAME##_linear_insert(i);                                                                                  \
    }                                                                                                                  \
}                                                                                                                      \
static inline void NAME##_sort(T* f, ptrdiff_t n, uint64_t* fallbacks)                                                        \
{                                                                                                                      \
    if(n == 0) return;                                                                                                 \
    NAME##_introsort(f, f + n, floorLog2((uint64_t)n) * 2, fallbacks);                                                 \
    if(n > 16) {                                                                                                       \
        NAME##_insertion_sort(f, f + 16);                                                                              \
        for(T* i = f + 16; i != f + n; ++i) NAME##_linear_insert(i);                                                   \
    } else NAME##_insertion_sort(f, f + n);                                                                            \
}

#define MARKER_LESS(x, y) ((x).kmerId < (y).kmerId)                 /* MarkerWithOrdinal::operator< */
#define VERTEX_LESS(x, y) ((x).o0 < (y).o0)                         /* pair<Vertex, Int> with every Int 0 */
#define HEAP_LESS(x, y) ((x).d > (y).d)                             /* OrderPairsByFirstOnlyGreater, src/orderPairs.hpp:35-42 */
DEFINE_STD_SORT(markers, PalMarker, MARKER_LESS)
DEFINE_STD_SORT(vertices, PalVertex, VERTEX_LESS)
DEFINE_STD_SORT(queue, PalHeapItem, HEAP_LESS)

/* McIlroy's adversary ("A Killer Adversary for Quicksort", 1999) against the std::sort restated above: the keys it
 * freezes make introsort use up its depth limit. */
static uint32_t* aqsVal; static uint32_t aqsGas, aqsSolid, aqsCandidate;
static int aqsCompare(uint32_t x, uint32_t y)
{
    if(aqsVal[x] == aqsGas && aqsVal[y] == aqsGas) aqsVal[x == aqsCandidate ? x : y] = aqsSolid++;
    if(aqsVal[x] == aqsGas) aqsCandidate = x; else if(aqsVal[y] == aqsGas) aqsCandidate = y;
    return aqsVal[x] < aqsVal[y] ? -1 : (aqsVal[x] > aqsVal[y] ? 1 : 0);
}
#define AQS_LESS(x, y) (aqsCompare((x), (y)) < 0)
DEFINE_STD_SORT(aqs, uint32_t, AQS_LESS)

void orc_sort_killer_keys(uint32_t n, uint32_t* keysOut)
{
    uint32_t* ptr = (uint32_t*)malloc(4ull * (n ? n : 1));
    aqsVal = keysOut; aqsGas = n; aqsSolid = 0; aqsCandidate = 0;
    for(uint32_t i = 0; i < n; i++) { ptr[i] = i; keysOut[i] = n; }
    uint64_t unused = 0;
    aqs_sort(ptr, n, &unused);
    for(uint32_t i = 0; i < n; i++) if(keysOut[i] == n) keysOut[i] = aqsSolid++;
    free(ptr);
}

/* std::sort of MarkerWithOrdinal rows by kmerId: the row's order and the heapsort-fallback count, for the tests. */
uint64_t orc_std_sort_markers(uint32_t* kmerIds, uint32_t* ordinals, uint64_t n)
{
    PalMarker* m = (PalMarker*)malloc(sizeof(PalMarker) * (n ? n : 1));
    for(uint64_t i = 0; i < n; i++) { m[i].kmerId = kmerIds[i]; m[i].ordinal = ordinals[i]; }
    uint64_t fallbacks = 0;
    markers_sort(m, (ptrdiff_t)n, &fallbacks);
    for(uint64_t i = 0; i < n; i++) { kmerIds[i] = m[i].kmerId; ordinals[i] = m[i].ordinal; }
    free(m);
    return fallbacks;
}

static int iabs(int x) { return x < 0 ? -x : x; }

typedef struct {
    PalVertex* v; uint64_t vCount, vCap;
    PalEdge* e; uint64_t eCount, eCap;
    uint32_t* corrected[2]; uint8_t* lowFrequency[2];
    uint64_t* first; uint64_t* lists;           /* CSR: first[V+3], lists[2E] */
    uint64_t* dist; uint64_t* pred; uint8_t* color;
    PalHeapItem* heap; uint64_t heapCap;
    uint64_t* path; uint64_t pathCount;
} PalWork;

static void* grow(void* p, uint64_t* cap, uint64_t need, size_t size)
{
    if(need <= *cap) return p;
    *cap = need + need / 2 + 16;
    return realloc(p, *cap * size);
}

/* AlignmentGraph::create (src/AlignmentGraph.cpp:58-136) and findShortestPath (src/shortestPath.hpp:65-161) for one read.
 * Leaves the path's graph vertices (without vStart and vFinish) in w->path. */
static void alignReadWithItself(PalWork* w, PalMarker* const m[2], const uint32_t n[2], uint32_t maxSkip32, uint32_t maxDrift32,
                                uint32_t maxMarkerFrequency, orc_palindromic_counters* k)
{
    const size_t maxSkip = maxSkip32, maxDrift = maxDrift32;
    /* createVertices (:156-265) */
    w->vCount = 0;
    for(int s = 0; s < 2; s++) {
        w->lowFrequency[s] = (uint8_t*)realloc(w->lowFrequency[s], n[s] + 1);
        w->corrected[s] = (uint32_t*)realloc(w->corrected[s], 4ull * (n[s] + 1));
        memset(w->lowFrequency[s], 1, n[s]);
    }
    uint32_t i0 = 0, i1 = 0;
    while(i0 < n[0] && i1 < n[1]) {
        if(m[0][i0].kmerId < m[1][i1].kmerId) i0++;
        else if(m[1][i1].kmerId < m[0][i0].kmerId) i1++;
        else {
            const uint32_t kmerId = m[0][i0].kmerId;
            uint32_t e0 = i0, e1 = i1;
            while(e0 < n[0] && m[0][e0].kmerId == kmerId) e0++;
            while(e1 < n[1] && m[1][e1].kmerId == kmerId) e1++;
            if(e0 - i0 > maxMarkerFrequency || e1 - i1 > maxMarkerFrequency) {
                for(uint32_t j = i0; j < e0; j++) w->lowFrequency[0][m[0][j].ordinal] = 0;
                for(uint32_t j = i1; j < e1; j++) w->lowFrequency[1][m[1][j].ordinal] = 0;
            } else {
                for(uint32_t j0 = i0; j0 < e0; j0++) for(uint32_t j1 = i1; j1 < e1; j1++) {
                    w->v = (PalVertex*)grow(w->v, &w->vCap, w->vCount + 1, sizeof(PalVertex));
                    w->v[w->vCount].o0 = m[0][j0].ordinal; w->v[w->vCount].o1 = m[1][j1].ordinal;
                    w->vCount++;
                }
            }
            i0 = e0; i1 = e1;
        }
    }
    for(int s = 0; s < 2; s++) {
        uint32_t c = 0;
        for(uint32_t j = 0; j < n[s]; j++) w->corrected[s][j] = w->lowFrequency[s][j] ? c++ : UINT32_MAX;
    }
    /* sortVertices (src/CompactUndirectedGraph.hpp:506-510), then vStart = V, vFinish = V + 1 (:84-85) */
    vertices_sort(w->v, (ptrdiff_t)w->vCount, &k->heapsortFallbacks);
    const uint64_t V = w->vCount, vStart = V, vFinish = V + 1, N = V + 2;
    k->vertices += V;

    /* createEdges (:294-397) */
    w->eCount = 0;
    for(uint64_t a = 0; a < V; a++) {
        const int cA0 = (int)w->corrected[0][w->v[a].o0], cA1 = (int)w->corrected[1][w->v[a].o1];
        for(uint64_t b = a + 1; b < V; b++) {
            const int cB0 = (int)w->corrected[0][w->v[b].o0];
            if(cB0 > cA0 + (int)maxSkip) break;
            const int cB1 = (int)w->corrected[1][w->v[b].o1];
            if(cB1 < cA1) continue;
            if((size_t)iabs(cB1 - cA1) > maxSkip) continue;
            if(maxDrift < maxSkip) {
                const int offsetA = cA0 - cA1, offsetB = cB0 - cB1;
                if((size_t)iabs(offsetA - offsetB) > maxDrift) continue;
            }
            w->e = (PalEdge*)grow(w->e, &w->eCap, w->eCount + 1, sizeof(PalEdge));
            PalEdge* e = &w->e[w->eCount++];
            e->a = (uint32_t)a; e->b = (uint32_t)b; e->w = (uint64_t)(size_t)(iabs(cB0 - cA0 - 1) + iabs(cB1 - cA1 - 1));
        }
    }
    w->e = (PalEdge*)grow(w->e, &w->eCap, w->eCount + 2 * V + 1, sizeof(PalEdge));
    for(uint64_t v = 0; v < V; v++) {
        const int c0 = (int)w->corrected[0][w->v[v].o0], c1 = (int)w->corrected[1][w->v[v].o1];
        PalEdge* e = &w->e[w->eCount++];
        e->a = (uint32_t)v; e->b = (uint32_t)vStart; e->w = (uint64_t)(size_t)(iabs(c0) + iabs(c1));
        e = &w->e[w->eCount++];
        e->a = (uint32_t)v; e->b = (uint32_t)vFinish; e->w = (uint64_t)(size_t)(iabs((int)n[0] - c0) + iabs((int)n[1] - c1));
    }
    const uint64_t E = w->eCount;
    k->edges += E;

    /* doneAddingEdges (src/CompactUndirectedGraph.hpp:537-583): each vertex's out-edges in increasing edge index.
     * No parallel edges: every pair edge joins a vertex to a later one and vStart, vFinish get one edge per vertex. */
    w->first = (uint64_t*)realloc(w->first, 8 * (N + 1));
    w->lists = (uint64_t*)realloc(w->lists, 8 * (2 * E + 1));
    memset(w->first, 0, 8 * (N + 1));
    for(uint64_t e = 0; e < E; e++) { w->first[w->e[e].a + 1]++; w->first[w->e[e].b + 1]++; }
    for(uint64_t v = 0; v < N; v++) w->first[v + 1] += w->first[v];
    uint64_t* fill = (uint64_t*)malloc(8 * (N + 1));
    memcpy(fill, w->first, 8 * (N + 1));
    for(uint64_t e = 0; e < E; e++) { w->lists[fill[w->e[e].a]++] = e; w->lists[fill[w->e[e].b]++] = e; }
    free(fill);

    /* findShortestPath(graph, vStart, vFinish) (src/shortestPath.hpp:65-161) */
    w->dist = (uint64_t*)realloc(w->dist, 8 * N);
    w->pred = (uint64_t*)realloc(w->pred, 8 * N);
    w->color = (uint8_t*)realloc(w->color, N);
    for(uint64_t v = 0; v < N; v++) { w->dist[v] = UINT64_MAX; w->pred[v] = UINT64_MAX; w->color[v] = 0; }
    w->pred[vStart] = vStart; w->dist[vStart] = 0;
    uint64_t q = 0;
    w->heap = (PalHeapItem*)grow(w->heap, &w->heapCap, 1, sizeof(PalHeapItem));
    w->heap[q].d = 0; w->heap[q].v = vStart; q++;                               /* push onto an empty heap */
    k->heapPushes++;
    w->pathCount = 0;
    while(q) {
        const PalHeapItem top = w->heap[0];
        if(q > 1) {                                                                /* pop_heap + pop_back */
            const PalHeapItem value = w->heap[q - 1];
            w->heap[q - 1] = w->heap[0];
            queue_adjust_heap(w->heap, 0, (ptrdiff_t)(q - 1), value);
        }
        q--;
        const uint64_t v0 = top.v;
        if(w->color[v0] == 1) continue;
        w->color[v0] = 1;
        if(v0 == vFinish) {
            uint64_t count = 0;
            for(uint64_t v = v0; ; v = w->pred[v]) { count++; if(v == vStart) break; }
            w->path = (uint64_t*)realloc(w->path, 8 * count);
            uint64_t i = count;
            for(uint64_t v = v0; ; v = w->pred[v]) { w->path[--i] = v; if(v == vStart) break; }
            /* drop vStart and vFinish (src/AlignmentGraph.cpp:121-128) */
            uint64_t out = 0;
            for(uint64_t j = 0; j < count; j++) if(w->path[j] != vStart && w->path[j] != vFinish) w->path[out++] = w->path[j];
            w->pathCount = out;
            return;
        }
        for(uint64_t p = w->first[v0]; p < w->first[v0 + 1]; p++) {
            const PalEdge* e = &w->e[w->lists[p]];
            const uint64_t v1 = (e->a == v0) ? e->b : e->a;
            if(w->color[v1] == 1) continue;
            const uint64_t d1 = top.d + e->w;
            if(d1 < w->dist[v1]) {
                w->heap = (PalHeapItem*)grow(w->heap, &w->heapCap, q + 1, sizeof(PalHeapItem));
                PalHeapItem item; item.d = d1; item.v = v1;
                queue_push_heap(w->heap, (ptrdiff_t)q, 0, item);                 /* push_back + push_heap */
                q++;
                k->heapPushes++;
                w->pred[v1] = v0; w->dist[v1] = d1;
            }
        }
    }
}

/* Assembler::flagPalindromicReadsThreadFunction (src/AssemblerAlign.cpp:704-770) for R reads given as marker rows
 * (toc uint64[2R+1], relative; read r = rows 2r and 2r+1).
 *   exactAll = 0: reads the prefilter proves not palindromic get flag 0 and their bounds as counts, as the GPU does;
 *   exactAll = 1: every read gets the graph and the path.
 * vBound/vNearBound/survives (optional): the prefilter's V, V_near and verdict per read. pathRead < R: its ordinals. */
int orc_flag_palindromic(uint64_t R, const uint64_t* toc, const uint32_t* kmerIds,
                         uint32_t maxSkip, uint32_t maxDrift, uint32_t maxMarkerFrequency,
                         double alignedFractionThreshold, double nearDiagonalFractionThreshold, uint32_t deltaThreshold,
                         int exactAll, uint8_t* flags, uint32_t* aligned, uint32_t* nearDiagonal,
                         uint64_t* vBound, uint64_t* vNearBound, uint8_t* survives,
                         uint64_t pathRead, uint32_t** pathOut, uint64_t* pathCount, orc_palindromic_counters* counters)
{
    PalWork w;
    memset(&w, 0, sizeof(w));
    orc_palindromic_counters k;
    memset(&k, 0, sizeof(k));
    PalMarker* m[2] = {NULL, NULL};
    uint64_t mCap[2] = {0, 0};
    for(uint64_t r = 0; r < R; r++) {
        uint32_t n[2];
        /* getMarkersSortedByKmerId (src/AssemblerMarkers.cpp:83-98) */
        for(int s = 0; s < 2; s++) {
            const uint64_t b = toc[2 * r + s];
            n[s] = (uint32_t)(toc[2 * r + s + 1] - b);
            m[s] = (PalMarker*)grow(m[s], &mCap[s], n[s] + 1, sizeof(PalMarker));
            for(uint32_t j = 0; j < n[s]; j++) { m[s][j].kmerId = kmerIds[b + j]; m[s][j].ordinal = j; }
            markers_sort(m[s], n[s], &k.heapsortFallbacks);
        }
        /* The prefilter: the path's vertices are distinct graph vertices, so aligned <= V and nearDiagonal <= V_near. */
        uint64_t V = 0, Vnear = 0;
        {
            uint32_t i0 = 0, i1 = 0;
            while(i0 < n[0] && i1 < n[1]) {
                if(m[0][i0].kmerId < m[1][i1].kmerId) i0++;
                else if(m[1][i1].kmerId < m[0][i0].kmerId) i1++;
                else {
                    const uint32_t kmerId = m[0][i0].kmerId;
                    uint32_t e0 = i0, e1 = i1;
                    while(e0 < n[0] && m[0][e0].kmerId == kmerId) e0++;
                    while(e1 < n[1] && m[1][e1].kmerId == kmerId) e1++;
                    if(e0 - i0 <= maxMarkerFrequency && e1 - i1 <= maxMarkerFrequency) {
                        V += (uint64_t)(e0 - i0) * (e1 - i1);
                        for(uint32_t j0 = i0; j0 < e0; j0++) for(uint32_t j1 = i1; j1 < e1; j1++) {
                            const uint32_t delta = (uint32_t)iabs((int32_t)m[0][j0].ordinal - (int32_t)m[1][j1].ordinal);
                            if(delta < deltaThreshold) Vnear++;
                        }
                    }
                    i0 = e0; i1 = e1;
                }
            }
        }
        const int rejected = ((double)V / (double)n[0] < alignedFractionThreshold) ||
                             ((double)Vnear / (double)n[0] < nearDiagonalFractionThreshold);
        if(vBound) vBound[r] = V;
        if(vNearBound) vNearBound[r] = Vnear;
        if(survives) survives[r] = (uint8_t)!rejected;
        if(rejected && !exactAll && r != pathRead) {
            flags[r] = 0; aligned[r] = (uint32_t)V; nearDiagonal[r] = (uint32_t)Vnear;
            continue;
        }
        k.exactReads++;
        alignReadWithItself(&w, m, n, maxSkip, maxDrift, maxMarkerFrequency, &k);
        /* src/AssemblerAlign.cpp:741-766 */
        uint64_t near = 0;
        for(uint64_t i = 0; i < w.pathCount; i++) {
            const PalVertex* v = &w.v[w.path[i]];
            const uint32_t delta = (uint32_t)iabs((int32_t)v->o0 - (int32_t)v->o1);
            if(delta < deltaThreshold) near++;
        }
        const double alignedFraction = (double)w.pathCount / (double)n[0];
        const double nearDiagonalFraction = (double)near / (double)n[0];
        flags[r] = (uint8_t)(!(alignedFraction < alignedFractionThreshold) && !(nearDiagonalFraction < nearDiagonalFractionThreshold));
        aligned[r] = (uint32_t)w.pathCount;
        nearDiagonal[r] = (uint32_t)near;
        if(r == pathRead) {
            uint32_t* out = (uint32_t*)malloc(8 * (w.pathCount ? w.pathCount : 1));
            for(uint64_t i = 0; i < w.pathCount; i++) { out[2 * i] = w.v[w.path[i]].o0; out[2 * i + 1] = w.v[w.path[i]].o1; }
            *pathOut = out;
            *pathCount = w.pathCount;
        }
    }
    free(m[0]); free(m[1]);
    free(w.v); free(w.e); free(w.first); free(w.lists); free(w.dist); free(w.pred); free(w.color); free(w.heap); free(w.path);
    for(int s = 0; s < 2; s++) { free(w.corrected[s]); free(w.lowFrequency[s]); }
    if(counters) *counters = k;
    return 0;
}
