/* TEST INFRASTRUCTURE. Sequential plain-C restatement of Assembler::createMarkerGraphVertices
 * (src/AssemblerMarkerGraph.cpp:38-518, threads :522-770), of findMarkerGraphReverseComplementVertices (:1134-1230) and of
 * PeakFinder (src/PeakFinder.cpp:23-198). Vertices are numbered in increasing order of their smallest marker id (a min-linking
 * union-find: the root of each set is its smallest marker); the reference's numbering follows its concurrent representatives.
 * Marker ids are 64-bit; markers are given as the Markers toc (2R+1 entries) and the k-mer ids. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

uint64_t orc_decompress_alignment(const uint8_t* s, uint64_t bytes, uint32_t* ordOut, uint64_t cap);   /* align_oracle.c */

#define MG_INVALID40 ((1ull << 40) - 1)

/* ---- PeakFinder -------------------------------------------------------------------------------------------------- */
typedef struct { uint64_t start, stop, left, right; int isMerged; uint64_t persistence; } mg_peak;

static const uint64_t* g_y;
static int byHeight(const void* pa, const void* pb)          /* :37-47: y descending, equal y by lower x */
{
    const uint64_t a = *(const uint64_t*)pa, b = *(const uint64_t*)pb;
    if(g_y[a] == g_y[b]) return a < b ? -1 : (a > b);
    return g_y[a] > g_y[b] ? -1 : 1;
}
static int byPersistence(const void* pa, const void* pb)     /* :131-144: persistence descending, equal by lower start */
{
    const mg_peak* a = (const mg_peak*)pa; const mg_peak* b = (const mg_peak*)pb;
    if(a->persistence == b->persistence) return a->start < b->start ? -1 : (a->start > b->start);
    return a->persistence > b->persistence ? -1 : 1;
}
static uint64_t area(const uint64_t* y, uint64_t xMin, uint64_t xMax)    /* :147-155 */
{
    uint64_t t = 0;
    for(uint64_t i = xMin; i <= xMax; i++) t += y[i];
    return t;
}

/* Returns 1 where the reference throws PeakFinderException (*observed = observedPercentArea), else 0 and *cutoff.
 * n = 0 (undefined in the reference: findPeaks reads peaks[0] of an empty vector) returns 1 with observed area 0. */
int orc_peak_finder_cutoff(const uint64_t* y, uint64_t n, double minAreaFraction, uint64_t startIndex, uint64_t* cutoff, double* observed)
{
    *observed = 0;
    if(n == 0) return 1;
    int64_t* peakIndex = malloc(8 * n);
    uint64_t* idx = malloc(8 * n);
    mg_peak* peaks = malloc(sizeof(mg_peak) * n);
    uint64_t np = 0;
    for(uint64_t i = 0; i < n; i++) { peakIndex[i] = -1; idx[i] = i; }
    g_y = y;
    qsort(idx, n, 8, byHeight);
    for(uint64_t t = 0; t < n; t++) {                                      /* :50-124 */
        const uint64_t i = idx[t];
        const int hasLeft = i > 0 && peakIndex[i - 1] >= 0;
        const int hasRight = i < n - 1 && peakIndex[i + 1] >= 0;
        if(!hasLeft && !hasRight) {
            mg_peak p = {i, 0, i, i, 0, 0};
            peaks[np++] = p;
            peakIndex[i] = (int64_t)(np - 1);
        } else if(hasLeft && !hasRight) {
            peaks[peakIndex[i - 1]].right = i;
            peakIndex[i] = peakIndex[i - 1];
        } else if(!hasLeft && hasRight) {
            peaks[peakIndex[i + 1]].left = i;
            peakIndex[i] = peakIndex[i + 1];
        } else {
            mg_peak* L = &peaks[peakIndex[i - 1]];
            mg_peak* Rp = &peaks[peakIndex[i + 1]];
            if(y[Rp->start] > y[L->start]) {
                Rp->left = L->left;
                peakIndex[i] = peakIndex[i + 1];
                L->right = i;
                peakIndex[L->left] = peakIndex[i + 1];
                peakIndex[L->right] = peakIndex[i + 1];
                L->stop = i; L->isMerged = 1;
                L->persistence = y[Rp->start] - y[i];                   /* :104, the surviving peak's height */
            } else {
                L->right = Rp->right;
                peakIndex[i] = peakIndex[i - 1];
                Rp->left = i;
                peakIndex[Rp->right] = peakIndex[i - 1];
                peakIndex[Rp->left] = peakIndex[i - 1];
                Rp->stop = i; Rp->isMerged = 1;
                Rp->persistence = y[Rp->start] - y[i];
            }
        }
    }
    peaks[0].persistence = y[peaks[0].start];                             /* :127 */
    int threw = 1;
    if(np >= 2) {                                                          /* :158-198 */
        qsort(peaks, np, sizeof(mg_peak), byPersistence);
        uint64_t leftBound, rightBound;
        if(peaks[1].start < peaks[0].start) { leftBound = peaks[1].right; rightBound = peaks[0].right; }
        else { leftBound = peaks[1].left; rightBound = peaks[1].right; }
        const uint64_t totalArea = area(y, startIndex, n - 1);
        const uint64_t peakArea = area(y, leftBound, rightBound);
        const double areaFraction = (double)peakArea / (double)totalArea;
        if(areaFraction > minAreaFraction) { *cutoff = leftBound; threw = 0; }
        else *observed = areaFraction;
    }
    free(peakIndex); free(idx); free(peaks);
    return threw;
}

/* ---- union-find ----------------------------------------------------------------------------------------------------- */
static uint64_t findRoot(uint64_t* P, uint64_t x)
{
    while(P[x] != x) { P[x] = P[P[x]]; x = P[x]; }
    return x;
}
static void unite(uint64_t* P, uint64_t a, uint64_t b)
{
    a = findRoot(P, a); b = findRoot(P, b);
    if(a == b) return;
    if(a < b) P[b] = a; else P[a] = b;
}
/* Assembler::findReverseComplement (src/AssemblerMarkers.cpp:140-153), given the oriented read of the marker. */
static uint64_t rcMarker(const uint64_t* toc, uint64_t o, uint64_t ordinal)
{
    return toc[o ^ 1] + (toc[o + 1] - toc[o] - 1 - ordinal);
}
static uint64_t orientedReadOf(const uint64_t* toc, uint64_t rows, uint64_t m)     /* last row with toc[row] <= m */
{
    uint64_t lo = 0, hi = rows;
    while(hi - lo > 1) { const uint64_t mid = lo + (hi - lo) / 2; if(toc[mid] <= m) lo = mid; else hi = mid; }
    return lo;
}

/* Status: 0 ok; 1 odd edge count; 2 a pair that is not an edge and its reverse complement; 3 unordered oriented read ids;
 * 4 alignmentId out of range; 5 k-mer ids differ.
 * params: minCoverage, maxCoverage, minCoveragePerStrand, allowDuplicateMarkers, peakFinderAreaStartIndex.
 * counts[12]: minCoverageUsed, peakFinderFailed, pairsUsed, pairsSkipped, alignedPairs, disjointSets, kept, bad, V,
 *             histogramSize, total vertex markers, (observed area fraction as the bits of a double).
 * Outputs (malloc'ed, orc_free): table uint64[M], vtoc uint64[V+1], vdata uint64[], histogram uint64[histogramSize]. */
int orc_create_marker_graph_vertices(const uint64_t* toc, uint64_t R, const uint32_t* kmerIds, const uint32_t* edges, uint64_t edgeCount,
                                     const uint64_t* ctoc, const uint8_t* cdata, uint64_t alignmentCount, const uint8_t* readFlags,
                                     const uint64_t* params, double peakFinderMinAreaFraction,
                                     uint64_t** tableOut, uint64_t** vtocOut, uint64_t** vdataOut, uint64_t** histOut, uint64_t* counts)
{
    const uint64_t rows = 2 * R, M = toc[rows];
    uint64_t minCoverage = params[0];
    const uint64_t maxCoverage = params[1], minCoveragePerStrand = params[2], allowDuplicateMarkers = params[3];
    memset(counts, 0, 12 * 8);
    if(edgeCount % 2) return 1;
    uint64_t* P = malloc(8 * (M + 1));
    for(uint64_t i = 0; i < M; i++) P[i] = i;
    uint32_t* ord = NULL;
    uint64_t ordCap = 0;
    for(uint64_t i = 0; i < edgeCount; i += 2) {                           /* :544-605 */
        const uint32_t* e = edges + 4 * i;
        const uint32_t* f = edges + 4 * (i + 1);
        if((f[0] ^ 1u) != e[0] || (f[1] ^ 1u) != e[1]) { free(P); free(ord); return 2; }
        if(e[3] >> 30) { counts[3]++; continue; }
        if(!(e[0] < e[1])) { free(P); free(ord); return 3; }
        if((readFlags[e[0] >> 1] | readFlags[e[1] >> 1]) & 2u) { counts[3]++; continue; }
        const uint64_t a = (uint64_t)e[2] | ((uint64_t)(e[3] & 0x3fffffffu) << 32);
        if(a >= alignmentCount) { free(P); free(ord); return 4; }
        counts[2]++;
        const uint64_t bytes = ctoc[a + 1] - ctoc[a];
        const uint64_t n = orc_decompress_alignment(cdata + ctoc[a], bytes, NULL, 0);        /* count, then decode */
        if(n + 1 > ordCap) { ordCap = n + 1; ord = realloc(ord, 8 * ordCap); }
        orc_decompress_alignment(cdata + ctoc[a], bytes, ord, ordCap);
        for(uint64_t j = 0; j < n; j++) {
            const uint64_t m0 = toc[e[0]] + ord[2 * j], m1 = toc[e[1]] + ord[2 * j + 1];
            if(kmerIds[m0] != kmerIds[m1]) { free(P); free(ord); return 5; }
            unite(P, m0, m1);
            unite(P, rcMarker(toc, e[0], ord[2 * j]), rcMarker(toc, e[1], ord[2 * j + 1]));
        }
        counts[4] += n;
    }
    free(ord);
    /* Sizes and histogram (:180-231). */
    uint64_t* size = calloc(M + 1, 8);
    for(uint64_t i = 0; i < M; i++) { P[i] = findRoot(P, i); size[P[i]]++; }
    uint64_t maxSize = 0;
    for(uint64_t i = 0; i < M; i++) if(size[i] > maxSize) maxSize = size[i];
    const uint64_t histSize = M ? maxSize + 1 : 0;
    uint64_t* hist = calloc(histSize + 1, 8);
    for(uint64_t i = 0; i < M; i++) if(size[i]) { hist[size[i]]++; counts[5]++; }
    if(minCoverage == 0) {                                                 /* :233-251 */
        uint64_t cutoff = 0;
        double observed = 0;
        if(orc_peak_finder_cutoff(hist, histSize, peakFinderMinAreaFraction, params[4], &cutoff, &observed)) {
            minCoverage = 5; counts[1] = 1; memcpy(&counts[11], &observed, 8);
        } else minCoverage = cutoff;
    }
    counts[0] = minCoverage;
    /* Kept sets in root order (:266-303); the markers of each, ascending (:324-345). */
    uint64_t* keptId = malloc(8 * (M + 1));
    uint64_t kept = 0;
    for(uint64_t i = 0; i < M; i++) keptId[i] = (size[i] && size[i] >= minCoverage && size[i] <= maxCoverage) ? kept++ : ~0ull;
    uint64_t* setOffset = calloc(kept + 1, 8);
    uint64_t* setCount = calloc(kept + 1, 8);
    for(uint64_t i = 0; i < M; i++) if(keptId[P[i]] != ~0ull) setOffset[keptId[P[i]] + 1]++;
    for(uint64_t k = 0; k < kept; k++) setOffset[k + 1] += setOffset[k];
    uint64_t* members = malloc(8 * (setOffset[kept] + 1));
    for(uint64_t i = 0; i < M; i++) {                                      /* ascending i: each set's markers come out sorted */
        const uint64_t k = keptId[P[i]];
        if(k != ~0ull) members[setOffset[k] + setCount[k]++] = i;
    }
    counts[6] = kept;
    /* Bad sets (:697-745) and the final numbering (:393-464). */
    uint64_t* vertexOf = malloc(8 * (kept + 1));
    uint64_t V = 0, vm = 0;
    for(uint64_t k = 0; k < kept; k++) {
        const uint64_t n = setOffset[k + 1] - setOffset[k];
        const uint64_t* m = members + setOffset[k];
        int bad = 0;
        if(n == 1) bad = 1 < minCoveragePerStrand;
        else {
            uint64_t byStrand[2] = {0, 0};
            for(uint64_t j = 0; j < n; j++) {
                const uint64_t o = orientedReadOf(toc, rows, m[j]);
                byStrand[o & 1]++;
                if(!allowDuplicateMarkers && j > 0 && (orientedReadOf(toc, rows, m[j - 1]) >> 1) == (o >> 1)) { bad = 1; break; }
            }
            if(!bad) bad = byStrand[0] < minCoveragePerStrand || byStrand[1] < minCoveragePerStrand;
        }
        if(bad) { vertexOf[k] = ~0ull; counts[7]++; }
        else { vertexOf[k] = V++; vm += n; }
    }
    uint64_t* table = malloc(8 * (M + 1));
    for(uint64_t i = 0; i < M; i++) {
        const uint64_t k = keptId[P[i]];
        table[i] = (k == ~0ull || vertexOf[k] == ~0ull) ? MG_INVALID40 : vertexOf[k];
    }
    uint64_t* vtoc = malloc(8 * (V + 1));
    uint64_t* vdata = malloc(8 * (vm + 1));
    vtoc[0] = 0;
    for(uint64_t k = 0, v = 0; k < kept; k++) {
        if(vertexOf[k] == ~0ull) continue;
        const uint64_t n = setOffset[k + 1] - setOffset[k];
        memcpy(vdata + vtoc[v], members + setOffset[k], 8 * n);
        vtoc[v + 1] = vtoc[v] + n;
        v++;
    }
    counts[8] = V; counts[9] = histSize; counts[10] = vm;
    free(P); free(size); free(keptId); free(setOffset); free(setCount); free(members); free(vertexOf);
    *tableOut = table; *vtocOut = vtoc; *vdataOut = vdata; *histOut = hist;
    return 0;
}

/* findMarkerGraphReverseComplementVertices (:1177-1230). Returns 0, or 1 when a vertex's reverse complemented markers are
 * not all on one (valid) vertex, 2 when rc(rc(v)) != v. */
int orc_find_rc_vertices(const uint64_t* toc, uint64_t R, const uint64_t* table, const uint64_t* vtoc, const uint64_t* vdata, uint64_t V,
                         uint64_t* rc)
{
    const uint64_t rows = 2 * R;
    for(uint64_t v = 0; v < V; v++) {
        uint64_t r = MG_INVALID40;
        for(uint64_t j = vtoc[v]; j < vtoc[v + 1]; j++) {
            const uint64_t m = vdata[j], o = orientedReadOf(toc, rows, m);
            const uint64_t t = table[rcMarker(toc, o, m - toc[o])];
            if(j == vtoc[v]) r = t;
            if(t == MG_INVALID40 || t >= V || t != r) return 1;
        }
        rc[v] = r;
    }
    for(uint64_t v = 0; v < V; v++) if(rc[rc[v]] != v) return 2;
    return 0;
}
