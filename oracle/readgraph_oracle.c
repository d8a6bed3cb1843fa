/* TEST INFRASTRUCTURE (oracle): CPU restatement of Assembler::createReadGraph, ReadGraph.creationMethod 0
 * (src/AssemblerReadGraph.cpp:35-175). Only tests/ may call it. Parity status: a restatement, pinned against the reference's
 * own code by tests/test_oracle_readgraph.py (oracle/ref_glue/ref_readgraph.cpp follows the member over the reference's
 * containers). It follows the reference's control flow with qsort in place of std::nth_element — the SET nth_element
 * leaves in the first maxAlignmentCount places is the same. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { uint32_t markerCount, alignmentId; } ReadAlignment;

/* std::greater<pair<uint32_t,uint32_t>>: descending by (markerCount, alignmentId) */
static int greaterFirst(const void* a, const void* b)
{
    const ReadAlignment* x = (const ReadAlignment*)a; const ReadAlignment* y = (const ReadAlignment*)b;
    if(x->markerCount != y->markerCount) return x->markerCount > y->markerCount ? -1 : 1;
    if(x->alignmentId != y->alignmentId) return x->alignmentId > y->alignmentId ? -1 : 1;
    return 0;
}

/* alignmentData: n 64-byte records (in/out: isInReadGraph). keep: uint8[n]. edges: room for 2n 16-byte records.
 * connToc: uint32[2*readCount+1], connData: uint32[4n]. *edgeCountOut: the number of edges. Returns 0, or 1 when a kept
 * alignment gives an edge, or a reverse-complement edge, whose oriented reads are not in increasing order: the reference's
 * SHASTA_ASSERT at src/AssemblerReadGraph.cpp:134,140 (readIds[0] > readIds[1], or a read aligned to itself). An alignment
 * that is not kept is never looked at there, so it may be unordered. */
static int createReadGraph(uint32_t* alignmentData, uint64_t n, uint64_t readCount, uint32_t maxAlignmentCount,
                           const uint8_t* eligible /* null: every alignment */,
                           uint8_t* keep, uint32_t* edges, uint64_t* edgeCountOut, uint32_t* connToc, uint32_t* connData)
{
    memset(keep, 0, n);
    /* the rows (readId, 0) of the alignment table: every alignment of the read (src/AssemblerAlign.cpp:509-571) */
    uint64_t* count = (uint64_t*)calloc(readCount + 1, sizeof(uint64_t));
    for(uint64_t a = 0; a < n; a++) {
        if(eligible && !eligible[a]) continue;          /* passesReadGraph2Criteria, src/AssemblerReadGraph2.cpp:218-221 */
        count[alignmentData[16 * a] + 1]++; count[alignmentData[16 * a + 1] + 1]++;
    }
    for(uint64_t r = 0; r < readCount; r++) count[r + 1] += count[r];
    ReadAlignment* all = (ReadAlignment*)malloc((2 * n + 1) * sizeof(ReadAlignment));
    uint64_t* fill = (uint64_t*)malloc((readCount + 1) * sizeof(uint64_t));
    memcpy(fill, count, (readCount + 1) * sizeof(uint64_t));
    for(uint64_t a = 0; a < n; a++) {
        if(eligible && !eligible[a]) continue;
        for(int side = 0; side < 2; side++) {
            ReadAlignment* p = all + fill[alignmentData[16 * a + side]]++;
            p->markerCount = alignmentData[16 * a + 9];         /* AlignmentInfo::markerCount */
            p->alignmentId = (uint32_t)a;
        }
    }
    /* :53-86 */
    for(uint64_t r = 0; r < readCount; r++) {
        ReadAlignment* row = all + count[r];
        uint64_t size = count[r + 1] - count[r];
        if(size > maxAlignmentCount) {
            qsort(row, size, sizeof(ReadAlignment), greaterFirst);
            size = maxAlignmentCount;
        }
        for(uint64_t k = 0; k < size; k++) keep[row[k].alignmentId] = 1;
    }
    free(all); free(fill); free(count);
    /* createReadGraphUsingSelectedAlignments :95-144 */
    uint64_t edgeCount = 0;
    *edgeCountOut = 0;
    for(uint64_t a = 0; a < n; a++) {
        uint32_t* rec = alignmentData + 16 * a;
        rec[15] = (rec[15] & ~1u) | keep[a];
        if(!keep[a]) continue;
        const uint32_t o0 = 2 * rec[0], o1 = 2 * rec[1] + ((rec[2] & 0xff) ? 0u : 1u);
        if(!(o0 < o1 && (o0 ^ 1u) < (o1 ^ 1u))) return 1;
        for(uint32_t k = 0; k < 2; k++) {
            uint32_t* e = edges + 4 * edgeCount;
            e[0] = o0 ^ k; e[1] = o1 ^ k; e[2] = (uint32_t)a; e[3] = 0;
            edgeCount++;
        }
    }
    /* connectivity :147-159. MemoryMapped::VectorOfVectors::store fills a row from its end
     * (src/MemoryMappedVectorOfVectors.hpp:384-387) and the edges are stored in increasing order, so every row lists its
     * edges in DECREASING edge index. */
    const uint64_t rows = 2 * readCount;
    memset(connToc, 0, (rows + 1) * sizeof(uint32_t));
    for(uint64_t i = 0; i < edgeCount; i++) { connToc[edges[4 * i] + 1]++; connToc[edges[4 * i + 1] + 1]++; }
    for(uint64_t r = 0; r < rows; r++) connToc[r + 1] += connToc[r];
    uint32_t* end = (uint32_t*)malloc((rows + 1) * sizeof(uint32_t));
    memcpy(end, connToc + 1, rows * sizeof(uint32_t));
    for(uint64_t i = 0; i < edgeCount; i++) {
        connData[--end[edges[4 * i]]] = (uint32_t)i;
        connData[--end[edges[4 * i + 1]]] = (uint32_t)i;
    }
    free(end);
    *edgeCountOut = edgeCount;
    return 0;
}

int orc_create_read_graph(uint32_t* alignmentData, uint64_t n, uint64_t readCount, uint32_t maxAlignmentCount,
                          uint8_t* keep, uint32_t* edges, uint64_t* edgeCount, uint32_t* connToc, uint32_t* connData)
{
    return createReadGraph(alignmentData, n, readCount, maxAlignmentCount, NULL, keep, edges, edgeCount, connToc, connData);
}

/* shasta::Histogram2 with dynamicBounds = true (src/Histogram.cpp:14-140), restated with the effect of its update():
 * growing to `index` bins and then incrementing bin `index` touches memory one past the end, so a sample whose index is not
 * below the current size is never counted. */
typedef struct { double start, binSize; uint64_t size, capacity; uint64_t* bins; } Hist;
static void histInit(Hist* h, double start, double stop, uint64_t binCount)
{
    h->start = start; h->binSize = (stop - start) / (double)binCount; h->size = binCount; h->capacity = binCount;
    h->bins = (uint64_t*)calloc(binCount ? binCount : 1, sizeof(uint64_t));
}
static void histUpdate(Hist* h, double x)
{
    const int64_t index = (int64_t)floor((x - h->start) / h->binSize);
    if(index < 0) return;
    if((uint64_t)index > h->size) {
        if((uint64_t)index > h->capacity) {
            uint64_t cap = h->capacity * 2 > (uint64_t)index ? h->capacity * 2 : (uint64_t)index;
            h->bins = (uint64_t*)realloc(h->bins, cap * sizeof(uint64_t));
            memset(h->bins + h->capacity, 0, (cap - h->capacity) * sizeof(uint64_t));
            h->capacity = cap;
        }
        h->size = (uint64_t)index;
    }
    if((uint64_t)index < h->size) h->bins[index]++;
}
static double histThreshold(const Hist* h, double fraction)
{
    uint64_t total = 0;
    for(uint64_t i = 0; i < h->size; i++) total += h->bins[i];
    double cumulativeSum = 0;
    uint64_t i;
    for(i = 0; i < h->size; i++) {
        cumulativeSum += (double)h->bins[i];
        if(cumulativeSum / (double)total >= fraction) break;
    }
    return h->start + h->binSize * (double)i + h->binSize / 2;
}
/* for the pin test against the compiled reference class */
double orc_histogram2_threshold(const double* x, uint64_t n, double start, double stop, uint64_t binCount, double fraction)
{
    Hist h; histInit(&h, start, stop, binCount);
    for(uint64_t i = 0; i < n; i++) histUpdate(&h, x[i]);
    const double t = histThreshold(&h, fraction);
    free(h.bins);
    return t;
}

typedef struct { double minAlignedFraction; uint32_t markerCount, maxDrift, maxSkip, trim; } Indicators;
/* AlignmentInfo accessors, src/Alignment.hpp:103-121, 252-284 */
static Indicators indicators(const uint32_t* rec)
{
    const uint32_t* d0 = rec + 3; const uint32_t* d1 = rec + 6;
    Indicators r;
    r.markerCount = rec[9]; r.maxSkip = rec[13]; r.maxDrift = rec[14];
    const double f0 = (double)r.markerCount / (double)(uint32_t)(d0[2] + 1 - d0[1]), f1 = (double)r.markerCount / (double)(uint32_t)(d1[2] + 1 - d1[1]);
    r.minAlignedFraction = f0 < f1 ? f0 : f1;
    const uint32_t l0 = d0[1], l1 = d1[1], r0 = d0[0] - 1 - d0[2], r1 = d1[0] - 1 - d1[2];
    const uint32_t leftTrim = l0 < l1 ? l0 : l1, rightTrim = r0 < r1 ? r0 : r1;
    r.trim = leftTrim > rightTrim ? leftTrim : rightTrim;
    return r;
}

/* createReadGraph2, src/AssemblerReadGraph2.cpp:99-248. percentiles: markerCount, alignedFraction, maxSkip, maxDrift, maxTrim.
 * criteria: double minAlignedFraction, then uint64 minAlignedMarkerCount, maxDrift, maxSkip, maxTrim (as 5 x 8 bytes). */
int orc_create_read_graph2(uint32_t* alignmentData, uint64_t n, uint64_t readCount, uint32_t maxAlignmentCount,
                           const double* percentiles, void* criteria,
                           uint8_t* keep, uint32_t* edges, uint64_t* edgeCount, uint32_t* connToc, uint32_t* connData)
{
    Hist af, mc, dr, sk, tr;
    histInit(&af, 0, 1, 100); histInit(&mc, 0, 3000, 300); histInit(&dr, 0, 100, 100); histInit(&sk, 0, 100, 100); histInit(&tr, 0, 100, 100);
    for(uint64_t i = 0; i < n; i++) {
        const Indicators a = indicators(alignmentData + 16 * i);
        histUpdate(&af, a.minAlignedFraction); histUpdate(&mc, a.markerCount); histUpdate(&dr, a.maxDrift);
        histUpdate(&sk, a.maxSkip); histUpdate(&tr, a.trim);
    }
    const double minAlignedFraction = histThreshold(&af, percentiles[1]);
    const uint64_t minAlignedMarkerCount = (uint64_t)round(histThreshold(&mc, percentiles[0]));
    const uint64_t maxDrift = (uint64_t)round(histThreshold(&dr, 1 - percentiles[3]));
    const uint64_t maxSkip = (uint64_t)round(histThreshold(&sk, 1 - percentiles[2]));
    const uint64_t maxTrim = (uint64_t)round(histThreshold(&tr, 1 - percentiles[4]));
    free(af.bins); free(mc.bins); free(dr.bins); free(sk.bins); free(tr.bins);
    memcpy(criteria, &minAlignedFraction, 8);
    memcpy((char*)criteria + 8, &minAlignedMarkerCount, 8); memcpy((char*)criteria + 16, &maxDrift, 8);
    memcpy((char*)criteria + 24, &maxSkip, 8); memcpy((char*)criteria + 32, &maxTrim, 8);
    uint8_t* eligible = (uint8_t*)malloc(n + 1);
    for(uint64_t i = 0; i < n; i++) {
        const Indicators a = indicators(alignmentData + 16 * i);
        eligible[i] = !(a.minAlignedFraction < minAlignedFraction) && !(a.markerCount < minAlignedMarkerCount) &&
                      !(a.maxDrift > maxDrift) && !(a.maxSkip > maxSkip) && !(a.trim > maxTrim);
    }
    const int status = createReadGraph(alignmentData, n, readCount, maxAlignmentCount, eligible, keep, edges, edgeCount, connToc, connData);
    free(eligible);
    return status;
}
