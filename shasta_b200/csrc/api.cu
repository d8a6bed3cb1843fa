// C ABI (include/shasta_b200.h): argument checking, exception -> status translation, marker upload.
#include "context.cuh"
#include <vector>
#include "compressed_alignment.cuh"
#include "lowhash_kernels.cuh"
#include "hostpool.cuh"
#include "digest.cuh"

#include <cstring>
#include <string>

namespace shb {

static thread_local std::string g_lastError;
void setLastError(const std::string& message) { g_lastError = message; }

void lowhash0(shb_context* c, const shb_lowhash_params& p, void** candidatesOut, uint64_t* candidateCountOut,
              uint64_t* statsOut, uint64_t* iterSummary, uint64_t maxIterSummary, shb_lowhash_result* result);

void computeAlignments(shb_context* c, const void* candidatesHost, uint64_t n, const shb_align_options& o,
                       void** alignmentDataOut, uint64_t* alignmentCountOut,
                       uint64_t** compressedTocOut, uint8_t** compressedDataOut, shb_align_result* result,
                       bool explicitOrientation);
void destroyAlignCache(shb_context* c);
void destroyLowhashState(shb_context* c);
void destroyDistState(shb_context* c);
void computeAlignmentTable(shb_context* c, const void* alignmentData, uint64_t n, uint64_t readCount, uint32_t** tocOut, uint32_t** dataOut);
void findMarkers(shb_context* c, uint32_t k, uint64_t readCount, const uint64_t* wordOffsets, const uint64_t* words,
                 const uint64_t* baseCounts, const uint8_t* kmerTable24, const uint32_t* isMarkerBitmap,
                 const uint8_t* readFlags, uint64_t** tocOut, uint8_t** data7Out, shb_marker_result* result);
void computeCandidateTable(shb_context* c, const void* candidates, uint64_t n, uint64_t readCount, uint64_t** tocOut, uint64_t** dataOut);
void createReadGraph(shb_context* c, void* alignmentData, uint64_t n, uint64_t readCount, uint32_t maxAlignmentCount,
                     const uint8_t* eligibleHost,
                     uint8_t** keepOut, void** edgesOut, uint64_t* edgeCountOut, uint32_t** connectivityTocOut, uint32_t** connectivityDataOut);
void flagPalindromicReads(shb_context* c, const shb_palindromic_params& p, uint8_t* flagsOut, uint32_t* alignedOut,
                          uint32_t* nearOut, shb_palindromic_result* result);
void palindromicReadAlignment(shb_context* c, uint64_t readId, const shb_palindromic_params& p, uint32_t** ordinals, uint64_t* count);
void readGraph2Criteria(const uint32_t* rec, uint64_t n, const double* percentiles, shb_read_graph2_criteria& out, std::vector<uint8_t>& eligible);
bool peakFinderCutoff(const uint64_t* y, uint64_t n, double minAreaFraction, uint64_t startIndex, uint64_t* cutoff, double* observed);
void createMarkerGraphVertices(shb_context* c, const shb_marker_graph_params& p, const uint32_t* edges, uint64_t edgeCount,
                               const uint64_t* ctoc, const uint8_t* cdata, uint64_t alignmentCount, const uint8_t* readFlags,
                               uint8_t** vertexTableOut, uint8_t** verticesTocOut, uint64_t** verticesDataOut, uint64_t** histogramOut,
                               shb_marker_graph_result* result);
void findMarkerGraphReverseComplementVertices(shb_context* c, const uint8_t* table5, const uint8_t* toc5, const uint64_t* vdata,
                                              uint64_t V, uint64_t** rcOut);
void createMarkerGraphEdges(shb_context* c, const uint8_t* table5, uint64_t tableCount, const uint8_t* toc5, const uint64_t* vdata,
                            uint64_t V, uint8_t** edgesOut, uint64_t** itocOut, uint8_t** idataOut, uint64_t** stocOut,
                            uint8_t** sdataOut, uint64_t** ttocOut, uint8_t** tdataOut, shb_marker_graph_edges_result* result);
void findMarkerGraphReverseComplementEdges(shb_context* c, const uint64_t* rcVertex, uint64_t V, const uint8_t* edges, uint64_t E,
                                           const uint64_t* itoc, const uint8_t* idata, const uint64_t* stoc, const uint8_t* sdata,
                                           uint64_t** rcOut, shb_marker_graph_edges_result* result);
void flagCrossStrandReadGraphEdges1(shb_context* c, int64_t maxDistance, uint32_t* edges, uint64_t edgeCount, const uint32_t* connToc,
                                    const uint32_t* connData, uint64_t readCount, uint32_t* rec, uint64_t alignmentCount,
                                    shb_cross_strand_result* result);
void flagChimericReads(shb_context* c, uint64_t maxDistance, const uint32_t* edges, uint64_t edgeCount, const uint32_t* connToc,
                       const uint32_t* connData, uint64_t readCount, uint8_t* readFlags, uint32_t* rec, uint64_t alignmentCount,
                       shb_chimeric_result* result);

template<class F> shb_status guarded(F&& f)
{
    try {
        f();
        return SHB_OK;
    } catch(const Error& e) {
        setLastError(e.what());
        return e.status;
    } catch(const std::exception& e) {
        setLastError(e.what());
        return SHB_ERR_INVALID;
    }
}

static void setCommonMarkerState(shb_context* c, uint64_t readCountTotal, uint64_t readBegin, uint64_t readEnd,
                                 const uint64_t* toc, const uint8_t* readFlags, uint64_t totalMarkerCount)
{
    SHB_REQUIRE(readBegin <= readEnd && readEnd <= readCountTotal, SHB_ERR_INVALID, "Invalid read range.");
    SHB_REQUIRE(toc != nullptr && (readFlags != nullptr || readCountTotal == 0), SHB_ERR_INVALID, "Null marker arrays.");
    const uint64_t rows = 2 * (readEnd - readBegin);
    SHB_REQUIRE(toc[0] == 0, SHB_ERR_INVALID, "The marker toc must be relative (toc[0] == 0).");
    for(uint64_t i = 0; i < rows; i++) {
        SHB_REQUIRE(toc[i] <= toc[i+1], SHB_ERR_INVALID, "The marker toc is not monotonic.");
    }
    c->markerGeneration++;
    c->readCountTotal = readCountTotal;
    c->readBegin = readBegin;
    c->readEnd = readEnd;
    c->totalMarkerCount = totalMarkerCount;
    c->localMarkerCount = toc[rows];
    c->tocHost.assign(toc, toc + rows + 1);
    c->readFlagsHost.assign(readFlags, readFlags + readCountTotal);
    c->toc.reserve(rows + 1);
    c->readFlags.reserve(readCountTotal + 1);
    SHB_CUDA(cudaMemcpyAsync(c->toc.get(), toc, (rows + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
    if(readCountTotal) {
        SHB_CUDA(cudaMemcpyAsync(c->readFlags.get(), readFlags, readCountTotal, cudaMemcpyHostToDevice, c->stream));
    }
}

} // namespace shb

using namespace shb;

extern "C" {

const char* shb_last_error(void) { return g_lastError.c_str(); }

shb_status shb_context_create(int device, shb_context** ctx)
{
    return guarded([&] {
        SHB_REQUIRE(ctx != nullptr, SHB_ERR_INVALID, "Null context pointer.");
        int count = 0;
        SHB_CUDA(cudaGetDeviceCount(&count));
        SHB_REQUIRE(device >= 0 && device < count, SHB_ERR_CUDA, "No such CUDA device.");
        cudaDeviceProp prop;
        SHB_CUDA(cudaGetDeviceProperties(&prop, device));
        SHB_REQUIRE(prop.major == 9 && prop.minor == 0, SHB_ERR_CUDA,
                    std::string("shasta_b200 is built for sm_90a (H100) only; device is sm_") + std::to_string(prop.major) + std::to_string(prop.minor));
        SHB_CUDA(cudaSetDevice(device));
        shb_context* c = new shb_context();
        c->device = device;
        SHB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
        SHB_CUDA(cudaStreamCreateWithFlags(&c->copyStream[0], cudaStreamNonBlocking));
        SHB_CUDA(cudaStreamCreateWithFlags(&c->copyStream[1], cudaStreamNonBlocking));
        c->scalars.reserve(shb::kScalarWords);     // never reallocated: device pointers into it are held across calls
        *ctx = c;
    });
}

void shb_context_destroy(shb_context* c)
{
    if(!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    destroyDistState(c);
    destroyAlignCache(c);
    destroyLowhashState(c);
    for(int i = 0; i < shb::kStageSlots; i++) { if(c->pinnedStage[i]) cudaFreeHost(c->pinnedStage[i]); if(c->stageEvent[i]) cudaEventDestroy(c->stageEvent[i]); }
    if(c->stream) cudaStreamDestroy(c->stream);
    for(int i = 0; i < 2; i++) if(c->copyStream[i]) cudaStreamDestroy(c->copyStream[i]);
    delete c;
}

void shb_free(void* p) { shb::HostPool::instance().release(p); }
void shb_trim_host_cache(void) { shb::HostPool::instance().trim(); }

shb_status shb_set_markers(shb_context* c, uint64_t readCountTotal, uint64_t readBegin, uint64_t readEnd,
                           const uint64_t* toc, const uint8_t* markerData7, const uint8_t* readFlags,
                           uint64_t totalMarkerCount)
{
    return guarded([&] {
        SHB_REQUIRE(c != nullptr, SHB_ERR_INVALID, "Null context.");
        SHB_CUDA(cudaSetDevice(c->device));
        c->haveMarkers = false;
        setCommonMarkerState(c, readCountTotal, readBegin, readEnd, toc, readFlags, totalMarkerCount);
        const uint64_t M = c->localMarkerCount;
        SHB_REQUIRE(markerData7 != nullptr || M == 0, SHB_ERR_INVALID, "Null marker data.");
        c->kmerIdsOwned.reserve(M + 64);
        // Stream the 7-byte records through two staging buffers; only the uint32 SoA stays resident.
        // SHB_MARKER_UPLOAD_CHUNK: test hook that shrinks the staging chunk so that small marker sets cross its seams.
        const uint64_t chunkMarkers = (uint64_t(envCount("SHB_MARKER_UPLOAD_CHUNK", 32u << 20)) + 1023) & ~1023ull;  // multiple of 1024
        const uint64_t chunkBytes = chunkMarkers * 7;
        DeviceBuffer<uint8_t> staging[2];
        for(uint64_t begin = 0, k = 0; begin < M; begin += chunkMarkers, k++) {
            const int b = int(k & 1);
            const uint64_t nMarkers = std::min(chunkMarkers, M - begin);
            const uint64_t nBytes = nMarkers * 7;
            if(!staging[b].get()) staging[b].reserve(std::min(chunkBytes, M * 7) + 16);
            cudaStream_t s = c->copyStream[b];
            SHB_CUDA(cudaMemcpyAsync(staging[b].get(), markerData7 + begin * 7, nBytes, cudaMemcpyHostToDevice, s));
            const uint64_t wordCount = (nBytes + 3) / 4;        // the last partial word is inside the +16 slack
            SHB_LAUNCH(extractKmerIdsKernel, ceilDiv(nMarkers, kExtractMarkersPerBlock), kExtractThreads, 0, s,
                       reinterpret_cast<const uint32_t*>(staging[b].get()), wordCount, nMarkers,
                       c->kmerIdsOwned.get() + begin);
        }
        SHB_CUDA(cudaStreamSynchronize(c->copyStream[0]));
        SHB_CUDA(cudaStreamSynchronize(c->copyStream[1]));
        SHB_CUDA(cudaStreamSynchronize(c->stream));
        c->kmerIds = c->kmerIdsOwned.get();
        c->haveMarkers = true;
    });
}

shb_status shb_set_markers_device(shb_context* c, uint64_t readCountTotal, uint64_t readBegin, uint64_t readEnd,
                                  const uint64_t* tocHost, const uint32_t* kmerIdsDevice,
                                  const uint8_t* readFlagsHost, uint64_t totalMarkerCount)
{
    return guarded([&] {
        SHB_REQUIRE(c != nullptr, SHB_ERR_INVALID, "Null context.");
        SHB_CUDA(cudaSetDevice(c->device));
        c->haveMarkers = false;
        setCommonMarkerState(c, readCountTotal, readBegin, readEnd, tocHost, readFlagsHost, totalMarkerCount);
        SHB_REQUIRE(kmerIdsDevice != nullptr || c->localMarkerCount == 0, SHB_ERR_INVALID, "Null k-mer id array.");
        SHB_CUDA(cudaStreamSynchronize(c->stream));
        c->kmerIdsOwned.release();
        c->kmerIds = kmerIdsDevice;
        c->haveMarkers = true;
    });
}

shb_status shb_lowhash0(shb_context* c, const shb_lowhash_params* params, void** candidates, uint64_t* candidateCount,
                        uint64_t* stats, uint64_t* iterSummary, uint64_t maxIterSummary, shb_lowhash_result* result)
{
    return guarded([&] {
        SHB_REQUIRE(c && params && candidates && candidateCount, SHB_ERR_INVALID, "Null argument.");
        lowhash0(c, *params, candidates, candidateCount, stats, iterSummary, maxIterSummary, result);
    });
}

shb_status shb_find_alignment_candidates_lowhash0(
    shb_context* c, uint64_t readCount, const uint64_t* toc, const uint8_t* markerData7, const uint8_t* readFlags,
    const shb_lowhash_params* params, void** candidates, uint64_t* candidateCount, uint64_t* stats,
    shb_lowhash_result* result)
{
    shb_status s = shb_set_markers(c, readCount, 0, readCount, toc, markerData7, readFlags, toc ? toc[2 * readCount] : 0);
    if(s != SHB_OK) return s;
    return shb_lowhash0(c, params, candidates, candidateCount, stats, nullptr, 0, result);
}

shb_status shb_markers_device(shb_context* c, void** kmerIdsDevice, uint64_t* localMarkerCount)
{
    return guarded([&] {
        SHB_REQUIRE(c && kmerIdsDevice && localMarkerCount, SHB_ERR_INVALID, "Null argument.");
        SHB_REQUIRE(c->haveMarkers, SHB_ERR_STATE, "Markers are not accessible.");
        *kmerIdsDevice = const_cast<uint32_t*>(c->kmerIds);
        *localMarkerCount = c->localMarkerCount;
    });
}

shb_status shb_compute_alignments(shb_context* c, const void* candidates, uint64_t candidateCount,
                                  const shb_align_options* options, void** alignmentData, uint64_t* alignmentCount,
                                  uint64_t** compressedToc, uint8_t** compressedData, shb_align_result* result)
{
    return guarded([&] {
        SHB_REQUIRE(c && options && alignmentData && alignmentCount && compressedToc && compressedData, SHB_ERR_INVALID, "Null argument.");
        computeAlignments(c, candidates, candidateCount, *options, alignmentData, alignmentCount, compressedToc, compressedData, result, false);
    });
}

shb_status shb_align_oriented_reads(shb_context* c, uint32_t orientedReadId0, uint32_t orientedReadId1,
                                    const shb_align_options* options, uint32_t** ordinals, uint64_t* markerCount,
                                    uint32_t* alignmentInfo13)
{
    return guarded([&] {
        SHB_REQUIRE(c && options && ordinals && markerCount, SHB_ERR_INVALID, "Null argument.");
        SHB_REQUIRE(orientedReadId0 != orientedReadId1, SHB_ERR_INVALID, "alignOrientedReads needs two different oriented reads.");
        const uint32_t strand0 = orientedReadId0 & 1u, strand1 = orientedReadId1 & 1u;
        const uint32_t cand[3] = {orientedReadId0 >> 1, orientedReadId1 >> 1, (strand0 == strand1 ? 1u : 0u) | (strand0 ? 0x100u : 0u)};
        void* rec = nullptr; uint64_t count = 0; uint64_t* toc = nullptr; uint8_t* data = nullptr;
        computeAlignments(c, cand, 1, *options, &rec, &count, &toc, &data, nullptr, true);
        HostResult recHold(rec), tocHold(toc), dataHold(data);
        *markerCount = 0;
        *ordinals = nullptr;
        if(alignmentInfo13) memset(alignmentInfo13, 0, 13 * sizeof(uint32_t));
        if(count == 1) {
            const uint32_t* w = static_cast<const uint32_t*>(rec);
            const uint64_t n = w[9];
            HostResult out(allocHostResult(8 * n + 8));
            SHB_REQUIRE(out.p != nullptr, SHB_ERR_OOM, "Out of host memory for the alignment.");
            // shasta::decompress (src/compressAlignment.cpp:73-137): the streaks become ordinal pairs, at most n of them written.
            const uint64_t bytes = toc[1] - toc[0];
            std::vector<uint8_t> s(data, data + bytes);
            s.resize(bytes + 8);                                // decodeStreak reads whole 8-byte words
            uint32_t* o = static_cast<uint32_t*>(out.p);
            uint64_t pos = 0, got = 0;
            uint32_t ordinal0 = 0, ordinal1 = 0;
            int32_t skip0, skip1; uint32_t len;
            while(pos < bytes && decodeStreak(s.data(), pos, bytes, skip0, skip1, len)) {
                ordinal0 += uint32_t(skip0); ordinal1 += uint32_t(skip1);
                for(uint32_t i = 0; i < len; i++, got++) if(got < n) { o[2 * got] = ordinal0 + i; o[2 * got + 1] = ordinal1 + i; }
                ordinal0 += len - 1; ordinal1 += len - 1;
            }
            SHB_REQUIRE(pos == bytes && got == n, SHB_ERR_CUDA, "Internal error: the compressed alignment does not decode to markerCount pairs.");
            if(alignmentInfo13) memcpy(alignmentInfo13, w + 3, 13 * sizeof(uint32_t));
            *markerCount = n;
            *ordinals = static_cast<uint32_t*>(out.take());
        }
    });
}

shb_status shb_compute_alignment_table(shb_context* c, const void* alignmentData, uint64_t alignmentCount, uint64_t readCount,
                                       uint32_t** tableToc, uint32_t** tableData)
{
    return guarded([&] {
        SHB_REQUIRE(c && tableToc && tableData && (alignmentData || alignmentCount == 0), SHB_ERR_INVALID, "Null argument.");
        computeAlignmentTable(c, alignmentData, alignmentCount, readCount, tableToc, tableData);
    });
}

shb_status shb_find_markers(shb_context* c, uint32_t k, uint64_t readCount, const uint64_t* readWordOffsets,
                            const uint64_t* readWords, const uint64_t* baseCounts, const uint8_t* kmerTable,
                            const uint32_t* isMarkerBitmap, const uint8_t* readFlags,
                            uint64_t** markerToc, uint8_t** markerData7, shb_marker_result* result)
{
    return guarded([&] {
        SHB_REQUIRE(c != nullptr, SHB_ERR_INVALID, "Null context.");
        findMarkers(c, k, readCount, readWordOffsets, readWords, baseCounts, kmerTable, isMarkerBitmap, readFlags, markerToc, markerData7, result);
    });
}

shb_status shb_compute_candidate_table(shb_context* c, const void* candidates, uint64_t candidateCount, uint64_t readCount,
                                       uint64_t** tableToc, uint64_t** tableData)
{
    return guarded([&] {
        SHB_REQUIRE(c && tableToc && tableData && (candidates || candidateCount == 0), SHB_ERR_INVALID, "Null argument.");
        computeCandidateTable(c, candidates, candidateCount, readCount, tableToc, tableData);
    });
}

shb_status shb_create_read_graph(shb_context* c, void* alignmentData, uint64_t alignmentCount, uint64_t readCount,
                                 uint32_t maxAlignmentCount, uint8_t** keep, void** edges, uint64_t* edgeCount,
                                 uint32_t** connectivityToc, uint32_t** connectivityData)
{
    return guarded([&] {
        SHB_REQUIRE(c && keep && edges && edgeCount && connectivityToc && connectivityData && (alignmentData || alignmentCount == 0),
                    SHB_ERR_INVALID, "Null argument.");
        createReadGraph(c, alignmentData, alignmentCount, readCount, maxAlignmentCount, nullptr, keep, edges, edgeCount, connectivityToc, connectivityData);
    });
}

shb_status shb_create_read_graph2(shb_context* c, void* alignmentData, uint64_t alignmentCount, uint64_t readCount,
                                  uint32_t maxAlignmentCount, double markerCountPercentile, double alignedFractionPercentile,
                                  double maxSkipPercentile, double maxDriftPercentile, double maxTrimPercentile,
                                  shb_read_graph2_criteria* criteria, uint8_t** keep, void** edges, uint64_t* edgeCount,
                                  uint32_t** connectivityToc, uint32_t** connectivityData)
{
    return guarded([&] {
        SHB_REQUIRE(c && criteria && keep && edges && edgeCount && connectivityToc && connectivityData && (alignmentData || alignmentCount == 0),
                    SHB_ERR_INVALID, "Null argument.");
        const double percentiles[5] = {markerCountPercentile, alignedFractionPercentile, maxSkipPercentile, maxDriftPercentile, maxTrimPercentile};
        std::vector<uint8_t> eligible;
        readGraph2Criteria(static_cast<const uint32_t*>(alignmentData), alignmentCount, percentiles, *criteria, eligible);
        eligible.push_back(0);      // never an empty array
        createReadGraph(c, alignmentData, alignmentCount, readCount, maxAlignmentCount, eligible.data(), keep, edges, edgeCount,
                        connectivityToc, connectivityData);
    });
}

shb_status shb_flag_palindromic_reads(shb_context* c, const shb_palindromic_params* params, uint8_t* readFlags,
                                      uint32_t* alignedMarkerCount, uint32_t* nearDiagonalMarkerCount,
                                      shb_palindromic_result* result)
{
    return guarded([&] {
        SHB_REQUIRE(c && params, SHB_ERR_INVALID, "Null argument.");
        flagPalindromicReads(c, *params, readFlags, alignedMarkerCount, nearDiagonalMarkerCount, result);
    });
}

shb_status shb_palindromic_read_alignment(shb_context* c, uint64_t readId, const shb_palindromic_params* params,
                                          uint32_t** ordinals, uint64_t* count)
{
    return guarded([&] {
        SHB_REQUIRE(c && params && ordinals && count, SHB_ERR_INVALID, "Null argument.");
        palindromicReadAlignment(c, readId, *params, ordinals, count);
    });
}

shb_status shb_flag_cross_strand_read_graph_edges1(shb_context* c, int64_t maxDistance, void* readGraphEdges, uint64_t edgeCount,
                                                   const uint32_t* connectivityToc, const uint32_t* connectivityData, uint64_t readCount,
                                                   void* alignmentData, uint64_t alignmentCount, shb_cross_strand_result* result)
{
    return guarded([&] {
        SHB_REQUIRE(c && (readGraphEdges || edgeCount == 0) && connectivityToc && (connectivityData || connectivityToc[2 * readCount] == 0) &&
                    (alignmentData || alignmentCount == 0), SHB_ERR_INVALID, "Null argument.");
        flagCrossStrandReadGraphEdges1(c, maxDistance, static_cast<uint32_t*>(readGraphEdges), edgeCount, connectivityToc, connectivityData,
                                       readCount, static_cast<uint32_t*>(alignmentData), alignmentCount, result);
    });
}

shb_status shb_flag_chimeric_reads(shb_context* c, uint64_t maxDistance, const void* readGraphEdges, uint64_t edgeCount,
                                   const uint32_t* connectivityToc, const uint32_t* connectivityData, uint64_t readCount,
                                   uint8_t* readFlags, void* alignmentData, uint64_t alignmentCount, shb_chimeric_result* result)
{
    return guarded([&] {
        SHB_REQUIRE(c && (readGraphEdges || edgeCount == 0) && connectivityToc && (connectivityData || connectivityToc[2 * readCount] == 0) &&
                    (readFlags || readCount == 0) && (alignmentData || alignmentCount == 0), SHB_ERR_INVALID, "Null argument.");
        flagChimericReads(c, maxDistance, static_cast<const uint32_t*>(readGraphEdges), edgeCount, connectivityToc, connectivityData,
                          readCount, readFlags, static_cast<uint32_t*>(alignmentData), alignmentCount, result);
    });
}

shb_status shb_create_marker_graph_vertices(shb_context* c, const shb_marker_graph_params* params, const void* readGraphEdges,
                                            uint64_t edgeCount, const uint64_t* compressedToc, const uint8_t* compressedData,
                                            uint64_t alignmentCount, const uint8_t* readFlags, uint8_t** vertexTable,
                                            uint8_t** verticesToc, uint64_t** verticesData, uint64_t** histogram,
                                            shb_marker_graph_result* result)
{
    return guarded([&] {
        SHB_REQUIRE(c && params && (readGraphEdges || edgeCount == 0) && compressedToc && (compressedData || alignmentCount == 0) &&
                    vertexTable && verticesToc && verticesData && histogram, SHB_ERR_INVALID, "Null argument.");
        SHB_REQUIRE(readFlags || (c->haveMarkers && c->readCountTotal == 0), SHB_ERR_INVALID, "Null argument.");
        createMarkerGraphVertices(c, *params, static_cast<const uint32_t*>(readGraphEdges), edgeCount, compressedToc, compressedData,
                                  alignmentCount, readFlags, vertexTable, verticesToc, verticesData, histogram, result);
    });
}

shb_status shb_find_marker_graph_reverse_complement_vertices(shb_context* c, const uint8_t* vertexTable, const uint8_t* verticesToc,
                                                             const uint64_t* verticesData, uint64_t vertexCount, uint64_t** rcVertex)
{
    return guarded([&] {
        SHB_REQUIRE(c && verticesToc && rcVertex && ((vertexTable && verticesData) || vertexCount == 0), SHB_ERR_INVALID, "Null argument.");
        findMarkerGraphReverseComplementVertices(c, vertexTable, verticesToc, verticesData, vertexCount, rcVertex);
    });
}

shb_status shb_create_marker_graph_edges(shb_context* c, const uint8_t* vertexTable, uint64_t vertexTableCount,
                                         const uint8_t* verticesToc, const uint64_t* verticesData, uint64_t vertexCount,
                                         uint8_t** edges, uint64_t** intervalsToc, uint8_t** intervalsData,
                                         uint64_t** bySourceToc, uint8_t** bySourceData, uint64_t** byTargetToc,
                                         uint8_t** byTargetData, shb_marker_graph_edges_result* result)
{
    return guarded([&] {
        SHB_REQUIRE(c && (vertexTable || vertexTableCount == 0) && verticesToc && (verticesData || vertexCount == 0) && edges &&
                    intervalsToc && intervalsData && bySourceToc && bySourceData && byTargetToc && byTargetData, SHB_ERR_INVALID,
                    "Null argument.");
        createMarkerGraphEdges(c, vertexTable, vertexTableCount, verticesToc, verticesData, vertexCount, edges, intervalsToc,
                               intervalsData, bySourceToc, bySourceData, byTargetToc, byTargetData, result);
    });
}

shb_status shb_find_marker_graph_reverse_complement_edges(shb_context* c, const uint64_t* rcVertex, uint64_t vertexCount,
                                                          const uint8_t* edges, uint64_t edgeCount, const uint64_t* intervalsToc,
                                                          const uint8_t* intervalsData, const uint64_t* bySourceToc,
                                                          const uint8_t* bySourceData, uint64_t** rcEdge,
                                                          shb_marker_graph_edges_result* result)
{
    return guarded([&] {
        SHB_REQUIRE(c && (rcVertex || vertexCount == 0) && (edges || edgeCount == 0) && intervalsToc && bySourceToc && rcEdge,
                    SHB_ERR_INVALID, "Null argument.");
        SHB_REQUIRE(intervalsData || intervalsToc[edgeCount] == 0, SHB_ERR_INVALID, "Null argument.");
        SHB_REQUIRE(bySourceData || bySourceToc[vertexCount] == 0, SHB_ERR_INVALID, "Null argument.");
        findMarkerGraphReverseComplementEdges(c, rcVertex, vertexCount, edges, edgeCount, intervalsToc, intervalsData, bySourceToc,
                                              bySourceData, rcEdge, result);
    });
}

int shb_peak_finder_cutoff(const uint64_t* histogram, uint64_t n, double minAreaFraction, uint64_t startIndex, uint64_t* cutoff,
                           double* observedAreaFraction)
{
    uint64_t x = 0;
    double observed = 0;
    const bool threw = peakFinderCutoff(histogram, n, minAreaFraction, startIndex, &x, &observed);
    if(cutoff) *cutoff = x;
    if(observedAreaFraction) *observedAreaFraction = observed;
    return threw ? 1 : 0;
}

shb_status shb_test_radix_sort(shb_context* c, uint64_t* keys, uint32_t* values, uint64_t n,
                               int lowBegin, int lowEnd, int highBegin, int highEnd)
{
    return guarded([&] {
        SHB_REQUIRE(c && (keys || n == 0), SHB_ERR_INVALID, "Null argument.");
        SHB_CUDA(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        DeviceBuffer<uint64_t> kA, kB;
        DeviceBuffer<uint32_t> vA, vB;
        kA.reserve(n + 1); kB.reserve(n + 1); vA.reserve(n + 1); vB.reserve(n + 1);
        SHB_CUDA(cudaMemcpyAsync(kA.get(), keys, 8 * n, cudaMemcpyHostToDevice, st));
        if(values) SHB_CUDA(cudaMemcpyAsync(vA.get(), values, 4 * n, cudaMemcpyHostToDevice, st));
        const int ranges[2][2] = {{lowBegin, lowEnd}, {highBegin, highEnd}};
        const int rangeCount = (highEnd > highBegin) ? 2 : 1;
        const bool inB = values ? radixSort<true>(kA.get(), kB.get(), vA.get(), vB.get(), n, ranges, rangeCount, c->sortWs, st)
                                : radixSort<false>(kA.get(), kB.get(), nullptr, nullptr, n, ranges, rangeCount, c->sortWs, st);
        SHB_CUDA(cudaMemcpyAsync(keys, inB ? kB.get() : kA.get(), 8 * n, cudaMemcpyDeviceToHost, st));
        if(values) SHB_CUDA(cudaMemcpyAsync(values, inB ? vB.get() : vA.get(), 4 * n, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
    });
}

uint64_t shb_digest_records(const uint32_t* records, uint64_t count, uint32_t words)
{
    uint64_t sum = 0;
    for(uint64_t i = 0; i < count; i++) {
        uint64_t h = kFnvOffset;
        for(uint32_t k = 0; k < words; k++) h = fnvWord(h, records[i * words + k]);
        sum += fnvFinish(h);
    }
    return sum;
}

uint64_t shb_digest_compressed(const uint32_t* alignmentData, uint64_t count, const uint64_t* compressedToc,
                               const uint8_t* compressedData)
{
    uint64_t sum = 0;
    for(uint64_t i = 0; i < count; i++) {
        uint64_t h = kFnvOffset;
        h = fnvWord(h, alignmentData[16 * i]); h = fnvWord(h, alignmentData[16 * i + 1]); h = fnvWord(h, alignmentData[16 * i + 2] & 0xffu);
        for(uint64_t p = compressedToc[i]; p < compressedToc[i + 1]; p++) h = fnvWord(h, compressedData[p]);
        sum += fnvFinish(h);
    }
    return sum;
}

} // extern "C"
