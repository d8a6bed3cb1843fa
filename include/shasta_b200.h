/*
 * shasta_b200 — C ABI of the H100-native implementation of Shasta's overlap-detection hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch types. Each entry point
 * cites the reference interface it replaces (paths relative to the chanzuckerberg/shasta tree).
 * The shared library is shasta_b200/lib/libshasta_b200.so (sm_90a only; there is no CPU fallback:
 * every compute entry point returns SHB_ERR_CUDA when no device is usable).
 *
 * Record layouts (SURVEY.md Appendix C):
 *   markers   : toc uint64[2R+1], row index = (readId<<1)|strand (src/ReadId.hpp:35-155);
 *               data = 7-byte CompressedMarker records {uint32 kmerId, uint24 position}
 *               (src/Marker.hpp:56-69), i.e. the payload of Data/Markers.toc + Data/Markers.data
 *   readFlags : 1 byte per read, bit0 = isPalindromic (src/ReadFlags.hpp:10-30)
 *   candidates: 12-byte OrientedReadPair {uint32 readIds[2]; uint8 isSameStrand; 3 pad}
 *               (src/OrientedReadPair.hpp:18-86); pad bytes are written as 0
 *   stats     : uint64[R][3] = ReadLowHashStatistics (src/LowHash0.cpp:386-393)
 */
#ifndef SHASTA_B200_H
#define SHASTA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    SHB_OK = 0,
    SHB_ERR_INVALID = 1,        /* bad argument; the message mirrors the reference's runtime_error text */
    SHB_ERR_CUDA = 2,           /* CUDA failure or no sm_90 device */
    SHB_ERR_OOM = 3,
    SHB_ERR_STATE = 4           /* call order violated (e.g. markers not uploaded) */
} shb_status;

typedef struct shb_context shb_context;

/* Message of the last error on the calling thread (std::runtime_error::what() equivalent). */
const char* shb_last_error(void);

/* One context per GPU / per process rank. device = CUDA ordinal. */
shb_status shb_context_create(int device, shb_context** ctx);
void shb_context_destroy(shb_context* ctx);

/* Free a host buffer returned by this library. Large buffers (>= 8 MiB) are kept on a free list and handed out
 * again by later calls (page-locked from their second use on, so that results arrive by direct DMA);
 * shb_trim_host_cache returns the cached buffers to the operating system. */
void shb_free(void* hostPtr);
void shb_trim_host_cache(void);

/* ------------------------------------------------------------------------------------------
 * Marker upload.  Replaces Assembler::accessMarkers (src/AssemblerMarkers.cpp, Data/Markers.*) +
 * LowHash0::createKmerIds (src/LowHash0.cpp:261-308): the 7-byte AoS records are streamed to the
 * device and converted to a uint32 k-mer id SoA that stays resident in HBM.
 *
 * readCountTotal = R of the whole assembly; [readBegin, readEnd) = the reads whose marker rows are
 * passed here (toc has 2*(readEnd-readBegin)+1 entries and is relative: toc[0] == 0). A single-GPU
 * run passes readBegin = 0, readEnd = readCountTotal. readFlags has readCountTotal entries.
 * totalMarkerCount = markers.totalSize() over ALL reads (enters the bucket-count rule,
 * src/LowHash0.cpp:73-76).
 */
shb_status shb_set_markers(shb_context* ctx,
                           uint64_t readCountTotal, uint64_t readBegin, uint64_t readEnd,
                           const uint64_t* toc, const uint8_t* markerData7,
                           const uint8_t* readFlags, uint64_t totalMarkerCount);

/* Same, with the k-mer ids already on the device (uint32 SoA, device pointer) — used by the
 * synthetic generator of bench.py. The library takes a copy-free reference; the caller keeps the
 * allocation alive until the context is destroyed or markers are replaced. tocHost is host memory. */
shb_status shb_set_markers_device(shb_context* ctx,
                                  uint64_t readCountTotal, uint64_t readBegin, uint64_t readEnd,
                                  const uint64_t* tocHost, const uint32_t* kmerIdsDevice,
                                  const uint8_t* readFlagsHost, uint64_t totalMarkerCount);

/* ------------------------------------------------------------------------------------------
 * Marker finding (SURVEY.md section 8f, rank 1: the producer of the path's input). Replaces Assembler::findMarkers ->
 * MarkerFinder (src/MarkerFinder.cpp:16-127, src/AssemblerMarkers.cpp): the reads go to the device as the reference
 * stores them (2 bits per base) and the markers of both strands are produced there, so the 7-byte records need not cross
 * PCIe at all when only the hot path follows.
 *   readWordOffsets : uint64[readCount+1], offsets in 64-bit words into readWords (the toc of Data/Reads)
 *   readWords       : LongBaseSequences payload (src/LongBaseSequence.hpp:33-41): per read, per 64 bases, the low bit plane
 *                     word then the high bit plane word, base 0 in the most significant bit; run-length encoded bases when the
 *                     assembly uses the RLE read representation
 *   baseCounts      : uint64[readCount]
 *   kmerTable       : 4^k KmerInfo records of 24 bytes (Data/Kmers, src/Kmer.hpp:23-38; only isMarker, byte 12, is read), or
 *                     NULL when isMarkerBitmap (4^k bits, bit i of word i/32 = k-mer i is a marker) is given instead
 *   readFlags       : 1 byte per read (Data/ReadFlags), kept for the LowHash step
 *   markerToc       : optional, receives uint64[2*readCount+1] (Data/Markers.toc payload); markerData7: optional, receives the
 *                     7-byte CompressedMarker records (Data/Markers.data payload). Free both with shb_free.
 * Afterwards the context holds the markers of all reads exactly as after shb_set_markers (k-mer id SoA resident in HBM).
 */
typedef struct {
    uint64_t readCount, baseCount, markerCount;     /* markerCount counts both strands */
    double   totalMs;                               /* device time incl. the host->device copies of the inputs */
    uint64_t kernelLaunches, h2dBytes;
} shb_marker_result;
shb_status shb_find_markers(shb_context* ctx, uint32_t k, uint64_t readCount, const uint64_t* readWordOffsets,
                            const uint64_t* readWords, const uint64_t* baseCounts, const uint8_t* kmerTable,
                            const uint32_t* isMarkerBitmap, const uint8_t* readFlags,
                            uint64_t** markerToc, uint8_t** markerData7, shb_marker_result* result);

/* ------------------------------------------------------------------------------------------
 * LowHash0.  Replaces Assembler::findAlignmentCandidatesLowHash0 (src/AssemblerLowHash.cpp:10-55,
 * declaration src/Assembler.hpp:688-699; Python binding src/PythonModule.cpp:218-228).
 * Field for field the reference's arguments; threadCount is accepted and ignored.
 */
typedef struct {
    uint64_t m;
    double   hashFraction;
    uint64_t minHashIterationCount;
    double   alignmentCandidatesPerRead;
    uint64_t log2MinHashBucketCount;
    uint64_t minBucketSize;
    uint64_t maxBucketSize;
    uint64_t minFrequency;
    uint64_t threadCount;
    /* 0: candidate counts are merged once after the last iteration (fast path; needs
     *    minHashIterationCount != 0).  1: merged after every iteration, which also yields the
     *    per-iteration "high frequency / total" summary of src/LowHash0.cpp:185-196.
     *    minHashIterationCount == 0 forces mode 1. */
    uint32_t perIterationMerge;
    uint32_t reserved;
} shb_lowhash_params;

typedef struct {
    uint64_t iterations;            /* iterations executed */
    uint64_t log2BucketCount;       /* after the rule of src/LowHash0.cpp:79-98 */
    uint64_t lowHashCount;          /* total low hashes over all iterations */
    uint64_t pairCount;             /* candidate pair hits generated over all iterations */
    uint64_t candidateCount;
    double   sweepMs;               /* device time of the hash sweep kernels (CUDA events) */
    double   totalMs;               /* device time of the whole call */
    uint64_t sweepLaunches;         /* number of sweep kernel launches */
    uint64_t kernelLaunches;        /* all kernels launched by the call */
    uint64_t candidateDigest;       /* order-independent digest of the emitted candidates (shb_digest_records of the
                                       12-byte records as 3 words), computed on the device; for sharded runs the sum
                                       of the ranks' digests (mod 2^64) equals the single-GPU digest */
} shb_lowhash_result;

/* One-shot single-GPU call on the markers held by ctx.
 *   candidates   : *candidates receives a host buffer of 12-byte OrientedReadPair records in the
 *                  reference order (readId0, then (readId1, strand)); free with shb_free.
 *   stats        : caller-allocated uint64[readCountTotal*3], or NULL.
 *   iterSummary  : optional uint64[2*maxIterSummary] (highFrequency,total) per iteration; only
 *                  filled in perIterationMerge mode.
 */
shb_status shb_lowhash0(shb_context* ctx, const shb_lowhash_params* params,
                        void** candidates, uint64_t* candidateCount,
                        uint64_t* stats, uint64_t* iterSummary, uint64_t maxIterSummary,
                        shb_lowhash_result* result);

/* Convenience: host buffers in, host buffers out (upload + LowHash0). This is the call a
 * reference maintainer binds (see INTEGRATION.md). */
shb_status shb_find_alignment_candidates_lowhash0(
    shb_context* ctx, uint64_t readCount, const uint64_t* toc, const uint8_t* markerData7,
    const uint8_t* readFlags, const shb_lowhash_params* params,
    void** candidates, uint64_t* candidateCount, uint64_t* stats, shb_lowhash_result* result);

/* ------------------------------------------------------------------------------------------
 * Staged LowHash0 for read-sharded multi-GPU runs (SURVEY.md section 8e). Each rank holds the marker rows of
 * a contiguous read range (shb_set_markers with readBegin/readEnd); buckets are owned by ranks; between the
 * sweep and the bucket inspection the low-hash entries are exchanged (all-to-all over NCCL, done by the host:
 * shasta_b200/distributed.py), and once at the end the per-owner pair counts are exchanged by readId0 range.
 * The single-GPU shb_lowhash0 is exactly  begin; { sweep; process_entries per slab }; emit.
 * All device pointers returned here are context scratch, valid until the next LowHash call on the context.
 */
shb_status shb_lowhash_begin(shb_context* ctx, const shb_lowhash_params* params, uint64_t* log2BucketCount);
/* pass 1 (src/LowHash0.cpp:314-360) for iterationCount (<= 16) consecutive iterations over the local reads.
 * lowHashCounts[s] receives the number of entries of slab s. */
shb_status shb_lowhash_sweep(shb_context* ctx, uint64_t iterationBegin, uint32_t iterationCount, uint64_t* lowHashCounts);
/* Slab s of the last sweep: keys uint64 (bucketId<<32 | hashHighBits), vals uint32 (orientedReadId). */
shb_status shb_lowhash_slab(shb_context* ctx, uint32_t slab, void** keysDevice, void** valsDevice);
/* Stable grouping of n (uint64 key, uint32 value) items by the `bits` (<= 8) key bits starting at `shift`;
 * counts[1<<bits] receives the group sizes; the grouped arrays are returned as device pointers. */
shb_status shb_device_partition(shb_context* ctx, void* keysDevice, void* valsDevice, uint64_t n, uint32_t shift,
                                uint32_t bits, uint64_t* counts, void** keysOutDevice, void** valsOutDevice);
/* passes 2+3 (src/LowHash0.cpp:365-484) on the entries of ONE iteration whose buckets this rank owns
 * (device arrays, clobbered): statistics, pair hits, accumulation. */
shb_status shb_lowhash_process_entries(shb_context* ctx, void* keysDevice, void* valsDevice, uint64_t n);
/* Merged local accumulator: uint64 pair keys (readId0<<32 | readId1<<1 | strand), uint32 counts. */
shb_status shb_lowhash_local_pairs(shb_context* ctx, void** pairKeysDevice, void** pairCountsDevice, uint64_t* n);
/* Replace the accumulator by the (pairKey,count) items received from all ranks for this rank's readId0 range. */
shb_status shb_lowhash_set_pairs(shb_context* ctx, const void* pairKeysDevice, const void* pairCountsDevice, uint64_t n);
/* Final merge and emission (src/LowHash0.cpp:204-214) of the accumulator: host buffer of 12-byte records. */
shb_status shb_lowhash_emit(shb_context* ctx, void** candidates, uint64_t* candidateCount);
/* Device pointer of the (partial) ReadLowHashStatistics, uint64[readCountTotal*3], for the final all-reduce. */
shb_status shb_lowhash_stats_device(shb_context* ctx, void** statsDevice);
/* Counters of the staged run so far (iterations is not tracked by the staged calls and is returned as 0). */
shb_status shb_lowhash_counters(shb_context* ctx, shb_lowhash_result* result);

/* ------------------------------------------------------------------------------------------
 * Alignments.  Replaces Assembler::computeAlignments (src/AssemblerAlign.cpp:208-304, declaration
 * src/Assembler.hpp:264-270; Python binding src/PythonModule.cpp:344-345).
 * shb_align_options mirrors AlignOptions field for field (src/AssemblerOptions.hpp:177-199); k is the
 * marker k-mer length (assemblerInfo->k): the method-3 downsampling hash kmerTable[kmerId].hash
 * (src/AssemblerKmers.cpp:182-186) is recomputed from it instead of reading the 4^k-entry Data/Kmers table.
 */
typedef struct {
    int32_t  alignMethod;            /* 3 (what every shipped conf selects), 4 (Align4) or 1 (unbanded SeqAn-style DP on all
                                        markers, src/AssemblerAlign1.cpp); 0 (AlignmentGraph) is not on the path */
    int32_t  maxSkip;
    int32_t  maxDrift;
    int32_t  maxTrim;
    int32_t  maxMarkerFrequency;     /* method 0 only; ignored */
    int32_t  minAlignedMarkerCount;
    double   minAlignedFraction;
    /* Scores of methods 1 and 3 (method 4 always scores 6/-1/-1). The DP runs in int32 with sentinels: a call is
       refused with SHB_ERR_INVALID unless max(|match|, |mismatch|, |gap|) * (2 * L + 16384) < 2^28, L = the markers
       of the longest read the call aligns (6/-1/-1: L up to 22.3 M). gapScore must not be positive. */
    int32_t  matchScore;
    int32_t  mismatchScore;
    int32_t  gapScore;
    double   downsamplingFactor;
    int32_t  bandExtend;
    int32_t  maxBand;
    int32_t  sameChannelReadAlignmentSuppressDeltaThreshold;    /* not used by computeAlignments */
    int32_t  suppressContainments;
    uint64_t align4DeltaX;
    uint64_t align4DeltaY;
    uint64_t align4MinEntryCountPerCell;
    uint64_t align4MaxDistanceFromBoundary;
    uint32_t k;
    uint32_t reserved;
} shb_align_options;

typedef struct {
    uint64_t candidateCount;
    uint64_t alignmentCount;        /* stored ("good") alignments */
    uint64_t skippedCount;          /* candidates the reference would skip with a logged exception */
    uint64_t dpCells;               /* DP cell updates performed (both stages) */
    double   dpMs;                  /* device time inside the DP kernels (CUDA events) */
    double   totalMs;               /* device time of the whole call */
    uint64_t kernelLaunches;
    double   outputCopyMs;          /* host wall time of the final device->host copy of the results */
    double   hostWallMs;            /* host wall time of the whole call */
    uint64_t dpUsefulCells;         /* ... of which in-band, in-matrix cells (what the reference's DP fills; dpCells also counts
                                       the padding of the band classes and the barrier offsets) */
    uint64_t tooWideCount;          /* candidates skipped because their unbanded stage needs a band wider than 16384 offsets
                                       (included in skippedCount; the reference has no such limit) */
    uint64_t workers;               /* host worker threads (streams) the batches were spread over */
    uint64_t alignmentDataDigest;   /* order-independent digests of the AlignmentData records (16 words each) and of the */
    uint64_t compressedDigest;      /* compressed alignments (pair + bytes), computed on the device: additive over any
                                       partition of the candidates (multi-GPU parity: sum of the ranks' digests) */
} shb_align_result;

/* The digest used above, on host buffers (for checking results that came from somewhere else, e.g. the CPU path):
 *   per record of `words` uint32 words: h = 0xcbf29ce484222325; for each word: h = (h ^ word) * 0x100000001b3;
 *   h ^= h >> 32;  the digest is the sum of the records' h (mod 2^64).                                              */
uint64_t shb_digest_records(const uint32_t* records, uint64_t count, uint32_t words);
/* Compressed alignments: per alignment the same FNV chain over readId0, readId1, isSameStrand (from its 64-byte
 * AlignmentData record) and then its compressed bytes one by one; summed. */
uint64_t shb_digest_compressed(const uint32_t* alignmentData, uint64_t count, const uint64_t* compressedToc,
                               const uint8_t* compressedData);

/* Computes the marker alignment of every candidate on the markers held by ctx (all reads must be
 * resident on this GPU).
 *   candidates      : n 12-byte OrientedReadPair records (host), readIds[0] < readIds[1].
 *   alignmentData   : receives a host buffer of 64-byte AlignmentData records (src/Alignment.hpp:419-447:
 *                     OrientedReadPair + AlignmentInfo; padding bytes 0), in candidate order (the
 *                     reference's order is thread-schedule dependent, any order is legal).
 *   compressedToc   : receives uint64[count+1]; compressedData: the concatenated shasta::compress bytes
 *                     (= Data/CompressedAlignments.toc/.data payload).
 * All three are freed with shb_free.
 */
shb_status shb_compute_alignments(shb_context* ctx, const void* candidates, uint64_t candidateCount,
                                  const shb_align_options* options,
                                  void** alignmentData, uint64_t* alignmentCount,
                                  uint64_t** compressedToc, uint8_t** compressedData,
                                  shb_align_result* result);

/* One pair of oriented reads, in exactly the orientation given (orientedReadId = (readId<<1)|strand). Replaces the
 * single-pair members Assembler::alignOrientedReads4 (src/AssemblerAlign4.cpp:13-61; Python src/PythonModule.cpp:302-327),
 * alignOrientedReads3 (src/AssemblerAlign3.cpp:23-313) and alignOrientedReads1 (src/AssemblerAlign1.cpp:129-148), selected by
 * options->alignMethod. The pair goes through the same device path as shb_compute_alignments, so the thresholds in
 * `options` apply (pass permissive ones for the unfiltered single-pair semantics of methods 1 and 3; Align4 applies the same
 * thresholds internally, src/Align4.cpp:944-985) and suppressContainments should be 0.
 *   ordinals      : receives uint32[2*markerCount] (ordinal0, ordinal1) pairs of the alignment, or NULL when no alignment
 *                   passes; free with shb_free.
 *   alignmentInfo : optional, 13 words = words 3..15 of the AlignmentData record (AlignmentInfo, src/Alignment.hpp:86-200).
 */
shb_status shb_align_oriented_reads(shb_context* ctx, uint32_t orientedReadId0, uint32_t orientedReadId1,
                                    const shb_align_options* options, uint32_t** ordinals, uint64_t* markerCount,
                                    uint32_t* alignmentInfo13);

/* Replaces Assembler::computeAlignmentTable (src/AssemblerAlign.cpp:509-571): for every oriented read the
 * indices of the alignments it is involved in (4 entries per alignment: both reads x both strands), each row
 * sorted by the other OrientedReadId (OrientedReadPair::getOther, src/OrientedReadPair.hpp:63-85).
 *   alignmentData : n 64-byte AlignmentData records (host); only readIds/isSameStrand are read.
 *   tableToc      : receives uint32[2*readCount+1]; tableData: uint32[4n]  (= Data/AlignmentTable.toc/.data
 *                   payload, VectorOfVectors<uint32_t,uint32_t>). Free both with shb_free.
 */
shb_status shb_compute_alignment_table(shb_context* ctx, const void* alignmentData, uint64_t alignmentCount,
                                       uint64_t readCount, uint32_t** tableToc, uint32_t** tableData);

/* Replaces AlignmentCandidates::computeCandidateTable (src/AssemblerAlignmentCandidates.cpp:379-448): for every
 * oriented read the indices of the candidates it is involved in (4 entries per candidate: both reads x both
 * strands), each row sorted by (other OrientedReadId, candidate index).
 *   candidates : n 12-byte OrientedReadPair records (host).
 *   tableToc   : receives uint64[2*readCount+1]; tableData: uint64[4n]  (= Data/CandidateTable.toc/.data payload,
 *                VectorOfVectors<uint64_t,uint64_t>, src/AlignmentCandidates.hpp:38). Free both with shb_free.
 */
shb_status shb_compute_candidate_table(shb_context* ctx, const void* candidates, uint64_t candidateCount,
                                       uint64_t readCount, uint64_t** tableToc, uint64_t** tableData);

// ---- flagPalindromicReads (src/AssemblerAlign.cpp:652-770) ----------------------------------------------------------
// The arguments of Assembler::flagPalindromicReads. threadCount is accepted and ignored.
typedef struct {
    uint32_t maxSkip, maxDrift, maxMarkerFrequency, deltaThreshold;
    double alignedFractionThreshold, nearDiagonalFractionThreshold;
    uint64_t threadCount;
} shb_palindromic_params;
typedef struct {
    uint64_t readCount, palindromicReadCount;
    uint64_t exactReadCount;        // reads the prefilter could not decide: they got the alignment graph and its path
    uint64_t vertexCount, edgeCount, heapPushCount, heapsortFallbackCount;     // over those reads
    double totalMs, exactMs;        // wall time of the call and of its exact phase
    uint64_t kernelLaunches;
} shb_palindromic_result;
// Flags the palindromic reads of the markers held by ctx (set by shb_set_markers* or shb_find_markers): bit 0 of every
// read's flags is reset, then set where the alignment of the read against its reverse complement (alignment method 0)
// passes both thresholds, exactly as the reference decides it. Bits 1-7 are kept. The context's flags are updated in
// place, so a following shb_lowhash0 / shb_compute_alignments sees them. readFlags (in/out, R bytes), alignedMarkerCount
// and nearDiagonalMarkerCount (R entries each) are optional. The counts are the reference's for the reads that got the
// alignment (exactReadCount of them, every read the reference flags among them); for every other read they are the
// bounds that decided it without an alignment: the number of alignment-graph vertices and of those within
// deltaThreshold of the diagonal, saturated to 32 bits. A context that holds only a read range returns SHB_ERR_STATE.
shb_status shb_flag_palindromic_reads(shb_context* ctx, const shb_palindromic_params* params, uint8_t* readFlags,
                                      uint32_t* alignedMarkerCount, uint32_t* nearDiagonalMarkerCount,
                                      shb_palindromic_result* result);
// The alignment of one read against its reverse complement that flagPalindromicReads uses (alignOrientedReads(readId, 0,
// readId, 1) with method 0): *ordinals = count (ordinal0, ordinal1) pairs, release with shb_free.
shb_status shb_palindromic_read_alignment(shb_context* ctx, uint64_t readId, const shb_palindromic_params* params,
                                          uint32_t** ordinals, uint64_t* count);

/* Replaces Assembler::createReadGraph, ReadGraph.creationMethod 0 (src/AssemblerReadGraph.cpp:35-175): for each read the
 * best maxAlignmentCount alignments by (markerCount, alignmentId), both descending, are kept; an alignment kept by either
 * of its reads becomes two read graph edges (the edge and its reverse complement), in alignmentId order.
 *   alignmentData    : n 64-byte AlignmentData records (host), IN/OUT: AlignmentInfo::isInReadGraph is set / cleared.
 *   keep             : receives uint8[n] (1 = used in the read graph).
 *   edges            : receives edgeCount 16-byte ReadGraphEdge records (src/ReadGraph.hpp:37-57) = Data/ReadGraphEdges payload.
 *   connectivityToc  : receives uint32[2*readCount+1]; connectivityData: uint32[2*edgeCount] = Data/ReadGraphConnectivity
 *                      (.toc/.data payload, VectorOfVectors<uint32_t,uint32_t>): per oriented read its edge indices, DECREASING
 *                      (the reference's VectorOfVectors::store fills each row from its end).
 * A kept alignment whose edge or reverse-complement edge is not ordered (readIds[0] > readIds[1], or a read aligned to
 * itself: the reference's SHASTA_ASSERT) returns SHB_ERR_INVALID naming the alignment; alignmentData is then left unchanged.
 * Free the four arrays with shb_free. (creationMethod 2: shb_create_read_graph2 below.)
 */
shb_status shb_create_read_graph(shb_context* ctx, void* alignmentData, uint64_t alignmentCount, uint64_t readCount,
                                 uint32_t maxAlignmentCount, uint8_t** keep, void** edges, uint64_t* edgeCount,
                                 uint32_t** connectivityToc, uint32_t** connectivityData);

/* Replaces Assembler::createReadGraph2, ReadGraph.creationMethod 2 (src/AssemblerReadGraph2.cpp:69-248): the selection of
 * shb_create_read_graph over the alignments that pass five thresholds read off histograms of the alignments' quality
 * indicators (setReadGraph2Criteria); `criteria` receives the thresholds (Assembler::actualMinAlignedFraction ...,
 * src/Assembler.hpp:154-158). Percentile arguments in the member's order; the other arguments as in shb_create_read_graph.
 */
typedef struct shb_read_graph2_criteria {
    double minAlignedFraction;
    uint64_t minAlignedMarkerCount, maxDrift, maxSkip, maxTrim;
} shb_read_graph2_criteria;
shb_status shb_create_read_graph2(shb_context* ctx, void* alignmentData, uint64_t alignmentCount, uint64_t readCount,
                                  uint32_t maxAlignmentCount, double markerCountPercentile, double alignedFractionPercentile,
                                  double maxSkipPercentile, double maxDriftPercentile, double maxTrimPercentile,
                                  shb_read_graph2_criteria* criteria, uint8_t** keep, void** edges, uint64_t* edgeCount,
                                  uint32_t** connectivityToc, uint32_t** connectivityData);

// ---- createMarkerGraphVertices (src/AssemblerMarkerGraph.cpp:38-770) ------------------------------------------------
// The arguments of Assembler::createMarkerGraphVertices (defaults src/AssemblerOptions.cpp:577-685: 10, 100, 0, 0, 0.08,
// 2). minCoverage 0 selects it from the disjoint-set size histogram with the reference's PeakFinder. threadCount is
// accepted and ignored.
typedef struct {
    uint64_t minCoverage, maxCoverage, minCoveragePerStrand;
    uint64_t allowDuplicateMarkers;         // 0 / 1
    double peakFinderMinAreaFraction;
    uint64_t peakFinderAreaStartIndex;
    uint64_t threadCount;
} shb_marker_graph_params;
typedef struct {
    uint64_t markerCount;
    uint64_t minCoverageUsed;               // Assembler::markerGraphMinCoverageUsed
    uint64_t peakFinderFailed;              // 1: the reference's PeakFinder throws here, minCoverage 5 was used
    double peakFinderObservedAreaFraction;  // PeakFinderException::observedPercentArea when it does
    uint64_t edgePairsUsed, edgePairsSkipped;   // skipped: crossesStrands, hasInconsistentAlignment or a chimeric read
    uint64_t alignedMarkerPairs;            // ordinal pairs decoded from the used alignments (two unions each)
    uint64_t disjointSetCount, keptDisjointSetCount, badDisjointSetCount, vertexCount;
    uint64_t histogramSize;                 // entries of *histogram: largest set size + 1 (0 without markers)
    uint64_t peakDeviceBytes;               // high-water mark of the device memory this call allocated (its own buffers and
                                            // the growth of the context's radix-sort workspace)
    double deviceMs, totalMs;               // device time line from the first to the last kernel; wall time of the call
    uint64_t kernelLaunches;
} shb_marker_graph_result;
/* Replaces Assembler::createMarkerGraphVertices on the markers held by ctx (every read: a context that holds a read range
 * returns SHB_ERR_STATE). Vertices are numbered in increasing order of their smallest marker id (the reference's order
 * depends on thread scheduling); the partition, each vertex's markers, the histogram and the counts are the reference's.
 *   readGraphEdges  : edgeCount 16-byte ReadGraphEdge records (Data/ReadGraphEdges payload), pairs (i, i+1), i even.
 *   compressedToc   : uint64[alignmentCount+1], compressedData: Data/CompressedAlignments payload.
 *   readFlags       : uint8[R] as in Data/ReadFlags (bit 1 = isChimeric) at call time.
 *   vertexTable     : receives Uint40[M] (5 bytes each, 2^40-1 = no vertex) = Data/MarkerGraphVertexTable payload.
 *   verticesToc     : receives Uint40[V+1]; verticesData: uint64[toc[V]] (= Data/MarkerGraphVertices.{toc,data}).
 *   histogram       : receives uint64[result->histogramSize]: the number of disjoint sets of each size.
 * Free the four arrays with shb_free. Inputs that trip one of the reference's assertions return SHB_ERR_INVALID (odd edge
 * count, a pair that is not an edge and its reverse complement, unordered oriented read ids, an alignmentId out of range,
 * aligned markers with different k-mer ids, and, beyond the reference's checks, a malformed compressed alignment). */
shb_status shb_create_marker_graph_vertices(shb_context* ctx, const shb_marker_graph_params* params, const void* readGraphEdges,
                                            uint64_t edgeCount, const uint64_t* compressedToc, const uint8_t* compressedData,
                                            uint64_t alignmentCount, const uint8_t* readFlags, uint8_t** vertexTable,
                                            uint8_t** verticesToc, uint64_t** verticesData, uint64_t** histogram,
                                            shb_marker_graph_result* result);
/* Replaces Assembler::findMarkerGraphReverseComplementVertices (:1134-1230) for vertices in any numbering (the reference's
 * own files included): rcVertex receives uint64[vertexCount], free with shb_free. A vertex whose reverse complemented
 * markers are not all on one vertex, or whose reverse complement's reverse complement is not itself, returns
 * SHB_ERR_INVALID. */
shb_status shb_find_marker_graph_reverse_complement_vertices(shb_context* ctx, const uint8_t* vertexTable, const uint8_t* verticesToc,
                                                             const uint64_t* verticesData, uint64_t vertexCount, uint64_t** rcVertex);
/* PeakFinder::findPeaks + findXCutoff (src/PeakFinder.cpp:23-198) on a histogram of n entries, host only. Returns 1 where
 * the reference throws PeakFinderException (*observedAreaFraction = its observedPercentArea), else 0 with *cutoff. n = 0,
 * undefined in the reference, returns 1 with observed area 0. */
int shb_peak_finder_cutoff(const uint64_t* histogram, uint64_t n, double minAreaFraction, uint64_t startIndex, uint64_t* cutoff,
                           double* observedAreaFraction);

/* ------------------------------------------------------------------------------------------
 * Read-sharded multi-GPU runs (SURVEY.md section 8e; BASELINE.json configs[2..4]): one process (and one context) per GPU,
 * NCCL over NVLink / NVSwitch for the two exchanges LowHash0 needs (bucket entries per iteration, pair counts once) and
 * for replicating the k-mer ids before the alignment step. NCCL is loaded at run time (libnccl.so.2); a host that
 * already has a communicator for these GPUs passes it with shb_dist_attach, otherwise rank 0 calls shb_dist_unique_id,
 * ships the 128 bytes to the other ranks by any means (MPI, a file, torch.distributed ...) and every rank calls
 * shb_dist_init (collective). The number of ranks must be a power of two. All shb_*_sharded calls are collective: every
 * rank makes the same calls in the same order.
 *   markers: each rank uploads the rows of its read range with shb_set_markers(readBegin, readEnd); the ranges must be
 *            contiguous in rank order and cover all reads.
 */
#define SHB_DIST_UNIQUE_ID_BYTES 128
shb_status shb_dist_unique_id(void* id128);
shb_status shb_dist_init(shb_context* ctx, int worldSize, int rank, const void* id128);
shb_status shb_dist_attach(shb_context* ctx, void* ncclComm /* ncclComm_t */, int worldSize, int rank);
void shb_dist_finalize(shb_context* ctx);

/* Assembler::findAlignmentCandidatesLowHash0 over the read shards (fixed minHashIterationCount). Rank g receives the g-th
 * contiguous block of the candidate list in the reference's order (the blocks are evened out on the device), free with
 * shb_free; stats (optional, uint64[readCountTotal*3]) receives the complete ReadLowHashStatistics on every rank;
 * result->candidateDigest is the digest of the slice this rank emitted: the ranks' digests sum (mod 2^64) to the digest of
 * the single-GPU run. */
shb_status shb_lowhash0_sharded(shb_context* ctx, const shb_lowhash_params* params, void** candidates, uint64_t* candidateCount,
                                uint64_t* stats, shb_lowhash_result* result);

/* Assembler::computeAlignments on this rank's block of candidates: the k-mer id shards of all ranks are gathered into this
 * GPU once per marker set (cached until shb_set_markers* is called again; collective only then), after which the call
 * is local. Same outputs as shb_compute_alignments. */
shb_status shb_compute_alignments_sharded(shb_context* ctx, const void* candidates, uint64_t candidateCount,
                                          const shb_align_options* options, void** alignmentData, uint64_t* alignmentCount,
                                          uint64_t** compressedToc, uint8_t** compressedData, shb_align_result* result);

typedef struct {
    double sweepSeconds, partitionSeconds, exchangeSeconds, processSeconds, finalSeconds, gatherSeconds, totalSeconds;
    uint64_t entriesReceived, pairsReceived;
} shb_dist_timing;
/* Host wall-clock breakdown of the last shb_lowhash0_sharded / marker gather on this rank (diagnostics). */
shb_status shb_dist_timing_get(shb_context* ctx, shb_dist_timing* timing);

/* ------------------------------------------------------------------------------------------
 * Bench / test utilities (not part of the reference's interface): the marker-space synthetic read
 * generator of shasta_b200/synth.py on the device, and helpers for the device buffers it returns.
 */
shb_status shb_synth_generate(shb_context* ctx, uint64_t seed, uint32_t k, double drop, double ins,
                              uint64_t genomeMarkers, const uint32_t* genomeKmerHost, const uint64_t* genomePosHost,
                              uint64_t readOffset /* global id of the first read generated here */, uint64_t readCount,
                              const int64_t* startHost, const int64_t* spanHost,
                              const uint8_t* revHost, uint64_t* tocOut /* 2*readCount+1, relative */,
                              uint32_t** kmerIdsDevice, uint8_t** data7Device /* may be NULL */);
shb_status shb_device_free(void* devicePtr);
/* Test hook for the library's radix sort (csrc/radix_sort.cuh): sorts n host (key, value) items in place, stably, on the
 * key bits [lowBegin, lowEnd) and then [highBegin, highEnd) (pass highEnd <= highBegin for a single range); values may be
 * NULL. */
shb_status shb_test_radix_sort(shb_context* ctx, uint64_t* keys, uint32_t* values, uint64_t n,
                               int lowBegin, int lowEnd, int highBegin, int highEnd);
/* Device pointer and length of the uint32 k-mer id SoA held by ctx (for the all-gather that replicates the
 * markers on every GPU before the alignment step). */
shb_status shb_markers_device(shb_context* ctx, void** kmerIdsDevice, uint64_t* localMarkerCount);
shb_status shb_copy_device_to_host(void* dstHost, const void* srcDevice, uint64_t bytes);

#ifdef __cplusplus
}
#endif
#endif
