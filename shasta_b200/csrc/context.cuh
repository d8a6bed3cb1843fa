// The per-GPU context behind the C ABI: device-resident markers and reusable workspaces.
#pragma once

#include "common.cuh"
#include "primitives.cuh"

#include <cstdlib>
#include <vector>

namespace shb {
// A positive count from the environment (the SHB_* test hooks that shrink batch and chunk sizes), else dflt.
inline uint32_t envCount(const char* name, uint32_t dflt)
{
    const char* v = std::getenv(name);
    if(!v) return dflt;
    const long x = std::strtol(v, nullptr, 10);
    return x > 0 ? uint32_t(x) : dflt;
}

constexpr int kMaxFusedIterations = 16;         // LowHash iterations hashed per pass over the k-mer ids (one slab each)
constexpr int kStageSlots = 8;                  // pinned staging chunks of the device -> host result copies (hostcopy.cuh)
constexpr uint64_t kStageBytes = 8ull << 20;

// The words of shb_context::scalars, the context's small device scratch for totals and counters. Every stage has slots of
// its own, so no two stages share a word whatever the order of the calls. The uint32 totals use the low half of their word.
enum ScalarSlot : uint32_t {
    kSlotSweepCounts = 0,                                       // lowhash: low hashes per fused iteration
    kSlotSegmentTotal = kSlotSweepCounts + kMaxFusedIterations, // lowhash: segments, high-frequency pairs (uint32)
    kSlotPairCursor,                                            // lowhash: pairs written
    kSlotPairHits,                                              // lowhash: pair hits (read with kSlotPairCursor in one copy)
    kSlotCandidateDigest,                                       // lowhash: digest of the emitted candidates (also read by dist.cu)
    kSlotPartitionCounts,                                       // devicePartition: one count per digit, 256 digits
    kSlotDownsampleTotal = kSlotPartitionCounts + 256,          // align: downsampled markers of a chunk (uint32)
    kSlotAlignmentDigests,                                      // align: AlignmentData digest, compressed alignment digest
    kSlotMarkerTotal = kSlotAlignmentDigests + 2,               // markers: markers of strand 0
    kSlotKeptAlignments,                                        // readgraph: alignments kept (uint32)
    kSlotBadConnectivity,                                       // readgraph_flags: bad ReadGraphConnectivity entries (uint32)
    kSlotMarkerGraphVertices,                                   // markergraph: errKmer, errFormat, alignedCount, maxSize, scan total, bigCount
    kSlotMarkerGraphRcErrors = kSlotMarkerGraphVertices + 6,    // markergraph: errMarker, errVertex
    kSlotMarkerGraphEdges = kSlotMarkerGraphRcErrors + 2,      // markergraph_edges: errMarker, errOrder, errVertex, longCount,
                                                                //   bigCount, saturated, edge total, interval total
    kSlotMarkerGraphRcEdges = kSlotMarkerGraphEdges + 8,        // markergraph_edges: errInput, errAssert, errNotFound, errRcRc
    kScalarSlotEnd = kSlotMarkerGraphRcEdges + 4
};
constexpr uint32_t kScalarWords = 512;                          // reserved once at context creation, never reallocated
static_assert(kScalarSlotEnd <= kScalarWords, "the scalar slots do not fit the reserved words");

// Device bytes a call holds, and their high-water mark.
struct Footprint {
    uint64_t live = 0, peak = 0;
    template<class T> void add(DeviceBuffer<T>& b, uint64_t n)
    {
        const uint64_t before = b.capacity();
        b.reserve(n);
        live += (b.capacity() - before) * sizeof(T);
        peak = std::max(peak, live);
    }
    template<class T> void drop(DeviceBuffer<T>& b) { live -= b.capacity() * sizeof(T); b.release(); }
};

struct LowHashAccumulator {
    uint64_t count = 0;     // reduced (pairKey, count) items in the acc ping-pong buffers
    bool inB = false;       // which of the acc ping-pong buffers holds the data
    bool sorted = false;    // the reduced items are one sorted run with unique keys (nothing left to merge)
    uint64_t rawCount = 0;  // raw pair hits (one key per hit, any order) of the iterations since the last reduction, in pairsA
    uint64_t rawLimit = 1ull << 31;     // reduce the raw hits when one more iteration would exceed this many (SHB_LOWHASH_RAW_LIMIT)
};
// State of one LowHash0 run (lowhashBegin ... lowhashEmitDevice in lowhash.cu), on one GPU (lowhash0) or on one rank of a
// read-sharded run (dist.cu).
struct LowHashState {
    shb_lowhash_params p{};
    uint64_t log2BucketCount = 0, bucketMask = 0, hashThreshold = 0, capacity = 0;
    uint32_t readBits = 1;
    uint32_t queueCapacityOverride = 0; // SHB_LOWHASH_QUEUE_CAPACITY (test hook), 0 = derived from hashFraction
    bool aggregateByRead = false;       // pair hits are counted per read in shared memory before they reach the accumulator
    LowHashAccumulator acc;
    uint64_t lowHashCount = 0, pairCount = 0, sweepLaunches = 0;
    uint64_t emittedCount = 0, candidateDigest = 0;     // of the last lowhashEmitDevice
    double sweepMs = 0.;
};
}

struct shb_context {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t copyStream[2] = {nullptr, nullptr};

    // ---- markers (a1, a4) -------------------------------------------------------------------
    bool haveMarkers = false;
    uint64_t markerGeneration = 0;      // bumped by every shb_set_markers*: invalidates derived caches
    uint64_t readCountTotal = 0;        // R of the whole assembly
    uint64_t readBegin = 0, readEnd = 0; // reads whose rows live on this GPU
    uint64_t totalMarkerCount = 0;      // over all reads (bucket-count rule)
    uint64_t localMarkerCount = 0;
    shb::DeviceBuffer<uint32_t> kmerIdsOwned;
    const uint32_t* kmerIds = nullptr;  // device, localMarkerCount entries (+ padding when owned)
    shb::DeviceBuffer<uint64_t> toc;    // device, relative, 2*(readEnd-readBegin)+1 entries
    shb::DeviceBuffer<uint8_t> readFlags; // device, readCountTotal entries
    std::vector<uint64_t> tocHost;      // host copy of the relative toc
    std::vector<uint8_t> readFlagsHost;

    // ---- shared workspaces --------------------------------------------------------------------
    shb::SortWorkspace sortWs;
    shb::DeviceBuffer<uint32_t> scanWs;
    shb::DeviceBuffer<unsigned long long> scalars;   // small device scratch for totals/counters: shb::ScalarSlot
    unsigned long long* scalar(shb::ScalarSlot slot) const { return scalars.get() + slot; }

    // ---- LowHash buffers (see lowhash.cu) -----------------------------------------------------
    shb::DeviceBuffer<uint64_t> sweepKeys;  shb::DeviceBuffer<uint32_t> sweepVals;
    shb::DeviceBuffer<uint32_t> sweepTileFirstRead;     // per sweep tile: the oriented read that holds its first position
    uint64_t sweepTileGeneration = ~0ull;               // markerGeneration the table was built for
    shb::DeviceBuffer<uint64_t> entryKeysTmp; shb::DeviceBuffer<uint32_t> entryValsTmp;
    shb::DeviceBuffer<uint32_t> flagsBuf, indexBuf, segStartBuf, countsBuf;
    shb::DeviceBuffer<uint64_t> pairsA, pairsB;
    shb::DeviceBuffer<uint64_t> accKeysA, accKeysB;
    shb::DeviceBuffer<uint32_t> accValsA, accValsB;
    shb::DeviceBuffer<unsigned long long> stats;
    shb::DeviceBuffer<uint32_t> candidatesDev;

    shb::DeviceBuffer<uint64_t> partKeys; shb::DeviceBuffer<uint32_t> partVals;
    void* lowhashState = nullptr;
    void* pinnedStage[shb::kStageSlots] = {};       // pinned staging ring of the device -> host result copies (hostcopy.cuh)
    cudaEvent_t stageEvent[shb::kStageSlots] = {};

    // ---- alignment cache (downsampled markers; see align.cu) ------------------------------------
    void* alignCache = nullptr;
    // ---- multi-GPU state (NCCL communicator, exchange buffers, gathered markers; see dist.cu) --------
    void* dist = nullptr;
};

namespace shb {
// The stages after the alignments work on the markers of every read.
inline void requireWholeAssembly(shb_context* c, const char* what)
{
    SHB_REQUIRE(c->haveMarkers, SHB_ERR_STATE, "No markers: call shb_set_markers* or shb_find_markers first.");
    SHB_REQUIRE(c->readBegin == 0 && c->readEnd == c->readCountTotal, SHB_ERR_STATE,
                std::string(what) + " needs the markers of every read on one context.");
}
}
