// LowHash0 on the GPU: host orchestration of the kernels in lowhash_kernels.cuh.
// Mirrors LowHash0::LowHash0 (src/LowHash0.cpp:23-257 of chanzuckerberg/shasta) step by step;
// see DESIGN.md for the data layout and the per-kernel roofline.
#include "context.cuh"
#include "lowhash_kernels.cuh"
#include "hostcopy.cuh"
#include "digest.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>

namespace shb {

thread_local uint64_t g_launchCount = 0;

namespace {

// Sizes of the fused-iteration groups the default feature length (m = 4, every shipped configuration) has a fully
// unrolled kernel for; the iteration loop of lowhash0 cuts the iterations into groups of these sizes.
const uint32_t kUnrolledGroups[] = {16, 10, 8, 4, 2, 1};

// Largest supported group that fits the remaining iterations and keeps the group's slabs (12 bytes per entry) within a
// fixed memory budget (HiFi at 2 M reads: 277 M entries per slab).
uint32_t nextSweepGroupImpl(uint64_t remaining, uint64_t slabCapacity)
{
    constexpr uint64_t kSlabBudgetBytes = 16ull << 30;
    const uint64_t fit = std::max<uint64_t>(1, kSlabBudgetBytes / (12ull * std::max<uint64_t>(slabCapacity, 1)));
    for(uint32_t g : kUnrolledGroups) if(g <= remaining && g <= fit) return g;
    return 1;
}

template<int MM, int KK> void launchSweepKernel(const SweepArgs& a, uint32_t blocks, cudaStream_t stream)
{
    const size_t dynamicBytes = size_t(a.queueCapacity) * 16;
    static size_t allowed = 0;          // per instantiation; the static part (tile + counters) is ~8.5 KB
    if(dynamicBytes > allowed) {
        SHB_CUDA(cudaFuncSetAttribute(lowhashSweepKernel<MM, KK>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(dynamicBytes)));
        allowed = dynamicBytes;
    }
    SHB_LAUNCH((lowhashSweepKernel<MM, KK>), blocks, kSweepThreads, dynamicBytes, stream, a);
}

void launchSweep(const SweepArgs& a, uint32_t blocks, cudaStream_t stream)
{
    if(a.m == 4) {
        switch(a.iterationCount) {
        case 16: launchSweepKernel<4, 16>(a, blocks, stream); return;
        case 10: launchSweepKernel<4, 10>(a, blocks, stream); return;
        case 8: launchSweepKernel<4, 8>(a, blocks, stream); return;
        case 4: launchSweepKernel<4, 4>(a, blocks, stream); return;
        case 2: launchSweepKernel<4, 2>(a, blocks, stream); return;
        case 1: launchSweepKernel<4, 1>(a, blocks, stream); return;
        default: break;
        }
    }
    switch(a.m) {
    case 1: launchSweepKernel<1, 0>(a, blocks, stream); break;
    case 2: launchSweepKernel<2, 0>(a, blocks, stream); break;
    case 3: launchSweepKernel<3, 0>(a, blocks, stream); break;
    case 4: launchSweepKernel<4, 0>(a, blocks, stream); break;
    case 5: launchSweepKernel<5, 0>(a, blocks, stream); break;
    case 6: launchSweepKernel<6, 0>(a, blocks, stream); break;
    case 7: launchSweepKernel<7, 0>(a, blocks, stream); break;
    case 8: launchSweepKernel<8, 0>(a, blocks, stream); break;
    default: launchSweepKernel<0, 0>(a, blocks, stream); break;
    }
}

// Sorted-by-key (keys[,vals]) -> head flags, exclusive segment index, segment starts.
// Returns the number of segments (one host sync) unless wantCount is false (then 0, no sync).
uint32_t buildSegments(shb_context* c, const uint64_t* sortedKeys, uint32_t n, int shift, bool wantCount = true)
{
    cudaStream_t st = c->stream;
    c->flagsBuf.reserve(n);
    c->indexBuf.reserve(n);
    c->segStartBuf.reserve(uint64_t(n) + 1);
    c->scanWs.reserve(scanWorkspaceElements(n));
    SHB_LAUNCH(headFlagsKernel, ceilDiv(n, 256), 256, 0, st, sortedKeys, n, shift, c->flagsBuf.get());
    uint32_t* total = reinterpret_cast<uint32_t*>(c->scalar(kSlotSegmentTotal));
    exclusiveScan<uint32_t>(c->flagsBuf.get(), c->indexBuf.get(), n, total, c->scanWs.get(), st);
    SHB_LAUNCH(segmentStartsKernel, ceilDiv(n, 256), 256, 0, st,
               (const uint32_t*)c->flagsBuf.get(), (const uint32_t*)c->indexBuf.get(), n, c->segStartBuf.get());
    return wantCount ? readBack(total, st) : 0u;
}

using Accumulator = LowHashAccumulator;

uint64_t* accKeys(shb_context* c, const Accumulator& a) { return a.inB ? c->accKeysB.get() : c->accKeysA.get(); }
uint32_t* accVals(shb_context* c, const Accumulator& a) { return a.inB ? c->accValsB.get() : c->accValsA.get(); }

void accReserve(shb_context* c, Accumulator& a, uint64_t n)
{
    // Keep both ping-pong buffers the same size; only the live one is preserved.
    if(a.inB) { c->accKeysB.reserve(n, true, c->stream); c->accValsB.reserve(n, true, c->stream); }
    else      { c->accKeysA.reserve(n, true, c->stream); c->accValsA.reserve(n, true, c->stream); }
}

// Sort the accumulated (pairKey,count) items by key and sum the counts of equal keys
// (the order-independent equivalent of LowHash0::merge, src/LowHash0.cpp:493-562; the uint16
// wrap-around is applied when the frequency is read, frequencyFlagsKernel).
void mergeAccumulator(shb_context* c, Accumulator& acc, uint32_t readBits)
{
    if(acc.count == 0 || acc.sorted) return;
    SHB_REQUIRE(acc.count < (1ull << 32), SHB_ERR_INVALID, "LowHash0: candidate accumulator exceeds 2^32-1 items.");
    const uint32_t n = uint32_t(acc.count);
    cudaStream_t st = c->stream;
    // The sort ping-pongs between A and B.
    uint64_t* kA = acc.inB ? c->accKeysB.get() : c->accKeysA.get();
    uint32_t* vA = acc.inB ? c->accValsB.get() : c->accValsA.get();
    DeviceBuffer<uint64_t>& otherK = acc.inB ? c->accKeysA : c->accKeysB;
    DeviceBuffer<uint32_t>& otherV = acc.inB ? c->accValsA : c->accValsB;
    otherK.reserve(n);
    otherV.reserve(n);
    const int ranges[2][2] = {{0, int(readBits) + 1}, {32, 32 + int(readBits)}};
    const bool flipped = radixSort<true>(kA, otherK.get(), vA, otherV.get(), n, ranges, 2, c->sortWs, st);
    if(flipped) acc.inB = !acc.inB;
    const uint64_t* sortedK = accKeys(c, acc);
    const uint32_t* sortedV = accVals(c, acc);
    const uint32_t numSeg = buildSegments(c, sortedK, n, 0);
    // Reduce into the other buffer pair.
    DeviceBuffer<uint64_t>& outK = acc.inB ? c->accKeysA : c->accKeysB;
    DeviceBuffer<uint32_t>& outV = acc.inB ? c->accValsA : c->accValsB;
    outK.reserve(numSeg);
    outV.reserve(numSeg);
    SHB_LAUNCH(segmentSumKernel, ceilDiv(numSeg, 256), 256, 0, st, sortedK, sortedV,
               (const uint32_t*)c->segStartBuf.get(), numSeg, outK.get(), outV.get());
    acc.inB = !acc.inB;
    acc.count = numSeg;
    acc.sorted = true;
}

// Raw pair hits are kept unsorted across iterations (one 8-byte key per hit) and reduced in one go: sort, run lengths,
// (pairKey, count) appended to the accumulator. When the accumulator was empty the result already is the merged table.
void reduceRawPairs(shb_context* c, Accumulator& acc, uint32_t readBits)
{
    if(acc.rawCount == 0) return;
    SHB_REQUIRE(acc.rawCount < (1ull << 32), SHB_ERR_INVALID, "LowHash0: more than 2^32-1 buffered candidate pair hits.");
    const uint32_t np = uint32_t(acc.rawCount);
    cudaStream_t st = c->stream;
    c->pairsB.reserve(np);
    const int pairRanges[2][2] = {{0, int(readBits) + 1}, {32, 32 + int(readBits)}};
    const bool inB = radixSort<false>(c->pairsA.get(), c->pairsB.get(), nullptr, nullptr, np, pairRanges, 2, c->sortWs, st);
    const uint64_t* sortedPairs = inB ? c->pairsB.get() : c->pairsA.get();
    const uint32_t numUnique = buildSegments(c, sortedPairs, np, 0);
    const bool first = (acc.count == 0);
    accReserve(c, acc, acc.count + numUnique);
    SHB_LAUNCH(uniqueCountsKernel, ceilDiv(numUnique, 256), 256, 0, st, sortedPairs,
               (const uint32_t*)c->segStartBuf.get(), numUnique,
               accKeys(c, acc) + acc.count, accVals(c, acc) + acc.count);
    if(std::getenv("SHB_LOWHASH_VERBOSE")) fprintf(stderr, "[shasta_b200] raw pair hits %u -> %u distinct pairs\n", np, numUnique);
    acc.count += numUnique;
    acc.sorted = first;
    acc.rawCount = 0;
    if(acc.count > (1ull << 30)) mergeAccumulator(c, acc, readBits);     // keep the accumulator below 2^32 items
}

uint64_t countHighFrequency(shb_context* c, const Accumulator& acc, uint64_t minFrequency, bool keepOffsets)
{
    if(acc.count == 0) return 0;
    const uint32_t n = uint32_t(acc.count);
    cudaStream_t st = c->stream;
    c->flagsBuf.reserve(n);
    c->indexBuf.reserve(n);
    c->scanWs.reserve(scanWorkspaceElements(n));
    SHB_LAUNCH(frequencyFlagsKernel, ceilDiv(n, 256), 256, 0, st, (const uint32_t*)accVals(c, acc), n, minFrequency, c->flagsBuf.get());
    uint32_t* total = reinterpret_cast<uint32_t*>(c->scalar(kSlotSegmentTotal));
    exclusiveScan<uint32_t>(c->flagsBuf.get(), c->indexBuf.get(), n, total, c->scanWs.get(), st);
    (void)keepOffsets;
    return readBack(total, st);
}

} // namespace

uint32_t nextSweepGroup(uint64_t remaining, uint64_t slabCapacity) { return nextSweepGroupImpl(remaining, slabCapacity); }


// ---------------------------------------------------------------------------------------------
// LowHash0 in stages. The single-GPU call (lowhash0) is begin -> { sweep -> processEntries per slab } -> emit; the
// read-sharded run (dist.cu) inserts the bucket exchange between sweep and processEntries and the pair exchange
// (localPairs -> setPairs) before emit.
LowHashState& lowhashState(shb_context* c)
{
    if(!c->lowhashState) c->lowhashState = new LowHashState();
    return *static_cast<LowHashState*>(c->lowhashState);
}
void destroyLowhashState(shb_context* c)
{
    if(c->lowhashState) { delete static_cast<LowHashState*>(c->lowhashState); c->lowhashState = nullptr; }
}

void lowhashBegin(shb_context* c, const shb_lowhash_params& p)
{
    SHB_REQUIRE(c->haveMarkers, SHB_ERR_STATE, "Markers are not accessible.");
    SHB_REQUIRE(p.m >= 1 && p.m <= 32, SHB_ERR_INVALID, "MinHash.m must be between 1 and 32 in this implementation.");
    SHB_REQUIRE(c->readCountTotal < (1ull << 31), SHB_ERR_INVALID, "Too many reads.");
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    LowHashState& S = lowhashState(c);
    S = LowHashState();
    S.p = p;
    // Count the pair hits per read before they reach the accumulator when one read pair collides many times per iteration
    // (hashFraction x overlap length: HiFi 0.05 -> ~25 hits per pair and iteration; at Nanopore's 0.01 both organisations
    // cost the same and the raw buffer is kept).
    S.aggregateByRead = p.hashFraction >= 0.03;
    if(const char* e = std::getenv("SHB_LOWHASH_AGGREGATE")) S.aggregateByRead = std::atoi(e) != 0;
    if(const char* e = std::getenv("SHB_LOWHASH_RAW_LIMIT")) {          // test hook: force the intermediate reductions
        const long long v = std::atoll(e);
        if(v > 0) S.acc.rawLimit = uint64_t(v);
    }
    // Test hook: the sweep's shared-memory queue holds this many low hashes per tile instead of the number derived from
    // hashFraction (lowhashSweep), clamped to 1 ... kSweepQueueMax; the hits beyond it take the sweep's inline path.
    if(const char* e = std::getenv("SHB_LOWHASH_QUEUE_CAPACITY")) {
        const long long v = std::atoll(e);
        if(v > 0) S.queueCapacityOverride = uint32_t(std::min<long long>(v, kSweepQueueMax));
    }
    g_launchCount = 0;
    const uint64_t R = c->readCountTotal;

    // Bucket-count rule, src/LowHash0.cpp:69-98.
    const uint64_t totalLowHashCountEstimate = uint64_t(p.hashFraction * double(c->totalMarkerCount));
    const uint32_t log2Estimate = totalLowHashCountEstimate ? uint32_t(64 - __builtin_clzll(totalLowHashCountEstimate)) : 0;
    uint64_t log2BucketCount = p.log2MinHashBucketCount;
    if(log2BucketCount == 0) log2BucketCount = 5 + log2Estimate;
    else SHB_REQUIRE(log2BucketCount >= log2Estimate, SHB_ERR_INVALID, "log2MinHashBucketCount is unreasonably small.");
    if(log2BucketCount > 31) log2BucketCount = 31;
    S.log2BucketCount = log2BucketCount;
    S.bucketMask = (1ull << log2BucketCount) - 1ull;
    // src/LowHash0.cpp:109
    S.hashThreshold = uint64_t(double(p.hashFraction) * double(std::numeric_limits<uint64_t>::max()));
    S.readBits = bitsFor(R ? R - 1 : 0);
    // Capacity of one iteration's low-hash slab.
    const uint64_t M = c->localMarkerCount;
    S.capacity = uint64_t(1.25 * p.hashFraction * double(M)) + 65536;
    if(S.capacity > M + 1) S.capacity = M + 1;
    c->stats.reserve(3 * R + 1);
    SHB_CUDA(cudaMemsetAsync(c->stats.get(), 0, (3 * R + 1) * sizeof(unsigned long long), st));
}

// pass 1 for `group` consecutive iterations in one pass over the local k-mer ids. counts[s] = low hashes of
// iteration iterationBegin+s; slab s = (sweepKeys + s*capacity, sweepVals + s*capacity).
void lowhashSweep(shb_context* c, uint64_t iterationBegin, uint32_t group, unsigned long long* counts)
{
    LowHashState& S = lowhashState(c);
    SHB_REQUIRE(group >= 1 && group <= (uint32_t)kMaxFusedIterations, SHB_ERR_INVALID, "Invalid iteration group.");
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const uint64_t M = c->localMarkerCount;
    EventTimer sweepTimer;
    for(;;) {
        c->sweepKeys.reserve(S.capacity * group);
        c->sweepVals.reserve(S.capacity * group);
        SHB_CUDA(cudaMemsetAsync(c->scalar(kSlotSweepCounts), 0, kMaxFusedIterations * sizeof(unsigned long long), st));
        SweepArgs a;
        a.kmerIds = c->kmerIds;
        a.markerCount = M;
        a.toc = c->toc.get();
        a.orientedReadCount = uint32_t(2 * (c->readEnd - c->readBegin));
        a.orientedReadBase = uint32_t(2 * c->readBegin);
        a.readFlags = c->readFlags.get();
        a.m = uint32_t(S.p.m);
        a.hashThreshold = S.hashThreshold;
        a.bucketMask = S.bucketMask;
        a.iterationBegin = uint32_t(iterationBegin);
        a.iterationCount = group;
        for(uint32_t k = 0; k < uint32_t(kMaxFusedIterations); k++) a.seeds[k] = (uint32_t(iterationBegin) + k) * 37u;
        a.keys = c->sweepKeys.get();
        a.vals = c->sweepVals.get();
        a.capacity = S.capacity;
        a.counts = c->scalar(kSlotSweepCounts);
        {
            const double expected = double(kSweepTile) * double(group) * S.p.hashFraction;
            a.queueCapacity = uint32_t(std::min<double>(kSweepQueueMax, std::max<double>(kSweepQueueMin, 1.5 * expected + 64.)));
            if(S.queueCapacityOverride) a.queueCapacity = S.queueCapacityOverride;
        }
        const uint32_t tileCount = uint32_t(ceilDiv(M, kSweepTile));
        if(tileCount && (c->sweepTileGeneration != c->markerGeneration || c->sweepTileFirstRead.capacity() < tileCount)) {
            c->sweepTileFirstRead.reserve(tileCount);
            SHB_LAUNCH(sweepTileReadsKernel, ceilDiv(tileCount, 256), 256, 0, st, (const uint64_t*)c->toc.get(), a.orientedReadCount,
                       tileCount, c->sweepTileFirstRead.get());
            c->sweepTileGeneration = c->markerGeneration;
        }
        a.tileFirstRead = c->sweepTileFirstRead.get();
        const bool run = M >= S.p.m && M > 0;
        if(run) {
            sweepTimer.start(st);
            launchSweep(a, ceilDiv(ceilDiv(M, kSweepTile), uint64_t(kSweepTilesPerBlock)), st);
            sweepTimer.stop(st);
            S.sweepLaunches++;
        }
        SHB_CUDA(cudaMemcpyAsync(counts, c->scalar(kSlotSweepCounts), group * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        if(run) S.sweepMs += sweepTimer.elapsedMs();
        const unsigned long long worst = *std::max_element(counts, counts + group);
        if(worst <= S.capacity) break;
        S.capacity = worst + worst / 8 + 1024;        // slab overflow: grow and redo this group
    }
}

// passes 2 and 3 on one iteration's entries (keys = bucketId<<32 | hashHigh, vals = orientedReadId), which must all
// belong to buckets owned by this GPU: bucket sort, per-read statistics, and the pair hits — appended raw to the pair
// buffer (sorted and counted once for many iterations) or, for HiFi-like hash fractions, counted per read in shared memory
// and appended as (pair, count) to the local accumulator. keysA/valsA are clobbered.
void lowhashProcessEntries(shb_context* c, uint64_t* keysA, uint32_t* valsA, uint64_t n64)
{
    LowHashState& S = lowhashState(c);
    SHB_REQUIRE(n64 < (1ull << 32), SHB_ERR_INVALID, "LowHash0: more than 2^32-1 low hashes in one iteration.");
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const shb_lowhash_params& p = S.p;
    const uint32_t n = uint32_t(n64);
    S.lowHashCount += n;
    if(n == 0) return;
    c->entryKeysTmp.reserve(n);
    c->entryValsTmp.reserve(n);
    const int bucketRange[1][2] = {{32, 32 + int(S.log2BucketCount)}};
    const bool inTmp = radixSort<true>(keysA, c->entryKeysTmp.get(), valsA, c->entryValsTmp.get(), n, bucketRange, 1, c->sortWs, st);
    const uint64_t* keys = inTmp ? c->entryKeysTmp.get() : keysA;
    const uint32_t* vals = inTmp ? c->entryValsTmp.get() : valsA;

    if(S.aggregateByRead) {
        // Entries grouped by read (stable sort of (readId, entry index)), each read's partners counted in shared memory.
        uint64_t* otherKeys = inTmp ? keysA : c->entryKeysTmp.get();
        uint32_t* otherVals = inTmp ? valsA : c->entryValsTmp.get();
        c->pairsA.reserve(n);           // bucket spans (uint2 per entry)
        c->pairsB.reserve(n);           // sort ping-pong
        c->countsBuf.reserve(n);
        uint2* span = reinterpret_cast<uint2*>(c->pairsA.get());
        SHB_LAUNCH(bucketSpanKernel, ceilDiv(n, 256), 256, 0, st, keys, vals, n, p.minBucketSize, p.maxBucketSize, c->stats.get(), span);
        SHB_LAUNCH(readKeysKernel, ceilDiv(n, 256), 256, 0, st, vals, n, otherKeys, otherVals);
        const int readRange[1][2] = {{0, int(S.readBits)}};
        const bool flipped = radixSort<true>(otherKeys, c->pairsB.get(), otherVals, c->countsBuf.get(), n, readRange, 1, c->sortWs, st);
        const uint64_t* sortedReadKeys = flipped ? c->pairsB.get() : otherKeys;
        const uint32_t* order = flipped ? c->countsBuf.get() : otherVals;
        const uint32_t numReads = buildSegments(c, sortedReadKeys, n, 0);
        unsigned long long* cursor = c->scalar(kSlotPairCursor);
        unsigned long long* hits = c->scalar(kSlotPairHits);
        uint32_t maxProbes = kPairTableMaxProbes;
        if(const char* e = std::getenv("SHB_LOWHASH_TABLE_PROBES")) maxProbes = uint32_t(std::max(1, std::atoi(e)));     // test hook: force the overflow path
        for(;;) {
            if(accKeys(c, S.acc) == nullptr) accReserve(c, S.acc, std::max<uint64_t>(S.acc.count + n, 1ull << 20));
            const uint64_t liveCapacity = S.acc.inB ? c->accKeysB.capacity() : c->accKeysA.capacity();
            const uint64_t room = liveCapacity - S.acc.count;
            SHB_CUDA(cudaMemsetAsync(cursor, 0, sizeof(unsigned long long), st));
            SHB_CUDA(cudaMemsetAsync(hits, 0, sizeof(unsigned long long), st));
            SHB_LAUNCH(readPairsKernel, ceilDiv(numReads, kPairTableWarps), kPairTableWarps * 32, 0, st, keys, vals, (const uint2*)span,
                       sortedReadKeys, order, (const uint32_t*)c->segStartBuf.get(), numReads, cursor, hits,
                       accKeys(c, S.acc) + S.acc.count, accVals(c, S.acc) + S.acc.count, (unsigned long long)room, maxProbes);
            static_assert(kSlotPairHits == kSlotPairCursor + 1, "cursor and hits are read in one copy");
            unsigned long long totals[2];      // cursor, hits
            SHB_CUDA(cudaMemcpyAsync(totals, cursor, sizeof(totals), cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaStreamSynchronize(st));
            if(totals[0] <= room) {
                S.acc.count += totals[0];
                if(totals[0]) S.acc.sorted = false;
                S.pairCount += totals[1];
                break;
            }
            accReserve(c, S.acc, S.acc.count + totals[0] + totals[0] / 16);
        }
        if(S.acc.count > (1ull << 30)) mergeAccumulator(c, S.acc, S.readBits);
        return;
    }

    // One pass: per-read statistics and the pair hits, appended (in any order) to the raw pair buffer; sorting and counting
    // happen once for many iterations. The pass reports the exact number of hits; if they did not fit, the buffer grows
    // (after a reduction of what it holds, when that would exceed the limit) and the pass runs again without the statistics.
    unsigned long long* cursor = c->scalar(kSlotPairCursor);
    if(c->pairsA.capacity() == 0) c->pairsA.reserve(1ull << 20);
    bool withStats = true;
    for(;;) {
        const uint64_t room = c->pairsA.capacity() - S.acc.rawCount;
        SHB_CUDA(cudaMemsetAsync(cursor, 0, sizeof(unsigned long long), st));
        SHB_LAUNCH(bucketPairsKernel, ceilDiv(n, 256), 256, 0, st, keys, vals, n, p.minBucketSize, p.maxBucketSize,
                   withStats ? c->stats.get() : (unsigned long long*)nullptr, cursor, c->pairsA.get() + S.acc.rawCount,
                   (unsigned long long)room);
        const unsigned long long np64 = readBack(cursor, st);
        SHB_REQUIRE(np64 < (1ull << 32), SHB_ERR_INVALID,
                    "LowHash0: more than 2^32-1 candidate pair hits in one iteration (maxBucketSize too large).");
        if(np64 <= room) {
            S.pairCount += np64;
            S.acc.rawCount += np64;
            break;
        }
        withStats = false;
        if(S.acc.rawCount && S.acc.rawCount + np64 > S.acc.rawLimit) reduceRawPairs(c, S.acc, S.readBits);
        const uint64_t iterations = std::max<uint64_t>(1, p.minHashIterationCount);
        const uint64_t want = S.acc.rawCount + np64;
        c->pairsA.reserve(std::max<uint64_t>(want + want / 32, std::min<uint64_t>(S.acc.rawLimit, (np64 + np64 / 8) * iterations)),
                          S.acc.rawCount != 0, st);
    }
    if(S.acc.rawCount > S.acc.rawLimit) reduceRawPairs(c, S.acc, S.readBits);
}

// Merge the local accumulator; returns its device arrays (valid until the next LowHash call on this context).
void lowhashLocalPairs(shb_context* c, uint64_t** keys, uint32_t** counts, uint64_t* n)
{
    LowHashState& S = lowhashState(c);
    SHB_CUDA(cudaSetDevice(c->device));
    reduceRawPairs(c, S.acc, S.readBits);
    mergeAccumulator(c, S.acc, S.readBits);
    *keys = accKeys(c, S.acc); *counts = accVals(c, S.acc); *n = S.acc.count;
}

// Replace the accumulator by externally supplied (pairKey,count) items (multi-GPU: what the other ranks sent).
void lowhashSetPairs(shb_context* c, const uint64_t* keys, const uint32_t* counts, uint64_t n)
{
    LowHashState& S = lowhashState(c);
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const uint64_t rawLimit = S.acc.rawLimit;
    S.acc = Accumulator();
    S.acc.rawLimit = rawLimit;
    accReserve(c, S.acc, n);
    if(n) {
        SHB_CUDA(cudaMemcpyAsync(accKeys(c, S.acc), keys, 8 * n, cudaMemcpyDeviceToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(accVals(c, S.acc), counts, 4 * n, cudaMemcpyDeviceToDevice, st));
        SHB_CUDA(cudaStreamSynchronize(st));
    }
    S.acc.count = n;
}

// Final merge + emission, src/LowHash0.cpp:204-214, left on the device: c->candidatesDev holds nOut 12-byte records.
// The digest of the emitted records is computed asynchronously into S.candidateDigest's device slot (kSlotCandidateDigest).
uint64_t lowhashEmitDevice(shb_context* c)
{
    LowHashState& S = lowhashState(c);
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    reduceRawPairs(c, S.acc, S.readBits);
    mergeAccumulator(c, S.acc, S.readBits);
    const uint64_t nOut = countHighFrequency(c, S.acc, S.p.minFrequency, true);
    unsigned long long* digestDev = c->scalar(kSlotCandidateDigest);
    SHB_CUDA(cudaMemsetAsync(digestDev, 0, sizeof(unsigned long long), st));
    if(nOut) {
        c->candidatesDev.reserve(3 * nOut);
        SHB_LAUNCH(emitCandidatesKernel, ceilDiv(S.acc.count, 256), 256, 0, st, (const uint64_t*)accKeys(c, S.acc),
                   (const uint32_t*)c->flagsBuf.get(), (const uint32_t*)c->indexBuf.get(), uint32_t(S.acc.count),
                   c->candidatesDev.get());
        SHB_LAUNCH(digestRecordsKernel, ceilDiv(nOut, 256), 256, 0, st, (const uint32_t*)c->candidatesDev.get(), nOut, 3u, digestDev);
    }
    S.emittedCount = nOut;
    return nOut;
}

// The scratch of a LowHash0 run stays allocated for the next run unless it is large (HiFi or 1 M Nanopore reads: tens of
// GB of pair buffers), in which case it is returned so that the alignment phase that follows finds room on an 80 GB H100.
void lowhashReleaseLargeScratch(shb_context* c)
{
    auto bytes = [](auto& b) { return uint64_t(b.capacity()) * sizeof(*b.get()); };
    const uint64_t total = bytes(c->pairsA) + bytes(c->pairsB) + bytes(c->flagsBuf) + bytes(c->indexBuf) + bytes(c->segStartBuf) +
                           bytes(c->countsBuf) + bytes(c->scanWs) + bytes(c->accKeysA) + bytes(c->accKeysB) + bytes(c->accValsA) +
                           bytes(c->accValsB) + bytes(c->entryKeysTmp) + bytes(c->entryValsTmp) + bytes(c->sweepKeys) +
                           bytes(c->sweepVals) + bytes(c->partKeys) + bytes(c->partVals);
    if(total < (32ull << 30)) return;
    SHB_CUDA(cudaStreamSynchronize(c->stream));
    c->pairsA.release(); c->pairsB.release(); c->flagsBuf.release(); c->indexBuf.release(); c->segStartBuf.release();
    c->countsBuf.release(); c->scanWs.release(); c->accKeysA.release(); c->accKeysB.release(); c->accValsA.release();
    c->accValsB.release(); c->entryKeysTmp.release(); c->entryValsTmp.release(); c->sweepKeys.release(); c->sweepVals.release();
    c->partKeys.release(); c->partVals.release();
    c->sortWs.status.release();
    LowHashState& S = lowhashState(c);
    const uint64_t rawLimit = S.acc.rawLimit;
    S.acc = LowHashAccumulator();
    S.acc.rawLimit = rawLimit;
}

// ... and copied to a host buffer (shb_free) of 12-byte records.
void lowhashEmit(shb_context* c, void** candidatesOut, uint64_t* candidateCountOut)
{
    LowHashState& S = lowhashState(c);
    const uint64_t nOut = lowhashEmitDevice(c);
    cudaStream_t st = c->stream;
    HostBlock host(nOut * 12);
    unsigned long long digest = 0;
    {
        // direct DMA into a page-locked block; into a pageable one through the staging ring, on three copier threads
        StagedCopier copier(c, st, 3);
        copyResult(copier, st, host, 0, reinterpret_cast<const uint8_t*>(c->candidatesDev.get()), nOut * 12);
        SHB_CUDA(cudaMemcpyAsync(&digest, c->scalar(kSlotCandidateDigest), sizeof(digest), cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        copier.finish();
    }
    S.candidateDigest = digest;
    *candidatesOut = host.owner.take();
    *candidateCountOut = nOut;
}

// One stable radix pass on `bits` key bits starting at `shift` (bits <= 8): groups the items by destination.
// counts[d] = items with digit d. Output pointers are context scratch, valid until the next call.
void devicePartition(shb_context* c, uint64_t* keys, uint32_t* vals, uint64_t n, uint32_t shift, uint32_t bits,
                     uint64_t* counts, uint64_t** keysOut, uint32_t** valsOut)
{
    SHB_REQUIRE(bits <= 8 && shift + bits <= 64, SHB_ERR_INVALID, "Invalid partition digit.");
    SHB_REQUIRE(n < (1ull << 32), SHB_ERR_INVALID, "Too many items to partition.");
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const uint32_t buckets = 1u << bits;
    for(uint32_t d = 0; d < buckets; d++) counts[d] = 0;
    if(n == 0 || bits == 0) {
        if(bits == 0) counts[0] = n;
        *keysOut = keys; *valsOut = vals;
        return;
    }
    c->partKeys.reserve(n);
    c->partVals.reserve(n);
    const int range[1][2] = {{int(shift), int(shift + bits)}};
    const bool inB = radixSort<true>(keys, c->partKeys.get(), vals, c->partVals.get(), n, range, 1, c->sortWs, st);
    uint64_t* sortedKeys = inB ? c->partKeys.get() : keys;
    // Digit boundaries by binary search on the host-visible sorted keys would need a copy; count on the device instead.
    unsigned long long* dCounts = c->scalar(kSlotPartitionCounts);
    SHB_CUDA(cudaMemsetAsync(dCounts, 0, buckets * sizeof(unsigned long long), st));
    SHB_LAUNCH(digitCountKernel, ceilDiv(n, 256), 256, 0, st, (const uint64_t*)sortedKeys, uint32_t(n), int(shift), buckets - 1u, dCounts);
    std::vector<unsigned long long> h(buckets);
    SHB_CUDA(cudaMemcpyAsync(h.data(), dCounts, buckets * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaStreamSynchronize(st));
    for(uint32_t d = 0; d < buckets; d++) counts[d] = h[d];
    *keysOut = sortedKeys;
    *valsOut = inB ? c->partVals.get() : vals;
}

// The whole LowHash0 computation on the markers held by the context (single GPU).
void lowhash0(shb_context* c, const shb_lowhash_params& p,
              void** candidatesOut, uint64_t* candidateCountOut,
              uint64_t* statsOut, uint64_t* iterSummary, uint64_t maxIterSummary,
              shb_lowhash_result* result)
{
    SHB_REQUIRE(c->haveMarkers, SHB_ERR_STATE, "Markers are not accessible.");
    SHB_REQUIRE(c->readBegin == 0 && c->readEnd == c->readCountTotal, SHB_ERR_STATE,
                "shb_lowhash0 needs all reads on this GPU (use shb_lowhash0_sharded otherwise).");
    const uint64_t R = c->readCountTotal;
    if(R == 0) {        // the reference would spin forever on 0/0 in its iteration control; return nothing
        *candidatesOut = malloc(1);
        *candidateCountOut = 0;
        if(result) memset(result, 0, sizeof(*result));
        return;
    }
    lowhashBegin(c, p);
    LowHashState& S = lowhashState(c);
    cudaStream_t st = c->stream;
    EventTimer totalTimer;
    totalTimer.start(st);
    const bool perIteration = (p.perIterationMerge != 0) || (p.minHashIterationCount == 0);

    uint64_t highFrequency = 0;
    uint64_t iteration = 0;
    for(;;) {
        // Iteration control, src/LowHash0.cpp:136-157.
        uint32_t group = 1;
        if(p.minHashIterationCount == 0) {
            const double current = 2. * double(highFrequency) / double(R);
            if(current >= p.alignmentCandidatesPerRead) break;
            // The reference spins forever when the target cannot be reached (src/LowHash0.cpp:137-149); give up instead.
            SHB_REQUIRE(iteration < 4096, SHB_ERR_INVALID,
                        "MinHash.alignmentCandidatesPerRead was not reached after 4096 LowHash iterations.");
        } else {
            if(iteration == p.minHashIterationCount) break;
            if(!perIteration) group = nextSweepGroup(p.minHashIterationCount - iteration, S.capacity);
        }
        unsigned long long counts[kMaxFusedIterations];
        lowhashSweep(c, iteration, group, counts);
        for(uint32_t s = 0; s < group; s++, iteration++) {
            lowhashProcessEntries(c, c->sweepKeys.get() + uint64_t(s) * S.capacity, c->sweepVals.get() + uint64_t(s) * S.capacity, counts[s]);
            if(perIteration) {
                reduceRawPairs(c, S.acc, S.readBits);
                mergeAccumulator(c, S.acc, S.readBits);
                highFrequency = countHighFrequency(c, S.acc, p.minFrequency, false);
                if(iterSummary && iteration < maxIterSummary) {
                    iterSummary[2 * iteration] = highFrequency;
                    iterSummary[2 * iteration + 1] = S.acc.count;
                }
            }
        }
    }

    lowhashEmit(c, candidatesOut, candidateCountOut);
    if(statsOut) {
        SHB_CUDA(cudaMemcpyAsync(statsOut, c->stats.get(), 3 * R * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    }
    totalTimer.stop(st);
    SHB_CUDA(cudaStreamSynchronize(st));
    const float totalMs = totalTimer.elapsedMs();
    lowhashReleaseLargeScratch(c);
    if(result) {
        result->iterations = iteration;
        result->log2BucketCount = S.log2BucketCount;
        result->lowHashCount = S.lowHashCount;
        result->pairCount = S.pairCount;
        result->candidateCount = *candidateCountOut;
        result->candidateDigest = S.candidateDigest;
        result->sweepMs = S.sweepMs;
        result->totalMs = totalMs;
        result->sweepLaunches = S.sweepLaunches;
        result->kernelLaunches = g_launchCount;
    }
}

} // namespace shb
