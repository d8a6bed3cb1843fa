// computeAlignments on the GPU: host orchestration (src/AssemblerAlign.cpp:208-495 of chanzuckerberg/shasta).
// Method 3: stage 1 (downsampled, unbanded) -> band -> stage 2 (banded, all markers) -> epilogue.
// Method 4: Align4 front end (cells/components) -> one banded DP per component -> best -> epilogue.
#include "context.cuh"
#include "align_kernels.cuh"
#include "hostcopy.cuh"
#include "digest.cuh"

#include <algorithm>
#include <atomic>
#include <exception>
#include <functional>
#include <memory>
#include <mutex>
#include <chrono>
#include <cstring>
#include <sys/mman.h>
#include <thread>
#include <limits>
#include <map>
#include <vector>

namespace shb {

extern thread_local uint64_t g_launchCount;

namespace {

// One launch per band class (dpClassAt). Wavefront classes run on groups of lanes in blocks of kDpMaxWarpsPerBlock
// warps, with no shared memory; the scan kernel (c = 0) takes as many warps as fit its shared memory.
uint32_t warpsForClass(const DpClass& k)
{
    if(k.c > 0) return kDpMaxWarpsPerBlock;
    // scan kernel: 3 * (wMax + 1) ints per warp; keep a block under ~200 KB of shared memory.
    const uint64_t perWarp = 3ull * (k.wMax + 1) * 4;
    const uint32_t w = uint32_t(std::min<uint64_t>(kDpMaxWarpsPerBlock, (200ull * 1024) / perWarp));
    return w ? w : 1;
}
size_t smemForClass(const DpClass& k, uint32_t warps) { return k.c > 0 ? 0 : size_t(warps) * 3 * (k.wMax + 1) * 4; }
// The scan kernels' dynamic shared memory limit is a per-function attribute shared by all host workers: it is always
// set to the largest class's need, never to the launch's own, so concurrent workers cannot lower it under each other.
size_t scanKernelSmemLimit()
{
    size_t most = 0;
    for(uint32_t k = 0; k < kDpClassCount; k++) most = std::max(most, smemForClass(dpClassAt(k), warpsForClass(dpClassAt(k))));
    return most;
}
constexpr uint32_t kMaxBandWidth = dpClassAt(kDpClassCount - 1).wMax;
// Launch geometry of a class: blocks of `warps` warps, 32 / lanes jobs per warp.
struct DpLaunch { uint32_t blocks, threads; size_t smem; };
DpLaunch dpLaunch(const DpClass& k, uint32_t jobs)
{
    const uint32_t warps = warpsForClass(k);
    return DpLaunch{ceilDiv(jobs, warps * (32 / k.lanes)), warps * 32, smemForClass(k, warps)};
}

// The banded DP kernel instantiation of band class k.
template<uint32_t K = 0, class... Args> void launchBanded(uint32_t k, const DpLaunch& l, cudaStream_t st, Args... args)
{
    if constexpr(K < kDpClassCount) {
        if(k != K) { launchBanded<K + 1>(k, l, st, args...); return; }
        constexpr DpClass cl = dpClassAt(K);
        if constexpr(cl.c == 0) {
            SHB_CUDA(cudaFuncSetAttribute(bandedAlignKernel<32, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(scanKernelSmemLimit())));
        }
        auto* kernel = &bandedAlignKernel<int(cl.lanes), int(cl.c)>;
        SHB_LAUNCH(kernel, l.blocks, l.threads, l.smem, st, args...);
    }
}
// Stage 1 of method 3 without a trace (downsampled reads of at most 512 markers): forward class k.
template<uint32_t K = 0, class... Args> void launchStage1Forward(uint32_t k, uint32_t jobs, cudaStream_t st, Args... args)
{
    if constexpr(K < kDpForwardClassCount) {
        if(k != K) { launchStage1Forward<K + 1>(k, jobs, st, args...); return; }
        constexpr DpForwardClass f = dpForwardClassAt(K);
        auto* kernel = &method3Stage1ForwardKernel<int(f.lanes), int(f.rows)>;
        SHB_LAUNCH(kernel, ceilDiv(jobs, kDpMaxWarpsPerBlock * (32 / f.lanes)), kDpMaxWarpsPerBlock * 32, 0, st, args...);
    }
}

// Buffers for one batch of candidates (both methods).
struct Batch {
    DeviceBuffer<uint32_t> cand, counts, infoWords, jobKeep, jobBytes, keep, keepIndex, bytes32, selected;
    DeviceBuffer<DpJob> jobs1, jobs;
    DeviceBuffer<unsigned long long> tw, twOff, outCnt, outOff, bytes64, bytesOff, scanWs64;
    DeviceBuffer<uint32_t> trace;
    DeviceBuffer<uint2> ordinals, runs;
    DeviceBuffer<int2> endCells;
    DeviceBuffer<uint32_t> runCounts;
    // method 4
    DeviceBuffer<unsigned long long> cellCnt, cellOff;
    DeviceBuffer<uint32_t> gridCounts, gridAux, gridList, componentCount, jobOffsets;
    DeviceBuffer<uint8_t> gridFlags;
    DeviceBuffer<int32_t> gridBands;
    // band-class ordering of the DP jobs
    DeviceBuffer<uint32_t> orderValsA, orderValsB;
    DeviceBuffer<uint64_t> orderKeysA, orderKeysB;
    const uint32_t* order = nullptr;
};

// Device-side counters of one worker (one unsigned long long each).
enum WorkerScalar { kScTotal64 = 0, kScTotal32 = 1, kScSkipped = 2, kScForwardCells = 3, kScTooWide = 4, kScBandCells = 5,
                    kScDigits = 16, kScCount = 16 + 256 };

// One host thread's private streams and scratch. computeAlignments runs the batches of a call on a few of these
// concurrently: while one worker waits for a device-side size (scratch is sized from scans on the device), the kernels of
// the others keep the GPU busy, so the host round trips leave the critical path.
struct AlignWorker {
    cudaStream_t stream = nullptr;
    // side streams: the band classes of one batch are independent launches (disjoint jobs and scratch), so the few
    // long jobs of the wide classes run beside the big narrow-band launch instead of after it
    static constexpr int kSideStreams = 3;
    cudaStream_t side[kSideStreams] = {nullptr, nullptr, nullptr};
    cudaEvent_t forkEv = nullptr, joinEv[kSideStreams] = {nullptr, nullptr, nullptr};
    // high-priority streams for the short latency-bound kernels (traceback, filter) that follow each DP chunk: their
    // blocks are scheduled ahead of the pending blocks of the other chunks' DP kernels
    static constexpr int kHiStreams = 4;
    cudaStream_t hiStream[kHiStreams] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t hiJoinEv[kHiStreams] = {nullptr, nullptr, nullptr, nullptr};
    std::vector<cudaEvent_t> unitEvents;
    cudaEvent_t dp1a = nullptr, dp1b = nullptr, dp2a = nullptr, dp2b = nullptr;
    Batch batch;
    SortWorkspace sortWs;
    DeviceBuffer<uint32_t> scanWs;
    DeviceBuffer<unsigned long long> scalars;
    // per call
    double dpMs = 0.;
    uint64_t traceWords = 0, launches = 0;

    void init()
    {
        if(stream) return;
        int least = 0, greatest = 0;
        SHB_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        SHB_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        SHB_CUDA(cudaEventCreateWithFlags(&forkEv, cudaEventDisableTiming));
        for(int i = 0; i < kSideStreams; i++) {
            SHB_CUDA(cudaStreamCreateWithFlags(&side[i], cudaStreamNonBlocking));
            SHB_CUDA(cudaEventCreateWithFlags(&joinEv[i], cudaEventDisableTiming));
        }
        for(int i = 0; i < kHiStreams; i++) {
            SHB_CUDA(cudaStreamCreateWithPriority(&hiStream[i], cudaStreamNonBlocking, greatest));
            SHB_CUDA(cudaEventCreateWithFlags(&hiJoinEv[i], cudaEventDisableTiming));
        }
        SHB_CUDA(cudaEventCreate(&dp1a)); SHB_CUDA(cudaEventCreate(&dp1b));
        SHB_CUDA(cudaEventCreate(&dp2a)); SHB_CUDA(cudaEventCreate(&dp2b));
        scalars.reserve(kScCount);
    }
    ~AlignWorker()
    {
        for(int i = 0; i < kHiStreams; i++) { if(hiStream[i]) cudaStreamDestroy(hiStream[i]); if(hiJoinEv[i]) cudaEventDestroy(hiJoinEv[i]); }
        for(cudaEvent_t e : unitEvents) cudaEventDestroy(e);
        for(int i = 0; i < kSideStreams; i++) { if(side[i]) cudaStreamDestroy(side[i]); if(joinEv[i]) cudaEventDestroy(joinEv[i]); }
        for(cudaEvent_t e : {forkEv, dp1a, dp1b, dp2a, dp2b}) if(e) cudaEventDestroy(e);
        if(stream) cudaStreamDestroy(stream);
    }
    unsigned long long* sc(int k) { return scalars.get() + k; }
};

// Derived per-marker data cached in the context (per marker generation), the workers, and the device-side result arena.
struct AlignCache {
    // method 3: downsampled marker CSR
    DeviceBuffer<uint64_t> dsToc;
    DeviceBuffer<uint32_t> dsKmer, dsOrdinal;
    uint32_t dsMaxRow = 0, dsK = 0;
    double dsFactor = -1.;
    uint64_t dsGeneration = ~0ull;
    // method 4: markers sorted by k-mer id within each oriented read
    DeviceBuffer<uint32_t> sortedKmer, sortedOrdinal;
    uint64_t sortedGeneration = ~0ull;
    uint64_t lengthCheckGeneration = ~0ull;
    uint64_t longestRead = 0;           // markers of the longest oriented read, for lengthCheckGeneration
    // workers and the device-side result accumulation: kept across calls so that a steady-state call does not allocate
    // or free device memory
    std::vector<std::unique_ptr<AlignWorker>> workers;
    DeviceBuffer<uint32_t> outRecords;
    DeviceBuffer<unsigned long long> outToc;
    DeviceBuffer<uint8_t> outData;
    cudaStream_t finalStream = nullptr;         // rebase / digest / device->host copy of the finished batches
    double lastBytesPerCandidate = 0.;          // compressed bytes per candidate of the previous call (sizes the data block)
    ~AlignCache() { if(finalStream) cudaStreamDestroy(finalStream); }
};

AlignCache& cache(shb_context* c)
{
    if(!c->alignCache) c->alignCache = new AlignCache();
    return *static_cast<AlignCache*>(c->alignCache);
}

// Runs launch(k, count, offset, stream) for every non-empty band class, cut into chunks of at most chunkMax jobs:
// the widest classes first, round-robin over the side streams and the worker's main stream, so that independent launches
// (disjoint jobs and scratch) overlap: the few long jobs of the wide classes run beside the big narrow-band launch,
// and the latency-bound traceback of one chunk runs beside the issue-bound DP of the next. The main stream continues
// after all of them.
template<class F> void forEachClassConcurrently(AlignWorker& w, const std::vector<uint64_t>& classCounts, uint32_t chunkMax, F launch)
{
    cudaStream_t st = w.stream;
    struct Unit { int k; uint32_t count; uint64_t offset; };
    std::vector<Unit> units;
    const int classCount = int(classCounts.size());
    std::vector<uint64_t> offsets(classCounts.size(), 0);
    for(int k = 1; k < classCount; k++) offsets[k] = offsets[k-1] + classCounts[k-1];
    for(int k = classCount - 1; k >= 0; k--) {
        const uint64_t count = classCounts[k];
        if(!count) continue;
        const uint64_t chunks = (count + chunkMax - 1) / chunkMax, per = (count + chunks - 1) / chunks;
        for(uint64_t begin = 0; begin < count; begin += per) units.push_back({k, uint32_t(std::min(per, count - begin)), offsets[k] + begin});
    }
    if(units.empty()) return;
    constexpr int kStreams = AlignWorker::kSideStreams + 1;      // the last one is the main stream
    bool used[AlignWorker::kSideStreams] = {false, false, false};
    if(units.size() > 1) SHB_CUDA(cudaEventRecord(w.forkEv, st));
    for(size_t u = 0; u < units.size(); u++) {
        // the last unit always goes to the main stream
        const int i = (u + 1 == units.size()) ? kStreams - 1 : int(u % kStreams);
        cudaStream_t s = st;
        if(i < AlignWorker::kSideStreams) {
            s = w.side[i];
            if(!used[i]) { SHB_CUDA(cudaStreamWaitEvent(s, w.forkEv, 0)); used[i] = true; }
        }
        launch(units[u].k, units[u].count, units[u].offset, s);
    }
    for(int i = 0; i < AlignWorker::kSideStreams; i++) {
        if(!used[i]) continue;
        SHB_CUDA(cudaEventRecord(w.joinEv[i], w.side[i]));
        SHB_CUDA(cudaStreamWaitEvent(st, w.joinEv[i], 0));
    }
}

void buildDownsampled(shb_context* c, uint32_t k, double factor)
{
    AlignCache& ds = cache(c);
    if(ds.dsK == k && ds.dsFactor == factor && ds.dsGeneration == c->markerGeneration && ds.dsToc.get()) return;
    cudaStream_t st = c->stream;
    const uint64_t M = c->localMarkerCount;
    const uint32_t rows = uint32_t(2 * c->readCountTotal);
    // src/AssemblerAlign3.cpp:71-72
    const uint32_t hashThreshold = uint32_t(factor * double(std::numeric_limits<uint32_t>::max()));
    ds.dsToc.reserve(uint64_t(rows) + 1);
    const uint32_t chunk = envCount("SHB_DOWNSAMPLE_CHUNK", 1u << 27);     // test hook: small sets cross chunk seams
    c->flagsBuf.reserve(std::min<uint64_t>(chunk, M) + 1);
    c->indexBuf.reserve(std::min<uint64_t>(chunk, M) + 1);
    c->scanWs.reserve(scanWorkspaceElements(chunk));
    // scalars: 512 entries, allocated once at context creation
    uint32_t* totalDev = reinterpret_cast<uint32_t*>(c->scalar(kSlotDownsampleTotal));
    // Pass 0 sizes the output exactly; pass 1 compacts.
    uint64_t total = 0;
    for(int pass = 0; pass < 2; pass++) {
        if(pass == 1) { ds.dsKmer.reserve(total + 1); ds.dsOrdinal.reserve(total + 1); }
        uint64_t running = 0;
        for(uint64_t begin = 0; begin < M; begin += chunk) {
            const uint32_t n = uint32_t(std::min<uint64_t>(chunk, M - begin));
            SHB_LAUNCH(downsampleFlagsKernel, ceilDiv(n, 256), 256, 0, st, c->kmerIds, begin, n, k, hashThreshold, c->flagsBuf.get());
            exclusiveScan<uint32_t>(c->flagsBuf.get(), c->indexBuf.get(), n, totalDev, c->scanWs.get(), st);
            const uint32_t t = readBack<uint32_t>(totalDev, st);
            if(pass == 1) {
                SHB_LAUNCH(downsampleCompactKernel, ceilDiv(n, 256), 256, 0, st, c->kmerIds, begin, n,
                           (const uint32_t*)c->flagsBuf.get(), (const uint32_t*)c->indexBuf.get(),
                           (const uint64_t*)c->toc.get(), rows, running, ds.dsKmer.get(), ds.dsOrdinal.get());
                SHB_LAUNCH(downsampleTocKernel, ceilDiv(uint64_t(rows) + 1, 256), 256, 0, st, (const uint64_t*)c->toc.get(), rows,
                           begin, n, (const uint32_t*)c->indexBuf.get(), running, running + t, ds.dsToc.get());
            }
            running += t;
        }
        total = running;
    }
    if(M == 0) SHB_CUDA(cudaMemsetAsync(ds.dsToc.get(), 0, (uint64_t(rows) + 1) * 8, st));
    // Longest downsampled row (diagnostics; candidates whose stage 1 is too wide are skipped one by one).
    std::vector<uint64_t> hostToc(uint64_t(rows) + 1);
    SHB_CUDA(cudaMemcpyAsync(hostToc.data(), ds.dsToc.get(), (uint64_t(rows) + 1) * 8, cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaStreamSynchronize(st));
    uint32_t maxRow = 0;
    for(uint32_t r = 0; r < rows; r++) maxRow = std::max<uint32_t>(maxRow, uint32_t(hostToc[r+1] - hostToc[r]));
    ds.dsMaxRow = maxRow; ds.dsK = k; ds.dsFactor = factor; ds.dsGeneration = c->markerGeneration;
}

} // namespace

// The markers of every row of the resident marker set sorted by k-mer id, chunk after chunk. A chunk is the longest run of
// rows, taken rowStep at a time, with at most chunkLimit markers, or rowStep rows of more. The chunk's (row - rowBegin) << 32 |
// k-mer id keys and its ordinals are radix-sorted on the low kmerBits bits and the row bits, and passed to
// sorted(keys, ordinals, rowBegin, rowEnd, markerBegin, n); with n = 0 the pointers are null. tooLong: the error for a chunk
// of 2^32 or more markers. The scratch is freed on return, after the stream has finished.
void sortMarkersByKmer(shb_context* c, uint32_t rowStep, uint64_t chunkLimit, uint32_t kmerBits, const char* tooLong,
                       const std::function<void(const uint64_t*, const uint32_t*, uint32_t, uint32_t, uint64_t, uint32_t)>& sorted)
{
    cudaStream_t st = c->stream;
    const uint32_t rows = uint32_t(2 * c->readCountTotal);
    const std::vector<uint64_t>& toc = c->tocHost;
    DeviceBuffer<uint64_t> keysA, keysB;
    DeviceBuffer<uint32_t> valsA, valsB;
    for(uint32_t rowBegin = 0; rowBegin < rows; ) {
        uint32_t rowEnd = rowBegin + rowStep;
        while(rowEnd < rows && toc[rowEnd + rowStep] - toc[rowBegin] <= chunkLimit) rowEnd += rowStep;
        const uint64_t markerBegin = toc[rowBegin];
        const uint64_t n64 = toc[rowEnd] - markerBegin;
        SHB_REQUIRE(n64 < (1ull << 32), SHB_ERR_INVALID, tooLong);
        const uint32_t n = uint32_t(n64);
        const uint64_t* keys = nullptr; const uint32_t* vals = nullptr;
        if(n) {
            keysA.reserve(n); keysB.reserve(n); valsA.reserve(n); valsB.reserve(n);
            SHB_LAUNCH(sortedMarkerKeysKernel, ceilDiv(n, 256), 256, 0, st, c->kmerIds, (const uint64_t*)c->toc.get(),
                       rowBegin, rowEnd, markerBegin, n, keysA.get(), valsA.get());
            const uint32_t rowBits = bitsFor(rowEnd - rowBegin - 1);
            const int ranges[2][2] = {{0, int(kmerBits)}, {32, 32 + int(rowBits)}};
            const bool inB = radixSort<true>(keysA.get(), keysB.get(), valsA.get(), valsB.get(), n, ranges, 2, c->sortWs, st);
            keys = inB ? keysB.get() : keysA.get();
            vals = inB ? valsB.get() : valsA.get();
        }
        sorted(keys, vals, rowBegin, rowEnd, markerBegin, n);
        rowBegin = rowEnd;
    }
    SHB_CUDA(cudaStreamSynchronize(st));
}

namespace {

// computeSortedMarkers (src/AssemblerAlign4.cpp:190-261): per oriented read, (kmerId, ordinal) sorted by kmerId.
void buildSortedMarkers(shb_context* c, uint32_t k)
{
    AlignCache& sc = cache(c);
    if(sc.sortedGeneration == c->markerGeneration && sc.sortedKmer.get()) return;
    cudaStream_t st = c->stream;
    const uint64_t M = c->localMarkerCount;
    sc.sortedKmer.reserve(M + 1);
    sc.sortedOrdinal.reserve(M + 1);
    const uint64_t chunkLimit = envCount("SHB_ALIGN4_SORT_CHUNK", 1u << 28);     // test hook: small sets make many row chunks
    sortMarkersByKmer(c, 1, chunkLimit, 2 * k, "An oriented read has more than 2^32-1 markers.",
                      [&](const uint64_t* keys, const uint32_t* vals, uint32_t, uint32_t, uint64_t markerBegin, uint32_t n) {
        if(!n) return;
        SHB_LAUNCH(sortedMarkerUnpackKernel, ceilDiv(n, 256), 256, 0, st, keys, n, sc.sortedKmer.get() + markerBegin);
        SHB_CUDA(cudaMemcpyAsync(sc.sortedOrdinal.get() + markerBegin, vals, 4ull * n, cudaMemcpyDeviceToDevice, st));
    });
    sc.sortedGeneration = c->markerGeneration;
}

// Groups the runnable jobs by band class (longest first inside a class). Returns per-class counts; b.order holds the
// job indices, class after class.
void buildClassOrder(AlignWorker& w, const DpJob* jobs, uint32_t nJobs, std::vector<uint64_t>& classCounts, bool forward = false)
{
    cudaStream_t st = w.stream;
    Batch& b = w.batch;
    classCounts.assign(kDpClassCount + (forward ? kDpForwardClassCount : 0), 0);
    if(nJobs == 0) return;
    b.orderKeysA.reserve(nJobs); b.orderKeysB.reserve(nJobs); b.orderValsA.reserve(nJobs); b.orderValsB.reserve(nJobs);
    SHB_LAUNCH(dpClassKeysKernel, ceilDiv(nJobs, 256), 256, 0, st, jobs, nJobs, forward, b.orderKeysA.get(), b.orderValsA.get());
    const int ranges[1][2] = {{0, kDpLengthKeyBits + kDpClassKeyBits}};
    const bool inB = radixSort<true>(b.orderKeysA.get(), b.orderKeysB.get(), b.orderValsA.get(), b.orderValsB.get(), nJobs, ranges, 1, w.sortWs, st);
    b.order = inB ? b.orderValsB.get() : b.orderValsA.get();
    unsigned long long* dCounts = w.sc(kScDigits);
    SHB_CUDA(cudaMemsetAsync(dCounts, 0, 256 * sizeof(unsigned long long), st));
    SHB_LAUNCH(digitCountKernel, ceilDiv(nJobs, 256), 256, 0, st, (const uint64_t*)(inB ? b.orderKeysB.get() : b.orderKeysA.get()), nJobs, kDpLengthKeyBits, kDpClassNone, dCounts);
    unsigned long long h[256];
    SHB_CUDA(cudaMemcpyAsync(h, dCounts, sizeof(h), cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaStreamSynchronize(st));
    for(size_t k = 0; k < classCounts.size(); k++) classCounts[k] = h[k];
}

// Runs the jobs of b.order class by class (classCounts from buildClassOrder), in chunks of at most chunkMax jobs.
// Band class k sits at index firstBanded + k: the DP of a chunk (group per job) on its stream, then its traceback (thread
// per job) and equal-k-mer filter (warp per job) on a high-priority stream. The classes below firstBanded (the forward
// classes of method 3's stage 1) go to launchOther(k, count, order, stream). The main stream continues after all of them.
// trace, endCells, runs, runCounts, ordinals and counts must be reserved for the jobs.
template<class F> void runDpClasses(AlignWorker& w, const std::vector<uint64_t>& classCounts, uint32_t chunkMax, uint32_t firstBanded,
                                    const DpJob* jobs, const uint32_t* sequences, DpScores scores, F launchOther)
{
    Batch& b = w.batch;
    BandedArgs g;
    g.kmerIds = sequences; g.scores = scores; g.fma = FmaUnits{1, 2, 4};
    size_t unit = 0;
    forEachClassConcurrently(w, classCounts, chunkMax, [&](int k, uint32_t count, uint64_t offset, cudaStream_t s) {
        const uint32_t* order = b.order + offset;
        if(uint32_t(k) < firstBanded) { launchOther(uint32_t(k), count, order, s); return; }
        const uint32_t cls = uint32_t(k) - firstBanded;
        BandedArgs gk = g;
        gk.n = count; gk.order = order; gk.wMax = dpClassAt(cls).wMax;
        launchBanded(cls, dpLaunch(dpClassAt(cls), count), s, gk, jobs, b.trace.get(), b.endCells.get());
        if(unit == w.unitEvents.size()) {
            cudaEvent_t e = nullptr;
            SHB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            w.unitEvents.push_back(e);
        }
        SHB_CUDA(cudaEventRecord(w.unitEvents[unit], s));
        cudaStream_t hs = w.hiStream[unit % AlignWorker::kHiStreams];
        SHB_CUDA(cudaStreamWaitEvent(hs, w.unitEvents[unit], 0));
        unit++;
        SHB_LAUNCH(tracebackKernel, ceilDiv(count, 128), 128, 0, hs, count, order, jobs, (const int2*)b.endCells.get(),
                   (const uint32_t*)b.trace.get(), b.runs.get(), b.runCounts.get());
        SHB_LAUNCH(filterStepsKernel, ceilDiv(count, 4), 128, 0, hs, count, order, jobs, sequences,
                   (const uint2*)b.runs.get(), (const uint32_t*)b.runCounts.get(), b.ordinals.get(), b.counts.get());
    });
    for(size_t i = 0; i < std::min<size_t>(unit, AlignWorker::kHiStreams); i++) {
        SHB_CUDA(cudaEventRecord(w.hiJoinEv[i], w.hiStream[i]));
        SHB_CUDA(cudaStreamWaitEvent(w.stream, w.hiJoinEv[i], 0));
    }
}

// Scratch offsets + the banded DP + traceback for nJobs jobs whose lo/hi/state are set.
void runBandedJobs(AlignWorker& w, uint32_t nJobs, const uint32_t* sequences, DpScores scores)
{
    cudaStream_t st = w.stream;
    Batch& b = w.batch;
    unsigned long long* total64 = w.sc(kScTotal64);
    b.scanWs64.reserve(scanWorkspaceElements(nJobs));
    b.twOff.reserve(nJobs); b.outOff.reserve(nJobs); b.counts.reserve(nJobs); b.endCells.reserve(nJobs); b.runCounts.reserve(nJobs);
    exclusiveScan<unsigned long long>(b.tw.get(), b.twOff.get(), nJobs, total64, b.scanWs64.get(), st);
    const unsigned long long traceWords = readBack<unsigned long long>(total64, st);
    exclusiveScan<unsigned long long>(b.outCnt.get(), b.outOff.get(), nJobs, total64, b.scanWs64.get(), st);
    const unsigned long long ordinalSlots = readBack<unsigned long long>(total64, st);
    b.trace.reserve(traceWords + 1);
    b.ordinals.reserve(ordinalSlots + 1);
    b.runs.reserve(ordinalSlots + 1);
    w.traceWords += traceWords;
    SHB_LAUNCH(setTraceOffsetsKernel, ceilDiv(nJobs, 256), 256, 0, st, b.jobs.get(), nJobs, (const unsigned long long*)b.twOff.get(),
               (const unsigned long long*)b.outOff.get());
    SHB_LAUNCH(bandCellsKernel, ceilDiv(nJobs, 256), 256, 0, st, (const DpJob*)b.jobs.get(), nJobs, w.sc(kScBandCells));
    SHB_CUDA(cudaMemsetAsync(b.counts.get(), 0, 4ull * nJobs, st));
    std::vector<uint64_t> classCounts;
    buildClassOrder(w, b.jobs.get(), nJobs, classCounts);
    SHB_CUDA(cudaEventRecord(w.dp2a, st));
    runDpClasses(w, classCounts, envCount("SHB_ALIGN_CHUNK", 32768), 0, b.jobs.get(), sequences, scores,
                 [](uint32_t, uint32_t, const uint32_t*, cudaStream_t) {});
    SHB_CUDA(cudaEventRecord(w.dp2b, st));
}

// What one call shares between its workers.
struct AlignCall {
    shb_context* c;
    AlignCache* ac;
    const uint32_t* cand; uint64_t n;
    shb_align_options o;
    bool method4;
    DpScores scores; FilterOptions fo;
    uint32_t batchMax;
    uint32_t align4SmemCells = kAlign4SmemCells;   // candidates with more existing cells take the global-memory path (SHB_ALIGN4_SMEM_CELLS: test hook)
    // batch dispenser (method 4 sizes a batch by its grid cells, so the cut is made under the lock, in order)
    std::mutex dispenserMutex;
    uint64_t nextBegin = 0, nextIndex = 0;
    // device-side result arena: segments in completion order + the ledger that puts them back into candidate order
    struct Segment { uint64_t recordBase = 0, kept = 0, byteBase = 0, bytes = 0; };
    std::mutex arenaMutex;
    std::map<uint64_t, Segment> ledger;     // by batch index (guarded by arenaMutex)
    uint64_t outCount = 0, outBytes = 0;
    // Finalisation in candidate order, as soon as a prefix of the batches is complete: rebase, digests and the device->host
    // copy run on their own stream beside the next batches.
    cudaStream_t finalStream = nullptr;
    unsigned long long* digests = nullptr;      // device, 2 words
    uint64_t nextToFinalise = 0, finalRecords = 0, finalBytes = 0;
    HostBlock* hostRecords = nullptr; HostBlock* hostToc = nullptr; HostBlock* hostData = nullptr;
    StagedCopier* copier = nullptr;
    // the compressed bytes go by direct DMA while they fit the page-locked data block; once they outgrow it, the copier
    // grows the block and fills the rest
    bool dataDirect = false;
    uint64_t dataDirectCapacity = 0;
    // failure of any worker stops the others
    std::atomic<bool> failed{false};
    std::exception_ptr error;
    std::mutex errorMutex;
};

// Next batch [begin, begin + nb) and its index; false when the candidates are exhausted.
bool nextBatch(AlignCall& call, uint64_t& begin, uint32_t& nb, uint64_t& index)
{
    std::lock_guard<std::mutex> lock(call.dispenserMutex);
    if(call.nextBegin >= call.n || call.failed.load()) return false;
    begin = call.nextBegin;
    nb = 0;
    if(call.method4) {
        const std::vector<uint64_t>& toc = call.c->tocHost;
        const uint64_t cellBudget = 768ull << 20;      // cells of grid scratch per batch (17 B each, per worker)
        uint64_t cells = 0;
        while(begin + nb < call.n && nb < call.batchMax) {
            const uint64_t i = begin + nb;
            const uint64_t o0 = 2ull * call.cand[3*i], o1 = 2ull * call.cand[3*i+1] + ((call.cand[3*i+2] & 0xff) ? 0 : 1);
            const uint64_t nx = toc[o0+1] - toc[o0], ny = toc[o1+1] - toc[o1];
            uint64_t cc = 2;
            if(nx && ny) cc += ((nx + ny - 2) / call.o.align4DeltaX + 1) * ((nx + ny - 2) / call.o.align4DeltaY + 1);
            if(nb && cells + cc > cellBudget) break;
            cells += cc; nb++;
        }
    } else nb = uint32_t(std::min<uint64_t>(call.batchMax, call.n - begin));
    index = call.nextIndex++;
    call.nextBegin += nb;
    return true;
}

// toc[k] += delta for the n entries of one segment.
__global__ void rebaseTocKernel(unsigned long long* __restrict__ toc, uint64_t n, long long delta)
{
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if(i < n) toc[i] = (unsigned long long)((long long)toc[i] + delta);
}

// Called with arenaMutex held, after a batch's segment has been recorded (and its write kernel has finished): finalises
// every segment whose predecessors are all complete. Everything is queued on call.finalStream.
void finaliseReadySegments(AlignCall& call)
{
    AlignCache& ac = *call.ac;
    cudaStream_t fs = call.finalStream;
    for(;;) {
        auto it = call.ledger.find(call.nextToFinalise);
        if(it == call.ledger.end()) break;
        const AlignCall::Segment& seg = it->second;
        if(seg.kept) {
            unsigned long long* segToc = ac.outToc.get() + seg.recordBase;
            const long long delta = (long long)call.finalBytes - (long long)seg.byteBase;     // the write kernel stored arena offsets
            if(delta) SHB_LAUNCH(rebaseTocKernel, ceilDiv(seg.kept, 256), 256, 0, fs, segToc, seg.kept, delta);
            SHB_LAUNCH(digestRecordsKernel, ceilDiv(seg.kept, 256), 256, 0, fs, (const uint32_t*)ac.outRecords.get() + 16 * seg.recordBase,
                       seg.kept, 16u, call.digests);
            SHB_LAUNCH(digestCompressedKernel, ceilDiv(seg.kept, 256), 256, 0, fs, (const uint32_t*)ac.outRecords.get() + 16 * seg.recordBase,
                       seg.kept, (const unsigned long long*)segToc, call.finalBytes + seg.bytes,
                       (const uint8_t*)ac.outData.get() + seg.byteBase - call.finalBytes, call.digests + 1);
            // The arena may move before a staged copy's DMA is queued: the copier looks the source up under arenaMutex.
            const AlignCache* acp = &ac;
            const uint64_t recordBase = seg.recordBase, byteBase = seg.byteBase;
            if(call.hostRecords->pageLocked) {
                SHB_CUDA(cudaMemcpyAsync(call.hostRecords->data() + 64 * call.finalRecords, ac.outRecords.get() + 16 * seg.recordBase, 64 * seg.kept, cudaMemcpyDeviceToHost, fs));
            } else call.copier->copy(*call.hostRecords, 64 * call.finalRecords,
                                     [acp, recordBase] { return reinterpret_cast<const uint8_t*>(acp->outRecords.get() + 16 * recordBase); }, 64 * seg.kept);
            if(call.hostToc->pageLocked) {
                SHB_CUDA(cudaMemcpyAsync(call.hostToc->data() + 8 * call.finalRecords, segToc, 8 * seg.kept, cudaMemcpyDeviceToHost, fs));
            } else call.copier->copy(*call.hostToc, 8 * call.finalRecords,
                                     [acp, recordBase] { return reinterpret_cast<const uint8_t*>(acp->outToc.get() + recordBase); }, 8 * seg.kept);
            if(call.dataDirect && call.finalBytes + seg.bytes > call.dataDirectCapacity) call.dataDirect = false;
            if(call.dataDirect) {
                SHB_CUDA(cudaMemcpyAsync(call.hostData->data() + call.finalBytes, ac.outData.get() + seg.byteBase, seg.bytes, cudaMemcpyDeviceToHost, fs));
            } else call.copier->copy(*call.hostData, call.finalBytes,
                                     [acp, byteBase] { return acp->outData.get() + byteBase; }, seg.bytes);
            call.finalRecords += seg.kept; call.finalBytes += seg.bytes;
        }
        call.nextToFinalise++;
    }
}

// One batch of candidates on one worker, up to the point where its kept alignments sit in the arena.
void processBatch(AlignCall& call, AlignWorker& w, uint64_t begin, uint32_t nb, uint64_t batchIndex)
{
    shb_context* c = call.c;
    AlignCache& ac = *call.ac;
    const shb_align_options& o = call.o;
    cudaStream_t st = w.stream;
    Batch& b = w.batch;
    unsigned long long* total64 = w.sc(kScTotal64);
    uint32_t* total32 = reinterpret_cast<uint32_t*>(w.sc(kScTotal32));

    b.cand.reserve(3ull * nb);
    SHB_CUDA(cudaMemcpyAsync(b.cand.get(), call.cand + 3 * begin, 12ull * nb, cudaMemcpyHostToDevice, st));
    b.keep.reserve(nb); b.keepIndex.reserve(nb); b.bytes32.reserve(nb); b.bytes64.reserve(nb); b.bytesOff.reserve(nb);
    b.scanWs64.reserve(scanWorkspaceElements(nb));
    w.scanWs.reserve(scanWorkspaceElements(std::max<uint64_t>(nb, 4096)));
    uint32_t nJobs = 0;
    const uint32_t* jobIndex = nullptr;
    bool stage1Timed = false;

    if(!call.method4) {
        // ---- methods 3 and 1 -----------------------------------------------------------------------
        const bool method1 = (o.alignMethod == 1);
        nJobs = nb;
        b.jobs1.reserve(nb); b.jobs.reserve(nb); b.tw.reserve(nb); b.twOff.reserve(nb); b.outCnt.reserve(nb);
        SHB_LAUNCH(method3SetupKernel, ceilDiv(nb, 256), 256, 0, st, (const uint32_t*)b.cand.get(), nb,
                   (const uint64_t*)c->toc.get(), method1 ? (const uint64_t*)nullptr : (const uint64_t*)ac.dsToc.get(), b.jobs1.get(), b.jobs.get(),
                   b.tw.get(), b.outCnt.get(), w.sc(kScForwardCells), kMaxBandWidth, w.sc(kScTooWide));
        if(!method1) {
            exclusiveScan<unsigned long long>(b.tw.get(), b.twOff.get(), nb, total64, b.scanWs64.get(), st);
            const unsigned long long traceWords1 = readBack<unsigned long long>(total64, st);
            b.trace.reserve(traceWords1 + 1);
            w.traceWords += traceWords1;
            // The jobs too long for the forward kernel keep their path's runs and kept steps in the candidate's stage-2
            // ordinal slots (min(nx, ny) is at least the number of downsampled diagonal steps).
            b.outOff.reserve(nb);
            exclusiveScan<unsigned long long>(b.outCnt.get(), b.outOff.get(), nb, total64, b.scanWs64.get(), st);
            const unsigned long long slots1 = readBack<unsigned long long>(total64, st);
            b.ordinals.reserve(slots1 + 1); b.runs.reserve(slots1 + 1);
            b.counts.reserve(nb); b.endCells.reserve(nb); b.runCounts.reserve(nb);
            SHB_LAUNCH(setTraceOffsetsKernel, ceilDiv(nb, 256), 256, 0, st, b.jobs1.get(), nb, (const unsigned long long*)b.twOff.get(),
                       (const unsigned long long*)b.outOff.get());
            Method3Args g1;
            g1.candidates = b.cand.get(); g1.candidateBegin = begin; g1.n = nb;
            g1.toc = c->toc.get(); g1.dsToc = ac.dsToc.get(); g1.dsKmer = ac.dsKmer.get(); g1.dsOrdinal = ac.dsOrdinal.get();
            g1.scores = call.scores; g1.bandExtend = o.bandExtend; g1.maxBand = o.maxBand;
            std::vector<uint64_t> classCounts1;
            buildClassOrder(w, b.jobs1.get(), nb, classCounts1, true);
            SHB_CUDA(cudaEventRecord(w.dp1a, st));
            // One launch per class: cutting stage 1 into SHB_ALIGN_CHUNK chunks measured slower on long reads
            // (bench.py --workload nanopore-ul-20k).
            runDpClasses(w, classCounts1, 0xffffffffu, kDpForwardClassCount, b.jobs1.get(), ac.dsKmer.get(), call.scores,
                         [&](uint32_t k, uint32_t count, const uint32_t* order, cudaStream_t s) {
                Method3Args gk = g1;
                gk.n = count; gk.order = order;
                launchStage1Forward(k, count, s, gk, (const DpJob*)b.jobs1.get(), b.jobs.get());
            });
            // The band of the jobs that took the trace path: they follow the forward classes in b.order.
            uint64_t forwardJobs = 0, tracedJobs = 0;
            for(uint32_t k = 0; k < classCounts1.size(); k++) (k < kDpForwardClassCount ? forwardJobs : tracedJobs) += classCounts1[k];
            if(tracedJobs) {
                SHB_LAUNCH(stage1BandKernel, ceilDiv(tracedJobs, 4), 128, 0, st, uint32_t(tracedJobs), b.order + forwardJobs,
                           (const DpJob*)b.jobs1.get(), (const uint32_t*)ac.dsOrdinal.get(), (const uint2*)b.ordinals.get(),
                           (const uint32_t*)b.runCounts.get(), (const uint32_t*)b.counts.get(), o.bandExtend, o.maxBand, b.jobs.get());
            }
            SHB_CUDA(cudaEventRecord(w.dp1b, st));
            stage1Timed = true;
            if(getenv("SHB_TRACE") && begin == 0) {        // band-width and active-column statistics of the first batch
                std::vector<DpJob> h(nb);
                SHB_CUDA(cudaMemcpyAsync(h.data(), b.jobs.get(), sizeof(DpJob) * nb, cudaMemcpyDeviceToHost, st));
                SHB_CUDA(cudaStreamSynchronize(st));
                uint64_t hist[12] = {0}, run = 0, cols = 0, fullCols = 0;
                for(const DpJob& j : h) {
                    if(j.state != kStateRun) continue;
                    run++;
                    const uint32_t wd = uint32_t(j.hi - j.lo + 1);
                    hist[std::min<uint32_t>(11, (wd + 7) / 8)]++;
                    cols += uint64_t(dpLastColumn(j.nx, j.ny, j.hi) - dpFirstColumn(j.lo)); fullCols += j.nx;
                }
                fprintf(stderr, "[shb] stage-2 jobs %llu of %u; band width histogram (bins of 8 offsets, last = wider):", (unsigned long long)run, nb);
                for(int k = 0; k < 12; k++) fprintf(stderr, " %llu", (unsigned long long)hist[k]);
                fprintf(stderr, "; active columns %.1f of %.1f per job\n", double(cols) / double(run ? run : 1), double(fullCols) / double(run ? run : 1));
            }
        }
        SHB_LAUNCH(stage2TraceWordsKernel, ceilDiv(nb, 256), 256, 0, st, (const DpJob*)b.jobs.get(), nb, b.tw.get());
        runBandedJobs(w, nJobs, c->kmerIds, call.scores);
        // Epilogue per job == per candidate.
        b.infoWords.reserve(13ull * nJobs);
        SHB_LAUNCH(alignmentInfoKernel, ceilDiv(nJobs, 4), 128, 0, st, nJobs, (const DpJob*)b.jobs.get(), (const uint2*)b.ordinals.get(),
                   (const uint32_t*)b.counts.get(), call.fo, b.infoWords.get(), b.keep.get(), b.bytes32.get(), w.sc(kScSkipped));
    } else {
        // ---- method 4 ---------------------------------------------------------------------------
        b.cellCnt.reserve(nb); b.cellOff.reserve(nb); b.componentCount.reserve(nb); b.jobOffsets.reserve(nb); b.selected.reserve(nb);
        SHB_LAUNCH(align4CellCountKernel, ceilDiv(nb, 256), 256, 0, st, (const uint32_t*)b.cand.get(), nb, (const uint64_t*)c->toc.get(),
                   uint32_t(o.align4DeltaX), uint32_t(o.align4DeltaY), b.cellCnt.get());
        exclusiveScan<unsigned long long>(b.cellCnt.get(), b.cellOff.get(), nb, total64, b.scanWs64.get(), st);
        const unsigned long long cells = readBack<unsigned long long>(total64, st);
        b.gridCounts.reserve(cells + 1); b.gridAux.reserve(cells + 1); b.gridList.reserve(cells + 1);
        b.gridFlags.reserve(cells + 1); b.gridBands.reserve(cells + 1);
        Align4Args g;
        g.candidates = b.cand.get(); g.n = nb; g.toc = c->toc.get();
        g.sortedKmer = ac.sortedKmer.get(); g.sortedOrdinal = ac.sortedOrdinal.get();
        g.deltaX = uint32_t(o.align4DeltaX); g.deltaY = uint32_t(o.align4DeltaY);
        g.minEntryCountPerCell = o.align4MinEntryCountPerCell; g.maxDistanceFromBoundary = o.align4MaxDistanceFromBoundary;
        g.maxBand = int64_t(uint64_t(o.maxBand));
        g.cellOffsets = b.cellOff.get(); g.counts = b.gridCounts.get(); g.aux = b.gridAux.get(); g.list = b.gridList.get();
        g.flags = b.gridFlags.get(); g.bands = b.gridBands.get(); g.componentCount = b.componentCount.get();
        SHB_LAUNCH(align4MatrixKernel, ceilDiv(nb, 4), 128, 0, st, g);
        SHB_LAUNCH(align4ComponentsKernel, ceilDiv(nb, kAlign4WarpsPerBlock), kAlign4WarpsPerBlock * 32, 0, st, g, call.align4SmemCells);
        exclusiveScan<uint32_t>(b.componentCount.get(), b.jobOffsets.get(), nb, total32, w.scanWs.get(), st);
        nJobs = readBack<uint32_t>(total32, st);
        if(nJobs) {
            b.jobs.reserve(nJobs); b.tw.reserve(nJobs); b.outCnt.reserve(nJobs);
            SHB_LAUNCH(align4MakeJobsKernel, ceilDiv(nb, 256), 256, 0, st, (const uint32_t*)b.cand.get(), nb, (const uint64_t*)c->toc.get(),
                       (const unsigned long long*)b.cellOff.get(), (const int32_t*)b.gridBands.get(),
                       (const uint32_t*)b.componentCount.get(), (const uint32_t*)b.jobOffsets.get(), b.jobs.get(), b.tw.get(), b.outCnt.get());
            runBandedJobs(w, nJobs, c->kmerIds, call.scores);
            b.infoWords.reserve(13ull * nJobs); b.jobKeep.reserve(nJobs); b.jobBytes.reserve(nJobs);
            // Align4's own filters (src/Align4.cpp:944-985), identical thresholds, no containment test.
            SHB_LAUNCH(alignmentInfoKernel, ceilDiv(nJobs, 4), 128, 0, st, nJobs, (const DpJob*)b.jobs.get(), (const uint2*)b.ordinals.get(),
                       (const uint32_t*)b.counts.get(), call.fo, b.infoWords.get(), b.jobKeep.get(), b.jobBytes.get(),
                       (unsigned long long*)nullptr);
        } else {
            b.infoWords.reserve(13); b.jobKeep.reserve(1); b.jobBytes.reserve(1); b.jobs.reserve(1); b.counts.reserve(1); b.ordinals.reserve(1);
        }
        SHB_LAUNCH(align4SelectKernel, ceilDiv(nb, 256), 256, 0, st, nb, (const uint32_t*)b.jobOffsets.get(),
                   (const uint32_t*)b.componentCount.get(), (const uint32_t*)b.jobKeep.get(), (const uint32_t*)b.infoWords.get(),
                   (const uint32_t*)b.jobBytes.get(), o.suppressContainments ? 1u : 0u, uint32_t(o.maxTrim),
                   b.selected.get(), b.keep.get(), b.bytes32.get());
        jobIndex = b.selected.get();
    }

    // ---- compaction + output of the kept alignments ---------------------------------------------------
    exclusiveScan<uint32_t>(b.keep.get(), b.keepIndex.get(), nb, total32, w.scanWs.get(), st);
    SHB_LAUNCH(widenKernel<uint32_t>, ceilDiv(nb, 256), 256, 0, st, (const uint32_t*)b.bytes32.get(), nb, b.bytes64.get());
    exclusiveScan<unsigned long long>(b.bytes64.get(), b.bytesOff.get(), nb, total64, b.scanWs64.get(), st);
    struct { unsigned long long bytes; uint32_t kept; } totals;
    SHB_CUDA(cudaMemcpyAsync(&totals.bytes, total64, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaMemcpyAsync(&totals.kept, total32, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaStreamSynchronize(st));
    const uint32_t kept = totals.kept;
    const unsigned long long bytes = totals.bytes;
    if(nJobs) {
        float ms = 0.f;
        SHB_CUDA(cudaEventElapsedTime(&ms, w.dp2a, w.dp2b));
        w.dpMs += ms;
    }
    if(stage1Timed) {
        float ms = 0.f;
        SHB_CUDA(cudaEventElapsedTime(&ms, w.dp1a, w.dp1b));
        w.dpMs += ms;
    }
    {
        // The arena may have to grow (realloc + copy): writers hold the lock until their kernel has finished, so nothing
        // is in flight into the arena while another worker moves it.
        std::lock_guard<std::mutex> lock(call.arenaMutex);
        AlignCall::Segment seg;
        seg.recordBase = call.outCount; seg.kept = kept; seg.byteBase = call.outBytes; seg.bytes = bytes;
        if(kept) {
            if(16ull * (call.outCount + kept) > ac.outRecords.capacity() || call.outCount + kept + 1 > ac.outToc.capacity() ||
               call.outBytes + bytes + 16 > ac.outData.capacity()) {
                SHB_CUDA(cudaStreamSynchronize(call.finalStream));       // the arena moves: nothing may still be reading it
            }
            ac.outRecords.reserve(16ull * (call.outCount + kept), true, st);
            ac.outToc.reserve(call.outCount + kept + 1, true, st);
            ac.outData.reserve(call.outBytes + bytes + 16, true, st);
            // compressedToc entries are written as arena offsets; computeAlignments rebases them once the final order of the
            // segments is known.
            SHB_LAUNCH(alignmentWriteKernel, ceilDiv(nb, 4), 128, 0, st, nb, (const uint32_t*)b.cand.get(), (const DpJob*)b.jobs.get(),
                       (const uint2*)b.ordinals.get(), (const uint32_t*)b.counts.get(), (const uint32_t*)b.infoWords.get(), jobIndex,
                       (const uint32_t*)b.keep.get(), (const uint32_t*)b.keepIndex.get(), (const unsigned long long*)b.bytesOff.get(),
                       call.outCount, call.outBytes, ac.outRecords.get(), ac.outToc.get(), ac.outData.get());
            SHB_CUDA(cudaStreamSynchronize(st));
            call.outCount += kept;
            call.outBytes += bytes;
        }
        call.ledger[batchIndex] = seg;
        finaliseReadySegments(call);
    }
}

void workerMain(AlignCall& call, AlignWorker& w)
{
    try {
        SHB_CUDA(cudaSetDevice(call.c->device));
        g_launchCount = 0;
        w.dpMs = 0.; w.traceWords = 0;
        SHB_CUDA(cudaMemsetAsync(w.scalars.get(), 0, kScCount * sizeof(unsigned long long), w.stream));
        uint64_t begin = 0, index = 0; uint32_t nb = 0;
        while(nextBatch(call, begin, nb, index)) processBatch(call, w, begin, nb, index);
        SHB_CUDA(cudaStreamSynchronize(w.stream));
    } catch(...) {
        std::lock_guard<std::mutex> lock(call.errorMutex);
        if(!call.error) call.error = std::current_exception();
        call.failed.store(true);
    }
    w.launches = g_launchCount;
}

} // namespace

void destroyAlignCache(shb_context* c)
{
    if(c->alignCache) { delete static_cast<AlignCache*>(c->alignCache); c->alignCache = nullptr; }
}


// explicitOrientation: the candidates may carry kCandidateStrand0Bit and need not satisfy readId0 < readId1
// (shb_align_oriented_reads); computeAlignments proper rejects both, like the reference (src/AssemblerAlign.cpp:378).
void computeAlignments(shb_context* c, const void* candidatesHost, uint64_t n, const shb_align_options& o,
                       void** alignmentDataOut, uint64_t* alignmentCountOut,
                       uint64_t** compressedTocOut, uint8_t** compressedDataOut, shb_align_result* result,
                       bool explicitOrientation)
{
    SHB_REQUIRE(c->haveMarkers, SHB_ERR_STATE, "Markers are not accessible.");
    SHB_REQUIRE(c->readBegin == 0 && c->readEnd == c->readCountTotal, SHB_ERR_STATE,
                "computeAlignments needs the markers of all reads on this GPU.");
    SHB_REQUIRE(o.alignMethod == 1 || o.alignMethod == 3 || o.alignMethod == 4, SHB_ERR_INVALID,
                "Only Align.alignMethod 1, 3 and 4 are implemented (0, the AlignmentGraph method, is not on the hot path).");
    SHB_REQUIRE(o.gapScore <= 0, SHB_ERR_INVALID, "Align.gapScore must not be positive.");
    SHB_REQUIRE(o.k >= 1 && o.k <= 16, SHB_ERR_INVALID, "Invalid k.");
    SHB_REQUIRE(n == 0 || candidatesHost != nullptr, SHB_ERR_INVALID, "Null candidates.");
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    g_launchCount = 0;
    const auto wall0 = std::chrono::steady_clock::now();
    EventTimer totalTimer;
    totalTimer.start(st);

    AlignCall call;
    call.c = c; call.ac = &cache(c); call.o = o; call.n = n;
    call.method4 = (o.alignMethod == 4);
    // src/AssemblerAlign.cpp:378 asserts readIds[0] < readIds[1].
    call.cand = static_cast<const uint32_t*>(candidatesHost);
    for(uint64_t i = 0; i < n; i++) {
        const uint32_t r0 = call.cand[3*i], r1 = call.cand[3*i+1], w = call.cand[3*i+2];
        if(explicitOrientation) SHB_REQUIRE(r0 < c->readCountTotal && r1 < c->readCountTotal && (w & ~(0xffu | kCandidateStrand0Bit)) == 0,
                                            SHB_ERR_INVALID, "Invalid oriented read pair.");
        else SHB_REQUIRE(r0 < r1 && r1 < c->readCountTotal && (w & 0xffffff00u) == 0, SHB_ERR_INVALID, "Invalid alignment candidate.");
    }

    AlignCache& ac = *call.ac;
    if(ac.lengthCheckGeneration != c->markerGeneration) {       // the traceback packs a run length above a 28-bit ordinal
        uint64_t longest = 0;                                   // (the reference's Uint24 positions cap a read at 2^24 markers anyway)
        for(size_t r = 0; r + 1 < c->tocHost.size(); r++) {
            SHB_REQUIRE(c->tocHost[r + 1] - c->tocHost[r] < (1ull << kRunLengthShift), SHB_ERR_INVALID, "A read has 2^28 or more markers.");
            longest = std::max<uint64_t>(longest, c->tocHost[r + 1] - c->tocHost[r]);
        }
        ac.longestRead = longest;
        ac.lengthCheckGeneration = c->markerGeneration;
    }
    // Methods 1 and 3 use the configured scores; Align4 hard-codes 6/-1/-1 (src/Align4.hpp:159-161: never overwritten).
    call.scores = call.method4 ? DpScores{6, -1, -1} : DpScores{o.matchScore, o.mismatchScore, o.gapScore};
    // Score range of the DP kernels. They run in int32 with sentinels instead of "have" flags: kNegInf = -2^29 starts every
    // cell outside the matrix, the two barrier offsets of the wavefront kernels enter with the gap score kGapBarrier = -2^28,
    // and the end cell starts at -2^30. With M = max(|match|, |mismatch|, |gap|), L = longest read and W = kMaxBandWidth,
    // their results equal exact arithmetic when M * (2L + W) < 2^28:
    //  - every in-band cell of the matrix lies on a diagonal that starts at a boundary cell (score 0) inside the band, so its
    //    exact score R satisfies |R| <= min(i, j) * M <= L * M, and every value in column i is at most i * M above anything
    //    that does not enter through a barrier;
    //  - an in-matrix cell only reads in-matrix cells and barriers (cells above the matrix feed only the row j = 0, which is
    //    reset to 0; cells below it feed nothing), and every barrier value is kNegInf plus the drift of at most L + 31
    //    columns (lanes start up to 31 columns early), or some earlier value plus kGapBarrier plus drift. Both are at most
    //    L * M - 2^28 < -L * M <= R: a barrier never wins, nor ties, against a real score, and so never changes a trace code;
    //  - the best end score is at least -L * M > -2^30, so it is always recorded;
    //  - values stay within [-2^29 - (L + 64) * M - 2^28, (L + 2) * M], and the scan kernel's A - e * gap (e < W) within
    //    (L + W + 1) * M of zero: nothing wraps.
    // Under 6/-1/-1 (the defaults, and Align4 always) this admits reads of up to 22.3 M markers, more than the reference's
    // 2^24-marker positions can hold; the 2^28-marker limit above alone would let a read exceed the sentinels.
    // L is the longest read in the context (cached above); only when that fails are the reads of this call's candidates
    // scanned, so that a context holding one very long read can still align the others.
    {
        const uint64_t M = uint64_t(std::max({std::abs(int64_t(call.scores.match)), std::abs(int64_t(call.scores.mismatch)),
                                              std::abs(int64_t(call.scores.gap))}));
        const auto fits = [M](uint64_t L) { return M * (2 * L + kMaxBandWidth) < (1ull << 28); };
        if(!fits(ac.longestRead)) {
            uint64_t longest = 0;
            for(uint64_t i = 0; i < n; i++) {
                for(int k = 0; k < 2; k++) {
                    const uint64_t o = 2ull * call.cand[3 * i + k];
                    longest = std::max<uint64_t>(longest, c->tocHost[o + 1] - c->tocHost[o]);
                }
            }
            SHB_REQUIRE(fits(longest), SHB_ERR_INVALID,
                        "Align scores too large for the reads: max(|matchScore|, |mismatchScore|, |gapScore|) * "
                        "(2 * longest read in markers + 16384) must be below 2^28.");
        }
    }
    if(call.method4) {
        SHB_REQUIRE(o.align4DeltaX >= 1 && o.align4DeltaY >= 1 && o.align4DeltaX < (1ull << 31) && o.align4DeltaY < (1ull << 31),
                    SHB_ERR_INVALID, "Invalid Align.align4.deltaX / deltaY.");
        buildSortedMarkers(c, o.k);
    } else if(o.alignMethod == 3) {
        buildDownsampled(c, o.k, o.downsamplingFactor);
    }
    const uint32_t maxStage2Width = uint32_t(std::max(0, o.maxBand)) + 3 + 64;     // W <= maxBand + 1, two barriers, padded to 64
    SHB_REQUIRE(maxStage2Width <= kMaxBandWidth, SHB_ERR_INVALID, "Align.maxBand too large for this implementation (limit 16317).");

    call.fo.minAlignedMarkerCount = uint64_t(o.minAlignedMarkerCount); call.fo.maxSkip = uint64_t(o.maxSkip);
    call.fo.maxDrift = uint64_t(o.maxDrift); call.fo.maxTrim = uint64_t(o.maxTrim);
    call.fo.minAlignedFraction = o.minAlignedFraction;
    call.fo.suppressContainments = (!call.method4 && o.suppressContainments) ? 1u : 0u;     // method 4 applies it after the selection

    // SHB_ALIGN_BATCH / SHB_ALIGN_CHUNK / SHB_ALIGN_WORKERS: test hooks that shrink the batch and chunk sizes so that small
    // inputs exercise the multi-batch, multi-chunk, multi-worker paths (tests/test_gpu_scale.py).
    call.batchMax = envCount("SHB_ALIGN_BATCH", call.method4 ? 32768 : (o.alignMethod == 1 ? 16384 : 262144));
    call.align4SmemCells = std::min<uint32_t>(kAlign4SmemCells, envCount("SHB_ALIGN4_SMEM_CELLS", kAlign4SmemCells));
    const uint64_t batchEstimate = (n + call.batchMax - 1) / call.batchMax;
    const uint32_t workerCount = uint32_t(std::max<uint64_t>(1, std::min<uint64_t>(envCount("SHB_ALIGN_WORKERS", 2), batchEstimate)));
    while(ac.workers.size() < workerCount) ac.workers.emplace_back(new AlignWorker());
    for(uint32_t k = 0; k < workerCount; k++) ac.workers[k]->init();
    if(!ac.finalStream) SHB_CUDA(cudaStreamCreateWithFlags(&ac.finalStream, cudaStreamNonBlocking));
    call.finalStream = ac.finalStream;
    call.digests = c->scalar(kSlotAlignmentDigests);
    SHB_CUDA(cudaMemsetAsync(call.digests, 0, 2 * sizeof(unsigned long long), st));
    // Host result blocks up front: records and toc by their upper bound (every candidate kept), the compressed bytes by the
    // previous call's bytes per candidate (a guess on the first call; the copier grows the block when it falls short). Only
    // the pages written are touched. The finished prefix of the batches is copied out while the later batches run: by direct
    // DMA into page-locked blocks (recycled ones), through the staging ring and four copier threads into the others.
    const uint64_t dataEstimate = n ? uint64_t((ac.lastBytesPerCandidate > 0. ? ac.lastBytesPerCandidate * 1.03 : 64.) * double(n)) + (1ull << 20) : 0;
    HostBlock recOut(64 * n), tocOut(8 * (n + 1)), dataOut(dataEstimate);
    StagedCopier copier(c, call.finalStream, 4, &call.arenaMutex);
    call.hostRecords = &recOut; call.hostToc = &tocOut; call.hostData = &dataOut; call.copier = &copier;
    call.dataDirect = dataOut.pageLocked; call.dataDirectCapacity = dataEstimate;
    SHB_CUDA(cudaStreamSynchronize(st));        // derived marker data ready before the workers read it

    if(n) {
        // Always on their own threads (also a single worker), so that the launch counters stay per thread.
        std::vector<std::thread> threads;
        for(uint32_t k = 0; k < workerCount; k++) threads.emplace_back([&call, &ac, k] { workerMain(call, *ac.workers[k]); });
        for(std::thread& t : threads) t.join();
        if(call.error) std::rethrow_exception(call.error);
    }

    // ---- results: the segments were rebased, digested and copied to the host in candidate order while the later batches were
    // still running (finaliseReadySegments); what is left is the copy of the last ones.
    const auto copy0 = std::chrono::steady_clock::now();
    SHB_CUDA(cudaStreamSynchronize(call.finalStream));
    copier.finish();
    const uint64_t count = call.outCount, outBytes = call.outBytes;
    SHB_REQUIRE(call.nextToFinalise == call.ledger.size() && call.finalRecords == count && call.finalBytes == outBytes, SHB_ERR_CUDA,
                "Internal error: not every batch was finalised.");
    if(n) ac.lastBytesPerCandidate = double(outBytes) / double(n);
    unsigned long long* digests = call.digests;
    // Counters of the workers.
    unsigned long long skipped = 0, forwardCells = 0, tooWide = 0, bandCells = 0, digestHost[2] = {0, 0};
    uint64_t traceWords = 0, launches = g_launchCount;
    double dpMs = 0.;
    for(uint32_t k = 0; k < workerCount && n; k++) {
        AlignWorker& w = *ac.workers[k];
        unsigned long long h[6];
        SHB_CUDA(cudaMemcpyAsync(h, w.scalars.get(), sizeof(h), cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        skipped += h[kScSkipped]; forwardCells += h[kScForwardCells]; tooWide += h[kScTooWide]; bandCells += h[kScBandCells];
        traceWords += w.traceWords; launches += w.launches; dpMs += w.dpMs;
    }
    SHB_CUDA(cudaMemcpyAsync(digestHost, digests, sizeof(digestHost), cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaStreamSynchronize(st));
    uint64_t* tocHostOut = reinterpret_cast<uint64_t*>(tocOut.data());
    tocHostOut[count] = outBytes;
    if(count == 0) tocHostOut[0] = 0;
    totalTimer.stop(st);
    SHB_CUDA(cudaStreamSynchronize(st));
    const float totalMs = totalTimer.elapsedMs();
    if(getenv("SHB_TRACE")) {
        fprintf(stderr, "[shb] computeAlignments: %u worker(s), %llu batches, %llu candidates skipped as too wide for the DP kernels\n",
                workerCount, (unsigned long long)call.ledger.size(), tooWide);
    }
    if(result) {
        memset(result, 0, sizeof(*result));
        result->candidateCount = n; result->alignmentCount = count; result->skippedCount = skipped;
        result->dpCells = 16ull * traceWords + forwardCells;
        result->dpUsefulCells = bandCells + forwardCells;
        result->tooWideCount = tooWide;
        result->dpMs = dpMs / double(workerCount); result->totalMs = totalMs; result->kernelLaunches = launches;
        result->alignmentDataDigest = digestHost[0]; result->compressedDigest = digestHost[1];
        result->workers = workerCount;
        result->outputCopyMs = msSince(copy0);
        result->hostWallMs = msSince(wall0);
    }
    *alignmentDataOut = recOut.owner.take(); *alignmentCountOut = count;
    *compressedTocOut = static_cast<uint64_t*>(tocOut.owner.take()); *compressedDataOut = static_cast<uint8_t*>(dataOut.owner.take());
}

} // namespace shb
