// Read-sharded multi-GPU LowHash0 + alignment behind the C ABI (SURVEY.md section 8e; BASELINE.json configs[2..4]).
// One process per GPU; the only collective library is NCCL (over NVLink / NVSwitch), resolved at run time with dlopen so
// that single-GPU users do not need it. The orchestration mirrors LowHash0::LowHash0 (src/LowHash0.cpp:23-257) with the
// two exchanges a sharded run needs:
//   * rank g holds the marker rows of a contiguous read range and hashes only those;
//   * LowHash buckets are owned by ranks: owner(bucketId) = bucketId >> (log2BucketCount - log2 W). After every sweep the
//     low-hash entries of each iteration are grouped by owner on the device (one radix pass) and exchanged with grouped
//     ncclSend/ncclRecv; a bucket is never split across ranks, so bucket sizes, per-read statistics and pair hits are
//     exact. The exchange of iteration k+1 runs on the communication stream while iteration k's buckets are inspected
//     on the compute stream;
//   * each owner accumulates (pair,count) over all iterations; once, at the end, the merged local lists are cut into
//     contiguous readId0 ranges of equal pair mass (histogram all-reduced over the ranks) and exchanged; the owner sums,
//     applies the uint16 wrap and the minFrequency threshold and emits its slice; the slices are then evened out to equal
//     contiguous blocks of the global order, on the device. Concatenating the ranks' outputs gives the reference's order;
//   * ReadLowHashStatistics are partial sums, all-reduced once;
//   * alignment: the k-mer id shards are gathered once per marker set (grouped ncclBroadcast, cached until the markers
//     change) into a second context that then aligns this rank's block of candidates; no collective in the loop.
// bench.py --gpus N, tests/run_distributed_gpu.py and a C++ host run this file on GPUs; tests/test_gpu_distributed.py runs it
// as a world of one.
#include "context.cuh"
#include "hostpool.cuh"

#include <dlfcn.h>
#include <nccl.h>

#include <chrono>
#include <cstring>
#include <string>
#include <vector>

namespace shb {

// internal entry points of lowhash.cu / api.cu / align.cu
LowHashState& lowhashState(shb_context* c);
void lowhashBegin(shb_context* c, const shb_lowhash_params& p);
void lowhashSweep(shb_context* c, uint64_t iterationBegin, uint32_t group, unsigned long long* counts);
void lowhashProcessEntries(shb_context* c, uint64_t* keysA, uint32_t* valsA, uint64_t n64);
void lowhashLocalPairs(shb_context* c, uint64_t** keys, uint32_t** counts, uint64_t* n);
void lowhashReleaseLargeScratch(shb_context* c);
void lowhashSetPairs(shb_context* c, const uint64_t* keys, const uint32_t* counts, uint64_t n);
uint64_t lowhashEmitDevice(shb_context* c);
uint32_t nextSweepGroup(uint64_t remaining, uint64_t slabCapacity);
void devicePartition(shb_context* c, uint64_t* keys, uint32_t* vals, uint64_t n, uint32_t shift, uint32_t bits,
                     uint64_t* counts, uint64_t** keysOut, uint32_t** valsOut);
void computeAlignments(shb_context* c, const void* candidatesHost, uint64_t n, const shb_align_options& o,
                       void** alignmentDataOut, uint64_t* alignmentCountOut,
                       uint64_t** compressedTocOut, uint8_t** compressedDataOut, shb_align_result* result,
                       bool explicitOrientation);
extern thread_local uint64_t g_launchCount;

namespace {

// The NCCL entry points used, resolved from libnccl.so.2 (already in the process when the host uses torch).
struct Nccl {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

Nccl& nccl()
{
    static Nccl n;
    if(n.handle) return n;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for(const char* name : names) { n.handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL); if(n.handle) break; }
    SHB_REQUIRE(n.handle != nullptr, SHB_ERR_STATE, "NCCL (libnccl.so.2) could not be loaded: the multi-GPU entry points need it.");
    auto sym = [&](const char* s) { void* p = dlsym(n.handle, s); SHB_REQUIRE(p != nullptr, SHB_ERR_STATE, std::string("NCCL symbol missing: ") + s); return p; };
    n.GetUniqueId = reinterpret_cast<decltype(n.GetUniqueId)>(sym("ncclGetUniqueId"));
    n.CommInitRank = reinterpret_cast<decltype(n.CommInitRank)>(sym("ncclCommInitRank"));
    n.CommDestroy = reinterpret_cast<decltype(n.CommDestroy)>(sym("ncclCommDestroy"));
    n.AllGather = reinterpret_cast<decltype(n.AllGather)>(sym("ncclAllGather"));
    n.AllReduce = reinterpret_cast<decltype(n.AllReduce)>(sym("ncclAllReduce"));
    n.Broadcast = reinterpret_cast<decltype(n.Broadcast)>(sym("ncclBroadcast"));
    n.Send = reinterpret_cast<decltype(n.Send)>(sym("ncclSend"));
    n.Recv = reinterpret_cast<decltype(n.Recv)>(sym("ncclRecv"));
    n.GroupStart = reinterpret_cast<decltype(n.GroupStart)>(sym("ncclGroupStart"));
    n.GroupEnd = reinterpret_cast<decltype(n.GroupEnd)>(sym("ncclGroupEnd"));
    n.GetErrorString = reinterpret_cast<decltype(n.GetErrorString)>(sym("ncclGetErrorString"));
    return n;
}

#define SHB_NCCL(call)                                                                          \
    do {                                                                                        \
        ncclResult_t shbNccl_ = (call);                                                         \
        if(shbNccl_ != ncclSuccess) throw ::shb::Error(SHB_ERR_CUDA, std::string(#call) + " failed at " + __FILE__ + ":" + \
            std::to_string(__LINE__) + ": " + nccl().GetErrorString(shbNccl_));                 \
    } while(0)

} // namespace

// Per-context distributed state.
struct DistState {
    ncclComm_t comm = nullptr;
    bool ownComm = false;
    int world = 1, rank = 0, log2World = 0;
    cudaStream_t commStream = nullptr;
    cudaEvent_t computeDone = nullptr;
    std::vector<cudaEvent_t> slabReady;
    // exchange buffers of one sweep group (per slab: what this rank sends, grouped by owner; what it receives)
    DeviceBuffer<uint64_t> sendKeys, recvKeys, pairSendKeys, pairRecvKeys;
    DeviceBuffer<uint32_t> sendVals, recvVals, pairSendVals, pairRecvVals, candRecv;
    DeviceBuffer<unsigned long long> countsDev;         // count matrices for the all-gathers
    // alignment: all reads' k-mer ids, gathered once per marker set
    shb_context* alignCtx = nullptr;
    DeviceBuffer<uint32_t> gathered;
    DeviceBuffer<unsigned long long> tocStage;
    uint64_t gatheredGeneration = ~0ull;
    shb_dist_timing timing{};
    ~DistState()
    {
        if(alignCtx) shb_context_destroy(alignCtx);
        for(cudaEvent_t e : slabReady) cudaEventDestroy(e);
        if(computeDone) cudaEventDestroy(computeDone);
        if(commStream) cudaStreamDestroy(commStream);
        if(comm && ownComm) nccl().CommDestroy(comm);
    }
};

DistState& distState(shb_context* c)
{
    SHB_REQUIRE(c->dist != nullptr, SHB_ERR_STATE, "shb_dist_init / shb_dist_attach was not called on this context.");
    return *static_cast<DistState*>(c->dist);
}

void destroyDistState(shb_context* c)
{
    if(c->dist) { delete static_cast<DistState*>(c->dist); c->dist = nullptr; }
}

namespace {

double seconds(std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b)
{
    return std::chrono::duration<double>(b - a).count();
}

void attach(shb_context* c, ncclComm_t comm, bool own, int world, int rank)
{
    SHB_REQUIRE(world >= 1 && rank >= 0 && rank < world, SHB_ERR_INVALID, "Invalid world size / rank.");
    int log2w = 0;
    while((1 << log2w) < world) log2w++;
    SHB_REQUIRE((1 << log2w) == world && world <= 256, SHB_ERR_INVALID,
                "The number of ranks must be a power of two (at most 256): bucket ownership is by the top bits of the bucket id.");
    destroyDistState(c);
    DistState* d = new DistState();
    c->dist = d;
    d->comm = comm; d->ownComm = own; d->world = world; d->rank = rank; d->log2World = log2w;
    SHB_CUDA(cudaSetDevice(c->device));
    SHB_CUDA(cudaStreamCreateWithFlags(&d->commStream, cudaStreamNonBlocking));
    SHB_CUDA(cudaEventCreateWithFlags(&d->computeDone, cudaEventDisableTiming));
    d->countsDev.reserve(uint64_t(world) * (kMaxFusedIterations * world + 512));
}

// All ranks learn every rank's `words` counters: out[r * words + k] = counter k of rank r (host vector).
std::vector<unsigned long long> allGatherCounts(shb_context* c, DistState& d, const std::vector<unsigned long long>& mine)
{
    const size_t words = mine.size();
    d.countsDev.reserve((uint64_t(d.world) + 1) * words);
    unsigned long long* send = d.countsDev.get();
    unsigned long long* recv = send + words;
    cudaStream_t st = d.commStream;
    SHB_CUDA(cudaMemcpyAsync(send, mine.data(), words * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
    SHB_NCCL(nccl().AllGather(send, recv, words, ncclUint64, d.comm, st));
    std::vector<unsigned long long> all(words * size_t(d.world));
    SHB_CUDA(cudaMemcpyAsync(all.data(), recv, all.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaStreamSynchronize(st));
    return all;
}

// Grouped variable-size exchange of one array: segment `dst` of `send` (sendCounts[dst] items from sendOffsets[dst]) goes
// to rank dst; what arrives from rank src lands at recvOffsets[src].
template<class T> void exchange(DistState& d, const T* send, const uint64_t* sendOffsets, const uint64_t* sendCounts,
                                T* recv, const uint64_t* recvOffsets, const uint64_t* recvCounts, ncclDataType_t type, cudaStream_t st)
{
    SHB_NCCL(nccl().GroupStart());
    for(int peer = 0; peer < d.world; peer++) {
        if(sendCounts[peer]) SHB_NCCL(nccl().Send(send + sendOffsets[peer], sendCounts[peer], type, peer, d.comm, st));
        if(recvCounts[peer]) SHB_NCCL(nccl().Recv(recv + recvOffsets[peer], recvCounts[peer], type, peer, d.comm, st));
    }
    SHB_NCCL(nccl().GroupEnd());
}

} // namespace

// LowHash0 over read shards. Every rank returns the g-th contiguous block of the global candidate list.
void lowhash0Sharded(shb_context* c, const shb_lowhash_params& p, void** candidatesOut, uint64_t* candidateCountOut,
                     uint64_t* statsOut, shb_lowhash_result* result)
{
    DistState& d = distState(c);
    SHB_REQUIRE(c->haveMarkers, SHB_ERR_STATE, "Markers are not accessible.");
    SHB_REQUIRE(p.minHashIterationCount != 0, SHB_ERR_INVALID,
                "The sharded LowHash0 needs a fixed MinHash.minHashIterationCount (every shipped configuration sets one): the "
                "candidate-driven stopping rule needs a merge over all ranks after every iteration.");
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream, cs = d.commStream;
    const int W = d.world, me = d.rank;
    const uint64_t R = c->readCountTotal;
    const auto t0 = std::chrono::steady_clock::now();
    d.timing = shb_dist_timing{};
    EventTimer total;
    total.start(st);

    lowhashBegin(c, p);
    LowHashState& S = lowhashState(c);
    SHB_REQUIRE(S.log2BucketCount >= uint64_t(d.log2World), SHB_ERR_INVALID, "Fewer LowHash buckets than ranks.");
    const uint32_t entryShift = uint32_t(32 + S.log2BucketCount - d.log2World);

    uint64_t iteration = 0;
    while(iteration < p.minHashIterationCount) {
        const uint32_t group = nextSweepGroup(p.minHashIterationCount - iteration, S.capacity);
        auto ta = std::chrono::steady_clock::now();
        unsigned long long counts[kMaxFusedIterations];
        lowhashSweep(c, iteration, group, counts);
        auto tb = std::chrono::steady_clock::now();
        d.timing.sweepSeconds += seconds(ta, tb);

        // Group every slab by bucket owner (one radix pass; the library's partition scratch is reused, so each slab's grouped
        // entries are staged in the send buffers) and collect the [slab][owner] count matrix.
        uint64_t sendTotal = 0;
        for(uint32_t s = 0; s < group; s++) sendTotal += counts[s];
        d.sendKeys.reserve(sendTotal + 1); d.sendVals.reserve(sendTotal + 1);
        std::vector<unsigned long long> mine(size_t(group) * W, 0);
        std::vector<uint64_t> slabSendBase(group + 1, 0);
        for(uint32_t s = 0; s < group; s++) {
            uint64_t cnt[256];
            uint64_t* pk = nullptr; uint32_t* pv = nullptr;
            devicePartition(c, c->sweepKeys.get() + uint64_t(s) * S.capacity, c->sweepVals.get() + uint64_t(s) * S.capacity, counts[s],
                            entryShift, uint32_t(d.log2World), cnt, &pk, &pv);
            for(int g = 0; g < W; g++) mine[size_t(s) * W + g] = (d.log2World == 0) ? counts[s] : cnt[g];
            slabSendBase[s + 1] = slabSendBase[s] + counts[s];
            if(counts[s]) {
                SHB_CUDA(cudaMemcpyAsync(d.sendKeys.get() + slabSendBase[s], pk, 8 * counts[s], cudaMemcpyDeviceToDevice, st));
                SHB_CUDA(cudaMemcpyAsync(d.sendVals.get() + slabSendBase[s], pv, 4 * counts[s], cudaMemcpyDeviceToDevice, st));
            }
        }
        SHB_CUDA(cudaEventRecord(d.computeDone, st));
        SHB_CUDA(cudaStreamWaitEvent(cs, d.computeDone, 0));
        auto tc = std::chrono::steady_clock::now();
        d.timing.partitionSeconds += seconds(tb, tc);

        // One count exchange for the whole group; then every slab's exchange is queued on the communication stream at once and
        // the compute stream inspects slab s as soon as its entries have arrived (exchange of s+1 overlaps the processing of s).
        const std::vector<unsigned long long> all = allGatherCounts(c, d, mine);       // [rank][slab][owner]
        std::vector<uint64_t> slabRecvBase(group + 1, 0);
        for(uint32_t s = 0; s < group; s++) {
            uint64_t n = 0;
            for(int src = 0; src < W; src++) n += all[(size_t(src) * group + s) * W + me];
            slabRecvBase[s + 1] = slabRecvBase[s] + n;
        }
        d.recvKeys.reserve(slabRecvBase[group] + 1); d.recvVals.reserve(slabRecvBase[group] + 1);
        while(d.slabReady.size() < group) {
            cudaEvent_t e = nullptr;
            SHB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            d.slabReady.push_back(e);
        }
        for(uint32_t s = 0; s < group; s++) {
            uint64_t sendOff[256], sendCnt[256], recvOff[256], recvCnt[256];
            uint64_t so = slabSendBase[s], ro = slabRecvBase[s];
            for(int g = 0; g < W; g++) {
                sendOff[g] = so; sendCnt[g] = mine[size_t(s) * W + g]; so += sendCnt[g];
                recvOff[g] = ro; recvCnt[g] = all[(size_t(g) * group + s) * W + me]; ro += recvCnt[g];
            }
            exchange<uint64_t>(d, d.sendKeys.get(), sendOff, sendCnt, d.recvKeys.get(), recvOff, recvCnt, ncclUint64, cs);
            exchange<uint32_t>(d, d.sendVals.get(), sendOff, sendCnt, d.recvVals.get(), recvOff, recvCnt, ncclUint32, cs);
            SHB_CUDA(cudaEventRecord(d.slabReady[s], cs));
        }
        auto td = std::chrono::steady_clock::now();
        d.timing.exchangeSeconds += seconds(tc, td);
        for(uint32_t s = 0; s < group; s++) {
            SHB_CUDA(cudaStreamWaitEvent(st, d.slabReady[s], 0));
            const uint64_t n = slabRecvBase[s + 1] - slabRecvBase[s];
            d.timing.entriesReceived += n;
            lowhashProcessEntries(c, d.recvKeys.get() + slabRecvBase[s], d.recvVals.get() + slabRecvBase[s], n);
        }
        SHB_CUDA(cudaStreamSynchronize(st));
        d.timing.processSeconds += seconds(td, std::chrono::steady_clock::now());
        iteration += group;
    }
    const auto tFinal = std::chrono::steady_clock::now();

    // Pair counts to the owner of readId0. Owners hold contiguous readId0 ranges (the concatenation of the ranks' candidates
    // stays sorted), but not equal ones: readId0 < readId1 puts most pairs on low read ids, so the ranges are cut on a fine
    // histogram (top bits of readId0, summed over the ranks) into groups of equal pair mass.
    const uint32_t readBits = bitsFor(R ? R - 1 : 0);
    const uint32_t fineBits = std::max<uint32_t>(uint32_t(d.log2World), std::min<uint32_t>(8, readBits));
    const uint32_t pairShift = 32 + (readBits > fineBits ? readBits - fineBits : 0);
    uint64_t* lk = nullptr; uint32_t* lv = nullptr; uint64_t ln = 0;
    lowhashLocalPairs(c, &lk, &lv, &ln);
    uint64_t fine[256];
    uint64_t* pk = nullptr; uint32_t* pv = nullptr;
    devicePartition(c, lk, lv, ln, pairShift, fineBits, fine, &pk, &pv);
    const uint32_t bins = 1u << fineBits;
    d.pairSendKeys.reserve(ln + 1); d.pairSendVals.reserve(ln + 1);
    if(ln) {
        SHB_CUDA(cudaMemcpyAsync(d.pairSendKeys.get(), pk, 8 * ln, cudaMemcpyDeviceToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(d.pairSendVals.get(), pv, 4 * ln, cudaMemcpyDeviceToDevice, st));
    }
    SHB_CUDA(cudaEventRecord(d.computeDone, st));
    SHB_CUDA(cudaStreamWaitEvent(cs, d.computeDone, 0));
    std::vector<unsigned long long> myHist(bins);
    for(uint32_t b = 0; b < bins; b++) myHist[b] = fine[b];
    const std::vector<unsigned long long> allHist = allGatherCounts(c, d, myHist);         // [rank][bin]
    std::vector<double> mass(bins, 0.);
    for(int r = 0; r < W; r++) for(uint32_t b = 0; b < bins; b++) mass[b] += double(allHist[size_t(r) * bins + b]);
    // contiguous bin ranges of (roughly) equal mass: boundary g = first bin whose cumulative mass reaches total * g / W
    std::vector<uint32_t> bound(W + 1, 0);
    {
        double totalMass = 0.;
        for(double m : mass) totalMass += m;
        double running = 0.;
        uint32_t b = 0;
        for(int g = 1; g < W; g++) {
            const double target = totalMass * double(g) / double(W);
            while(b < bins && running < target) running += mass[b++];
            bound[g] = b;
        }
        bound[W] = bins;
        for(int g = 1; g <= W; g++) bound[g] = std::max(bound[g], bound[g - 1]);
    }
    {
        uint64_t sendOff[256], sendCnt[256], recvOff[256], recvCnt[256];
        uint64_t so = 0, ro = 0;
        for(int g = 0; g < W; g++) {
            uint64_t n = 0;
            for(uint32_t b = bound[g]; b < bound[g + 1]; b++) n += fine[b];
            sendOff[g] = so; sendCnt[g] = n; so += n;
            uint64_t rn = 0;
            for(uint32_t b = bound[me]; b < bound[me + 1]; b++) rn += allHist[size_t(g) * bins + b];
            recvOff[g] = ro; recvCnt[g] = rn; ro += rn;
        }
        d.pairRecvKeys.reserve(ro + 1); d.pairRecvVals.reserve(ro + 1);
        exchange<uint64_t>(d, d.pairSendKeys.get(), sendOff, sendCnt, d.pairRecvKeys.get(), recvOff, recvCnt, ncclUint64, cs);
        exchange<uint32_t>(d, d.pairSendVals.get(), sendOff, sendCnt, d.pairRecvVals.get(), recvOff, recvCnt, ncclUint32, cs);
        SHB_CUDA(cudaStreamSynchronize(cs));
        d.timing.pairsReceived = ro;
        lowhashSetPairs(c, d.pairRecvKeys.get(), d.pairRecvVals.get(), ro);
    }
    const uint64_t emitted = lowhashEmitDevice(c);
    // ReadLowHashStatistics: partial sums over the bucket owners.
    SHB_CUDA(cudaEventRecord(d.computeDone, st));
    SHB_CUDA(cudaStreamWaitEvent(cs, d.computeDone, 0));
    SHB_NCCL(nccl().AllReduce(c->stats.get(), c->stats.get(), 3 * R, ncclUint64, ncclSum, d.comm, cs));

    // Even out the slices: rank g ends up with the g-th contiguous block of the concatenation (the order is kept).
    const std::vector<unsigned long long> allEmitted = allGatherCounts(c, d, std::vector<unsigned long long>{emitted});
    uint64_t totalCandidates = 0, myBegin = 0;
    for(int r = 0; r < W; r++) { if(r < me) myBegin += allEmitted[r]; totalCandidates += allEmitted[r]; }
    auto blockBegin = [&](int g) { return totalCandidates * uint64_t(g) / uint64_t(W); };
    const uint64_t outCount = blockBegin(me + 1) - blockBegin(me);
    d.candRecv.reserve(3 * outCount + 3);
    {
        uint64_t sendOff[256], sendCnt[256], recvOff[256], recvCnt[256];
        uint64_t ro = 0;
        for(int g = 0; g < W; g++) {
            // what of my slice [myBegin, myBegin + emitted) falls into block g
            const uint64_t lo = std::min(std::max(blockBegin(g), myBegin), myBegin + emitted);
            const uint64_t hi = std::min(std::max(blockBegin(g + 1), myBegin), myBegin + emitted);
            sendOff[g] = 3 * (lo - myBegin); sendCnt[g] = 3 * (hi - lo);
            // what of rank g's slice falls into my block
            uint64_t gBegin = 0;
            for(int r = 0; r < g; r++) gBegin += allEmitted[r];
            const uint64_t gEnd = gBegin + uint64_t(allEmitted[g]);
            const uint64_t rlo = std::min(std::max(blockBegin(me), gBegin), gEnd);
            const uint64_t rhi = std::min(std::max(blockBegin(me + 1), gBegin), gEnd);
            recvOff[g] = ro; recvCnt[g] = 3 * (rhi - rlo); ro += recvCnt[g];
        }
        exchange<uint32_t>(d, c->candidatesDev.get(), sendOff, sendCnt, d.candRecv.get(), recvOff, recvCnt, ncclUint32, cs);
    }
    HostResult host(allocHostResult(outCount * 12));
    SHB_REQUIRE(host.p != nullptr, SHB_ERR_OOM, "Out of host memory for the alignment candidates.");
    if(outCount) SHB_CUDA(cudaMemcpyAsync(host.p, d.candRecv.get(), outCount * 12, cudaMemcpyDeviceToHost, cs));
    if(statsOut) SHB_CUDA(cudaMemcpyAsync(statsOut, c->stats.get(), 3 * R * sizeof(uint64_t), cudaMemcpyDeviceToHost, cs));
    unsigned long long digest = 0;
    SHB_CUDA(cudaMemcpyAsync(&digest, c->scalar(kSlotCandidateDigest), sizeof(digest), cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaStreamSynchronize(cs));
    total.stop(st);
    SHB_CUDA(cudaStreamSynchronize(st));
    S.candidateDigest = digest;
    lowhashReleaseLargeScratch(c);
    d.timing.finalSeconds = seconds(tFinal, std::chrono::steady_clock::now());
    d.timing.totalSeconds = seconds(t0, std::chrono::steady_clock::now());
    const float totalMs = total.elapsedMs();
    if(result) {
        memset(result, 0, sizeof(*result));
        result->iterations = iteration; result->log2BucketCount = S.log2BucketCount; result->lowHashCount = S.lowHashCount;
        result->pairCount = S.pairCount; result->candidateCount = outCount; result->sweepMs = S.sweepMs; result->totalMs = totalMs;
        result->sweepLaunches = S.sweepLaunches; result->kernelLaunches = g_launchCount;
        result->candidateDigest = digest;          // of the slice this rank EMITTED (the ranks' digests sum to the global one)
    }
    *candidatesOut = host.take();
    *candidateCountOut = outCount;
}

// All reads' k-mer ids on this GPU (second context), gathered once per marker set.
shb_context* gatherMarkers(shb_context* c)
{
    DistState& d = distState(c);
    SHB_REQUIRE(c->haveMarkers, SHB_ERR_STATE, "Markers are not accessible.");
    if(d.alignCtx && d.gatheredGeneration == c->markerGeneration) return d.alignCtx;
    SHB_CUDA(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    cudaStream_t cs = d.commStream;
    const int W = d.world;
    const uint64_t R = c->readCountTotal;
    if(!d.alignCtx) SHB_REQUIRE(shb_context_create(c->device, &d.alignCtx) == SHB_OK, SHB_ERR_CUDA, shb_last_error());
    // sizes: local marker count and local read range of every rank
    const std::vector<unsigned long long> info =
        allGatherCounts(c, d, std::vector<unsigned long long>{c->localMarkerCount, c->readBegin, c->readEnd});
    uint64_t totalMarkers = 0;
    for(int r = 0; r < W; r++) {
        totalMarkers += info[3 * r];
        SHB_REQUIRE(info[3 * r + 1] == (r ? info[3 * (r - 1) + 2] : 0ull), SHB_ERR_INVALID, "The ranks' read ranges are not contiguous in rank order.");
    }
    SHB_REQUIRE(info[3 * (W - 1) + 2] == R, SHB_ERR_INVALID, "The ranks' read ranges do not cover all reads.");
    d.gathered.reserve(totalMarkers + 64);
    d.tocStage.reserve(2 * R + 2);
    SHB_CUDA(cudaStreamSynchronize(c->stream));
    // k-mer ids and relative tocs, rank after rank (variable sizes: one broadcast per source, grouped)
    SHB_NCCL(nccl().GroupStart());
    uint64_t markerOffset = 0;
    for(int r = 0; r < W; r++) {
        const uint64_t n = info[3 * r], rows = 2 * (info[3 * r + 2] - info[3 * r + 1]);
        if(n) SHB_NCCL(nccl().Broadcast(c->kmerIds, d.gathered.get() + markerOffset, n, ncclUint32, r, d.comm, cs));
        // toc rows of rank r go to tocStage[2*readBegin_r + 1 ...] (relative to rank r's first marker; rebased on the host)
        if(rows) SHB_NCCL(nccl().Broadcast(c->toc.get() + 1, d.tocStage.get() + 2 * info[3 * r + 1] + 1, rows, ncclUint64, r, d.comm, cs));
        markerOffset += n;
    }
    SHB_NCCL(nccl().GroupEnd());
    std::vector<uint64_t> toc(2 * R + 1, 0);
    if(R) SHB_CUDA(cudaMemcpyAsync(toc.data() + 1, d.tocStage.get() + 1, 2 * R * sizeof(uint64_t), cudaMemcpyDeviceToHost, cs));
    SHB_CUDA(cudaStreamSynchronize(cs));
    markerOffset = 0;
    for(int r = 0; r < W; r++) {
        for(uint64_t row = 2 * info[3 * r + 1] + 1; row <= 2 * info[3 * r + 2]; row++) toc[row] += markerOffset;
        markerOffset += info[3 * r];
    }
    SHB_REQUIRE(shb_set_markers_device(d.alignCtx, R, 0, R, toc.data(), d.gathered.get(), c->readFlagsHost.data(), totalMarkers) == SHB_OK,
                SHB_ERR_CUDA, shb_last_error());
    d.gatheredGeneration = c->markerGeneration;
    d.timing.gatherSeconds = seconds(t0, std::chrono::steady_clock::now());
    return d.alignCtx;
}

} // namespace shb

using namespace shb;

namespace shb {
template<class F> shb_status guardedDist(F&& f)
{
    try { f(); return SHB_OK; }
    catch(const Error& e) { setLastError(e.what()); return e.status; }
    catch(const std::exception& e) { setLastError(e.what()); return SHB_ERR_INVALID; }
}
}

extern "C" {

shb_status shb_dist_unique_id(void* id128)
{
    return guardedDist([&] {
        SHB_REQUIRE(id128 != nullptr, SHB_ERR_INVALID, "Null argument.");
        static_assert(sizeof(ncclUniqueId) == SHB_DIST_UNIQUE_ID_BYTES, "ncclUniqueId is 128 bytes");
        ncclUniqueId id;
        SHB_NCCL(nccl().GetUniqueId(&id));
        memcpy(id128, &id, sizeof(id));
    });
}

shb_status shb_dist_init(shb_context* c, int world, int rank, const void* id128)
{
    return guardedDist([&] {
        SHB_REQUIRE(c && id128, SHB_ERR_INVALID, "Null argument.");
        SHB_CUDA(cudaSetDevice(c->device));
        ncclUniqueId id;
        memcpy(&id, id128, sizeof(id));
        ncclComm_t comm = nullptr;
        SHB_NCCL(nccl().CommInitRank(&comm, world, id, rank));
        attach(c, comm, true, world, rank);
    });
}

shb_status shb_dist_attach(shb_context* c, void* ncclComm, int world, int rank)
{
    return guardedDist([&] {
        SHB_REQUIRE(c && ncclComm, SHB_ERR_INVALID, "Null argument.");
        nccl();
        attach(c, static_cast<ncclComm_t>(ncclComm), false, world, rank);
    });
}

void shb_dist_finalize(shb_context* c)
{
    if(!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    destroyDistState(c);
}

shb_status shb_lowhash0_sharded(shb_context* c, const shb_lowhash_params* params, void** candidates, uint64_t* candidateCount,
                                uint64_t* stats, shb_lowhash_result* result)
{
    return guardedDist([&] {
        SHB_REQUIRE(c && params && candidates && candidateCount, SHB_ERR_INVALID, "Null argument.");
        lowhash0Sharded(c, *params, candidates, candidateCount, stats, result);
    });
}

shb_status shb_compute_alignments_sharded(shb_context* c, const void* candidates, uint64_t candidateCount,
                                          const shb_align_options* options, void** alignmentData, uint64_t* alignmentCount,
                                          uint64_t** compressedToc, uint8_t** compressedData, shb_align_result* result)
{
    return guardedDist([&] {
        SHB_REQUIRE(c && options && alignmentData && alignmentCount && compressedToc && compressedData, SHB_ERR_INVALID, "Null argument.");
        shb_context* a = gatherMarkers(c);
        computeAlignments(a, candidates, candidateCount, *options, alignmentData, alignmentCount, compressedToc, compressedData, result, false);
    });
}

shb_status shb_dist_timing_get(shb_context* c, shb_dist_timing* timing)
{
    return guardedDist([&] {
        SHB_REQUIRE(c && timing, SHB_ERR_INVALID, "Null argument.");
        *timing = distState(c).timing;
    });
}

} // extern "C"
