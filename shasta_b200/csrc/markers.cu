// MarkerFinder on the GPU (SURVEY.md section 8f, rank 1): src/MarkerFinder.cpp:16-127 of chanzuckerberg/shasta.
// Input: the run-length encoded reads exactly as the reference stores them (LongBaseSequences, src/LongBaseSequence.hpp:33-41:
// per read two uint64 words per 64 bases, low bit plane then high bit plane, base 0 in the most significant bit) and the
// marker k-mer table (only KmerInfo::isMarker is read, src/Kmer.hpp:23-38). Output: the markers of both strands
// (src/MarkerFinder.cpp:92-100: strand 1 = reversed order, reverse-complemented k-mers, position baseCount - k - position)
// as the resident uint32 k-mer id SoA the rest of the path works on, and on request the 7-byte CompressedMarker records
// + toc for Data/Markers. The reads cross PCIe as 2 bits per base instead of 7 bytes per marker and strand.
//
//   markerMaskKernel   one thread per 64-base block: the k-mer id of each of its positions (two funnel shifts over the bit
//                      planes: id = (highPlaneBits << k) | lowPlaneBits, src/ShortBaseSequence.hpp:92-107), one bit-test in
//                      the 4^k-bit isMarker bitmap (L2 resident: 32 MB for k = 14), a 64-bit mask and its population count;
//   (exclusive scan of the counts over the blocks)
//   markerWriteKernel  one thread per block again: expands the mask into both strands' rows.
#include "context.cuh"
#include "hostpool.cuh"

#include <cstring>
#include <vector>

namespace shb {

extern thread_local uint64_t g_launchCount;

namespace {

// The read a 64-base block belongs to: largest r with blockStart[r] <= g (blockStart = word offsets / 2).
__device__ __forceinline__ uint32_t readOfBlock(const uint64_t* __restrict__ wordOffsets, uint32_t readCount, uint64_t g)
{
    uint32_t lo = 0, hi = readCount;
    while(hi - lo > 1) {
        const uint32_t mid = lo + ((hi - lo) >> 1);
        if((wordOffsets[mid] >> 1) <= g) lo = mid; else hi = mid;
    }
    return lo;
}

// k consecutive bits of a bit plane starting at base `offset` of the block (base 0 = most significant bit), continuing
// into the next block's word when they straddle.
__device__ __forceinline__ uint32_t planeBits(uint64_t w, uint64_t next, uint32_t offset, uint32_t k)
{
    uint64_t v = w << offset;
    if(offset) v |= next >> (64u - offset);
    return uint32_t(v >> (64u - k));
}

struct MarkerArgs {
    const uint64_t* words;          // all reads' bit-plane words
    const uint64_t* wordOffsets;    // [readCount + 1], in words
    const uint64_t* baseCounts;     // [readCount]
    const uint32_t* isMarkerBits;   // 4^k bits
    uint32_t readCount, k;
    uint64_t blockCount;            // total 64-base blocks = wordOffsets[readCount] / 2
};

__global__ void markerMaskKernel(MarkerArgs a, unsigned long long* __restrict__ masks, uint32_t* __restrict__ counts)
{
    const uint64_t g = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if(g >= a.blockCount) return;
    const uint32_t r = readOfBlock(a.wordOffsets, a.readCount, g);
    const uint64_t firstBlock = a.wordOffsets[r] >> 1, endBlock = a.wordOffsets[r + 1] >> 1;
    const uint64_t baseCount = a.baseCounts[r];
    const uint64_t base0 = (g - firstBlock) * 64;            // position of the block's first base in the read
    const uint64_t lowW = a.words[2 * g], highW = a.words[2 * g + 1];
    const bool hasNext = g + 1 < endBlock;
    const uint64_t lowN = hasNext ? a.words[2 * g + 2] : 0ull, highN = hasNext ? a.words[2 * g + 3] : 0ull;
    unsigned long long mask = 0;
    if(baseCount >= a.k) {                                   // "avoid pathological case", src/MarkerFinder.cpp:78
        const uint64_t lastPosition = baseCount - a.k;      // last position that starts a k-mer
        for(uint32_t o = 0; o < 64 && base0 + o <= lastPosition; o++) {
            const uint32_t kmerId = (planeBits(highW, highN, o, a.k) << a.k) | planeBits(lowW, lowN, o, a.k);
            if((a.isMarkerBits[kmerId >> 5] >> (kmerId & 31u)) & 1u) mask |= 1ull << o;
        }
    }
    masks[g] = mask;
    counts[g] = uint32_t(__popcll(mask));
}

// markerBefore[g] = exclusive scan of counts (markers of strand 0 before block g, over all reads).
__global__ void markerWriteKernel(MarkerArgs a, const unsigned long long* __restrict__ masks, const unsigned long long* __restrict__ markerBefore,
                                  unsigned long long totalMarkersOneStrand, uint32_t* __restrict__ kmerIds /* both strands */,
                                  uint8_t* __restrict__ data7 /* may be null */, unsigned long long* __restrict__ toc /* 2R+1 */)
{
    const uint64_t g = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if(g >= a.blockCount) return;
    const uint32_t r = readOfBlock(a.wordOffsets, a.readCount, g);
    const uint64_t firstBlock = a.wordOffsets[r] >> 1, endBlock = a.wordOffsets[r + 1] >> 1;
    const uint64_t readBefore = markerBefore[firstBlock];                                       // strand-0 markers of earlier reads
    const uint64_t readCountMarkers = ((endBlock < a.blockCount) ? markerBefore[endBlock] : totalMarkersOneStrand) - readBefore;
    const uint64_t row0 = 2 * readBefore, row1 = row0 + readCountMarkers;                      // both strands of a read are adjacent rows
    if(g == firstBlock) {
        toc[2ull * r] = row0; toc[2ull * r + 1] = row1;
        if(r + 1 == a.readCount) toc[2ull * a.readCount] = 2 * totalMarkersOneStrand;
    }
    unsigned long long mask = masks[g];
    if(!mask) return;
    const uint64_t baseCount = a.baseCounts[r];
    const uint64_t base0 = (g - firstBlock) * 64;
    const uint64_t lowW = a.words[2 * g], highW = a.words[2 * g + 1];
    const bool hasNext = g + 1 < endBlock;
    const uint64_t lowN = hasNext ? a.words[2 * g + 2] : 0ull, highN = hasNext ? a.words[2 * g + 3] : 0ull;
    uint64_t ordinal = markerBefore[g] - readBefore;          // ordinal of the block's first marker in strand 0
    while(mask) {
        const uint32_t o = uint32_t(__ffsll((long long)mask)) - 1u;
        mask &= mask - 1ull;
        const uint32_t kmerId = (planeBits(highW, highN, o, a.k) << a.k) | planeBits(lowW, lowN, o, a.k);
        const uint32_t position = uint32_t(base0 + o);
        const uint64_t i0 = row0 + ordinal, i1 = row1 + (readCountMarkers - 1 - ordinal);
        const uint32_t rc = reverseComplementKmer(kmerId, a.k);
        const uint32_t position1 = uint32_t(baseCount - a.k - position);
        kmerIds[i0] = kmerId;
        kmerIds[i1] = rc;
        if(data7) {
            uint8_t* p0 = data7 + 7 * i0; uint8_t* p1 = data7 + 7 * i1;
            p0[0] = uint8_t(kmerId); p0[1] = uint8_t(kmerId >> 8); p0[2] = uint8_t(kmerId >> 16); p0[3] = uint8_t(kmerId >> 24);
            p0[4] = uint8_t(position); p0[5] = uint8_t(position >> 8); p0[6] = uint8_t(position >> 16);
            p1[0] = uint8_t(rc); p1[1] = uint8_t(rc >> 8); p1[2] = uint8_t(rc >> 16); p1[3] = uint8_t(rc >> 24);
            p1[4] = uint8_t(position1); p1[5] = uint8_t(position1 >> 8); p1[6] = uint8_t(position1 >> 16);
        }
        ordinal++;
    }
}

} // namespace

// The markers of reads [0, readCount) become the context's resident marker set (as after shb_set_markers with all reads on
// this GPU). tocOut / data7Out: optional host copies (shb_free).
void findMarkers(shb_context* c, uint32_t k, uint64_t readCount, const uint64_t* wordOffsets, const uint64_t* words,
                 const uint64_t* baseCounts, const uint8_t* kmerTable24, const uint32_t* isMarkerBitmap,
                 const uint8_t* readFlags, uint64_t** tocOut, uint8_t** data7Out, shb_marker_result* result)
{
    SHB_REQUIRE(k >= 1 && k <= 16, SHB_ERR_INVALID, "Invalid k.");
    SHB_REQUIRE(readCount < (1ull << 31), SHB_ERR_INVALID, "Too many reads.");
    SHB_REQUIRE(wordOffsets && baseCounts && (words || wordOffsets[readCount] == 0) && (kmerTable24 || isMarkerBitmap) && (readFlags || readCount == 0),
                SHB_ERR_INVALID, "Null argument.");
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    g_launchCount = 0;
    const uint64_t wordCount = wordOffsets[readCount];
    for(uint64_t r = 0; r < readCount; r++) {
        const uint64_t need = baseCounts[r] ? 2 * (((baseCounts[r] - 1) >> 6) + 1) : 0;         // LongBaseSequenceView::wordCount
        SHB_REQUIRE(wordOffsets[r + 1] - wordOffsets[r] == need, SHB_ERR_INVALID, "Read words and base counts are inconsistent.");
        SHB_REQUIRE(baseCounts[r] < (1ull << 24), SHB_ERR_INVALID, "A read has 2^24 or more bases (marker positions are 24 bits, src/Marker.hpp:62-64).");
    }
    const uint64_t blockCount = wordCount / 2;
    EventTimer timer;
    timer.start(st);

    // isMarker bitmap: 4^k bits
    const uint64_t kmerCount = 1ull << (2 * k);
    const uint64_t bitmapWords = (kmerCount + 31) / 32;
    std::vector<uint32_t> bitmapHost;
    if(!isMarkerBitmap) {
        bitmapHost.assign(bitmapWords, 0u);
        for(uint64_t i = 0; i < kmerCount; i++) if(kmerTable24[24 * i + 12]) bitmapHost[i >> 5] |= 1u << (i & 31);    // KmerInfo::isMarker
        isMarkerBitmap = bitmapHost.data();
    }
    DeviceBuffer<uint32_t> dBitmap, dCounts;
    DeviceBuffer<uint64_t> dWords, dOffsets, dBaseCounts;
    DeviceBuffer<unsigned long long> dMasks, dBefore, dCounts64, dScanWs, dToc;
    dBitmap.reserve(bitmapWords); dWords.reserve(wordCount + 4); dOffsets.reserve(readCount + 1); dBaseCounts.reserve(readCount + 1);
    dMasks.reserve(blockCount + 1); dCounts.reserve(blockCount + 1); dCounts64.reserve(blockCount + 1); dBefore.reserve(blockCount + 1);
    dScanWs.reserve(scanWorkspaceElements(blockCount + 1)); dToc.reserve(2 * readCount + 1);
    SHB_CUDA(cudaMemcpyAsync(dBitmap.get(), isMarkerBitmap, bitmapWords * 4, cudaMemcpyHostToDevice, st));
    if(wordCount) SHB_CUDA(cudaMemcpyAsync(dWords.get(), words, wordCount * 8, cudaMemcpyHostToDevice, st));
    SHB_CUDA(cudaMemcpyAsync(dOffsets.get(), wordOffsets, (readCount + 1) * 8, cudaMemcpyHostToDevice, st));
    if(readCount) SHB_CUDA(cudaMemcpyAsync(dBaseCounts.get(), baseCounts, readCount * 8, cudaMemcpyHostToDevice, st));

    MarkerArgs a;
    a.words = dWords.get(); a.wordOffsets = dOffsets.get(); a.baseCounts = dBaseCounts.get(); a.isMarkerBits = dBitmap.get();
    a.readCount = uint32_t(readCount); a.k = k; a.blockCount = blockCount;
    unsigned long long* totalDev = c->scalar(kSlotMarkerTotal);
    SHB_CUDA(cudaMemsetAsync(totalDev, 0, sizeof(unsigned long long), st));
    if(blockCount) {
        SHB_LAUNCH(markerMaskKernel, ceilDiv(blockCount, 128), 128, 0, st, a, dMasks.get(), dCounts.get());
        SHB_LAUNCH(widenKernel<uint64_t>, ceilDiv(blockCount, 256), 256, 0, st, (const uint32_t*)dCounts.get(), blockCount, dCounts64.get());
        exclusiveScan<unsigned long long>(dCounts64.get(), dBefore.get(), blockCount, totalDev, dScanWs.get(), st);
    }
    const unsigned long long totalOneStrand = readBack(totalDev, st);
    const uint64_t M = 2 * totalOneStrand;

    c->haveMarkers = false;
    c->kmerIdsOwned.reserve(M + 64);
    DeviceBuffer<uint8_t> dData7;
    if(data7Out) dData7.reserve(7 * M + 16);
    if(readCount == 0) SHB_CUDA(cudaMemsetAsync(dToc.get(), 0, sizeof(unsigned long long), st));
    if(blockCount) {
        SHB_LAUNCH(markerWriteKernel, ceilDiv(blockCount, 128), 128, 0, st, a, (const unsigned long long*)dMasks.get(),
                   (const unsigned long long*)dBefore.get(), totalOneStrand, c->kmerIdsOwned.get(), data7Out ? dData7.get() : (uint8_t*)nullptr,
                   dToc.get());
    }
    // Reads without a single 64-base block (baseCount 0) own no thread: their toc entries are filled on the host below.
    std::vector<uint64_t> toc(2 * readCount + 1, 0);
    SHB_CUDA(cudaMemcpyAsync(toc.data(), dToc.get(), (2 * readCount + 1) * 8, cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaStreamSynchronize(st));
    toc[2 * readCount] = M;
    for(uint64_t r = readCount; r-- > 0; ) {
        if(wordOffsets[r + 1] == wordOffsets[r]) { toc[2 * r] = toc[2 * r + 2]; toc[2 * r + 1] = toc[2 * r + 2]; }
    }
    HostResult tocHost(tocOut ? allocHostResult(8 * (2 * readCount + 1)) : nullptr), dataHost(data7Out ? allocHostResult(7 * M + 8) : nullptr);
    if(tocOut) { SHB_REQUIRE(tocHost.p, SHB_ERR_OOM, "Out of host memory for the marker toc."); memcpy(tocHost.p, toc.data(), 8 * (2 * readCount + 1)); }
    if(data7Out) {
        SHB_REQUIRE(dataHost.p, SHB_ERR_OOM, "Out of host memory for the markers.");
        if(M) SHB_CUDA(cudaMemcpyAsync(dataHost.p, dData7.get(), 7 * M, cudaMemcpyDeviceToHost, st));
    }
    // Install as the context's marker set (all reads on this GPU).
    c->markerGeneration++;
    c->readCountTotal = readCount; c->readBegin = 0; c->readEnd = readCount;
    c->totalMarkerCount = M; c->localMarkerCount = M;
    c->tocHost = toc;
    c->readFlagsHost.assign(readFlags, readFlags + readCount);
    c->toc.reserve(2 * readCount + 1);
    c->readFlags.reserve(readCount + 1);
    SHB_CUDA(cudaMemcpyAsync(c->toc.get(), toc.data(), (2 * readCount + 1) * 8, cudaMemcpyHostToDevice, st));
    if(readCount) SHB_CUDA(cudaMemcpyAsync(c->readFlags.get(), readFlags, readCount, cudaMemcpyHostToDevice, st));
    timer.stop(st);
    SHB_CUDA(cudaStreamSynchronize(st));
    c->kmerIds = c->kmerIdsOwned.get();
    c->haveMarkers = true;
    const float ms = timer.elapsedMs();
    if(result) {
        result->readCount = readCount; result->baseCount = 0;
        for(uint64_t r = 0; r < readCount; r++) result->baseCount += baseCounts[r];
        result->markerCount = M; result->totalMs = ms; result->kernelLaunches = g_launchCount;
        result->h2dBytes = wordCount * 8 + bitmapWords * 4 + (readCount + 1) * 8 + readCount * 9;
    }
    if(tocOut) *tocOut = static_cast<uint64_t*>(tocHost.take());
    if(data7Out) *data7Out = static_cast<uint8_t*>(dataHost.take());
}

} // namespace shb
