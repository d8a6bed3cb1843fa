// LowHash0 device kernels (sm_90a). Reference: src/LowHash0.cpp (chanzuckerberg/shasta).
//   extractKmerIdsKernel    <- LowHash0::createKmerIds            src/LowHash0.cpp:261-308
//   lowhashSweepKernel      <- LowHash0::pass1ThreadFunction       src/LowHash0.cpp:314-360
//                              + MurmurHash64A                     src/MurmurHash2.cpp:96-137
//   bucket*Kernel           <- pass2 / pass3                       src/LowHash0.cpp:365-484
//   candidate kernels       <- merge + final emission              src/LowHash0.cpp:204-214, 493-562
#pragma once

#include "common.cuh"
#include "context.cuh"

namespace shb {

// ---------------------------------------------------------------------------------------------
// a4. 7-byte CompressedMarker AoS -> uint32 kmerId SoA.
// The byte stream is read as aligned 32-bit words (coalesced), staged in shared memory, and each
// k-mer id is re-assembled with a funnel shift. One block converts 1024 markers (7168 bytes).
constexpr int kExtractThreads = 256;
constexpr int kExtractMarkersPerBlock = 1024;

static __global__ void __launch_bounds__(kExtractThreads)
extractKmerIdsKernel(const uint32_t* __restrict__ words, uint64_t wordCount, uint64_t markerCount,
                     uint32_t* __restrict__ kmerIds)
{
    constexpr int kWords = kExtractMarkersPerBlock * 7 / 4;          // 1792
    __shared__ uint32_t sm[kWords + 1];
    const uint64_t wordBase = uint64_t(blockIdx.x) * kWords;
    for(int w = threadIdx.x; w < kWords + 1; w += kExtractThreads) {
        const uint64_t gw = wordBase + w;
        sm[w] = (gw < wordCount) ? words[gw] : 0u;
    }
    __syncthreads();
    const uint64_t markerBase = uint64_t(blockIdx.x) * kExtractMarkersPerBlock;
#pragma unroll
    for(int i = 0; i < kExtractMarkersPerBlock / kExtractThreads; i++) {
        const int local = i * kExtractThreads + threadIdx.x;
        const uint64_t g = markerBase + local;
        if(g < markerCount) {
            const int byteOffset = local * 7;
            const int w = byteOffset >> 2;
            const int shift = (byteOffset & 3) * 8;
            kmerIds[g] = __funnelshift_r(sm[w], sm[w + 1], shift);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// a5. Hash sweep. Every marker position p is treated as the start of a feature (m consecutive
// k-mer ids = 4m bytes); MurmurHash64A of the feature is evaluated for up to kMaxFusedIterations
// seeds (= LowHash iterations, seed = 37*iteration) per pass over the k-mer ids: the per-block
// mixing of the 64-bit words does not depend on the seed, so K iterations cost one read of the
// k-mer ids and (m/2)*2 + 3K 64-bit multiplies per feature instead of K*(m+3).
// Only hashes below the threshold (about hashFraction of them) look up which oriented read they
// belong to (binary search in the toc) and whether the feature lies inside one non-palindromic read.
constexpr int kSweepThreads = 256;
constexpr int kSweepPositionsPerThread = 8;
constexpr int kSweepTile = kSweepThreads * kSweepPositionsPerThread;      // 2048 positions per block
// Low hashes queued per block before the (slow) inline path: sized by the host from the expected 2048 * K * hashFraction
// (205 for K = 10 and hashFraction 0.01; 1640 for K = 16 and the HiFi configuration's 0.05) with 50 % slack.
constexpr uint32_t kSweepQueueMin = 256, kSweepQueueMax = 6144;
constexpr int kMaxTemplatedM = 8;
constexpr int kSweepTileReads = 32;                   // toc entries staged per tile (more reads than that: global binary search)

struct SweepArgs {
    const uint32_t* kmerIds;        // local k-mer ids
    uint64_t markerCount;           // local marker count
    const uint64_t* toc;            // local toc, relative, orientedReadCount+1 entries
    uint32_t orientedReadCount;     // local oriented reads
    uint32_t orientedReadBase;      // global id of local oriented read 0
    const uint8_t* readFlags;       // global, indexed by global readId
    uint32_t m;
    uint64_t hashThreshold;
    uint64_t bucketMask;
    uint32_t iterationBegin;
    uint32_t iterationCount;        // <= kMaxFusedIterations
    uint64_t* keys;                 // iterationCount slabs of `capacity` entries
    uint32_t* vals;
    uint64_t capacity;
    unsigned long long* counts;     // [iterationCount]
    uint32_t queueCapacity;         // entries of the shared-memory low-hash queue (16 bytes each, dynamic shared memory)
    const uint32_t* tileFirstRead;  // per tile: largest local oriented read r with toc[r] <= first position of the tile
    uint32_t seeds[kMaxFusedIterations];    // MurmurHash seed of every fused iteration, (iterationBegin + s) * 37: read straight
                                            // from the constant bank by the hot loop's xor
};

// tileFirstRead[t] for every sweep tile (built once per marker set).
static __global__ void sweepTileReadsKernel(const uint64_t* __restrict__ toc, uint32_t orientedReadCount, uint32_t tileCount,
                                            uint32_t* __restrict__ tileFirstRead);

// 64-bit values as two 32-bit halves: the hash is pure 32-bit integer work on this machine, and keeping the halves apart
// stops the compiler from routing them through 64-bit adds with carry chains.
struct U64Halves { uint32_t lo, hi; };
__device__ __forceinline__ U64Halves halves(uint64_t x) { return U64Halves{uint32_t(x), uint32_t(x >> 32)}; }
__device__ __forceinline__ uint64_t whole(U64Halves x) { return (uint64_t(x.hi) << 32) | x.lo; }

// x * 0xc6a4a7935bd1e995 (mod 2^64): one wide multiply and two multiply-adds into the high word.
__device__ __forceinline__ U64Halves mulM(U64Halves x)
{
    U64Halves r;
    asm("{\n\t.reg .u64 w;\n\tmul.wide.u32 w, %2, 0x5bd1e995;\n\tmov.b64 {%0, %1}, w;\n\t"
        "mad.lo.u32 %1, %2, 0xc6a4a793, %1;\n\tmad.lo.u32 %1, %3, 0x5bd1e995, %1;\n\t}"
        : "=&r"(r.lo), "=&r"(r.hi) : "r"(x.lo), "r"(x.hi));       // early clobber: x.lo is read again after r.lo is written
    return r;
}
__device__ __forceinline__ uint64_t mulM(uint64_t x) { return whole(mulM(halves(x))); }

__device__ __forceinline__ uint64_t murmurMix(uint64_t k)
{
    U64Halves h = mulM(halves(k));
    h.lo ^= h.hi >> 15;                 // k ^= k >> 47
    return whole(mulM(h));
}

// MurmurHash64A of one feature for one seed, given the seed-independent mixed blocks and tail, up to but NOT including
// the final `h ^= h >> 47`: that last step only touches the low 17 bits, so the high word — all the threshold test of the
// hot loop looks at — is already final. h0 = (seed ^ len*M) ^ mixed[0] when the feature has at least one block.
template<int MM> __device__ __forceinline__ U64Halves murmurAlmost(U64Halves h, const uint64_t* mixed, uint32_t blocks, bool hasTail, uint64_t tail)
{
    if(MM >= 2) {
        h = mulM(h);
#pragma unroll
        for(int b = 1; b < MM / 2; b++) { h.lo ^= uint32_t(mixed[b]); h.hi ^= uint32_t(mixed[b] >> 32); h = mulM(h); }
    } else if(MM == 0) {
        if(blocks) {
            h = mulM(h);
            for(uint32_t b = 1; b < blocks; b++) { h.lo ^= uint32_t(mixed[b]); h.hi ^= uint32_t(mixed[b] >> 32); h = mulM(h); }
        }
    }
    if(hasTail) { h.lo ^= uint32_t(tail); h.hi ^= uint32_t(tail >> 32); h = mulM(h); }
    h.lo ^= h.hi >> 15;                 // h ^= h >> 47
    h = mulM(h);
    return h;
}

// The complete MurmurHash64A of the feature of m k-mer ids at w (src/MurmurHash2.cpp:96-140 on 4*m bytes), seed < 2^32.
template<int MM> __device__ __forceinline__ uint64_t featureHash(const uint32_t* w, uint32_t m, uint32_t seed, uint64_t lenTimesM)
{
    const uint32_t blocks = (MM > 0) ? uint32_t(MM / 2) : (m >> 1);
    U64Halves h = halves(lenTimesM);
    h.lo ^= seed;
    for(uint32_t b = 0; b < blocks; b++) {
        const U64Halves k = halves(murmurMix(uint64_t(w[2*b]) | (uint64_t(w[2*b + 1]) << 32)));
        h.lo ^= k.lo; h.hi ^= k.hi;
        h = mulM(h);
    }
    if(m & 1u) { h.lo ^= w[m - 1]; h = mulM(h); }
    h.lo ^= h.hi >> 15;
    h = mulM(h);
    h.lo ^= h.hi >> 15;
    return whole(h);
}

static __global__ void sweepTileReadsKernel(const uint64_t* __restrict__ toc, uint32_t orientedReadCount, uint32_t tileCount,
                                            uint32_t* __restrict__ tileFirstRead)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if(t >= tileCount) return;
    tileFirstRead[t] = rowOf(toc, 0u, orientedReadCount, uint64_t(t) * kSweepTile);         // toc[0] = 0
}

// Which oriented read does marker position p belong to, and is the feature starting at p valid
// (inside one read, read not palindromic: src/LowHash0.cpp:325,337,344)? Returns the LOCAL
// oriented read index or 0xffffffff.
__device__ __forceinline__ uint32_t resolveFeature(const SweepArgs& a, uint64_t p, uint32_t m)
{
    const uint32_t lo = rowOf(a.toc, 0u, a.orientedReadCount, p);
    const bool inside = (p + m <= a.toc[lo + 1]);
    const bool palindromic = (a.readFlags[(a.orientedReadBase + lo) >> 1] & 1u) != 0;
    return (inside && !palindromic) ? lo : 0xffffffffu;
}

// The hot loop hashes every position for every seed of the launch and tests only the HIGH word of the hash against the
// threshold (one compare), collecting the (position, seed) pairs that pass (about hashFraction of them) in bit masks. They
// are queued in shared memory once per tile; all the work on them (complete hash, exact test, toc binary search, validity,
// output slot) is done afterwards by all threads of the block over the queue, one entry per lane, so a warp never
// serialises behind one lane's rare path.
// KK > 0: the number of fused iterations is a compile-time constant (fully unrolled seed loop); KK == 0: a.iterationCount.
constexpr int kSweepTilesPerBlock = 4;      // consecutive tiles per block: the next tile streams into shared memory (cp.async)
                                            // while the current one is hashed

__device__ __forceinline__ void cpAsync16(void* smemDst, const void* globalSrc)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(uint32_t(__cvta_generic_to_shared(smemDst))), "l"(globalSrc) : "memory");
}
__device__ __forceinline__ void cpAsyncCommitAndWaitNone() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cpAsyncWaitAll() { asm volatile("cp.async.wait_all;" ::: "memory"); }

template<int MM, int KK> __global__ void __launch_bounds__(kSweepThreads)
lowhashSweepKernel(const SweepArgs a)
{
    constexpr int kHalo = 2 * kMaxFusedIterations;       // >= any supported m (generic path caps m at 32)
    __shared__ __align__(16) uint32_t skBuf[2][kSweepTile + kHalo];
    extern __shared__ uint64_t queueHash[];              // a.queueCapacity low hashes queued per block, then per entry:
    uint32_t* queueMeta = reinterpret_cast<uint32_t*>(queueHash + a.queueCapacity);   // in: local | s<<16   out: rank within (block, seed) | s<<24, or ~0
    uint32_t* queueRead = queueMeta + a.queueCapacity;                               // oriented read (global)
    __shared__ uint32_t queueCountBuf[2];
    __shared__ unsigned long long tileTocBuf[2][kSweepTileReads + 1];      // toc[tileFirstRead + k]
    __shared__ uint32_t tileFirstReadBuf[2];
    __shared__ uint32_t seedCountBuf[2][kMaxFusedIterations];
    __shared__ unsigned long long seedBase[kMaxFusedIterations];

    const uint64_t M = 0xc6a4a7935bd1e995ull;
    const uint32_t m = (MM > 0) ? uint32_t(MM) : a.m;
    const uint32_t tileCount = uint32_t((a.markerCount + kSweepTile - 1) / kSweepTile);
    const uint32_t firstTile = blockIdx.x * kSweepTilesPerBlock;
    const uint32_t lastTile = min(firstTile + uint32_t(kSweepTilesPerBlock), tileCount);
    const uint32_t K = (KK > 0) ? uint32_t(KK) : a.iterationCount;
    const uint64_t lenTimesM = uint64_t(4u * m) * M;
    const uint64_t threshold = a.hashThreshold;
    const uint32_t thresholdHigh = uint32_t(threshold >> 32);
    const uint32_t seed0 = a.iterationBegin * 37u;                    // iteration * 37 fits 32 bits

    // Streams tile t into buffer `buf`: full, 16-byte aligned tiles with cp.async (no registers, no wait here); the last or
    // a misaligned tile with plain loads. Also stages the toc entries of the reads that cover the tile: a tile of 2048
    // positions spans a few reads, so the oriented read of a queued position is found in a shared-memory copy of the toc
    // entries from the tile's first read on (the first read of every tile comes from a table built once per marker set)
    // instead of a 21-step binary search in global memory per low hash.
    auto prefetchTile = [&](uint32_t t, int buf) {
        const uint64_t base = uint64_t(t) * kSweepTile;
        uint32_t* dst = skBuf[buf];
        if(base + kSweepTile <= a.markerCount && (reinterpret_cast<uintptr_t>(a.kmerIds + base) & 15u) == 0) {
            const uint4* src = reinterpret_cast<const uint4*>(a.kmerIds + base);
            cpAsync16(reinterpret_cast<uint4*>(dst) + threadIdx.x, src + threadIdx.x);
            cpAsync16(reinterpret_cast<uint4*>(dst) + threadIdx.x + kSweepThreads, src + threadIdx.x + kSweepThreads);
            if(threadIdx.x < kHalo) { const uint64_t g = base + kSweepTile + threadIdx.x; dst[kSweepTile + threadIdx.x] = (g < a.markerCount) ? a.kmerIds[g] : 0u; }
        } else {
            for(int i = threadIdx.x; i < kSweepTile + kHalo; i += kSweepThreads) {
                const uint64_t g = base + i;
                dst[i] = (g < a.markerCount) ? a.kmerIds[g] : 0u;
            }
        }
        cpAsyncCommitAndWaitNone();
        if(threadIdx.x >= kSweepThreads - 32) {          // the last warp (the first ones own the halo loads)
            const unsigned lane = threadIdx.x & 31u;
            const uint32_t lo = a.tileFirstRead[t];
            tileTocBuf[buf][lane] = a.toc[min(lo + lane, a.orientedReadCount)];
            if(lane == 0) { tileTocBuf[buf][kSweepTileReads] = a.toc[min(lo + uint32_t(kSweepTileReads), a.orientedReadCount)]; tileFirstReadBuf[buf] = lo; }
        }
    };

    if(threadIdx.x < 2 * kMaxFusedIterations) (&seedCountBuf[0][0])[threadIdx.x] = 0;
    if(threadIdx.x < 2) queueCountBuf[threadIdx.x] = 0;
    if(firstTile < lastTile) prefetchTile(firstTile, 0);

    for(uint32_t tile = firstTile; tile < lastTile; tile++) {
    const int cur = int(tile - firstTile) & 1;
    cpAsyncWaitAll();
    __syncthreads();            // tile `tile` is in skBuf[cur]; everybody is done with the previous tile (buffer cur ^ 1, the queue)
    if(tile + 1 < lastTile) prefetchTile(tile + 1, cur ^ 1);
    if(tile != firstTile) {     // counters of the other parity: last used by the previous tile, next used by the next one
        if(threadIdx.x < kMaxFusedIterations) seedCountBuf[cur ^ 1][threadIdx.x] = 0;
        if(threadIdx.x == 0) queueCountBuf[cur ^ 1] = 0;
    }
    const uint32_t* sk = skBuf[cur];
    uint32_t& queueCount = queueCountBuf[cur];
    uint32_t* seedCount = seedCountBuf[cur];
    const unsigned long long* tileToc = tileTocBuf[cur];
    const uint32_t tileFirstRead = tileFirstReadBuf[cur];
    const uint64_t tileBase = uint64_t(tile) * kSweepTile;

    static_assert(kSweepPositionsPerThread <= 8 && kMaxFusedIterations <= 16, "hit masks: 16 bits x 8 positions");
    uint64_t hitsA = 0, hitsB = 0;
#pragma unroll 1
    for(int slot = 0; slot < kSweepPositionsPerThread; slot++) {
        const int local = slot * kSweepThreads + threadIdx.x;
        const uint64_t p = tileBase + local;
        if(p + m > a.markerCount) continue;

        // Seed-independent part: mixed 64-bit blocks (little-endian pairs of k-mer ids) and tail.
        uint64_t mixed[(MM > 0) ? ((MM / 2) > 0 ? (MM / 2) : 1) : 16];
        const uint32_t blocks = m >> 1;
        if(MM > 0) {
#pragma unroll
            for(int b = 0; b < MM / 2; b++) {
                const uint64_t w = uint64_t(sk[local + 2*b]) | (uint64_t(sk[local + 2*b + 1]) << 32);
                mixed[b] = murmurMix(w);
            }
        } else {
            for(uint32_t b = 0; b < blocks; b++) {
                const uint64_t w = uint64_t(sk[local + 2*b]) | (uint64_t(sk[local + 2*b + 1]) << 32);
                mixed[b] = murmurMix(w);
            }
        }
        const bool hasTail = (m & 1u) != 0;
        const uint64_t tail = hasTail ? uint64_t(sk[local + m - 1]) : 0ull;
        // h after the first block's xor = (seed ^ len*M) ^ mixed[0]; the seed only reaches the low word.
        const uint64_t x0 = blocks ? (lenTimesM ^ mixed[0]) : lenTimesM;

        // Hot loop: hash for every seed and remember WHICH seeds passed the high-word test in a bit mask (no divergent work
        // here: a warp step in which one of the 32 lanes has a hit would otherwise drag the whole warp through the rare path,
        // and with hashFraction 0.01 and 10 seeds that is nearly every step).
        uint32_t hitMask = 0;
#pragma unroll
        for(uint32_t s = 0; s < ((KK > 0) ? uint32_t(KK) : K); s++) {
            const U64Halves h = murmurAlmost<MM>(U64Halves{uint32_t(x0) ^ a.seeds[s], uint32_t(x0 >> 32)}, mixed, blocks, hasTail, tail);
            // hitMask |= (h.hi <= thresholdHigh) << s, as one compare and one predicated or
            asm("{\n\t.reg .pred q;\n\tsetp.le.u32 q, %1, %2;\n\t@q or.b32 %0, %0, %3;\n\t}" : "+r"(hitMask) : "r"(h.hi), "r"(thresholdHigh), "r"(1u << s));
        }
        // 16 mask bits per position, four positions per word.
        if(slot < 4) hitsA |= uint64_t(hitMask) << (16 * slot);
        else hitsB |= uint64_t(hitMask) << (16 * (slot - 4));
    }
    // The hits of all the thread's positions are queued in one go (the warp loops as often as its busiest lane has hits in
    // the whole tile, not once per position); only (position, seed) is queued: the hash is recomputed, lane-dense, below.
    for(;;) {
        uint32_t bit;
        if(hitsA) { bit = uint32_t(__ffsll((long long)hitsA)) - 1u; hitsA &= hitsA - 1ull; }
        else if(hitsB) { bit = 64u + uint32_t(__ffsll((long long)hitsB)) - 1u; hitsB &= hitsB - 1ull; }
        else break;
        const uint32_t local = (bit >> 4) * kSweepThreads + threadIdx.x, s = bit & 15u;
        const uint32_t q = atomicAdd(&queueCount, 1u);
        if(q < a.queueCapacity) queueMeta[q] = local | (s << 16);
        else {
            // Queue full (cannot happen for the sizes the host derives from hashFraction unless the data are pathological):
            // do the rare path inline.
            const uint64_t hash = featureHash<MM>(sk + local, m, seed0 + 37u * s, lenTimesM);
            if(hash >= threshold) continue;
            const uint32_t o = resolveFeature(a, tileBase + local, m);
            if(o != 0xffffffffu) {
                const unsigned long long gi = atomicAdd(&a.counts[s], 1ull);
                if(gi < a.capacity) {
                    a.keys[uint64_t(s) * a.capacity + gi] = ((hash & a.bucketMask) << 32) | (hash >> 32);
                    a.vals[uint64_t(s) * a.capacity + gi] = a.orientedReadBase + o;
                }
            }
        }
    }
    __syncthreads();

    // Queue pass A: resolve each queued low hash to its oriented read, rank it within (block, seed).
    const uint32_t nq = min(queueCount, a.queueCapacity);
    for(uint32_t q = threadIdx.x; q < nq; q += kSweepThreads) {
        const uint32_t meta = queueMeta[q];
        const uint32_t local = meta & 0xffffu, s = meta >> 16;
        // The complete hash and the exact test (the hot loop looked at the high word only).
        const uint64_t hash = featureHash<MM>(sk + local, m, seed0 + 37u * s, lenTimesM);
        uint32_t o = 0xffffffffu;
        if(hash < threshold) {
            const uint64_t p = tileBase + local;
            int k = 0;
#pragma unroll 1
            while(k < kSweepTileReads && tileToc[k + 1] <= p) k++;          // largest k with toc[first + k] <= p
            const uint32_t r = tileFirstRead + uint32_t(k);
            if(k == kSweepTileReads || r >= a.orientedReadCount) o = resolveFeature(a, p, m);      // beyond the staged entries
            else {
                const bool inside = (p + m <= tileToc[k + 1]);
                const bool palindromic = (a.readFlags[(a.orientedReadBase + r) >> 1] & 1u) != 0;
                o = (inside && !palindromic) ? r : 0xffffffffu;
            }
        }
        queueHash[q] = hash;
        if(o != 0xffffffffu) {
            queueMeta[q] = atomicAdd(&seedCount[s], 1u) | (s << 24);
            queueRead[q] = a.orientedReadBase + o;
        } else {
            queueMeta[q] = 0xffffffffu;
        }
    }
    __syncthreads();
    if(threadIdx.x < K) {
        const uint32_t c = seedCount[threadIdx.x];
        seedBase[threadIdx.x] = c ? atomicAdd(&a.counts[threadIdx.x], (unsigned long long)c) : 0ull;
    }
    __syncthreads();
    // Queue pass B: write (bucketId<<32 | hashHigh, orientedReadId) to the iteration's slab.
    for(uint32_t q = threadIdx.x; q < nq; q += kSweepThreads) {
        const uint32_t meta = queueMeta[q];
        if(meta == 0xffffffffu) continue;
        const uint32_t s = meta >> 24;
        const unsigned long long gi = seedBase[s] + (meta & 0xffffffu);
        if(gi < a.capacity) {
            const uint64_t h = queueHash[q];
            a.keys[uint64_t(s) * a.capacity + gi] = ((h & a.bucketMask) << 32) | (h >> 32);
            a.vals[uint64_t(s) * a.capacity + gi] = queueRead[q];
        }
    }
    }   // tiles of this block
}

// ---------------------------------------------------------------------------------------------
// a7/a8. Bucket inspection in ONE pass. Entries (key = bucketId<<32 | hashHigh, val = orientedReadId) are sorted by
// bucketId. One thread per entry e0:
//   * finds its bucket by walking left and right over equal bucket ids, giving up once the bucket is known to be larger
//     than maxBucketSize (buckets are a handful of entries; no head flags / scan / segment table);
//   * classifies the bucket size (sparse / good / crowded) into readLowHashStatistics (pass2, src/LowHash0.cpp:386-393);
//   * for buckets whose size is in [max(2,minBucketSize), maxBucketSize], counts the entries with equal hashHigh and
//     readId1 > readId0 (pass3, src/LowHash0.cpp:430-458), reserves room for them in the raw pair buffer (one atomic per
//     warp on `cursor`) and writes (readId0, readId1, strand). The order of the raw pair hits is arbitrary: they are sorted
//     and counted later. Hits that do not fit below `capacity` are not written; *cursor still ends up as the exact total,
//     so the host can grow the buffer and run the pass again (with stats == nullptr).
static __global__ void __launch_bounds__(256)
bucketPairsKernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint32_t n,
                  uint64_t minBucketSize, uint64_t maxBucketSize,
                  unsigned long long* __restrict__ stats,          // may be null
                  unsigned long long* __restrict__ cursor,         // pair hits reserved so far
                  uint64_t* __restrict__ pairsOut, unsigned long long capacity)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned lane = threadIdx.x & 31u;
    uint32_t count = 0, begin = 0, end = 0, oread0 = 0, hashHigh0 = 0;
    if(i < n) {
        const uint64_t key0 = keys[i];
        const uint32_t bucket = uint32_t(key0 >> 32);
        hashHigh0 = uint32_t(key0);
        oread0 = vals[i];
        begin = i; end = i + 1;
        uint64_t size = 1;          // exact when <= maxBucketSize, else maxBucketSize + 1 = "crowded"
        while(size <= maxBucketSize && begin > 0 && uint32_t(keys[begin - 1] >> 32) == bucket) { begin--; size++; }
        while(size <= maxBucketSize && end < n && uint32_t(keys[end] >> 32) == bucket) { end++; size++; }
        const uint32_t readId0 = oread0 >> 1;
        if(stats) {
            const int cls = (size < minBucketSize) ? 0 : ((size > maxBucketSize) ? 2 : 1);
            atomicAdd(&stats[3ull * readId0 + cls], 1ull);
        }
        const uint64_t lowest = minBucketSize > 2 ? minBucketSize : 2;
        if(size >= lowest && size <= maxBucketSize) {
            for(uint32_t j = begin; j < end; j++) {
                if(uint32_t(keys[j]) == hashHigh0 && (vals[j] >> 1) > readId0) count++;
            }
        } else end = begin;         // nothing to emit
    }
    // Room for the warp's hits: exclusive prefix over the lanes + one atomic.
    uint32_t inclusive = count;
#pragma unroll
    for(int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inclusive, d);
        if(lane >= unsigned(d)) inclusive += t;
    }
    const uint32_t warpTotal = __shfl_sync(0xffffffffu, inclusive, 31);
    if(warpTotal == 0) return;
    unsigned long long base = 0;
    if(lane == 31) base = atomicAdd(cursor, (unsigned long long)warpTotal);
    base = __shfl_sync(0xffffffffu, base, 31);
    unsigned long long out = base + (inclusive - count);
    if(count == 0 || out + count > capacity) return;
    const uint32_t readId0 = oread0 >> 1;
    for(uint32_t j = begin; j < end; j++) {
        if(uint32_t(keys[j]) != hashHigh0) continue;
        const uint32_t oread1 = vals[j];
        const uint32_t readId1 = oread1 >> 1;
        if(readId1 <= readId0) continue;
        const uint32_t strand = (oread0 ^ oread1) & 1u;        // 0 = same strand
        pairsOut[out++] = (uint64_t(readId0) << 32) | (uint64_t(readId1) << 1) | strand;
    }
}

// ---------------------------------------------------------------------------------------------
// a7/a8 for configurations in which one overlapping read pair collides in MANY buckets of the same iteration (HiFi:
// hashFraction 0.05 on low-error reads gives ~25 hits per pair and iteration, 3.3 G hits per iteration at 2 M reads): the
// hits are counted per read in a shared-memory hash table, and only (pair, count) leaves the kernel.
//   bucketSpanKernel    per entry: statistics as in bucketPairsKernel, and the entry's bucket [begin, begin + size) when the
//                       bucket is eligible for pair generation (size 0 otherwise);
//   readKeysKernel      (readId, entry index) for the stable sort that groups the entries by read;
//   readPairsKernel     one warp per read: visits the buckets of the read's entries, counts the partners (readId1 > readId0,
//                       equal hashHigh) in the table, then writes the table's (pair, count) items at a slot range reserved
//                       with one atomic; *hits accumulates the number of hits counted (the reference's pair hits).
static __global__ void __launch_bounds__(256)
bucketSpanKernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint32_t n,
                 uint64_t minBucketSize, uint64_t maxBucketSize, unsigned long long* __restrict__ stats, uint2* __restrict__ span)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n) return;
    const uint32_t bucket = uint32_t(keys[i] >> 32);
    uint32_t begin = i, end = i + 1;
    uint64_t size = 1;          // exact when <= maxBucketSize, else maxBucketSize + 1 = "crowded"
    while(size <= maxBucketSize && begin > 0 && uint32_t(keys[begin - 1] >> 32) == bucket) { begin--; size++; }
    while(size <= maxBucketSize && end < n && uint32_t(keys[end] >> 32) == bucket) { end++; size++; }
    if(stats) {
        const int cls = (size < minBucketSize) ? 0 : ((size > maxBucketSize) ? 2 : 1);
        atomicAdd(&stats[3ull * (vals[i] >> 1) + cls], 1ull);
    }
    const uint64_t lowest = minBucketSize > 2 ? minBucketSize : 2;
    const bool eligible = size >= lowest && size <= maxBucketSize;
    span[i] = make_uint2(begin, eligible ? uint32_t(size) : 0u);
}

static __global__ void readKeysKernel(const uint32_t* __restrict__ vals, uint32_t n, uint64_t* __restrict__ readKeys, uint32_t* __restrict__ index)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n) return;
    readKeys[i] = uint64_t(vals[i] >> 1);
    index[i] = i;
}

constexpr uint32_t kPairTableSlots = 512;           // per warp; a power of two (a read has ~40 - 300 partners per iteration)
constexpr uint32_t kPairTableLog2Slots = 9;
constexpr uint32_t kPairTableWarps = 8;
constexpr uint32_t kPairTableEmpty = 0xffffffffu;   // never a key: readId1 < 2^31
constexpr uint32_t kPairTableMaxProbes = 24;

static __global__ void __launch_bounds__(kPairTableWarps * 32)
readPairsKernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, const uint2* __restrict__ span,
                const uint64_t* __restrict__ sortedReadKeys, const uint32_t* __restrict__ order,
                const uint32_t* __restrict__ segStart, uint32_t numReads,
                unsigned long long* __restrict__ cursor, unsigned long long* __restrict__ hits,
                uint64_t* __restrict__ outKeys, uint32_t* __restrict__ outCounts, unsigned long long capacity, uint32_t maxProbes)
{
    __shared__ uint32_t tableKeyAll[kPairTableWarps][kPairTableSlots];
    __shared__ uint32_t tableCountAll[kPairTableWarps][kPairTableSlots];
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t seg = blockIdx.x * kPairTableWarps + warp;
    if(seg >= numReads) return;
    uint32_t* tableKey = tableKeyAll[warp];
    uint32_t* tableCount = tableCountAll[warp];
#pragma unroll
    for(uint32_t s = lane; s < kPairTableSlots; s += 32) { tableKey[s] = kPairTableEmpty; tableCount[s] = 0; }
    __syncwarp();
    const uint32_t a = segStart[seg], b = segStart[seg + 1];
    const uint32_t readId0 = uint32_t(sortedReadKeys[a]);
    uint32_t myHits = 0;
    // 32 entries of the read at a time (one per lane), then entry by entry with the bucket's members spread over the lanes:
    // the member loads are coalesced, and every lane works on every bucket.
    for(uint32_t e0 = a; e0 < b; e0 += 32) {
        uint32_t begin = 0, size = 0, hashHigh0 = 0, oread0 = 0;
        if(e0 + lane < b) {
            const uint32_t i = order[e0 + lane];
            const uint2 sp = span[i];
            begin = sp.x; size = sp.y;
            if(size) { hashHigh0 = uint32_t(keys[i]); oread0 = vals[i]; }
        }
        unsigned live = __ballot_sync(0xffffffffu, size != 0);
        while(live) {
            const int t = __ffs(int(live)) - 1;
            live &= live - 1u;
            const uint32_t tBegin = __shfl_sync(0xffffffffu, begin, t), tSize = __shfl_sync(0xffffffffu, size, t);
            const uint32_t tHash = __shfl_sync(0xffffffffu, hashHigh0, t), tRead = __shfl_sync(0xffffffffu, oread0, t);
            for(uint32_t j = tBegin + lane; j < tBegin + tSize; j += 32) {
                if(uint32_t(keys[j]) != tHash) continue;
                const uint32_t oread1 = vals[j];
                const uint32_t readId1 = oread1 >> 1;
                if(readId1 <= readId0) continue;
                const uint32_t k = (readId1 << 1) | ((tRead ^ oread1) & 1u);       // strand bit 0 = same strand
                myHits++;
                uint32_t slot = (k * 2654435761u) >> (32 - kPairTableLog2Slots);
                uint32_t probes = 0;
                for(;;) {
                    const uint32_t prev = atomicCAS(&tableKey[slot], kPairTableEmpty, k);
                    if(prev == kPairTableEmpty || prev == k) { atomicAdd(&tableCount[slot], 1u); break; }
                    slot = (slot + 1u) & (kPairTableSlots - 1u);
                    if(++probes >= maxProbes) {
                        // Table (nearly) full: this hit goes out on its own; the merge adds the counts up.
                        const unsigned long long at = atomicAdd(cursor, 1ull);
                        if(at < capacity) { outKeys[at] = (uint64_t(readId0) << 32) | k; outCounts[at] = 1u; }
                        break;
                    }
                }
            }
        }
    }
    __syncwarp();
    // Occupied slots -> output: count them, reserve, write.
    uint32_t occupied = 0;
#pragma unroll
    for(uint32_t s = lane; s < kPairTableSlots; s += 32) occupied += (tableKey[s] != kPairTableEmpty) ? 1u : 0u;
    uint32_t inclusive = occupied, hitSum = myHits;
#pragma unroll
    for(int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inclusive, d);
        if(lane >= unsigned(d)) inclusive += t;
    }
#pragma unroll
    for(int d = 16; d > 0; d >>= 1) hitSum += __shfl_down_sync(0xffffffffu, hitSum, d);
    const uint32_t total = __shfl_sync(0xffffffffu, inclusive, 31);
    if(lane == 0 && hitSum) atomicAdd(hits, (unsigned long long)hitSum);
    if(total == 0) return;
    unsigned long long base = 0;
    if(lane == 31) base = atomicAdd(cursor, (unsigned long long)total);
    base = __shfl_sync(0xffffffffu, base, 31);
    if(base + total > capacity) return;
    unsigned long long out = base + (inclusive - occupied);
    for(uint32_t s = lane; s < kPairTableSlots; s += 32) {
        const uint32_t k = tableKey[s];
        if(k != kPairTableEmpty) { outKeys[out] = (uint64_t(readId0) << 32) | k; outCounts[out] = tableCount[s]; out++; }
    }
}

// Sorted pair keys -> unique keys with multiplicities.
static __global__ void uniqueCountsKernel(const uint64_t* __restrict__ sortedKeys, const uint32_t* __restrict__ segStart,
                                   uint32_t numSegments, uint64_t* __restrict__ outKeys, uint32_t* __restrict__ outCounts)
{
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if(s >= numSegments) return;
    const uint32_t b = segStart[s];
    outKeys[s] = sortedKeys[b];
    outCounts[s] = segStart[s + 1] - b;
}

// Sorted (key,count) items with duplicate keys -> unique keys with summed counts.
static __global__ void segmentSumKernel(const uint64_t* __restrict__ sortedKeys, const uint32_t* __restrict__ sortedCounts,
                                 const uint32_t* __restrict__ segStart, uint32_t numSegments,
                                 uint64_t* __restrict__ outKeys, uint32_t* __restrict__ outCounts)
{
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if(s >= numSegments) return;
    const uint32_t b = segStart[s], e = segStart[s + 1];
    uint32_t sum = 0;
    for(uint32_t j = b; j < e; j++) sum += sortedCounts[j];
    outKeys[s] = sortedKeys[b];
    outCounts[s] = sum;
}

// flags[i] = (uint16(count[i]) >= minFrequency)   — the frequency is a wrapping uint16 in the
// reference (src/LowHash0.hpp:116, src/LowHash0.cpp:207,521).
static __global__ void frequencyFlagsKernel(const uint32_t* __restrict__ counts, uint32_t n, uint64_t minFrequency,
                                     uint32_t* __restrict__ flags)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n) return;
    flags[i] = (uint64_t(counts[i] & 0xffffu) >= minFrequency) ? 1u : 0u;
}

// Compact the flagged keys into 12-byte OrientedReadPair records (src/OrientedReadPair.hpp:18-86).
static __global__ void emitCandidatesKernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ flags,
                                     const uint32_t* __restrict__ offsets, uint32_t n, uint32_t* __restrict__ out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n || !flags[i]) return;
    const uint64_t key = keys[i];
    const uint64_t o = offsets[i];
    out[3*o + 0] = uint32_t(key >> 32);
    out[3*o + 1] = uint32_t(key & 0xffffffffull) >> 1;
    out[3*o + 2] = (key & 1ull) ? 0u : 1u;          // byte 0 = isSameStrand, bytes 1..3 = 0
}

} // namespace shb
