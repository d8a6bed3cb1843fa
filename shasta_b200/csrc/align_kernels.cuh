// Marker-space alignment kernels (sm_90a). Reference: chanzuckerberg/shasta
//   downsampling hash            src/AssemblerKmers.cpp:182-186, src/MurmurHash2.cpp:37-88
//   method 3 (two-stage banded)  src/AssemblerAlign3.cpp:23-313
//   overlap DP + traceback       call sites src/AssemblerAlign3.cpp:117-122,254-260, src/Align4.cpp:1027-1033
//                                 (SeqAn in the reference; rule set of SURVEY.md Appendix A)
//   AlignmentInfo / filters      src/Alignment.cpp:67-113, src/AssemblerAlign.cpp:438-483
//   compress                     src/compressAlignment.cpp:11-70
#pragma once

#include "common.cuh"
#include "compressed_alignment.cuh"
#include "primitives.cuh"
#include "../../include/shb_dp_policy.h"

namespace shb {

// ---------------------------------------------------------------------------------------------
// kmerTable[kmerId].hash without the 4^k table: MurmurHash2(&n, 8, 13477), n = kmerId + rc(kmerId).
__device__ __forceinline__ uint32_t kmerDownsamplingHash(uint32_t kmer, uint32_t k)
{
    const uint64_t n = uint64_t(kmer) + uint64_t(reverseComplementKmer(kmer, k));
    const uint32_t m = 0x5bd1e995u;
    uint32_t h = 13477u ^ 8u;
    uint32_t k1 = uint32_t(n);
    k1 *= m; k1 ^= k1 >> 24; k1 *= m;
    h *= m; h ^= k1;
    uint32_t k2 = uint32_t(n >> 32);
    k2 *= m; k2 ^= k2 >> 24; k2 *= m;
    h *= m; h ^= k2;
    h ^= h >> 13; h *= m; h ^= h >> 15;
    return h;
}

static __global__ void downsampleFlagsKernel(const uint32_t* __restrict__ kmerIds, uint64_t begin, uint32_t n,
                                             uint32_t k, uint32_t hashThreshold, uint32_t* __restrict__ flags)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n) return;
    flags[i] = (kmerDownsamplingHash(kmerIds[begin + i], k) < hashThreshold) ? 1u : 0u;
}

// Compact the downsampled markers of a chunk: dsKmer / dsOrdinal at (dsBase + exclusive index).
static __global__ void downsampleCompactKernel(const uint32_t* __restrict__ kmerIds, uint64_t begin, uint32_t n,
                                               const uint32_t* __restrict__ flags, const uint32_t* __restrict__ index,
                                               const uint64_t* __restrict__ toc, uint32_t orientedReadCount, uint64_t dsBase,
                                               uint32_t* __restrict__ dsKmer, uint32_t* __restrict__ dsOrdinal)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n || !flags[i]) return;
    const uint64_t p = begin + i;
    const uint32_t lo = rowOf(toc, 0u, orientedReadCount, p);
    const uint64_t d = dsBase + index[i];
    dsKmer[d] = kmerIds[p];
    dsOrdinal[d] = uint32_t(p - toc[lo]);
}

// dsToc[o] = number of downsampled markers before row o's first marker. Rows starting in this chunk.
static __global__ void downsampleTocKernel(const uint64_t* __restrict__ toc, uint32_t orientedReadCount,
                                           uint64_t begin, uint32_t n, const uint32_t* __restrict__ index,
                                           uint64_t dsBase, uint64_t dsTotalAfterChunk, uint64_t* __restrict__ dsToc)
{
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if(o > orientedReadCount) return;
    const uint64_t p = toc[o];
    if(p >= begin && p < begin + n) dsToc[o] = dsBase + index[p - begin];
    else if(p == begin + n) dsToc[o] = dsTotalAfterChunk;       // rows starting exactly at the chunk end (or the final sentinel)
}

// ---------------------------------------------------------------------------------------------
// One DP job = one overlap alignment of sequence a (horizontal, index i) against b (vertical, j)
// restricted to the band lo <= i - j <= hi (already clipped to the matrix).
struct DpJob {
    uint64_t aOffset, bOffset;      // into the sequence array
    uint32_t nx, ny;
    int32_t lo, hi;
    uint64_t traceOffset;           // in 32-bit words
    uint64_t outOffset;             // stage 2: in ordinal pairs
    uint32_t state;                 // 0 = run, others = skip (see kState*)
    uint32_t pad;
};
constexpr uint32_t kStateRun = 0, kStateEmpty = 1, kStateSkipped = 2;

struct DpScores { int32_t match, mismatch, gap; };

// The two oriented reads of candidate p (src/AssemblerAlign.cpp:381-382): (readId0, strand 0) and (readId1, sameStrand ? 0 : 1).
// Bit 8 of the third word (never set by computeAlignments' callers: the record's padding is zero) flips both strands: the
// single-pair entry point shb_align_oriented_reads uses it to align a pair in exactly the orientation it was given.
constexpr uint32_t kCandidateStrand0Bit = 0x100u;
__device__ __forceinline__ void candidateOrientedReads(const uint32_t* __restrict__ candidates, uint64_t p, uint64_t& o0, uint64_t& o1)
{
    const uint32_t r0 = candidates[3ull * p], r1 = candidates[3ull * p + 1], w = candidates[3ull * p + 2];
    const uint32_t strand0 = (w & kCandidateStrand0Bit) ? 1u : 0u;
    const bool same = (w & 0xffu) != 0;
    o0 = 2ull * r0 + strand0;
    o1 = 2ull * r1 + (same ? strand0 : 1u - strand0);
}

constexpr int32_t kNegInf = -(1 << 29);
constexpr int kDpMaxWarpsPerBlock = 4;

// Tie-break rules (include/shb_dp_policy.h, shared with the CPU oracle): which move wins when two give the same score.
//   viaGap  : the cell takes the better gap move g = gapIn + gap instead of the diagonal move
//   horzWins: of the two gap inputs the horizontal one is taken
__device__ __forceinline__ bool dpViaGap(int32_t g, int32_t diag) { return SHB_DP_DIAG_WINS_TIES ? (g > diag) : (g >= diag); }
__device__ __forceinline__ bool dpHorzWins(int32_t horzIn, int32_t vertIn) { return SHB_DP_VERT_BEFORE_HORZ ? (horzIn > vertIn) : (horzIn >= vertIn); }
// End cell: candidate (s2,i2,j2) replaces (s,i,j)? Column-major visiting order = (i, then j) ascending.
__device__ __forceinline__ bool dpEndCellBetter(int32_t s2, int32_t i2, int32_t j2, int32_t s, int32_t i, int32_t j)
{
    if(s2 != s) return s2 > s;
    return SHB_DP_END_FIRST_MAX ? (i2 < i || (i2 == i && j2 < j)) : (i2 > i || (i2 == i && j2 > j));
}
constexpr int32_t kEndCellNone = SHB_DP_END_FIRST_MAX ? 0x7fffffff : -1;        // bestI / bestJ of "no candidate yet"

// Physical band layout of the wavefront kernels: band offset e = j - i + hi in [0, W) sits at physical offset p = e + 1;
// p = 0 and p = W + 1 are BARRIER offsets whose gap score is "minus infinity", so that nothing flows around the band
// edges; physical offsets beyond W + 1 are padding that only the barrier ever reads.
//
// Band classes, one launch each. A wavefront class (c > 0) runs a job on a group of `lanes` lanes, each owning two
// sub-chunks of c physical offsets, so it holds W + 2 <= wMax = 2 * lanes * c. Narrow bands run on groups of 8 lanes
// (four jobs per warp, widths 32, 48, ..., 128), wider ones on a whole warp; c = 0 is the shared-memory scan kernel.
// The padded width of a job (its trace row length) is W + 2 rounded up to 2 * lanes.
struct DpClass { uint32_t wMax, lanes, c; };
constexpr uint32_t kDpClassCount = 17, kDpGroupClassCount = 7;
__host__ __device__ constexpr DpClass dpClassAt(uint32_t k)
{
    const uint32_t m = k - kDpGroupClassCount;                          // whole-warp classes: c = 3, 4, 6, 8, 12, 16
    const uint32_t warpC = m < 2 ? m + 3u : m < 4 ? 2u * m + 2u : 4u * m - 4u;
    return k < kDpGroupClassCount ? DpClass{16u * (k + 2u), 8u, k + 2u}
         : m < 6 ? DpClass{64u * warpC, 32u, warpC}
         : DpClass{2048u << (m - 6u), 32u, 0u};
}
struct DpShape { uint32_t cls, lanes, c, wpad; };
// The class of a band lo..hi (the last class, with a padded width beyond its wMax, for bands too wide for any).
__host__ __device__ inline DpShape dpBandShape(int32_t lo, int32_t hi)
{
    const uint32_t need = uint32_t(hi - lo + 1) + 2u;
    uint32_t k = 0;
    while(k + 1 < kDpClassCount && need > dpClassAt(k).wMax) k++;
    const DpClass cl = dpClassAt(k);
    return DpShape{k, cl.lanes, cl.c, (need + 2u * cl.lanes - 1u) & ~(2u * cl.lanes - 1u)};
}
constexpr int32_t kGapBarrier = -(1 << 28);
// Columns of the matrix that hold at least one in-band cell: max(0, lo) <= i <= min(nx, ny + hi). The wavefront kernel
// only visits these (a band that enters through the top edge or leaves through the bottom edge skips the rest).
__host__ __device__ inline int32_t dpFirstColumn(int32_t lo) { return lo > 0 ? lo : 0; }
__host__ __device__ inline int32_t dpLastColumn(uint32_t nx, uint32_t ny, int32_t hi)
{
    const int64_t bottom = int64_t(ny) + hi;
    return int32_t(bottom < int64_t(nx) ? bottom : int64_t(nx));
}
// Trace layout of both DP kernels: word (t >> 4) * wpad + p holds the 2-bit codes of 16 steps t at physical offset
// p = e + 1, newest step in the low bits (step t at bits 2 * (15 - t % 16)). The step of cell (i, p): the wavefront kernels
// store by step, and lane p / (2C) reaches column i in step i - iFirst + p / (2C); the scan kernel stores by column, t = i.
struct DpTraceSteps {
    int32_t iFirst;
    uint32_t reciprocal;            // p / (2C) == (p * reciprocal) >> 16 for p < 1024; 0 for the scan kernel
    __host__ __device__ uint32_t step(int32_t i, uint32_t p) const { return uint32_t(i - iFirst) + ((p * reciprocal) >> 16); }
};
__host__ __device__ inline DpTraceSteps dpTraceSteps(const DpShape& s, int32_t lo)
{
    return s.c ? DpTraceSteps{dpFirstColumn(lo), (65536u + 2u * s.c - 1u) / (2u * s.c)} : DpTraceSteps{0, 0u};
}
__host__ __device__ inline uint64_t dpTraceWords(uint32_t nx, uint32_t ny, int32_t lo, int32_t hi)
{
    const DpShape s = dpBandShape(lo, hi);
    uint64_t columns = nx;                                              // scan kernel: by-column layout over all columns
    if(s.c) {
        const int64_t active = int64_t(dpLastColumn(nx, ny, hi)) - dpFirstColumn(lo);
        columns = uint64_t(active > 0 ? active : 0);
    }
    // Rows of the by-step layout: columns + 1 steps plus the lane skew, and one spare row that the traceback may read.
    return ((columns + s.lanes + 15u) / 16u + 1u) * s.wpad;
}

// Warp-cooperative banded overlap DP. Band offset e = j - i + hi in [0, W). Lanes own e % 32.
//   hPrev/hCur : shared memory, Wpad + 1 ints each (sentinel at Wpad).   traceAcc: Wpad words.
//   trace      : global scratch, dpTraceWords() words, in the layout and code format of the wavefront kernels
//                (DpTraceSteps, systolicSubChunk) with step t = column i: word (i/16)*Wpad + e + 1 holds the codes of
//                columns 16*(i/16) .. +15 for band offset e, column i at bits 2*(15 - i%16); boundary cells are diagonal.
// Tie-break and end-cell rules: SURVEY.md Appendix A (diag > vertical > horizontal; first strict maximum in
// column-major order over last-row / last-column cells).
__device__ inline void bandedOverlapDp(const uint32_t* __restrict__ a, uint32_t nx, const uint32_t* __restrict__ b, uint32_t ny,
                                       int32_t lo, int32_t hi, DpScores sc,
                                       int32_t* hPrev, int32_t* hCur, uint32_t* traceAcc, uint32_t* __restrict__ trace,
                                       int32_t& bestScore, int32_t& bestI, int32_t& bestJ)
{
    const unsigned lane = threadIdx.x & 31u;
    const int32_t W = hi - lo + 1;
    const int32_t Wpad = int32_t(dpBandShape(lo, hi).wpad);
    const int32_t chunks = Wpad >> 5;

    bestScore = kNegInf * 2; bestI = -1; bestJ = -1;
    for(int32_t e = lane; e <= Wpad; e += 32) { hPrev[e] = kNegInf; hCur[e] = kNegInf; }
    for(int32_t e = lane; e < Wpad; e += 32) traceAcc[e] = 0;
    __syncwarp();

    for(int32_t i = 0; i <= int32_t(nx); i++) {
        const uint32_t ai = (i > 0) ? a[i - 1] : 0u;
        int32_t carry = kNegInf;                         // H of offset e-1 (previous chunk's last lane)
        int32_t carryP = kNegInf * 2;                    // running prefix maximum of A(e) - e*gap
        const bool lastColumn = (i == int32_t(nx));
        const int32_t eLastRow = int32_t(ny) - i + hi;   // band offset of row j = ny in this column
        for(int32_t c = 0; c < chunks; c++) {
            const int32_t e = (c << 5) + int32_t(lane);
            const int32_t j = e + i - hi;
            const bool valid = (e < W) && (j >= 0) && (j <= int32_t(ny));
            int32_t A = kNegInf, diag = kNegInf, horz = kNegInf;
            const bool boundary = (i == 0) || (j == 0);
            if(valid) {
                if(boundary) A = 0;
                else {
                    diag = hPrev[e] + ((ai == b[j - 1]) ? sc.match : sc.mismatch);
                    horz = hPrev[e + 1] + sc.gap;        // (i-1, j); sentinel / out-of-band entries hold kNegInf
                    A = max(diag, horz);
                }
            }
            // Vertical moves: H(e) = max(A(e), H(e-1) + gap)  ==  e*gap + prefixmax(A(e') - e'*gap).
            int32_t P = A - e * sc.gap;
#pragma unroll
            for(int d = 1; d < 32; d <<= 1) {
                const int32_t t = __shfl_up_sync(0xffffffffu, P, d);
                if(lane >= (unsigned)d) P = max(P, t);
            }
            P = max(P, carryP);
            int32_t H = P + e * sc.gap;
            if(!valid) H = kNegInf;
            if(valid && boundary) H = 0;
            // Trace code.
            int32_t below = __shfl_up_sync(0xffffffffu, H, 1);       // H(e-1) = cell (i, j-1)
            if(lane == 0) below = carry;
            uint32_t code = 0;
            if(valid && !boundary) {
                const int32_t vert = below + sc.gap;
                const bool horzWins = dpHorzWins(horz, vert);
                code = dpViaGap(max(horz, vert), diag) ? (horzWins ? 3u : 1u) : 0u;
            }
            hCur[e] = H;
            uint32_t acc = (traceAcc[e] << 2) | code;
            traceAcc[e] = acc;
            if((i & 15) == 15 || lastColumn) {
                const uint32_t filled = uint32_t(i & 15) + 1u;       // columns accumulated in this word
                // e + 1 == Wpad would be the next job's trace; W + 2 <= Wpad keeps every in-band offset below it
                if(e + 1 < Wpad) trace[uint64_t(i >> 4) * uint32_t(Wpad) + uint32_t(e + 1)] = acc << (2u * (16u - filled));
                traceAcc[e] = 0;
            }
            carry = __shfl_sync(0xffffffffu, H, 31);
            carryP = __shfl_sync(0xffffffffu, P, 31);
            // End-cell candidates: row ny in every column, all rows in the last column.
            if(lastColumn) {
                int32_t mx = valid ? H : kNegInf * 2;
#pragma unroll
                for(int d = 16; d > 0; d >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
                const unsigned who = __ballot_sync(0xffffffffu, valid && H == mx);
                if(who && (SHB_DP_END_FIRST_MAX ? (mx > bestScore) : (mx >= bestScore))) {
                    const int pick = SHB_DP_END_FIRST_MAX ? (__ffs(who) - 1) : (31 - __clz(who));
                    bestScore = mx; bestI = i; bestJ = ((c << 5) + pick) + i - hi;
                }
            } else if(eLastRow >= (c << 5) && eLastRow < (c << 5) + 32 && eLastRow < W && eLastRow >= 0) {
                const int32_t s = __shfl_sync(0xffffffffu, H, eLastRow & 31);
                if(SHB_DP_END_FIRST_MAX ? (s > bestScore) : (s >= bestScore)) { bestScore = s; bestI = i; bestJ = int32_t(ny); }
            }
        }
        __syncwarp();
        int32_t* t = hPrev; hPrev = hCur; hCur = t;
    }
}

// ---------------------------------------------------------------------------------------------
// Register-resident wavefront version of the same DP for bands of up to 2*G*C - 2 offsets, run by a group of G lanes
// (G = 8 or 32, C <= 16). The 2*G*C PHYSICAL offsets (band offset e at p = e + 1, barriers at p = 0 and p = W + 1, see
// dpBandShape) are cut into 2G sub-chunks of C consecutive offsets; lane l of the group owns sub-chunks 2l ("A") and
// 2l+1 ("B"). Cell (i, p) depends on (i-1, p),
// (i-1, p+1) and (i, p-1), so sub-chunk s can process column i at step T = 2i + s: on even steps every lane advances its A
// sub-chunk, on odd steps its B sub-chunk (no divergence, every lane busy every step), and the only inter-lane traffic is
// one shuffle per half-step (the neighbouring sub-chunk's boundary score). All scores of the previous column live in
// registers; no shared memory, no scan.
// Same recurrence, tie-break and end-cell rules as bandedOverlapDp (bit-identical results, tested against the oracle); the
// end cell is selected with the order-independent formulation of dpEndCellBetter.
//
// Per-offset constants of a sub-chunk, fixed for the whole job. The cell of band offset e is inside the matrix for
// columns first <= i <= min(nx, ny + hi - e), where first = max(0, hi - e); in column `first` it is a boundary cell
// (i == 0 or j == 0, score 0). gap = the gap score, or kGapBarrier for the two barrier offsets: a barrier cell can only
// be entered by a gap move, so its score is "minus infinity" plus something bounded, whatever its neighbours hold, and
// no finite score ever passes through it; no per-cell clamp and no special case for the first / last lane is needed
// (lane 0's first offset and lane G-1's last offset are barrier or padding, so the values their shuffles wrap around
// are never used by an in-band cell).
template<int C> struct SubChunkLimits { int32_t first[C]; int32_t gap[C]; };

template<int C> __device__ __forceinline__ void initSubChunkLimits(SubChunkLimits<C>& lim, int32_t p0, int32_t W, int32_t hi, int32_t gap)
{
#pragma unroll
    for(int c = 0; c < C; c++) {
        const int32_t e = p0 + c - 1;
        lim.first[c] = (e >= 0 && e < W) ? max(0, hi - e) : 0x7fffffff;
        lim.gap[c] = (e == -1 || e == W) ? kGapBarrier : gap;
    }
}

// Trace layout of the wavefront kernel: the codes are stored by STEP, not by column. Lane l works on column
// i = t2 - l in step t2, and every lane stores the codes of its last 16 steps in the same step (t2 % 16 == 15), so the
// stores are group-uniform and coalesced: word (t2 >> 4) * Wpad + p holds, at bits 2 * (15 - t2 % 16), the code of cell
// (t2 - p / (2C), p) (DpTraceSteps).

// One sub-chunk (C consecutive physical offsets) of column i. Straight-line code for the common interior cell; cells
// outside the matrix are NOT masked: above the matrix they only ever combine "minus infinity" values (kNegInf plus a
// bounded drift), below the matrix their values are never read by an in-matrix cell, and their trace codes are never
// visited by the traceback. bw[] = b[j-1] for the C offsets (sentinel outside the row).
// Boundary = false leaves out the test for the boundary cell (i == 0 or j == 0): for columns past max(0, hi).
// The wavefront kernels are bound by the integer-ALU pipe (compares, selects, min/max); the FMA pipe idles. The adds of
// the recurrence and the trace bookkeeping are therefore written as integer multiply-adds with run-time multipliers
// (a kernel argument the compiler cannot fold): IMAD issues on the FMA pipe. FmaUnits = {1, 2, 4}.
struct FmaUnits { int32_t one, two, four; };
// Sub-chunk widths up to this one run their 16-step blocks fully unrolled, with the trace codes added in place.
constexpr int kDpInPlaceTraceMaxC = 4;
__device__ __forceinline__ int32_t fmaPipeAdd(int32_t a, int32_t b, int32_t one)
{
    int32_t r;
    asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(one), "r"(b));
    return r;
}
__device__ __forceinline__ uint32_t fmaPipeMul(uint32_t a, uint32_t b)
{
    uint32_t r;
    asm("mad.lo.u32 %0, %1, %2, 0;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
// acc += v if x == y (compare on the ALU pipe, the predicated add on the FMA pipe)
__device__ __forceinline__ void fmaPipeAddIfEqual(int32_t& acc, uint32_t x, uint32_t y, int32_t v, int32_t one)
{
    asm("{\n\t.reg .pred q;\n\tsetp.eq.u32 q, %1, %2;\n\t@q mad.lo.s32 %0, %3, %4, %0;\n\t}" : "+r"(acc) : "r"(x), "r"(y), "r"(v), "r"(one));
}
// acc += a * b if x > y (x >= y when OrEqual), signed
template<bool OrEqual> __device__ __forceinline__ void fmaPipeAddIfGreater(uint32_t& acc, int32_t x, int32_t y, int32_t a, int32_t b)
{
    if(OrEqual) asm("{\n\t.reg .pred q;\n\tsetp.ge.s32 q, %1, %2;\n\t@q mad.lo.u32 %0, %3, %4, %0;\n\t}" : "+r"(acc) : "r"(x), "r"(y), "r"(a), "r"(b));
    else asm("{\n\t.reg .pred q;\n\tsetp.gt.s32 q, %1, %2;\n\t@q mad.lo.u32 %0, %3, %4, %0;\n\t}" : "+r"(acc) : "r"(x), "r"(y), "r"(a), "r"(b));
}

// Trace words of the wavefront kernels: a shift register of 2-bit codes, newest step in the low bits:
//   bit 0 = the cell took a gap move (its score is gapIn + gap, not the diagonal's), bit 1 = the horizontal input was the
//   larger gap input (meaningful when bit 0 is set). After the 16 steps of a block, step s of the block sits at bits
//   2 * (15 - s).
// Step >= 0: the step's position in its 16-step block is a compile-time constant (fully unrolled block) and the trace word
// was cleared at the start of the block, so the code is added in place (one multiply-add less per cell than shifting the
// register); Step < 0: shift register.
template<int C, bool Boundary, int Step = -1> __device__ __forceinline__ void systolicSubChunk(
    int32_t (&H)[C], uint32_t (&Tr)[C], const SubChunkLimits<C>& lim, int32_t i, uint32_t ai,
    int32_t below /* H(i, p0-1) */, int32_t top /* H(i-1, p0+C) */, const uint32_t* bw, DpScores sc, FmaUnits u)
{
    constexpr int32_t kCodeUnit = (Step >= 0) ? int32_t(1u << (2 * (15 - (Step >= 0 ? Step : 0)))) : 1;      // bit 0 of this step's code
    int32_t vertIn = below;
    const int32_t matchBonus = sc.match - sc.mismatch;
#pragma unroll
    for(int c = 0; c < C; c++) {
        int32_t diag = fmaPipeAdd(H[c], sc.mismatch, u.one);                    // from H(i-1, p)
        fmaPipeAddIfEqual(diag, ai, bw[c], matchBonus, u.one);
        const int32_t horzIn = (c + 1 < C) ? H[c + 1] : top;                    // H(i-1, p+1); vertIn = H(i, p-1)
        // max(diag, vert, horz) as one max and one add-max; the tie order (include/shb_dp_policy.h) only enters the trace.
        const int32_t gapIn = max(vertIn, horzIn);
        int32_t h = __viaddmax_s32(gapIn, lim.gap[c], diag);
        uint32_t tr = (Step >= 0) ? Tr[c] : fmaPipeMul(Tr[c], uint32_t(u.four));      // shift the older codes up by two bits
        if(Step >= 0) {
            if(SHB_DP_DIAG_WINS_TIES) fmaPipeAddIfGreater<false>(tr, h, diag, u.one, kCodeUnit);
            else fmaPipeAddIfGreater<true>(tr, fmaPipeAdd(gapIn, lim.gap[c], u.one), diag, u.one, kCodeUnit);
            fmaPipeAddIfGreater<!SHB_DP_VERT_BEFORE_HORZ>(tr, horzIn, vertIn, u.one, 2 * kCodeUnit);
        } else {
            if(SHB_DP_DIAG_WINS_TIES) fmaPipeAddIfGreater<false>(tr, h, diag, u.one, u.one);
            else fmaPipeAddIfGreater<true>(tr, fmaPipeAdd(gapIn, lim.gap[c], u.one), diag, u.one, u.one);
            fmaPipeAddIfGreater<!SHB_DP_VERT_BEFORE_HORZ>(tr, horzIn, vertIn, u.one, u.two);
        }
        Tr[c] = tr;
        if(Boundary) h = (i == lim.first[c]) ? 0 : h;
        H[c] = h;
        vertIn = h;
    }
}

// End-cell candidates of one sub-chunk in column i (rare: only the lanes whose offsets touch the last row or the
// last column get here). bestJ is tracked as j + hi (fixed up by the caller). e0 = band offset of the sub-chunk's first
// physical offset (p0 - 1).
template<int C> __device__ __forceinline__ void systolicEndCells(
    const int32_t (&H)[C], const SubChunkLimits<C>& lim, int32_t e0, int32_t i, int32_t cStar /* offset index on row ny */,
    int32_t nx, int32_t& bestScore, int32_t& bestI, int32_t& bestJ)
{
#pragma unroll
    for(int c = 0; c < C; c++) {
        // the cell on the last row j == ny of this column, and every in-matrix cell (j <= ny) of the last column
        const bool lastRow = (c == cStar);
        const bool lastColumn = (i == nx) && (c <= cStar) && (lim.first[c] <= nx);
        if((lastRow || lastColumn) && i >= lim.first[c]) {                  // first == INT_MAX outside the band
            const int32_t h = H[c];
            const int32_t jPlusHi = e0 + c + i;
            if(dpEndCellBetter(h, i, jPlusHi, bestScore, bestI, bestJ)) { bestScore = h; bestI = i; bestJ = jPlusHi; }
        }
    }
}

// State of one job's wavefront, all in registers.
template<int C> struct SystolicState {
    int32_t HA[C], HB[C];
    uint32_t TA[C], TB[C];
    SubChunkLimits<C> limA, limB;
    uint32_t bw[2 * C];             // b[j-1] of the lane's 2C offsets in the current column (sliding window)
    int32_t i;                      // column of this lane in the current step
    const uint32_t* ap;             // &a[i - 1]
    const uint32_t* bNext;          // &b[jA - 1 + 2C]: the element that enters the window in the next step
    int32_t jNext;                  // its index (jA - 1 + 2C), for the range test
    int32_t bestScore, bestI, bestJ;
};

// 16 steps. Checked = false: no boundary cell and no end cell can occur in these steps for any lane, and every k-mer
// the lanes load lies inside its row (see the block ranges in bandedOverlapDpSystolic), so the loads are unconditional.
template<int G, int C, bool Checked, int Step> __device__ __forceinline__ void systolicStep(
    SystolicState<C>& s, int32_t eA, int32_t eB, int32_t rowEndA, int32_t nx, int32_t ny, DpScores sc, FmaUnits fu)
{
    uint32_t ai = 0xfffffffeu;
    uint32_t bIn = 0xffffffffu;                     // enters the window after this step
    if(Checked) {
        if(uint32_t(s.i - 1) < uint32_t(nx)) ai = __ldg(s.ap);
        if(uint32_t(s.jNext) < uint32_t(ny)) bIn = __ldg(s.bNext);
    } else {
        ai = __ldg(s.ap);
        bIn = __ldg(s.bNext);
    }
    // Even step: sub-chunk A of column i. Its vertical input is the last offset of lane-1's B at column i
    // (lane 0: its own value comes back, which only the barrier offset p = 0 reads).
    const int32_t below = __shfl_up_sync(0xffffffffu, s.HB[C - 1], 1, G);
    systolicSubChunk<C, Checked, Step>(s.HA, s.TA, s.limA, s.i, ai, below, s.HB[0], s.bw, sc, fu);
    // Odd step: sub-chunk B of column i. Its horizontal input is the first offset of lane+1's A at column i-1
    // (lane G-1: its own value comes back, read only by barrier / padding offsets).
    const int32_t top = __shfl_down_sync(0xffffffffu, s.HA[0], 1, G);
    systolicSubChunk<C, Checked, Step>(s.HB, s.TB, s.limB, s.i, ai, s.HA[C - 1], top, s.bw + C, sc, fu);
    if(Checked) {
        // End-cell bookkeeping for both sub-chunks: offsets eA + cStar (row ny) and, in column nx, all rows.
        const int32_t cStar = rowEndA - s.i;
        if((uint32_t(cStar) < uint32_t(2 * C) || s.i == nx) && uint32_t(s.i) <= uint32_t(nx)) {
            systolicEndCells<C>(s.HA, s.limA, eA, s.i, cStar, nx, s.bestScore, s.bestI, s.bestJ);
            systolicEndCells<C>(s.HB, s.limB, eB, s.i, cStar - C, nx, s.bestScore, s.bestI, s.bestJ);
        }
    }
    // Next column: every offset moves one row down.
#pragma unroll
    for(int k = 0; k + 1 < 2 * C; k++) s.bw[k] = s.bw[k + 1];
    s.bw[2 * C - 1] = bIn;
    s.i++; s.ap++; s.bNext++; s.jNext++;
}

template<int G, int C, bool Checked, int... Steps> __device__ __forceinline__ void systolicStepsInPlace(
    SystolicState<C>& s, int32_t eA, int32_t eB, int32_t rowEndA, int32_t nx, int32_t ny, DpScores sc, FmaUnits fu,
    std::integer_sequence<int, Steps...>)
{
    (systolicStep<G, C, Checked, Steps>(s, eA, eB, rowEndA, nx, ny, sc, fu), ...);
}

template<int G, int C, bool Checked> __device__ __forceinline__ void systolicBlock(
    SystolicState<C>& s, int32_t eA, int32_t eB, int32_t rowEndA, int32_t nx, int32_t ny, DpScores sc, FmaUnits fu)
{
    if constexpr(C <= kDpInPlaceTraceMaxC) {
        // Fully unrolled: every step adds its trace code at its own bit position of a cleared word.
#pragma unroll
        for(int c = 0; c < C; c++) { s.TA[c] = 0; s.TB[c] = 0; }
        systolicStepsInPlace<G, C, Checked>(s, eA, eB, rowEndA, nx, ny, sc, fu, std::make_integer_sequence<int, 16>{});
    } else {
        constexpr int kUnroll = (C <= 4) ? 4 : (C <= 8) ? 2 : 1;
#pragma unroll kUnroll
        for(int step = 0; step < 16; step++) systolicStep<G, C, Checked, -1>(s, eA, eB, rowEndA, nx, ny, sc, fu);
    }
}

// The DP of one job on a group of G lanes (G = 32: the whole warp). All 32 lanes of the warp must call it together (the
// shuffles and the block schedule are warp-wide); live = false marks a group without a job (nx = ny = 0, no trace), which
// steps along without storing anything. bestScore / bestI / bestJ end up in every lane of the group.
template<int G, int C> __device__ inline void bandedOverlapDpSystolic(
    const uint32_t* __restrict__ a, uint32_t nxU, const uint32_t* __restrict__ b, uint32_t nyU, int32_t lo, int32_t hi, bool live,
    DpScores sc, FmaUnits fu, uint32_t* __restrict__ trace, int32_t& bestScore, int32_t& bestI, int32_t& bestJ)
{
    const int32_t lane = int32_t(threadIdx.x & unsigned(G - 1));
    const int32_t nx = int32_t(nxU), ny = int32_t(nyU);
    const int32_t W = hi - lo + 1;
    const uint32_t WpadJob = dpBandShape(lo, hi).wpad;
    SystolicState<C> s;
    const int32_t pA = (2 * lane) * C, pB = (2 * lane + 1) * C;         // physical offsets of the lane's sub-chunks
    const int32_t eA = pA - 1, eB = pB - 1;                             // ... as band offsets
#pragma unroll
    for(int c = 0; c < C; c++) { s.HA[c] = kNegInf; s.HB[c] = kNegInf; s.TA[c] = 0; s.TB[c] = 0; }
    initSubChunkLimits<C>(s.limA, pA, W, hi, sc.gap);
    initSubChunkLimits<C>(s.limB, pB, W, hi, sc.gap);
    s.bestScore = kNegInf * 2; s.bestI = kEndCellNone; s.bestJ = kEndCellNone;
    // Only the columns iFirst..iLast hold in-band cells. Column of this lane in step t2 is i = iFirst + t2 - lane;
    // the row of its first offset in that column is jA = eA + i - hi.
    const int32_t iFirst = dpFirstColumn(lo), iLast = dpLastColumn(nxU, nyU, hi);
    s.i = iFirst - lane;
    const int32_t jA = eA + s.i - hi;
    s.ap = a + (int64_t(s.i) - 1);
#pragma unroll
    for(int k = 0; k < 2 * C; k++) {
        const int32_t idx = jA - 1 + k;
        s.bw[k] = 0xffffffffu;
        if(uint32_t(idx) < uint32_t(ny)) s.bw[k] = __ldg(b + idx);
    }
    s.jNext = jA - 1 + 2 * C;
    s.bNext = b + int64_t(s.jNext);
    const int32_t rowEndA = ny + hi - eA;                   // the column in which offset eA reaches the last row
    // Steps run in blocks of 16 (one trace word per offset and block); the last block may run past the step in which
    // lane G-1 reaches column iLast: the cells beyond it feed nothing and their trace codes are never read.
    const int32_t blocks = live ? (iLast - iFirst + G + 15) >> 4 : 0;
    // Boundary cells only occur in columns <= max(0, hi), which lane G-1 leaves after step max(0, hi) - iFirst + G-1.
    // End cells (row ny, column nx) first occur in step min(nx - iFirst, ny + hi - iFirst - 2GC + G): lane 0 reaching
    // column nx, or lane G-1's last offset reaching row ny. The blocks in between run without either test, and in them
    // every lane's column satisfies max(0, hi) < i < nx and every window row (including the element prefetched for the
    // next step) satisfies 1 <= j <= ny, so their loads need no range test: lane 0's barrier offset p = 0 sits on row
    // i - hi - 1 >= 1 because lane 0 is G-1 >= 7 columns ahead of lane G-1, and lane G-1's prefetch index 2GC - 2 + i - hi
    // is at most ny - 1 up to step ny + hi - iFirst - 2GC + G.
    // Several groups share a warp: a block runs unchecked only if it does so for every group, and a group without a job
    // runs every block checked (its loads stay inside its empty rows: none).
    int32_t headBlocks = live ? ((max(0, hi) - iFirst + G - 1) >> 4) + 1 : INT32_MAX;
    const int32_t firstEndStep = min(nx - iFirst, ny + hi - iFirst - 2 * G * C + G);
    int32_t tailBlock = max(0, firstEndStep) >> 4;
    int32_t warpBlocks = blocks;
    if constexpr(G < 32) {
        headBlocks = __reduce_max_sync(0xffffffffu, headBlocks);
        tailBlock = __reduce_min_sync(0xffffffffu, tailBlock);
        warpBlocks = __reduce_max_sync(0xffffffffu, blocks);
    }
    uint32_t* row = trace;
    for(int32_t blk = 0; blk < warpBlocks; blk++, row += WpadJob) {
        if(blk < headBlocks || blk >= tailBlock) systolicBlock<G, C, true>(s, eA, eB, rowEndA, nx, ny, sc, fu);
        else systolicBlock<G, C, false>(s, eA, eB, rowEndA, nx, ny, sc, fu);
        // Group-uniform, coalesced trace store of the block's 16 steps (a group past its last block only steps along).
        if(blk < blocks) {
#pragma unroll
            for(int c = 0; c < C; c++) {
                if(uint32_t(pA + c) < WpadJob) row[pA + c] = s.TA[c];
                if(uint32_t(pB + c) < WpadJob) row[pB + c] = s.TB[c];
            }
        }
    }
    bestScore = s.bestScore; bestI = s.bestI; bestJ = s.bestJ;
    if(bestI != kEndCellNone) bestJ -= hi;          // bestJ was tracked as j + hi
    // Group reduction of the end cell.
#pragma unroll
    for(int d = G / 2; d > 0; d >>= 1) {
        const int32_t s2 = __shfl_xor_sync(0xffffffffu, bestScore, d);
        const int32_t i2 = __shfl_xor_sync(0xffffffffu, bestI, d);
        const int32_t j2 = __shfl_xor_sync(0xffffffffu, bestJ, d);
        if(dpEndCellBetter(s2, i2, j2, bestScore, bestI, bestJ)) { bestScore = s2; bestI = i2; bestJ = j2; }
    }
    if(bestI == kEndCellNone) { bestI = -1; bestJ = -1; }
    __syncwarp();
}

// ---------------------------------------------------------------------------------------------
// Method 3, stage 1 (src/AssemblerAlign3.cpp:62-239): unbanded DP on the downsampled markers, then the band for stage 2.
// Most jobs take method3Stage1ForwardKernel; the others run bandedAlignKernel, tracebackKernel and filterStepsKernel on
// the downsampled markers, and stage1BandKernel derives their band.
struct Method3Args {
    const uint32_t* candidates;     // n x 3 (readId0, readId1, isSameStrand)
    uint64_t candidateBegin; uint32_t n;
    const uint32_t* order;          // job indices of this launch's band class, longest first; n = how many
    const uint64_t* toc;            // global rows (all reads)
    const uint64_t* dsToc; const uint32_t* dsKmer; const uint32_t* dsOrdinal;
    DpScores scores;
    int32_t bandExtend, maxBand;
};

// The stage-2 job of a candidate from its stage-1 path (src/AssemblerAlign3.cpp:185-191, 222-239): the smallest and
// largest ordinal offset over the matching diagonal steps (INT32_MAX / INT32_MIN when none matches), widened by
// bandExtend with the 32-bit wrap-around of the compiled reference, then clipped to the matrix.
__device__ inline void setStage2Band(DpJob& j2, bool diagonalStep, int32_t offsetMin, int32_t offsetMax, int32_t bandExtend, int32_t maxBand)
{
    if(!diagonalStep) { j2.state = kStateEmpty; return; }                                                          // :185-191
    const int32_t bandMin = int32_t(uint32_t(offsetMin) - uint32_t(bandExtend));
    const int32_t bandMax = int32_t(uint32_t(offsetMax) + uint32_t(bandExtend));
    if(int32_t(uint32_t(bandMax) - uint32_t(bandMin)) > maxBand) j2.state = kStateEmpty;
    else if(bandMin > bandMax || bandMax < -int32_t(j2.ny) || bandMin > int32_t(j2.nx)) j2.state = kStateSkipped;  // SeqAn MinValue -> throw
    else {
        j2.lo = max(bandMin, -int32_t(j2.ny));
        j2.hi = min(bandMax, int32_t(j2.nx));
        j2.state = kStateRun;
    }
}

// The job of this lane's group in a kernel that runs 32/G jobs per warp (slots in launch order). A group without a
// runnable job gets an empty one (live = false). Returns false when the whole warp has nothing to run.
template<int G> __device__ __forceinline__ bool dpGroupJob(const uint32_t* __restrict__ order, uint32_t n, const DpJob* __restrict__ jobs,
                                                           uint32_t& warpSlot, uint32_t& p, DpJob& job, bool& live)
{
    warpSlot = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * (32u / G);
    if(warpSlot >= n) return false;
    const uint32_t slot = warpSlot + (threadIdx.x & 31u) / G;
    live = false;
    p = 0;
    if(slot < n) {
        p = order[slot];
        job = jobs[p];
        live = job.state == kStateRun;
    }
    if(!live) { job = DpJob{}; job.state = kStateEmpty; }
    return __any_sync(0xffffffffu, live);
}

// Resident blocks per SM the register allocation of the wavefront kernels aims for (the narrow classes are issue-bound and
// want the warps).
constexpr int dpMinBlocks(int C) { return C <= 2 ? 6 : C == 3 ? 5 : C == 4 ? 4 : C <= 8 ? 2 : 1; }

// Method 3, stage 1 without a trace: the unbanded DP on the downsampled markers only has to deliver the smallest and
// largest ordinal offset over the matching diagonal steps of the optimal path (src/AssemblerAlign3.cpp:193-239), so
// every cell carries that pair along with its score and inherits it from the predecessor the recurrence picks: the
// same information a traceback from that cell would collect, with no trace to write or walk.
// Layout: a job runs on a group of G lanes (G = 8, 16 or 32; 32/G jobs per warp). Lane l of the group owns the R
// consecutive rows j = R*l + 1 .. R*l + R of b (its k-mers and ordinals stay in registers), and in step t works on column
// i = t - l + 1; the only inter-lane traffic is lane l-1's last row (score and pair) of the same column, one step
// earlier. Rows beyond ny and columns outside 1..nx are dead: nothing live reads them.
// Covers ny <= G*R (R <= 16); longer downsampled reads take the trace path (bandedAlignKernel). Same recurrence, tie-break and
// end-cell rules as bandedOverlapDp.
// The (smallest, largest) matching ordinal offset of a path travels as ONE packed value: low half = the smallest offset,
// high half = MINUS the largest, both as signed 16-bit numbers, so that one packed minimum (VIMNMX.S16x2) updates both and
// one select moves both. Offsets are differences of marker ordinals: the forward kernel therefore only takes pairs whose
// reads have at most kStage1ForwardMaxMarkers markers (the others take the trace path).
constexpr uint32_t kPairNoDiagonalStep = 0x7fff7fffu;   // path without diagonal steps
constexpr uint32_t kPairNoMatchingStep = 0x7fff7ffeu;   // ... with diagonal steps, none of them on equal k-mers
constexpr uint32_t kStage1ForwardMaxRows = 512;
constexpr uint32_t kStage1ForwardMaxMarkers = 32000;

__device__ __forceinline__ uint32_t packedAdd16(uint32_t x, uint32_t y)
{
    uint32_t r;
    asm("add.s16x2 %0, %1, %2;" : "=r"(r) : "r"(x), "r"(y));
    return r;
}
__device__ __forceinline__ uint32_t packOffsetPair(int32_t lowHalf, int32_t highHalf)
{
    return (uint32_t(lowHalf) & 0xffffu) | (uint32_t(highHalf) << 16);
}

template<int G, int R> __global__ void __launch_bounds__(kDpMaxWarpsPerBlock * 32)
method3Stage1ForwardKernel(Method3Args g, const DpJob* __restrict__ jobs1, DpJob* __restrict__ jobs2)
{
    const int32_t lane = int32_t(threadIdx.x & unsigned(G - 1));
    uint32_t warpSlot, p;
    DpJob job;
    bool live;
    if(!dpGroupJob<G>(g.order, g.n, jobs1, warpSlot, p, job, live)) return;
    const uint32_t* __restrict__ a = g.dsKmer + job.aOffset;
    const uint32_t* __restrict__ oa = g.dsOrdinal + job.aOffset;
    const int32_t nx = int32_t(job.nx), ny = int32_t(job.ny);
    const DpScores sc = g.scores;

    // This lane's rows of b. boP = (-ordinal, +ordinal) so that (ordinal_a, -ordinal_a) + boP = (offset, -offset).
    uint32_t bk[R], boP[R];
    int32_t H[R];
    uint32_t P[R];                              // column i-1 (then i) of the own rows; column 0 is the boundary
#pragma unroll
    for(int r = 0; r < R; r++) {
        const int32_t j = R * lane + r + 1;
        bk[r] = 0xffffffffu; boP[r] = 0;
        if(j <= ny) {
            bk[r] = __ldg(g.dsKmer + job.bOffset + (j - 1));
            const int32_t ob = int32_t(__ldg(g.dsOrdinal + job.bOffset + (j - 1)));
            boP[r] = packOffsetPair(-ob, ob);
        }
        H[r] = 0; P[r] = kPairNoDiagonalStep;
    }
    const int32_t lastLane = live ? (ny - 1) / R : 0, rLast = live ? (ny - 1) % R : -1;        // where row ny lives
    int32_t upH = 0;                                                    // row R*lane of the previous column
    uint32_t upP = kPairNoDiagonalStep;
    int32_t bestScore = 0, bestI = kEndCellNone, bestJ = kEndCellNone;
    uint32_t bestP = kPairNoDiagonalStep;

    int32_t steps = nx + lastLane;                                      // lanes beyond lastLane only hold dead rows
    if constexpr(G < 32) steps = __reduce_max_sync(0xffffffffu, steps);  // a group past its last step only steps along
#pragma unroll 2
    for(int32_t t = 0; t < steps; t++) {
        // Row R*lane of the current column: lane-1's last row, computed one step ago (row 0 for lane 0).
        int32_t inH = __shfl_up_sync(0xffffffffu, H[R - 1], 1, G);
        uint32_t inP = __shfl_up_sync(0xffffffffu, P[R - 1], 1, G);
        if(lane == 0) { inH = 0; inP = kPairNoDiagonalStep; }
        const int32_t i = t - lane + 1;
        if(uint32_t(i - 1) < uint32_t(nx)) {
            const uint32_t ai = __ldg(a + (i - 1));
            const int32_t ao = int32_t(__ldg(oa + (i - 1)));
            const uint32_t aoP = packOffsetPair(ao, -ao);
            int32_t dH = upH; uint32_t dP = upP;                        // (i-1, j-1)
            int32_t vH = inH; uint32_t vP = inP;                        // (i, j-1)
#pragma unroll
            for(int r = 0; r < R; r++) {
                const int32_t hH = H[r]; const uint32_t hP = P[r];      // (i-1, j)
                const bool eq = (ai == bk[r]);
                const int32_t diag = dH + (eq ? sc.match : sc.mismatch);
                const int32_t gapIn = max(vH, hH);
                const int32_t h = __viaddmax_s32(gapIn, sc.gap, diag);  // tie order: include/shb_dp_policy.h
                const bool viaGap = SHB_DP_DIAG_WINS_TIES ? (h > diag) : (gapIn + sc.gap >= diag), viaHorz = dpHorzWins(hH, vH);
                // a diagonal step: the pair of the diagonal predecessor, extended by this step's offset if the k-mers are equal
                const uint32_t stepP = __vmins2(dP, eq ? packedAdd16(aoP, boP[r]) : kPairNoMatchingStep);
                const uint32_t gapP = viaHorz ? hP : vP;
                const uint32_t pr = viaGap ? gapP : stepP;
                dH = hH; dP = hP;
                vH = h; vP = pr;
                H[r] = h; P[r] = pr;
            }
            // End-cell candidates in column-major order: row ny of the columns before nx, then every row of column nx (the
            // cell (nx, ny) is visited once, after the rows below it). The boundary cell (0, ny) scores 0 and comes
            // first: the start value (score 0, no cell) stands for it, so under the first-maximum rule only positive scores
            // win. The boundary cell (nx, 0) comes after the row-ny cells of the columns before nx: see below the loop.
            if(lane == lastLane && i != nx) {
                int32_t h = 0; uint32_t pr = 0;
                switch(rLast) {                  // group-uniform; a jump instead of R selects per value
#define SHB_PICK_ROW(k) case k: if constexpr(k < R) { h = H[k]; pr = P[k]; } break;
                SHB_PICK_ROW(0) SHB_PICK_ROW(1) SHB_PICK_ROW(2) SHB_PICK_ROW(3) SHB_PICK_ROW(4) SHB_PICK_ROW(5) SHB_PICK_ROW(6) SHB_PICK_ROW(7)
                SHB_PICK_ROW(8) SHB_PICK_ROW(9) SHB_PICK_ROW(10) SHB_PICK_ROW(11) SHB_PICK_ROW(12) SHB_PICK_ROW(13) SHB_PICK_ROW(14) SHB_PICK_ROW(15)
#undef SHB_PICK_ROW
                default: break;
                }
                if(SHB_DP_END_FIRST_MAX ? (h > bestScore) : (h >= bestScore)) { bestScore = h; bestI = i; bestJ = ny; bestP = pr; }
            }
            if(i == nx) {
#pragma unroll
                for(int r = 0; r < R; r++) {
                    const int32_t j = R * lane + r + 1;
                    if(j <= ny && (SHB_DP_END_FIRST_MAX ? (H[r] > bestScore) : (H[r] >= bestScore))) { bestScore = H[r]; bestI = i; bestJ = j; bestP = P[r]; }
                }
            }
        }
        upH = inH; upP = inP;
    }
    if constexpr(!SHB_DP_END_FIRST_MAX) {
        // Under the last-maximum rule the boundary cell (nx, 0) (score 0, empty path) wins a tie with a row-ny cell of an
        // earlier column. It joins here, after the per-lane updates above (whose >= would let such a row-ny cell replace
        // it), and the reduction below orders it among the lanes' candidates.
        if(lane == 0 && dpEndCellBetter(0, nx, 0, bestScore, bestI, bestJ)) { bestScore = 0; bestI = nx; bestJ = 0; bestP = kPairNoDiagonalStep; }
    }
    // Maximum score, then the visiting order of the end-cell rule (over the lanes of the group).
#pragma unroll
    for(int d = G / 2; d > 0; d >>= 1) {
        const int32_t s2 = __shfl_xor_sync(0xffffffffu, bestScore, d);
        const int32_t i2 = __shfl_xor_sync(0xffffffffu, bestI, d);
        const int32_t j2 = __shfl_xor_sync(0xffffffffu, bestJ, d);
        const uint32_t p2 = __shfl_xor_sync(0xffffffffu, bestP, d);
        if(dpEndCellBetter(s2, i2, j2, bestScore, bestI, bestJ)) {
            bestScore = s2; bestI = i2; bestJ = j2; bestP = p2;
        }
    }
    if(lane == 0 && live) {
        DpJob j2 = jobs2[p];
        const uint32_t lowHalf = bestP & 0xffffu;
        const bool noMatch = lowHalf == (kPairNoMatchingStep & 0xffffu);
        setStage2Band(j2, bestI != kEndCellNone && lowHalf != (kPairNoDiagonalStep & 0xffffu),
                      noMatch ? INT32_MAX : int32_t(int16_t(lowHalf)), noMatch ? INT32_MIN : -int32_t(int16_t(bestP >> 16)),
                      g.bandExtend, g.maxBand);
        jobs2[p] = j2;
    }
}

// Stage 2 / generic banded alignment on full marker rows, in three launches:
//   bandedAlignKernel<G,C> one group of G lanes per job: the DP; writes the trace and the end cell;
//   tracebackKernel        one THREAD per job: walks the trace (a serial, latency-bound pointer chase that a warp could
//                          only execute redundantly on its 32 lanes) and writes every diagonal step, last step first;
//   filterStepsKernel      one warp per job: keeps the steps on equal k-mers; counts[p] receives how many.
struct BandedArgs {
    uint32_t n;
    const uint32_t* order;          // job indices of this launch's band class, longest first; n = how many
    const uint32_t* kmerIds;
    DpScores scores;
    FmaUnits fma;                   // {1, 2, 4}: run-time multipliers of the FMA-pipe adds
    uint32_t wMax;                  // widest padded band of this launch's class (sizes the scan kernel's shared memory)
};

template<int G, int C> __global__ void __launch_bounds__(kDpMaxWarpsPerBlock * 32, dpMinBlocks(C))
bandedAlignKernel(BandedArgs g, const DpJob* __restrict__ jobs, uint32_t* __restrict__ trace, int2* __restrict__ endCells)
{
    extern __shared__ int32_t smem[];
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & unsigned(G - 1);
    uint32_t warpSlot, p;
    DpJob job;
    bool live;
    if(!dpGroupJob<G>(g.order, g.n, jobs, warpSlot, p, job, live)) return;
    const uint32_t* a = g.kmerIds + job.aOffset;
    const uint32_t* b = g.kmerIds + job.bOffset;
    int32_t bestScore, bestI, bestJ;
    if constexpr(C > 0) {
        bandedOverlapDpSystolic<G, C>(a, job.nx, b, job.ny, job.lo, job.hi, live, g.scores, g.fma, live ? trace + job.traceOffset : nullptr,
                                      bestScore, bestI, bestJ);
        (void)warp;
    } else {
        static_assert(C > 0 || G == 32, "the scan kernel runs one job per warp");
        const uint32_t stride = g.wMax + 1;
        int32_t* hPrev = smem + warp * 3 * stride;
        int32_t* hCur = hPrev + stride;
        uint32_t* traceAcc = reinterpret_cast<uint32_t*>(hCur + stride);
        bandedOverlapDp(a, job.nx, b, job.ny, job.lo, job.hi, g.scores, hPrev, hCur, traceAcc, trace + job.traceOffset,
                        bestScore, bestI, bestJ);
    }
    if(lane == 0 && live) endCells[p] = make_int2(bestI, bestJ);
}

// A run of consecutive diagonal steps (x0 - k, y0 - k), k = 0 .. length-1, as the traceback emits it (last step first):
// .x = x0 | (length - 1) << 28, .y = y0. Reads have fewer than 2^28 markers (checked by the host).
constexpr uint32_t kRunLengthShift = 28, kRunOrdinalMask = (1u << kRunLengthShift) - 1u;

__device__ __forceinline__ void prefetchL1(const void* p) { asm volatile("prefetch.global.L1 [%0];" :: "l"(p)); }

static __global__ void __launch_bounds__(128)
tracebackKernel(uint32_t n, const uint32_t* __restrict__ order, const DpJob* __restrict__ jobs, const int2* __restrict__ endCells,
                const uint32_t* __restrict__ trace, uint2* __restrict__ runs, uint32_t* __restrict__ runCounts)
{
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if(slot >= n) return;
    const uint32_t p = order[slot];             // neighbouring threads: same band class, similar length
    const DpJob job = jobs[p];
    const int2 end = endCells[p];
    int32_t i = end.x, j = end.y;
    uint32_t count = 0;
    if(job.state == kStateRun && i > 0 && j > 0) {
        const DpShape shape = dpBandShape(job.lo, job.hi);
        const uint32_t Wpad = shape.wpad;
        const DpTraceSteps steps = dpTraceSteps(shape, job.lo);
        const uint32_t* __restrict__ tr = trace + job.traceOffset;
        uint2* __restrict__ out = runs + job.outOffset;
        const int32_t hi = job.hi;
        // One dependent load per iteration; the threads of a warp stay in step (one run or one gap step per iteration).
        uint32_t lastBlock = 0xffffffffu;
        while(i > 0 && j > 0) {
            const uint32_t off = uint32_t(j - i + hi) + 1u;                    // physical offset (barrier at 0)
            const uint32_t t = steps.step(i, off);
            const uint32_t block = t >> 4;
            const uint32_t word = tr[uint64_t(block) * Wpad + off];
            // The walk is a chain of dependent loads, and each 16-step block of the trace is a new DRAM line: ask for the
            // lines of the two blocks above (same offset; the path drifts by a few offsets per block) when a block is entered.
            if(block != lastBlock) {
                lastBlock = block;
                if(block >= 1) prefetchL1(tr + uint64_t(block - 1) * Wpad + off);
                if(block >= 2) prefetchL1(tr + uint64_t(block - 2) * Wpad + off);
            }
            // Diagonal steps stay on the same offset: a run of them is a run of codes without the gap bit going down this
            // word. Bit 0: gap move, bit 1: horizontal; step s of the word at bits 2 * (15 - s).
            const uint32_t q = t & 15u;
            const uint32_t w = word >> (2u * (15u - q));
            const uint32_t gaps = w & 0x55555555u & (q == 15u ? 0xffffffffu : ((1u << (2u * (q + 1u))) - 1u));
            const int32_t run = min(gaps ? ((__ffs(int(gaps)) - 1) >> 1) : int32_t(q) + 1, min(i, j));
            if(run > 0) {
                out[count++] = make_uint2(uint32_t(i - 1) | (uint32_t(run - 1) << kRunLengthShift), uint32_t(j - 1));
                i -= run; j -= run;
            } else if(w & 2u) i--;
            else j--;
        }
    }
    runCounts[p] = count;
}

// Expands the runs of one job (warp per job) into its diagonal steps and keeps, in order, those on equal k-mers
// (src/AssemblerAlign3.cpp:279-295, src/Align4.cpp:1052-1068); counts[p] receives how many.
static __global__ void __launch_bounds__(128)
filterStepsKernel(uint32_t n, const uint32_t* __restrict__ order, const DpJob* __restrict__ jobs, const uint32_t* __restrict__ kmerIds,
                  const uint2* __restrict__ runs, const uint32_t* __restrict__ runCounts, uint2* __restrict__ ordinals,
                  uint32_t* __restrict__ counts)
{
    const uint32_t slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if(slot >= n) return;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t p = order[slot];
    const DpJob job = jobs[p];
    const uint32_t* __restrict__ a = kmerIds + job.aOffset;
    const uint32_t* __restrict__ b = kmerIds + job.bOffset;
    const uint2* __restrict__ in = runs + job.outOffset;
    uint2* __restrict__ out = ordinals + job.outOffset;
    const uint32_t nRuns = runCounts[p];
    uint32_t count = 0;
    for(uint32_t base = 0; base < nRuns; base += 32) {
        // One run per lane; exclusive prefix of the run lengths = index of each run's first step in this group.
        const uint32_t r = base + lane;
        uint2 d = make_uint2(0, 0);
        uint32_t length = 0;
        if(r < nRuns) { d = in[r]; length = (d.x >> kRunLengthShift) + 1u; }
        const uint32_t x0 = d.x & kRunOrdinalMask, y0 = d.y;
        uint32_t inclusive = length;
#pragma unroll
        for(int s = 1; s < 32; s <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, inclusive, s);
            if(lane >= uint32_t(s)) inclusive += v;
        }
        const uint32_t total = __shfl_sync(0xffffffffu, inclusive, 31);
        const uint32_t first = inclusive - length;
        for(uint32_t s0 = 0; s0 < total; s0 += 32) {
            const uint32_t step = s0 + lane;
            // The run that holds this step: the last lane whose first step is <= step (binary search over the lanes;
            // empty trailing lanes have first == total > step).
            uint32_t owner = 0;
#pragma unroll
            for(int w = 16; w > 0; w >>= 1) {
                const uint32_t probe = owner + uint32_t(w);
                const uint32_t v = __shfl_sync(0xffffffffu, first, int(probe & 31u));
                if(v <= step) owner = probe;
            }
            const uint32_t k = step - __shfl_sync(0xffffffffu, first, int(owner));
            const uint32_t x = __shfl_sync(0xffffffffu, x0, int(owner)) - k;
            const uint32_t y = __shfl_sync(0xffffffffu, y0, int(owner)) - k;
            const bool keep = step < total && a[x] == b[y];
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            if(keep) out[count + __popc(m & ((1u << lane) - 1u))] = make_uint2(x, y);
            count += __popc(m);
        }
    }
    if(lane == 0) counts[p] = count;
}

// Method 3, stage 1 of the jobs that took the trace path, after filterStepsKernel on the downsampled markers: the stage-2
// band from the ordinal offsets of the kept steps (runCounts[p] == 0: the path has no diagonal step). One warp per job.
static __global__ void __launch_bounds__(128)
stage1BandKernel(uint32_t n, const uint32_t* __restrict__ order, const DpJob* __restrict__ jobs1, const uint32_t* __restrict__ dsOrdinal,
                 const uint2* __restrict__ ordinals, const uint32_t* __restrict__ runCounts, const uint32_t* __restrict__ counts,
                 int32_t bandExtend, int32_t maxBand, DpJob* __restrict__ jobs2)
{
    const uint32_t slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if(slot >= n) return;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t p = order[slot];
    const DpJob j1 = jobs1[p];
    const uint32_t* __restrict__ oa = dsOrdinal + j1.aOffset;
    const uint32_t* __restrict__ ob = dsOrdinal + j1.bOffset;
    const uint2* __restrict__ kept = ordinals + j1.outOffset;
    const uint32_t count = counts[p];
    int32_t offsetMin = INT32_MAX, offsetMax = INT32_MIN;
    for(uint32_t k = lane; k < count; k += 32) {
        const uint2 s = kept[k];
        const int32_t off = int32_t(oa[s.x]) - int32_t(ob[s.y]);
        offsetMin = min(offsetMin, off);
        offsetMax = max(offsetMax, off);
    }
#pragma unroll
    for(int d = 16; d > 0; d >>= 1) {
        offsetMin = min(offsetMin, __shfl_xor_sync(0xffffffffu, offsetMin, d));
        offsetMax = max(offsetMax, __shfl_xor_sync(0xffffffffu, offsetMax, d));
    }
    if(lane == 0) {
        DpJob j2 = jobs2[p];
        setStage2Band(j2, runCounts[p] != 0, offsetMin, offsetMax, bandExtend, maxBand);
        jobs2[p] = j2;
    }
}

// ---------------------------------------------------------------------------------------------
// Epilogue, one thread per candidate: AlignmentInfo::create (src/Alignment.cpp:67-113), the filters of
// computeAlignmentsThreadFunction (src/AssemblerAlign.cpp:438-483) and the compressed size
// (src/compressAlignment.cpp:11-70). ordinals are stored last-first; entry k of the alignment is
// ord[count-1-k].
struct FilterOptions {
    uint64_t minAlignedMarkerCount, maxSkip, maxDrift, maxTrim;
    double minAlignedFraction;
    uint32_t suppressContainments;
};

// Warp-cooperative walk over the streaks of an alignment (stored last-first). For chunk-of-32 position k the lane
// gets: o = entry k, whether k is the TAIL of a streak (last pair of a run of consecutive diagonal steps), and for
// tails the streak's first index. Used by both epilogue kernels.
struct StreakLane { uint2 o, prev; bool valid, tail; uint32_t start; };

__device__ __forceinline__ StreakLane streakChunk(const uint2* __restrict__ ord, uint32_t count, uint32_t base, uint32_t& carryStart)
{
    const unsigned lane = threadIdx.x & 31u;
    const uint32_t k = base + lane;
    StreakLane r;
    r.valid = k < count;
    r.o = make_uint2(0, 0); r.prev = make_uint2(0, 0);
    uint2 next = make_uint2(0, 0);
    if(r.valid) {
        r.o = ord[count - 1 - k];
        if(k) r.prev = ord[count - k];
        if(k + 1 < count) next = ord[count - 2 - k];
    }
    const bool head = r.valid && (k == 0 || r.o.x != r.prev.x + 1 || r.o.y != r.prev.y + 1);
    r.tail = r.valid && (k + 1 == count || next.x != r.o.x + 1 || next.y != r.o.y + 1);
    const unsigned headMask = __ballot_sync(0xffffffffu, head);
    const unsigned below = headMask & (0xffffffffu >> (31u - lane));       // heads at lanes <= this one
    r.start = below ? (base + 31u - uint32_t(__clz(below))) : carryStart;
    if(headMask) carryStart = base + 31u - uint32_t(__clz(headMask));
    return r;
}

// info words = the 13 words [3..15] of the 64-byte AlignmentData record. One WARP per job.
static __global__ void __launch_bounds__(128)
alignmentInfoKernel(uint32_t n, const DpJob* __restrict__ jobs, const uint2* __restrict__ ordinals,
                    const uint32_t* __restrict__ counts, FilterOptions f,
                    uint32_t* __restrict__ infoWords, uint32_t* __restrict__ keep,
                    uint32_t* __restrict__ compressedBytes, unsigned long long* __restrict__ skippedCounter)
{
    const unsigned lane = threadIdx.x & 31u;
    const uint32_t p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if(p >= n) return;
    const DpJob job = jobs[p];
    if(lane == 0) { keep[p] = 0; compressedBytes[p] = 0; }
    if(job.state == kStateSkipped && skippedCounter && lane == 0) atomicAdd(skippedCounter, 1ull);
    if(job.state != kStateRun) return;
    const uint32_t count = counts[p];
    if(count == 0) return;                               // empty alignments are never stored
    const uint2* ord = ordinals + job.outOffset;
    int32_t mn = INT32_MAX, mx = INT32_MIN;
    uint32_t maxSkip = 0, maxDrift = 0, bytes = 0;
    long long sum = 0;
    uint32_t carryStart = 0;
    for(uint32_t base = 0; base < count; base += 32) {
        const StreakLane s = streakChunk(ord, count, base, carryStart);
        if(s.valid) {
            const int32_t off = int32_t(s.o.x) - int32_t(s.o.y);
            mn = min(mn, off); mx = max(mx, off); sum += off;
            if(base + lane) {
                maxSkip = max(maxSkip, uint32_t(abs(int32_t(s.o.x) - int32_t(s.prev.x))));
                maxSkip = max(maxSkip, uint32_t(abs(int32_t(s.o.y) - int32_t(s.prev.y))));
                maxDrift = max(maxDrift, uint32_t(abs(off - (int32_t(s.prev.x) - int32_t(s.prev.y)))));
            }
        }
        if(s.tail) {
            const uint2 first = ord[count - 1 - s.start];
            const uint2 before = s.start ? ord[count - s.start] : make_uint2(0, 0);
            bytes += compressedStreakBytes(int32_t(first.x) - int32_t(before.x), int32_t(first.y) - int32_t(before.y),
                                           base + lane - s.start + 1);
        }
    }
#pragma unroll
    for(int d = 16; d > 0; d >>= 1) {
        mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, d));
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
        maxSkip = max(maxSkip, __shfl_xor_sync(0xffffffffu, maxSkip, d));
        maxDrift = max(maxDrift, __shfl_xor_sync(0xffffffffu, maxDrift, d));
        bytes += __shfl_xor_sync(0xffffffffu, bytes, d);
        sum += __shfl_xor_sync(0xffffffffu, sum, d);
    }
    if(lane != 0) return;
    const uint2 first = ord[count - 1], last = ord[0];
    // Filters, in the reference's order.
    if(uint64_t(count) < f.minAlignedMarkerCount) return;
    const double frac0 = double(count) / double(last.x + 1 - first.x);
    const double frac1 = double(count) / double(last.y + 1 - first.y);
    if(min(frac0, frac1) < f.minAlignedFraction) return;
    const uint32_t leftTrim = min(first.x, first.y);
    const uint32_t rightTrim = min(job.nx - 1 - last.x, job.ny - 1 - last.y);
    if(leftTrim > f.maxTrim || rightTrim > f.maxTrim) return;
    if(uint64_t(maxSkip) > f.maxSkip) return;
    if(uint64_t(maxDrift) > f.maxDrift) return;
    if(f.suppressContainments) {
        const uint32_t mt = uint32_t(f.maxTrim);
        if((first.x <= mt && job.nx - 1 - last.x <= mt) || (first.y <= mt && job.ny - 1 - last.y <= mt)) return;
    }
    uint32_t* w = infoWords + 13ull * p;
    w[0] = job.nx; w[1] = first.x; w[2] = last.x;
    w[3] = job.ny; w[4] = first.y; w[5] = last.y;
    w[6] = count; w[7] = uint32_t(mn); w[8] = uint32_t(mx);
    w[9] = uint32_t(int32_t(round(double(sum) / double(count))));
    w[10] = maxSkip; w[11] = maxDrift; w[12] = 0;
    keep[p] = 1;
    compressedBytes[p] = bytes;
}

// One WARP per kept candidate: 64-byte AlignmentData record + compressed alignment bytes.
// jobIndex maps a candidate to the DP job that produced its alignment (NULL = identity, method 3).
static __global__ void __launch_bounds__(128)
alignmentWriteKernel(uint32_t n, const uint32_t* __restrict__ candidates, const DpJob* __restrict__ jobs,
                     const uint2* __restrict__ ordinals, const uint32_t* __restrict__ counts,
                     const uint32_t* __restrict__ infoWords, const uint32_t* __restrict__ jobIndex,
                     const uint32_t* __restrict__ keep,
                     const uint32_t* __restrict__ keepIndex, const unsigned long long* __restrict__ byteOffsets,
                     uint64_t recordBase, uint64_t byteBase,
                     uint32_t* __restrict__ records, unsigned long long* __restrict__ compressedToc,
                     uint8_t* __restrict__ compressedData)
{
    const unsigned lane = threadIdx.x & 31u;
    const uint32_t p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if(p >= n || !keep[p]) return;
    const uint32_t j = jobIndex ? jobIndex[p] : p;
    const uint64_t r = recordBase + keepIndex[p];
    uint32_t* rec = records + 16ull * r;
    if(lane < 3) rec[lane] = (lane == 2) ? (candidates[3ull * p + 2] & 0xffu) : candidates[3ull * p + lane];
    else if(lane < 16) rec[lane] = infoWords[13ull * j + (lane - 3)];
    const uint64_t byteOffset = byteBase + byteOffsets[p];
    if(lane == 0) compressedToc[r] = byteOffset;
    uint8_t* out = compressedData + byteOffset;
    const uint32_t count = counts[j];
    const uint2* ord = ordinals + jobs[j].outOffset;
    uint32_t carryStart = 0, written = 0;
    for(uint32_t base = 0; base < count; base += 32) {
        const StreakLane s = streakChunk(ord, count, base, carryStart);
        int32_t skip0 = 0, skip1 = 0;
        uint32_t len = 0, bytes = 0;
        if(s.tail) {
            const uint2 first = ord[count - 1 - s.start];
            const uint2 before = s.start ? ord[count - s.start] : make_uint2(0, 0);
            skip0 = int32_t(first.x) - int32_t(before.x);
            skip1 = int32_t(first.y) - int32_t(before.y);
            len = base + lane - s.start + 1;
            bytes = compressedStreakBytes(skip0, skip1, len);
        }
        // Exclusive prefix of the streak sizes inside the chunk.
        uint32_t inc = bytes;
#pragma unroll
        for(int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
            if(lane >= (unsigned)d) inc += t;
        }
        if(s.tail) writeCompressedStreak(out + written + inc - bytes, skip0, skip1, len);
        written += __shfl_sync(0xffffffffu, inc, 31);
    }
}

} // namespace shb

namespace shb {

// Per-candidate job setup (src/AssemblerAlign.cpp:376-382): oriented reads (readId0, strand 0) and
// (readId1, sameStrand ? 0 : 1); stage-1 job on the downsampled rows, stage-2 job skeleton on the full rows.
// maxWidth: widest padded band the DP kernels take (kMaxBandWidth); a candidate whose unbanded stage needs more is
// skipped and counted (tooWide), not the whole call (the reference has no such limit: documented deviation).
// dsToc == nullptr: method 1 (src/AssemblerAlign1.cpp:129-148), no stage 1, the stage-2 job covers the whole matrix.
static __global__ void method3SetupKernel(const uint32_t* __restrict__ candidates, uint32_t n,
                                          const uint64_t* __restrict__ toc, const uint64_t* __restrict__ dsToc,
                                          DpJob* __restrict__ jobs1, DpJob* __restrict__ jobs2,
                                          unsigned long long* __restrict__ traceWords1, unsigned long long* __restrict__ outCount,
                                          unsigned long long* __restrict__ forwardCells, uint32_t maxWidth,
                                          unsigned long long* __restrict__ tooWide)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if(p >= n) return;
    uint64_t o0, o1;
    candidateOrientedReads(candidates, p, o0, o1);
    DpJob j1, j2;
    if(dsToc == nullptr) {
        j2.aOffset = toc[o0]; j2.nx = uint32_t(toc[o0 + 1] - toc[o0]);
        j2.bOffset = toc[o1]; j2.ny = uint32_t(toc[o1 + 1] - toc[o1]);
        j2.lo = -int32_t(j2.ny); j2.hi = int32_t(j2.nx); j2.traceOffset = 0; j2.outOffset = 0; j2.pad = 0;
        j2.state = (j2.nx == 0 || j2.ny == 0) ? kStateEmpty : kStateRun;
        if(j2.state == kStateRun && dpBandShape(j2.lo, j2.hi).wpad > maxWidth) { j2.state = kStateSkipped; atomicAdd(tooWide, 1ull); }
        jobs2[p] = j2;
        outCount[p] = min(j2.nx, j2.ny);
        return;
    }
    j1.aOffset = dsToc[o0]; j1.nx = uint32_t(dsToc[o0 + 1] - dsToc[o0]);
    j1.bOffset = dsToc[o1]; j1.ny = uint32_t(dsToc[o1 + 1] - dsToc[o1]);
    j1.lo = -int32_t(j1.ny); j1.hi = int32_t(j1.nx);
    j1.traceOffset = 0; j1.outOffset = 0;
    j1.state = (j1.nx == 0 || j1.ny == 0) ? kStateEmpty : kStateRun;       // src/AssemblerAlign3.cpp:100-106
    j2.aOffset = toc[o0]; j2.nx = uint32_t(toc[o0 + 1] - toc[o0]);
    j2.bOffset = toc[o1]; j2.ny = uint32_t(toc[o1 + 1] - toc[o1]);
    j2.lo = 0; j2.hi = 0; j2.traceOffset = 0; j2.outOffset = 0; j2.pad = 0;
    // Only the jobs that the forward kernel cannot take need a trace: too many downsampled rows, or reads so long that an
    // ordinal offset does not fit the kernel's 16-bit offset pair. pad = 1 marks the forward-kernel jobs for the class sort.
    const bool forward = j1.ny <= kStage1ForwardMaxRows && max(j2.nx, j2.ny) <= kStage1ForwardMaxMarkers;
    j1.pad = forward ? 1u : 0u;
    if(j1.state == kStateRun && !forward && dpBandShape(j1.lo, j1.hi).wpad > maxWidth) {
        j1.state = kStateSkipped; atomicAdd(tooWide, 1ull);
    }
    j2.state = (j1.state == kStateEmpty) ? kStateEmpty : kStateSkipped;     // stage 1 overwrites it when it runs
    jobs1[p] = j1; jobs2[p] = j2;
    traceWords1[p] = (j1.state == kStateRun && !forward) ? dpTraceWords(j1.nx, j1.ny, j1.lo, j1.hi) : 0ull;
    if(j1.state == kStateRun && forward) atomicAdd(forwardCells, (unsigned long long)j1.nx * j1.ny);
    outCount[p] = min(j2.nx, j2.ny);
}

static __global__ void setTraceOffsetsKernel(DpJob* __restrict__ jobs, uint32_t n, const unsigned long long* __restrict__ traceOffsets,
                                             const unsigned long long* __restrict__ outOffsets)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if(p >= n) return;
    jobs[p].traceOffset = traceOffsets[p];
    jobs[p].outOffset = outOffsets[p];
}

// Classes of the forward kernel (method 3, stage 1 without a trace): groups of `lanes` lanes with `rows` rows per lane
// hold ny <= lanes * rows downsampled markers: steps of 8 rows up to 128 on groups of 8 lanes, of 16 up to 256 on groups
// of 16, then 384 and 512 on whole warps.
struct DpForwardClass { uint32_t lanes, rows; };
constexpr uint32_t kDpForwardClassCount = 26;
__host__ __device__ constexpr DpForwardClass dpForwardClassAt(uint32_t k)
{
    return k < 16 ? DpForwardClass{8u, k + 1u} : k < 24 ? DpForwardClass{16u, k - 7u} : DpForwardClass{32u, k == 24 ? 12u : 16u};
}
static_assert(dpForwardClassAt(kDpForwardClassCount - 1).lanes * dpForwardClassAt(kDpForwardClassCount - 1).rows == kStage1ForwardMaxRows,
              "the forward classes cover every row count the forward kernel takes");

constexpr int kDpLengthKeyBits = 10, kDpClassKeyBits = 6;
constexpr uint32_t kDpLengthKeyMax = (1u << kDpLengthKeyBits) - 1u, kDpClassNone = (1u << kDpClassKeyBits) - 1u;
static_assert(kDpForwardClassCount + kDpClassCount < kDpClassNone, "class key too narrow");

// Sort key of a DP job: class, then longest first (load balance inside a launch; the jobs that share a warp differ by
// less than one 16-step block). Band class: dpBandShape; jobs that do not run get class kDpClassNone.
// forward (method 3, stage 1): the jobs marked for the forward kernel take its classes (dpForwardClassAt), the others
// their band class, shifted up by kDpForwardClassCount.
static __global__ void dpClassKeysKernel(const DpJob* __restrict__ jobs, uint32_t n, bool forward, uint64_t* __restrict__ keys,
                                         uint32_t* __restrict__ vals)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if(p >= n) return;
    const DpJob j = jobs[p];
    uint32_t cls = kDpClassNone;
    if(j.state == kStateRun) {
        if(forward && j.pad) {                  // marked by method3SetupKernel: few enough rows and short enough reads
            for(uint32_t k = 0; k < kDpForwardClassCount; k++) {
                const DpForwardClass f = dpForwardClassAt(k);
                if(j.ny <= f.lanes * f.rows) { cls = k; break; }
            }
        } else {
            const DpShape s = dpBandShape(j.lo, j.hi);
            if(s.wpad <= dpClassAt(s.cls).wMax) cls = (forward ? kDpForwardClassCount : 0u) + s.cls;
        }
    }
    // 16-bit key (two radix passes): class, then the number of columns the kernel visits in units of 16, longest first.
    const int32_t active = dpLastColumn(j.nx, j.ny, j.hi) - dpFirstColumn(j.lo);
    const uint32_t length = min(uint32_t(active > 0 ? active : 0) >> 4, kDpLengthKeyMax);
    keys[p] = (uint64_t(cls) << kDpLengthKeyBits) | uint64_t(kDpLengthKeyMax - length);
    vals[p] = p;
}

static __global__ void stage2TraceWordsKernel(const DpJob* __restrict__ jobs, uint32_t n, unsigned long long* __restrict__ traceWords)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if(p >= n) return;
    const DpJob j = jobs[p];
    traceWords[p] = (j.state == kStateRun) ? dpTraceWords(j.nx, j.ny, j.lo, j.hi) : 0ull;
}

// In-band, in-matrix cells of the banded jobs (what the reference's DP fills): per column i the rows max(0, i - hi) ..
// min(ny, i - lo). counter += the total over the runnable jobs.
static __global__ void bandCellsKernel(const DpJob* __restrict__ jobs, uint32_t n, unsigned long long* __restrict__ counter)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long cells = 0;
    if(p < n) {
        const DpJob j = jobs[p];
        if(j.state == kStateRun) {
            // Sum over the columns a..b of  min(ny, i - lo) - max(0, i - hi) + 1  (positive for every such column), as two
            // arithmetic series: the bottom edge grows with i up to column ny + lo, the top edge from column hi + 1 on.
            const long long nx = j.nx, ny = j.ny, lo = j.lo, hi = j.hi;
            const long long a = max(0ll, lo), b = min(nx, ny + hi);
            if(b >= a) {
                long long total = b - a + 1;                                    // the "+ 1" of every column
                const long long c = min(b, ny + lo);                            // last column whose bottom edge is i - lo
                if(c >= a) total += (c - a + 1) * (a + c) / 2 - lo * (c - a + 1);
                total += (b - max(c, a - 1)) * ny;                               // columns with bottom edge ny
                const long long d = max(a, hi + 1);                             // first column whose top edge is i - hi
                if(d <= b) total -= (b - d + 1) * (d + b) / 2 - hi * (b - d + 1);
                cells = (unsigned long long)total;
            }
        }
    }
#pragma unroll
    for(int d = 16; d > 0; d >>= 1) cells += __shfl_xor_sync(0xffffffffu, cells, d);
    if((threadIdx.x & 31u) == 0 && cells) atomicAdd(counter, cells);
}

} // namespace shb

// =============================================================================================
// Method 4 (Align4) front end — src/Align4.cpp:195-868, one warp per candidate.
// Only the NUMBER of alignment-matrix entries per (iX,iY) cell matters to the reference (createCells,
// :380-436), so the sparse matrix is a dense count grid in global scratch. Then: cell flags, forward /
// backward reachability (children (iX+{0,1}, iY+{-1,0,1}), :682-787), 8-neighbourhood components of the
// active cells (:792-868) and one band per component (:890-934), in raster order of each component's
// first cell (the reference's order depends on std::unordered_map iteration; it only matters when two kept
// components tie on markerCount, see DESIGN.md).
namespace shb {

struct Align4Args {
    const uint32_t* candidates; uint32_t n;
    const uint64_t* toc;
    const uint32_t* sortedKmer; const uint32_t* sortedOrdinal;     // per oriented read, sorted by kmerId
    uint32_t deltaX, deltaY;
    uint64_t minEntryCountPerCell, maxDistanceFromBoundary;
    int64_t maxBand;
    const unsigned long long* cellOffsets;      // per candidate: first cell of its scratch (exclusive scan of cell counts)
    uint32_t* counts;       // per cell: match count, later component label / YMin
    uint32_t* aux;          // per cell: YMax per component root
    uint32_t* list;         // per cell: compact list of existing cells (raster indices)
    uint8_t* flags;         // per cell: 1 exists, 2 nearLeftOrTop, 4 nearRightOrBottom, 8 forward, 16 backward
    int32_t* bands;         // per cell: (bandMin, bandMax) per component, compact, 2 ints each
    uint32_t* componentCount;   // per candidate
};

__device__ __forceinline__ void align4GridSize(uint32_t nx, uint32_t ny, uint32_t deltaX, uint32_t deltaY, uint32_t& nIX, uint32_t& nIY)
{
    if(nx == 0 || ny == 0) { nIX = 0; nIY = 0; return; }
    const uint32_t sizeXY = nx + ny - 1;
    nIX = (sizeXY - 1) / deltaX + 1;
    nIY = (sizeXY - 1) / deltaY + 1;
}

static __global__ void align4CellCountKernel(const uint32_t* __restrict__ candidates, uint32_t n, const uint64_t* __restrict__ toc,
                                             uint32_t deltaX, uint32_t deltaY, unsigned long long* __restrict__ cellCounts)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if(p >= n) return;
    uint64_t o0, o1;
    candidateOrientedReads(candidates, p, o0, o1);
    uint32_t nIX, nIY;
    align4GridSize(uint32_t(toc[o0 + 1] - toc[o0]), uint32_t(toc[o1 + 1] - toc[o1]), deltaX, deltaY, nIX, nIY);
    cellCounts[p] = (unsigned long long)nIX * nIY + 2;      // +2: room for one degenerate band
}

__device__ __forceinline__ void align4Getxy(int32_t X, int32_t Y, int32_t nx, int32_t& x, int32_t& y)
{
    x = (X - Y + nx - 1) / 2;       // C division truncates toward zero, as in src/Align4.cpp:183-191
    y = (X + Y - nx + 1) / 2;
}

// The cell that holds alignment-matrix entry (x, y) of a grid with nIX cells per row.
struct Align4Grid {
    uint32_t nx, ny, nIX, nIY, nCells;
    uint64_t aBegin, bBegin, base;
};
__device__ __forceinline__ Align4Grid align4Grid(const Align4Args& g, uint32_t p)
{
    uint64_t o0, o1;
    candidateOrientedReads(g.candidates, p, o0, o1);
    Align4Grid r;
    r.aBegin = g.toc[o0]; r.bBegin = g.toc[o1];
    r.nx = uint32_t(g.toc[o0 + 1] - r.aBegin); r.ny = uint32_t(g.toc[o1 + 1] - r.bBegin);
    align4GridSize(r.nx, r.ny, g.deltaX, g.deltaY, r.nIX, r.nIY);
    r.nCells = r.nIX * r.nIY;
    r.base = g.cellOffsets[p];
    return r;
}

// Cell flags of createCells (:380-436): 1 exists, 2|8 near the left / top boundary (forward seeds), 4 near right / bottom.
__device__ __forceinline__ uint8_t align4CellFlags(const Align4Args& g, const Align4Grid& G, uint32_t iX, uint32_t iY)
{
    const int32_t nx = int32_t(G.nx), ny = int32_t(G.ny);
    int32_t x, y;
    align4Getxy(int32_t(iX * g.deltaX), int32_t((iY + 1) * g.deltaY), nx, x, y);
    const uint32_t dLeft = x < 0 ? 0u : uint32_t(x);
    align4Getxy(int32_t((iX + 1) * g.deltaX), int32_t(iY * g.deltaY), nx, x, y);
    const uint32_t dRight = (x >= nx - 1) ? 0u : uint32_t(nx - 1 - x);
    align4Getxy(int32_t(iX * g.deltaX), int32_t(iY * g.deltaY), nx, x, y);
    const uint32_t dTop = y < 0 ? 0u : uint32_t(y);
    align4Getxy(int32_t((iX + 1) * g.deltaX), int32_t((iY + 1) * g.deltaY), nx, x, y);
    const uint32_t dBottom = (y >= ny - 1) ? 0u : uint32_t(ny - 1 - y);
    uint8_t f = 1;
    if(uint64_t(dLeft) < g.maxDistanceFromBoundary || uint64_t(dTop) < g.maxDistanceFromBoundary) f |= 2 | 8;   // seeds are forward accessible
    if(uint64_t(dRight) < g.maxDistanceFromBoundary || uint64_t(dBottom) < g.maxDistanceFromBoundary) f |= 4;
    return f;
}

// Front end, kernel 1 of 2, one warp per candidate: createAlignmentMatrix (:195-267) as a dense grid of entry counts in
// global scratch. Every pair of equal k-mers (x in read 0, y in read 1) adds one entry to cell (X/deltaX, Y/deltaY),
// X = x + y, Y = y + nx - 1 - x. The cell whose count reaches the existence threshold of createCells is appended (in
// any order) to the candidate's cell list; listCount (= componentCount[p] until kernel 2 overwrites it) counts them.
static __global__ void __launch_bounds__(128) align4MatrixKernel(Align4Args g)
{
    const unsigned lane = threadIdx.x & 31u;
    const uint32_t p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if(p >= g.n) return;
    const Align4Grid G = align4Grid(g, p);
    const uint32_t nx = G.nx, ny = G.ny, nIX = G.nIX, nCells = G.nCells;
    uint32_t* counts = g.counts + G.base;
    uint32_t* list = g.list + G.base;
    uint8_t* flags = g.flags + G.base;
    if(lane == 0) g.componentCount[p] = 0;
    if(nCells == 0) return;
    for(uint32_t i = lane; i < nCells; i += 32) { counts[i] = 0; flags[i] = 0; }
    __syncwarp();
    // A cell exists when its count is positive and not below minEntryCountPerCell (:398-402).
    const int64_t minEntries = int64_t(g.minEntryCountPerCell);
    const uint32_t threshold = minEntries <= 1 ? 1u : (minEntries > int64_t(0xffffffffu) ? 0xffffffffu : uint32_t(minEntries));
    const uint32_t* sa = g.sortedKmer + G.aBegin; const uint32_t* oa = g.sortedOrdinal + G.aBegin;
    const uint32_t* sb = g.sortedKmer + G.bBegin; const uint32_t* ob = g.sortedOrdinal + G.bBegin;
    for(uint32_t t = lane; t < nx; t += 32) {
        const uint32_t kmer = sa[t];
        uint32_t lo = 0, hi = ny;               // lower bound of kmer in sb
        while(lo < hi) { const uint32_t mid = (lo + hi) >> 1; if(sb[mid] < kmer) lo = mid + 1; else hi = mid; }
        const uint32_t x = oa[t];
        for(uint32_t q = lo; q < ny && sb[q] == kmer; q++) {
            const uint32_t y = ob[q];
            const uint32_t X = x + y, Y = nx + y - x - 1;
            const uint32_t cell = (Y / g.deltaY) * nIX + X / g.deltaX;
            if(atomicAdd(&counts[cell], 1u) + 1u == threshold) list[atomicAdd(&g.componentCount[p], 1u)] = cell;
        }
    }
}

// Front end, kernel 2 of 2, one warp per candidate: cell flags, forward / backward reachability, components, bands.
// A true overlap leaves a few cells per grid column (100 - 300 for a pair of ultra-long reads, out of 10^4 - 10^5 grid
// cells), and the three fixpoints over them are chains of dependent neighbour reads: with the existing cells in shared
// memory (sorted raster indices, an 8-neighbour slot table built once by binary search, flags, labels) a sweep costs
// shared-memory latencies instead of global ones. Candidates with more existing cells than fit take the global path.
// Both paths run the same steps (align4ComponentBands) through a view of where the cells are stored.
constexpr uint32_t kAlign4SmemCells = 512;
constexpr uint32_t kAlign4WarpsPerBlock = 2;
constexpr uint16_t kAlign4NoSlot = 0xffffu;

// A candidate's existing cells as kernel 2 sees them. Cell t of the list in raster order has the id id(t); ids increase
// in raster order. neighbour(c, k) is the id of the cell at (iX + k % 3 - 1, iY + k / 3 - 1) of cell c, or kNone; a
// cell that does not exist has flags 0. The flags, the label and the YMax of a component root are stored by id;
// activeLabel(q) is the label of q if q is active, else kNone.
// Shared memory: the id is the cell's slot in the sorted list, neighbours come from the slot table (existing cells only).
struct Align4SharedCells {
    using Id = uint32_t;
    static constexpr Id kNone = kAlign4NoSlot;
    const uint32_t* sRow; const uint16_t (*sNbr)[9]; uint8_t* sFlag; uint16_t* sLabel; uint32_t* sYMax;
    __device__ Id id(uint32_t t) const { return t; }
    __device__ uint32_t row(Id c) const { return sRow[c]; }
    __device__ Id neighbour(Id c, int k) const { return sNbr[c][k]; }
    __device__ uint8_t& flag(Id c) const { return sFlag[c]; }
    __device__ uint16_t& label(Id c) const { return sLabel[c]; }
    __device__ Id activeLabel(Id c) const { return sLabel[c]; }            // inactive cells carry kNone
    __device__ uint32_t& yMax(Id c) const { return sYMax[c]; }
};
// The dense grid in global scratch: the id is the raster index. A cell that does not exist keeps its entry count in
// counts[], so only an active cell's counts[] is a label.
struct Align4GridCells {
    using Id = uint32_t;
    static constexpr Id kNone = 0xffffffffu;
    const uint32_t* list; uint32_t nIX, nIY; uint8_t* flags; uint32_t* counts; uint32_t* aux;
    __device__ Id id(uint32_t t) const { return list[t]; }
    __device__ uint32_t row(Id c) const { return c / nIX; }
    __device__ Id neighbour(Id c, int k) const
    {
        const int32_t qX = int32_t(c % nIX) + k % 3 - 1, qY = int32_t(c / nIX) + k / 3 - 1;
        return (uint32_t(qX) >= nIX || uint32_t(qY) >= nIY) ? kNone : uint32_t(qY) * nIX + uint32_t(qX);
    }
    __device__ uint8_t& flag(Id c) const { return flags[c]; }
    __device__ Id& label(Id c) const { return counts[c]; }
    __device__ Id activeLabel(Id c) const { return (flags[c] & 24) == 24 ? counts[c] : kNone; }
    __device__ uint32_t& yMax(Id c) const { return aux[c]; }
};

// forwardSearch (:682-729): a cell is forward accessible (flag 8) if one of its parents (iX - {0,1}, iY - {-1,0,1}) is.
// backwardSearch (:736-787): a cell is backward accessible (flag 16) if one of its children (iX + {0,1}, iY + {-1,0,1}) is.
template<bool kForward, class Cells>
__device__ __forceinline__ void align4Search(const Cells& v, uint32_t n)
{
    constexpr uint8_t kBit = kForward ? 8 : 16;
    for(;;) {
        bool changed = false;
        for(uint32_t t = threadIdx.x & 31u; t < n; t += 32) {
            const typename Cells::Id c = v.id(t);
            const uint8_t f = v.flag(c);
            if(f & kBit) continue;
            bool reach = false;
#pragma unroll
            for(int e = 0; e < 5; e++) {
                constexpr int kParents[5] = {7, 6, 3, 1, 0}, kChildren[5] = {8, 7, 5, 2, 1};
                const typename Cells::Id q = v.neighbour(c, kForward ? kParents[e] : kChildren[e]);
                if(q != Cells::kNone && (v.flag(q) & kBit)) reach = true;
            }
            if(reach) { v.flag(c) = f | kBit; changed = true; }
        }
        __syncwarp();
        if(!__any_sync(0xffffffffu, changed)) break;
    }
}

// Kernel 2 after the cell flags, on the n cells of the view: reachability, components of the active cells, and one band
// per component into the candidate's bands; componentCount[p] = the number of bands.
template<class Cells>
__device__ __forceinline__ void align4ComponentBands(const Cells& v, uint32_t n, const Align4Args& g, uint32_t p, const Align4Grid& G)
{
    using Id = typename Cells::Id;
    const unsigned lane = threadIdx.x & 31u;
    align4Search<true>(v, n);
    // backwardSearch seeds: near right / bottom and forward accessible.
    for(uint32_t t = lane; t < n; t += 32) {
        const Id c = v.id(t);
        const uint8_t f = v.flag(c);
        if((f & 4) && (f & 8)) v.flag(c) = f | 16;
    }
    __syncwarp();
    align4Search<false>(v, n);
    // Connected components of the active cells (8-neighbourhood): min-label propagation. Ids are in raster order, so a
    // component's label ends up as the id of its first cell in raster order, its root.
    for(uint32_t t = lane; t < n; t += 32) {
        const Id c = v.id(t);
        v.label(c) = ((v.flag(c) & 24) == 24) ? c : Cells::kNone;
        v.yMax(c) = 0;
    }
    __syncwarp();
    for(;;) {
        bool changed = false;
        for(uint32_t t = lane; t < n; t += 32) {
            const Id c = v.id(t);
            const Id label = v.label(c);
            if(label == Cells::kNone) continue;
            Id best = label;
#pragma unroll
            for(int k = 0; k < 9; k++) {
                if(k == 4) continue;
                const Id q = v.neighbour(c, k);
                if(q != Cells::kNone) best = min(best, v.activeLabel(q));     // kNone is the largest value
            }
            if(best < label) { v.label(c) = best; changed = true; }
        }
        __syncwarp();
        if(!__any_sync(0xffffffffu, changed)) break;
    }
    // YMax per component at its root; the root's own row is its YMin.
    for(uint32_t t = lane; t < n; t += 32) {
        const Id c = v.id(t);
        const Id label = v.label(c);
        if(label != Cells::kNone) atomicMax(&v.yMax(label), v.row(c));
    }
    __syncwarp();
    // One band per component (:890-934), components in raster order of their first cell; too-wide bands dropped.
    int32_t* bands = g.bands + G.base;
    const uint32_t nx = G.nx;
    uint32_t nBands = 0;
    for(uint32_t t0 = 0; t0 < n; t0 += 32) {
        const uint32_t t = t0 + lane;
        bool emit = false;
        int32_t bandMin = 0, bandMax = 0;
        if(t < n) {
            const Id c = v.id(t);
            if(v.label(c) == c) {
                const uint32_t YMin = v.row(c) * g.deltaY, YMax = (v.yMax(c) + 1) * g.deltaY - 1;
                bandMin = int32_t(nx) - 1 - int32_t(YMax);
                bandMax = int32_t(nx) - 1 - int32_t(YMin);
                emit = !(int64_t(bandMax - bandMin + 1) > g.maxBand);
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, emit);
        if(emit) {
            const uint32_t slot = nBands + __popc(m & ((1u << lane) - 1u));
            bands[2 * slot] = bandMin;
            bands[2 * slot + 1] = bandMax;
        }
        nBands += __popc(m);
    }
    __syncwarp();
    if(lane == 0) g.componentCount[p] = nBands;
}

// Kernel 2 on the dense global grid (any number of existing cells): createCells (:380-436) writes the flags, and a scan
// of the grid lists the existing cells in raster order. Out of line, so that the shared-memory path keeps its registers.
__device__ __noinline__ void align4GridComponents(const Align4Args& g, uint32_t p, const Align4Grid& G)
{
    const unsigned lane = threadIdx.x & 31u;
    const uint32_t nCells = G.nCells;
    uint32_t* list = g.list + G.base;
    const Align4GridCells v{list, G.nIX, G.nIY, g.flags + G.base, g.counts + G.base, g.aux + G.base};
    uint32_t listSize = 0;
    for(uint32_t i0 = 0; i0 < nCells; i0 += 32) {
        const uint32_t i = i0 + lane;
        bool exists = false;
        if(i < nCells) {
            const uint32_t cnt = v.counts[i];
            exists = cnt > 0 && !(int64_t(cnt) < int64_t(g.minEntryCountPerCell));
            if(exists) v.flags[i] = align4CellFlags(g, G, i % G.nIX, i / G.nIX);
        }
        const unsigned m = __ballot_sync(0xffffffffu, exists);
        if(exists) list[listSize + __popc(m & ((1u << lane) - 1u))] = i;
        listSize += __popc(m);
    }
    __syncwarp();
    align4ComponentBands(v, listSize, g, p, G);
}

static __global__ void __launch_bounds__(kAlign4WarpsPerBlock * 32) align4ComponentsKernel(Align4Args g, uint32_t smemCells)
{
    __shared__ uint32_t sIdxAll[kAlign4WarpsPerBlock][kAlign4SmemCells];          // raster index, later the cell's row iY
    __shared__ uint32_t sYMaxAll[kAlign4WarpsPerBlock][kAlign4SmemCells];
    __shared__ uint16_t sNbrAll[kAlign4WarpsPerBlock][kAlign4SmemCells][9];       // slot of neighbour (oY+1)*3 + (oX+1)
    __shared__ uint16_t sLabelAll[kAlign4WarpsPerBlock][kAlign4SmemCells];
    __shared__ uint8_t sFlagAll[kAlign4WarpsPerBlock][kAlign4SmemCells];
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t p = blockIdx.x * kAlign4WarpsPerBlock + warp;
    if(p >= g.n) return;
    const Align4Grid G = align4Grid(g, p);
    if(G.nCells == 0) { if(lane == 0) g.componentCount[p] = 0; return; }
    const uint32_t n = g.componentCount[p];                 // existing cells (kernel 1)
    if(n > smemCells) { align4GridComponents(g, p, G); return; }
    if(n == 0) return;                                      // no cells, no components: componentCount[p] is already 0
    uint32_t* sIdx = sIdxAll[warp]; uint32_t* sYMax = sYMaxAll[warp];
    uint16_t (*sNbr)[9] = sNbrAll[warp]; uint16_t* sLabel = sLabelAll[warp]; uint8_t* sFlag = sFlagAll[warp];
    const uint32_t nIX = G.nIX, nIY = G.nIY;

    // The cell list in raster order: bitonic sort of the (padded) list.
    uint32_t P = 32;
    while(P < n) P <<= 1;
    const uint32_t* list = g.list + G.base;
    for(uint32_t t = lane; t < P; t += 32) sIdx[t] = t < n ? list[t] : 0xffffffffu;
    __syncwarp();
    for(uint32_t k = 2; k <= P; k <<= 1) {
        for(uint32_t j = k >> 1; j > 0; j >>= 1) {
            for(uint32_t t = lane; t < P; t += 32) {
                const uint32_t u = t ^ j;
                if(u > t) {
                    const uint32_t a = sIdx[t], b = sIdx[u];
                    if((a > b) == ((t & k) == 0)) { sIdx[t] = b; sIdx[u] = a; }
                }
            }
            __syncwarp();
        }
    }
    // Flags and the neighbour slots.
    for(uint32_t t = lane; t < n; t += 32) {
        const uint32_t i = sIdx[t];
        const uint32_t iX = i % nIX, iY = i / nIX;
        sFlag[t] = align4CellFlags(g, G, iX, iY);
#pragma unroll
        for(int oY = -1; oY <= 1; oY++) {
#pragma unroll
            for(int oX = -1; oX <= 1; oX++) {
                uint16_t slot = kAlign4NoSlot;
                const int32_t qX = int32_t(iX) + oX, qY = int32_t(iY) + oY;
                if((oX || oY) && qX >= 0 && qY >= 0 && qX < int32_t(nIX) && qY < int32_t(nIY)) {
                    const uint32_t j = uint32_t(qY) * nIX + uint32_t(qX);
                    uint32_t lo = 0, hi = n;        // lower bound of j in sIdx[0, n)
                    while(lo < hi) { const uint32_t mid = (lo + hi) >> 1; if(sIdx[mid] < j) lo = mid + 1; else hi = mid; }
                    if(lo < n && sIdx[lo] == j) slot = uint16_t(lo);
                }
                sNbr[t][(oY + 1) * 3 + (oX + 1)] = slot;
            }
        }
    }
    __syncwarp();
    for(uint32_t t = lane; t < n; t += 32) sIdx[t] /= nIX;          // from here on only the row is needed
    __syncwarp();
    align4ComponentBands(Align4SharedCells{sIdx, sNbr, sFlag, sLabel, sYMax}, n, g, p, G);
}

// Expand (candidate, component) into DP jobs. jobOffsets = exclusive scan of componentCount.
static __global__ void align4MakeJobsKernel(const uint32_t* __restrict__ candidates, uint32_t n, const uint64_t* __restrict__ toc,
                                            const unsigned long long* __restrict__ cellOffsets, const int32_t* __restrict__ bands,
                                            const uint32_t* __restrict__ componentCount, const uint32_t* __restrict__ jobOffsets,
                                            DpJob* __restrict__ jobs, unsigned long long* __restrict__ traceWords,
                                            unsigned long long* __restrict__ outCount)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if(p >= n) return;
    uint64_t o0, o1;
    candidateOrientedReads(candidates, p, o0, o1);
    DpJob j;
    j.aOffset = toc[o0]; j.nx = uint32_t(toc[o0 + 1] - toc[o0]);
    j.bOffset = toc[o1]; j.ny = uint32_t(toc[o1 + 1] - toc[o1]);
    j.traceOffset = 0; j.outOffset = 0; j.pad = p;
    const int32_t* b = bands + cellOffsets[p];
    const uint32_t first = jobOffsets[p];
    for(uint32_t c = 0; c < componentCount[p]; c++) {
        const int32_t bandMin = b[2 * c], bandMax = b[2 * c + 1];
        // SeqAn returns MinValue when the band misses the matrix: "SeqAn banded alignment computation failed."
        // and the component yields an empty alignment (src/Align4.cpp:1034-1036).
        const bool misses = bandMin > bandMax || bandMax < -int32_t(j.ny) || bandMin > int32_t(j.nx);
        j.lo = max(bandMin, -int32_t(j.ny));
        j.hi = min(bandMax, int32_t(j.nx));
        j.state = misses ? kStateEmpty : kStateRun;
        jobs[first + c] = j;
        traceWords[first + c] = misses ? 0ull : dpTraceWords(j.nx, j.ny, j.lo, j.hi);
        outCount[first + c] = min(j.nx, j.ny);
    }
}

// Per candidate: among its jobs kept by the Align4-internal filters, the one with the most aligned markers
// (first wins ties, src/Align4.cpp:128-147); then the driver's own filter chain, which only adds the
// containment test (src/AssemblerAlign.cpp:438-473). selected[p] = job index or 0xffffffff.
static __global__ void align4SelectKernel(uint32_t n, const uint32_t* __restrict__ jobOffsets, const uint32_t* __restrict__ componentCount,
                                          const uint32_t* __restrict__ jobKeep, const uint32_t* __restrict__ jobInfoWords,
                                          const uint32_t* __restrict__ jobBytes, uint32_t suppressContainments, uint32_t maxTrim,
                                          uint32_t* __restrict__ selected, uint32_t* __restrict__ keep, uint32_t* __restrict__ bytes)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if(p >= n) return;
    uint32_t best = 0xffffffffu, bestCount = 0;
    const uint32_t first = jobOffsets[p];
    for(uint32_t c = 0; c < componentCount[p]; c++) {
        const uint32_t j = first + c;
        if(!jobKeep[j]) continue;
        const uint32_t markerCount = jobInfoWords[13ull * j + 6];
        if(best == 0xffffffffu || markerCount > bestCount) { best = j; bestCount = markerCount; }
    }
    uint32_t k = best != 0xffffffffu;
    if(k && suppressContainments) {
        const uint32_t* w = jobInfoWords + 13ull * best;
        const bool c0 = w[1] <= maxTrim && w[0] - 1 - w[2] <= maxTrim;
        const bool c1 = w[4] <= maxTrim && w[3] - 1 - w[5] <= maxTrim;
        if(c0 || c1) k = 0;
    }
    selected[p] = k ? best : 0xffffffffu;
    keep[p] = k;
    bytes[p] = k ? jobBytes[best] : 0u;
}

// (rowIndex<<32 | kmerId, ordinal) keys for the per-read sort of computeSortedMarkers (src/AssemblerAlign4.cpp:190-261),
// for sortMarkersByKmer (align.cu).
static __global__ void sortedMarkerKeysKernel(const uint32_t* __restrict__ kmerIds, const uint64_t* __restrict__ toc,
                                              uint32_t rowBegin, uint32_t rowEnd, uint64_t markerBegin, uint32_t n,
                                              uint64_t* __restrict__ keys, uint32_t* __restrict__ ordinals)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n) return;
    const uint64_t p = markerBegin + i;
    const uint32_t lo = rowOf(toc, rowBegin, rowEnd, p);
    keys[i] = (uint64_t(lo - rowBegin) << 32) | kmerIds[p];
    ordinals[i] = uint32_t(p - toc[lo]);
}

static __global__ void sortedMarkerUnpackKernel(const uint64_t* __restrict__ keys, uint32_t n, uint32_t* __restrict__ sortedKmer)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i < n) sortedKmer[i] = uint32_t(keys[i]);
}

} // namespace shb
