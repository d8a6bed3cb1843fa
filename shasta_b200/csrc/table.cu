// computeAlignmentTable (src/AssemblerAlign.cpp:509-571) and computeCandidateTable
// (src/AssemblerAlignmentCandidates.cpp:379-448) on the GPU: 4 (row, other, index) entries per oriented read pair,
// stable radix sort by (row, other), row starts by binary search. The two tables differ only in the record they read the
// pair from (64-byte AlignmentData / 12-byte OrientedReadPair) and in the integer width of the output
// (VectorOfVectors<uint32_t,uint32_t> / VectorOfVectors<uint64_t,uint64_t>).
#include "context.cuh"
#include "hostpool.cuh"

#include <cstring>
#include <string>

namespace shb {
namespace {

// records: `stride` words per item, words 0..2 = readId0, readId1, isSameStrand.
__global__ void pairTableKeysKernel(const uint32_t* __restrict__ records, uint32_t stride, uint32_t n, uint64_t* __restrict__ keys,
                                    uint32_t* __restrict__ vals)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n) return;
    const uint32_t r0 = records[uint64_t(stride) * i], r1 = records[uint64_t(stride) * i + 1];
    const bool same = (records[uint64_t(stride) * i + 2] & 0xffu) != 0;
    const uint32_t o0 = 2 * r0, o1 = 2 * r1 + (same ? 0u : 1u);
    // Generated in item order; the sort is stable, so equal (row, other) keep increasing item index
    // (the reference sorts pair<OrientedReadId, index>).
    keys[4ull * i + 0] = (uint64_t(o0) << 32) | o1;            vals[4ull * i + 0] = i;
    keys[4ull * i + 1] = (uint64_t(o1) << 32) | o0;            vals[4ull * i + 1] = i;
    keys[4ull * i + 2] = (uint64_t(o0 ^ 1u) << 32) | (o1 ^ 1u); vals[4ull * i + 2] = i;
    keys[4ull * i + 3] = (uint64_t(o1 ^ 1u) << 32) | (o0 ^ 1u); vals[4ull * i + 3] = i;
}

// T = uint32_t (alignment table) or unsigned long long (candidate table).
template<class T> void computePairTable(shb_context* c, const uint32_t* rec, uint32_t stride, uint64_t n, uint64_t readCount,
                                        T** tocOut, T** dataOut, const char* what)
{
    SHB_REQUIRE(4 * n < (1ull << 32), SHB_ERR_INVALID, std::string("Too many ") + what + " for one table sort (limit 2^30-1).");
    SHB_REQUIRE(readCount < (1ull << 31), SHB_ERR_INVALID, "Too many reads.");
    SHB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const uint32_t rows = uint32_t(2 * readCount);
    HostResult tocHost(allocHostResult(sizeof(T) * (uint64_t(rows) + 1))), dataHost(allocHostResult(sizeof(T) * (4 * n + 1)));
    SHB_REQUIRE(tocHost.p && dataHost.p, SHB_ERR_OOM, "Out of host memory for the table.");
    if(n == 0) {
        memset(tocHost.p, 0, sizeof(T) * (uint64_t(rows) + 1));
        *tocOut = static_cast<T*>(tocHost.take()); *dataOut = static_cast<T*>(dataHost.take());
        return;
    }
    for(uint64_t i = 0; i < n; i++) {
        SHB_REQUIRE(rec[stride*i] < readCount && rec[stride*i+1] < readCount, SHB_ERR_INVALID,
                    std::string("One of the ") + what + " refers to a read that does not exist.");
    }
    DeviceBuffer<uint32_t> dRec, valsA, valsB;
    DeviceBuffer<T> dToc, dWide;
    DeviceBuffer<uint64_t> keysA, keysB;
    const uint32_t entries = uint32_t(4 * n);
    dRec.reserve(uint64_t(stride) * n); keysA.reserve(entries); keysB.reserve(entries); valsA.reserve(entries); valsB.reserve(entries);
    dToc.reserve(uint64_t(rows) + 1);
    SHB_CUDA(cudaMemcpyAsync(dRec.get(), rec, 4ull * stride * n, cudaMemcpyHostToDevice, st));
    SHB_LAUNCH(pairTableKeysKernel, ceilDiv(n, 256), 256, 0, st, (const uint32_t*)dRec.get(), stride, uint32_t(n), keysA.get(), valsA.get());
    const uint32_t rowBits = bitsFor(rows ? rows - 1 : 0);
    const int ranges[2][2] = {{0, int(rowBits)}, {32, 32 + int(rowBits)}};
    const bool inB = radixSort<true>(keysA.get(), keysB.get(), valsA.get(), valsB.get(), entries, ranges, 2, c->sortWs, st);
    SHB_LAUNCH((rowStartsKernel<T>), ceilDiv(uint64_t(rows) + 1, 256), 256, 0, st, (const uint64_t*)(inB ? keysB.get() : keysA.get()),
               entries, rows, dToc.get());
    SHB_CUDA(cudaMemcpyAsync(tocHost.p, dToc.get(), sizeof(T) * (uint64_t(rows) + 1), cudaMemcpyDeviceToHost, st));
    const uint32_t* sortedVals = inB ? valsB.get() : valsA.get();
    if(sizeof(T) == 4) {
        SHB_CUDA(cudaMemcpyAsync(dataHost.p, sortedVals, 4ull * entries, cudaMemcpyDeviceToHost, st));
    } else {
        dWide.reserve(entries);
        SHB_LAUNCH(widenKernel<uint32_t>, ceilDiv(entries, 256), 256, 0, st, sortedVals, entries, (unsigned long long*)dWide.get());
        SHB_CUDA(cudaMemcpyAsync(dataHost.p, dWide.get(), 8ull * entries, cudaMemcpyDeviceToHost, st));
    }
    SHB_CUDA(cudaStreamSynchronize(st));
    *tocOut = static_cast<T*>(tocHost.take()); *dataOut = static_cast<T*>(dataHost.take());
}

} // namespace

void computeAlignmentTable(shb_context* c, const void* alignmentData, uint64_t n, uint64_t readCount,
                           uint32_t** tocOut, uint32_t** dataOut)
{
    computePairTable<uint32_t>(c, static_cast<const uint32_t*>(alignmentData), 16, n, readCount, tocOut, dataOut, "alignments");
}

void computeCandidateTable(shb_context* c, const void* candidates, uint64_t n, uint64_t readCount,
                           uint64_t** tocOut, uint64_t** dataOut)
{
    unsigned long long* toc = nullptr; unsigned long long* data = nullptr;
    computePairTable<unsigned long long>(c, static_cast<const uint32_t*>(candidates), 3, n, readCount, &toc, &data, "candidates");
    *tocOut = reinterpret_cast<uint64_t*>(toc); *dataOut = reinterpret_cast<uint64_t*>(data);
}

} // namespace shb
