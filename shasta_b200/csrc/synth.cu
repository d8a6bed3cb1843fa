// Bench/test utility: the marker-space synthetic read generator of shasta_b200/synth.py on the GPU.
// Produces bit-identical data (every random draw is splitmix64(seed, stream, i, j)); the per-read
// window (start, span, strand) and the genome arrays are computed on the host by synth.py and passed in.
// This is input generation for bench.py and the tests, not part of the reference's hot path.
#include "context.cuh"

namespace shb {
namespace {

__host__ __device__ inline uint64_t mix64(uint64_t seed, uint64_t stream, uint64_t a, uint64_t b)
{
    uint64_t x = (seed ^ (stream * 0x9E3779B97F4A7C15ull)) + a * 0xBF58476D1CE4E5B9ull + b * 0x94D049BB133111EBull;
    x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 27; x *= 0x94D049BB133111EBull;
    x ^= x >> 31;
    return x;
}
__device__ inline double unitOf(uint64_t x) { return double(x >> 11) * (1.0 / 9007199254740992.0); }

struct SynthArgs {
    uint64_t seed; uint32_t k; double drop; double ins;
    const uint32_t* genomeKmer; const uint64_t* genomePos;
    uint64_t readCount; const int64_t* start; const int64_t* span; const uint8_t* rev;
    uint64_t readOffset;            // global id of local read 0 (the RNG is keyed by the global read id)
};

// One block per read: number of markers of the read (kept genome markers + inserted markers).
__global__ void __launch_bounds__(256) synthCountKernel(SynthArgs a, uint64_t* counts)
{
    __shared__ uint32_t smem[8];
    const uint64_t local = blockIdx.x;
    const uint64_t r = local + a.readOffset;
    const int64_t start = a.start[local], span = a.span[local];
    uint32_t c = 0;
    for(int64_t j = threadIdx.x; j < span; j += 256) {
        const uint64_t g = uint64_t(start + j);
        c += (unitOf(mix64(a.seed, 5, r, g)) >= a.drop) ? 1u : 0u;
        c += (unitOf(mix64(a.seed, 6, r, g)) < a.ins) ? 1u : 0u;
    }
    uint32_t total;
    blockExclusiveScan256<uint32_t>(c, total, smem);
    if(threadIdx.x == 0) counts[local] = total;
}

// One block per read: fill both strand rows. toc is the final (2R+1) table.
__global__ void __launch_bounds__(256) synthFillKernel(SynthArgs a, const uint64_t* toc, uint32_t* kmerOut, uint32_t* posOut)
{
    __shared__ uint32_t smem[8];
    const uint64_t local = blockIdx.x;
    const uint64_t r = local + a.readOffset;
    const int64_t start = a.start[local], span = a.span[local];
    const bool rev = a.rev[local] != 0;
    const uint64_t row0 = toc[2*local], row1 = toc[2*local+1];
    const uint64_t n = row1 - row0;
    const uint64_t base = a.genomePos[start];
    const uint64_t totalLen = (a.genomePos[start + span - 1] - base) + a.k + 2;
    const uint64_t k4 = 1ull << (2 * a.k);
    uint32_t running = 0;
    for(int64_t j0 = 0; j0 < span; j0 += 256) {
        const int64_t j = j0 + threadIdx.x;
        bool keep = false, insm = false;
        uint64_t g = 0;
        if(j < span) {
            g = uint64_t(start + j);
            keep = unitOf(mix64(a.seed, 5, r, g)) >= a.drop;
            insm = unitOf(mix64(a.seed, 6, r, g)) < a.ins;
        }
        uint32_t total;
        const uint32_t slot = running + blockExclusiveScan256<uint32_t>((keep ? 1u : 0u) + (insm ? 1u : 0u), total, smem);
        running += total;
        if(j < span) {
            const uint64_t pg = a.genomePos[g] - base;
            for(int e = 0; e < 2; e++) {
                if(e == 0 ? !keep : !insm) continue;
                const uint32_t s = slot + ((e == 1 && keep) ? 1u : 0u);
                uint32_t km = (e == 0) ? a.genomeKmer[g] : uint32_t(mix64(a.seed, 7, r, g) % k4);
                uint64_t ps = (e == 0) ? pg : pg + 1;
                // Strand-0 row index/content (a reverse-strand read is stored reversed + reverse complemented).
                uint64_t i0 = s;
                if(rev) { i0 = n - 1 - s; km = reverseComplementKmer(km, a.k); ps = totalLen - a.k - ps; }
                kmerOut[row0 + i0] = km;
                posOut[row0 + i0] = uint32_t(ps);
                // Strand-1 row = strand-0 row reversed and reverse complemented (src/MarkerFinder.cpp:92-100).
                kmerOut[row1 + (n - 1 - i0)] = reverseComplementKmer(km, a.k);
                posOut[row1 + (n - 1 - i0)] = uint32_t(totalLen - a.k - ps);
            }
        }
    }
}

// (kmerId, position) SoA -> 7-byte CompressedMarker records (src/Marker.hpp:56-69).
__global__ void packMarkersKernel(const uint32_t* kmer, const uint32_t* pos, uint64_t n, uint8_t* out)
{
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if(i >= n) return;
    const uint32_t k = kmer[i], p = pos[i];
    uint8_t* o = out + 7 * i;
    o[0] = uint8_t(k); o[1] = uint8_t(k >> 8); o[2] = uint8_t(k >> 16); o[3] = uint8_t(k >> 24);
    o[4] = uint8_t(p); o[5] = uint8_t(p >> 8); o[6] = uint8_t(p >> 16);
}

} // namespace
} // namespace shb

using namespace shb;

extern "C" {

// Device-memory helpers for callers that hold generated data.
shb_status shb_device_free(void* p)
{
    cudaFree(p);
    return SHB_OK;
}

shb_status shb_copy_device_to_host(void* dstHost, const void* srcDevice, uint64_t bytes)
{
    return cudaMemcpy(dstHost, srcDevice, bytes, cudaMemcpyDeviceToHost) == cudaSuccess ? SHB_OK : SHB_ERR_CUDA;
}

// See shasta_b200/synth.py generate(): same data, produced on the device.
//   tocOut        : host, 2R+1 entries (absolute).
//   kmerIdsDevice : receives a device allocation of uint32[M] (free with shb_device_free).
//   data7Device   : if not NULL receives a device allocation of the 7-byte records (7*M bytes).
shb_status shb_synth_generate(shb_context* c, uint64_t seed, uint32_t k, double drop, double ins,
                              uint64_t genomeMarkers, const uint32_t* genomeKmerHost, const uint64_t* genomePosHost,
                              uint64_t readOffset, uint64_t readCount,
                              const int64_t* startHost, const int64_t* spanHost, const uint8_t* revHost,
                              uint64_t* tocOut, uint32_t** kmerIdsDevice, uint8_t** data7Device)
{
    try {
        SHB_REQUIRE(c && tocOut && kmerIdsDevice, SHB_ERR_INVALID, "Null argument.");
        SHB_CUDA(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        DeviceBuffer<uint32_t> gk; DeviceBuffer<uint64_t> gp, counts;
        DeviceBuffer<int64_t> start, span; DeviceBuffer<uint8_t> rev;
        gk.reserve(genomeMarkers); gp.reserve(genomeMarkers);
        start.reserve(readCount); span.reserve(readCount); rev.reserve(readCount); counts.reserve(readCount);
        SHB_CUDA(cudaMemcpyAsync(gk.get(), genomeKmerHost, genomeMarkers * 4, cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(gp.get(), genomePosHost, genomeMarkers * 8, cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(start.get(), startHost, readCount * 8, cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(span.get(), spanHost, readCount * 8, cudaMemcpyHostToDevice, st));
        SHB_CUDA(cudaMemcpyAsync(rev.get(), revHost, readCount, cudaMemcpyHostToDevice, st));
        SynthArgs a{seed, k, drop, ins, gk.get(), gp.get(), readCount, start.get(), span.get(), rev.get(), readOffset};
        std::vector<uint64_t> hostCounts(readCount);
        if(readCount) {
            SHB_LAUNCH(synthCountKernel, (unsigned)readCount, 256, 0, st, a, counts.get());
            SHB_CUDA(cudaMemcpyAsync(hostCounts.data(), counts.get(), readCount * 8, cudaMemcpyDeviceToHost, st));
        }
        SHB_CUDA(cudaStreamSynchronize(st));
        tocOut[0] = 0;
        for(uint64_t r = 0; r < readCount; r++) {
            tocOut[2*r+1] = tocOut[2*r] + hostCounts[r];
            tocOut[2*r+2] = tocOut[2*r+1] + hostCounts[r];
        }
        const uint64_t M = tocOut[2*readCount];
        DeviceBuffer<uint64_t> toc; toc.reserve(2*readCount + 1);
        SHB_CUDA(cudaMemcpyAsync(toc.get(), tocOut, (2*readCount + 1) * 8, cudaMemcpyHostToDevice, st));
        uint32_t* kmer = nullptr; uint32_t* pos = nullptr;
        SHB_CUDA(cudaMalloc(&kmer, (M + 64) * 4));
        SHB_CUDA(cudaMalloc(&pos, (M + 64) * 4));
        if(readCount) SHB_LAUNCH(synthFillKernel, (unsigned)readCount, 256, 0, st, a, (const uint64_t*)toc.get(), kmer, pos);
        if(data7Device) {
            uint8_t* d7 = nullptr;
            SHB_CUDA(cudaMalloc(&d7, M * 7 + 64));
            if(M) SHB_LAUNCH(packMarkersKernel, ceilDiv(M, 256), 256, 0, st, (const uint32_t*)kmer, (const uint32_t*)pos, M, d7);
            *data7Device = d7;
        }
        SHB_CUDA(cudaStreamSynchronize(st));
        cudaFree(pos);
        *kmerIdsDevice = kmer;
        return SHB_OK;
    } catch(const Error& e) {
        setLastError(e.what());
        return e.status;
    }
}

} // extern "C"
