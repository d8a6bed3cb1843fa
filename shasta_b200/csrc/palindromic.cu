// flagPalindromicReads on the GPU (src/AssemblerAlign.cpp:652-770 of chanzuckerberg/shasta).
//
// Phase A, every read: the k-mer ids of each oriented read are radix-sorted, strand 0 is merge-joined against strand 1, and
// V (the alignment graph's vertex count: pairs of equal k-mers from streaks no longer than maxMarkerFrequency) and V_near
// (those with |ordinal0 - ordinal1| < deltaThreshold) are counted. The path's vertices are distinct graph vertices, so
// aligned <= V and nearDiagonal <= V_near; the reference's own double expressions on V and V_near then prove most reads
// "not palindromic" without a graph.
// Phase B, the remaining reads: one warp per read builds the reference's graph and runs its Dijkstra exactly.
#include "context.cuh"
#include "hostpool.cuh"
#include "palindromic_kernels.cuh"

#include <chrono>
#include <cstring>
#include <functional>
#include <vector>

namespace shb {

extern thread_local uint64_t g_launchCount;

void sortMarkersByKmer(shb_context* c, uint32_t rowStep, uint64_t chunkLimit, uint32_t kmerBits, const char* tooLong,
                       const std::function<void(const uint64_t*, const uint32_t*, uint32_t, uint32_t, uint64_t, uint32_t)>& sorted);

namespace {

using namespace pal;

// ---- phase A -------------------------------------------------------------------------------------------------------
// One thread per read: the merge join of createVertices (src/AlignmentGraph.cpp:179-249), counting only.
__global__ void palPrefilterKernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ordinals,
                                   const uint64_t* __restrict__ toc, uint64_t readBegin, uint64_t readEnd, uint64_t markerBegin,
                                   uint32_t maxMarkerFrequency, uint32_t deltaThreshold, double alignedFractionThreshold,
                                   double nearDiagonalFractionThreshold, unsigned long long* __restrict__ vBound, unsigned long long* __restrict__ vNearBound,
                                   uint8_t* __restrict__ survives)
{
    const uint64_t r = readBegin + blockIdx.x * uint64_t(blockDim.x) + threadIdx.x;
    if(r >= readEnd) return;
    const uint64_t b0 = toc[2 * r] - markerBegin, b1 = toc[2 * r + 1] - markerBegin;
    const uint32_t n0 = uint32_t(toc[2 * r + 1] - toc[2 * r]), n1 = uint32_t(toc[2 * r + 2] - toc[2 * r + 1]);
    uint64_t V = 0, Vnear = 0;
    uint32_t i0 = 0, i1 = 0;
    while(i0 < n0 && i1 < n1) {
        const uint32_t k0 = uint32_t(keys[b0 + i0]), k1 = uint32_t(keys[b1 + i1]);
        if(k0 < k1) i0++;
        else if(k1 < k0) i1++;
        else {
            uint32_t e0 = i0 + 1, e1 = i1 + 1;
            while(e0 < n0 && uint32_t(keys[b0 + e0]) == k0) e0++;
            while(e1 < n1 && uint32_t(keys[b1 + e1]) == k0) e1++;
            if(e0 - i0 <= maxMarkerFrequency && e1 - i1 <= maxMarkerFrequency) {
                V += uint64_t(e0 - i0) * (e1 - i1);
                for(uint32_t j0 = i0; j0 < e0; j0++) {
                    const int32_t o0 = int32_t(ordinals[b0 + j0]);
                    for(uint32_t j1 = i1; j1 < e1; j1++) {
                        const uint32_t delta = uint32_t(abs(o0 - int32_t(ordinals[b1 + j1])));
                        if(delta < deltaThreshold) Vnear++;
                    }
                }
            }
            i0 = e0; i1 = e1;
        }
    }
    // src/AssemblerAlign.cpp:741-766 with aligned <= V and nearDiagonal <= V_near. n0 = 0 gives NaN: not rejected.
    const bool rejected = (double(V) / double(n0) < alignedFractionThreshold) || (double(Vnear) / double(n0) < nearDiagonalFractionThreshold);
    vBound[r] = V;
    vNearBound[r] = Vnear;
    survives[r] = rejected ? 0 : 1;
}

// ---- phase B -------------------------------------------------------------------------------------------------------
struct PalJob {
    uint64_t readId;
    uint32_t n0, n1;
    uint64_t vCap;                  // bound on the vertex count used to size the phase-1 scratch
    uint64_t off1;                  // bytes into arena 1: markers[n0+n1], corrected[n0+n1], vertices[vCap], pairCount[vCap]
    uint64_t off2;                  // bytes into arena 2 (see palPathKernel)
    uint64_t pathOff;               // Vertex entries into the path buffer; ~0 = no path wanted
    // written by the kernels
    uint64_t V, pairEdges, heapPushes;
    uint32_t aligned, nearDiagonal, fallbacks, flag;
};

__host__ __device__ inline uint64_t align16(uint64_t x) { return (x + 15) & ~15ull; }
__host__ __device__ inline uint64_t arena1Bytes(uint64_t n, uint64_t vCap) { return align16(8 * n) + align16(4 * n) + align16(8 * vCap) + align16(4 * vCap); }
__host__ __device__ inline uint64_t arena2Bytes(uint64_t V, uint64_t pairEdges)
{
    const uint64_t E = pairEdges + 2 * V, N = V + 2;
    return align16(16 * E) + align16(4 * (N + 1)) + align16(4 * (N + 1)) + align16(4 * 2 * E) + align16(8 * N) + align16(4 * N) + align16(N) +
           align16(16 * (2 * E + 1));
}

// One warp per read: getMarkersSortedByKmerId (src/AssemblerMarkers.cpp:83-98), createVertices (src/AlignmentGraph.cpp:
// 156-265), sortVertices (src/CompactUndirectedGraph.hpp:506-510), and the number of pair edges each vertex starts
// (createEdges, src/AlignmentGraph.cpp:308-371).
__global__ void palVerticesKernel(PalJob* __restrict__ jobs, uint32_t jobCount, uint8_t* __restrict__ arena,
                                  const uint32_t* __restrict__ kmerIds, const uint64_t* __restrict__ toc,
                                  uint32_t maxSkip32, uint32_t maxDrift32, uint32_t maxMarkerFrequency)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t j = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if(j >= jobCount) return;
    PalJob& job = jobs[j];
    const uint32_t n[2] = {job.n0, job.n1};
    uint8_t* base = arena + job.off1;
    Marker* m[2]; m[0] = reinterpret_cast<Marker*>(base); m[1] = m[0] + n[0];
    uint32_t* corr[2]; corr[0] = reinterpret_cast<uint32_t*>(base + align16(8ull * (n[0] + n[1]))); corr[1] = corr[0] + n[0];
    Vertex* vert = reinterpret_cast<Vertex*>(reinterpret_cast<uint8_t*>(corr[0]) + align16(4ull * (n[0] + n[1])));
    uint32_t* pairCount = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(vert) + align16(8 * job.vCap));
    for(int s = 0; s < 2; s++) {
        const uint64_t b = toc[2 * job.readId + s];
        for(uint32_t i = lane; i < n[s]; i += 32) { m[s][i] = Marker{kmerIds[b + i], i}; corr[s][i] = 1; }
    }
    __syncwarp();
    uint64_t V = 0;
    if(lane == 0) {
        uint32_t fallbacks = stdSort(m[0], n[0], MarkerLess()) + stdSort(m[1], n[1], MarkerLess());
        uint32_t i0 = 0, i1 = 0;
        while(i0 < n[0] && i1 < n[1]) {
            if(m[0][i0].kmerId < m[1][i1].kmerId) i0++;
            else if(m[1][i1].kmerId < m[0][i0].kmerId) i1++;
            else {
                const uint32_t kmerId = m[0][i0].kmerId;
                uint32_t e0 = i0, e1 = i1;
                while(e0 < n[0] && m[0][e0].kmerId == kmerId) e0++;
                while(e1 < n[1] && m[1][e1].kmerId == kmerId) e1++;
                if(e0 - i0 > maxMarkerFrequency || e1 - i1 > maxMarkerFrequency) {
                    for(uint32_t q = i0; q < e0; q++) corr[0][m[0][q].ordinal] = 0;
                    for(uint32_t q = i1; q < e1; q++) corr[1][m[1][q].ordinal] = 0;
                } else {
                    for(uint32_t q0 = i0; q0 < e0; q0++) for(uint32_t q1 = i1; q1 < e1; q1++) vert[V++] = Vertex{m[0][q0].ordinal, m[1][q1].ordinal};
                }
                i0 = e0; i1 = e1;
            }
        }
        for(int s = 0; s < 2; s++) {            // correctedOrdinals
            uint32_t c = 0;
            for(uint32_t i = 0; i < n[s]; i++) corr[s][i] = corr[s][i] ? c++ : 0xffffffffu;
        }
        fallbacks += stdSort(vert, int64_t(V), VertexLess());
        job.V = V;
        job.fallbacks = fallbacks;
    }
    V = __shfl_sync(0xffffffffu, V, 0);
    __syncwarp();
    const int maxSkip = int(maxSkip32);
    const bool driftTest = maxDrift32 < maxSkip32;
    unsigned long long pairs = 0;
    for(uint64_t a = lane; a < V; a += 32) {
        const int cA0 = int(corr[0][vert[a].o0]), cA1 = int(corr[1][vert[a].o1]);
        uint32_t count = 0;
        for(uint64_t b = a + 1; b < V; b++) {
            const int cB0 = int(corr[0][vert[b].o0]);
            if(cB0 > cA0 + maxSkip) break;
            const int cB1 = int(corr[1][vert[b].o1]);
            if(cB1 < cA1) continue;
            if(uint32_t(abs(cB1 - cA1)) > maxSkip32) continue;
            if(driftTest && uint32_t(abs((cA0 - cA1) - (cB0 - cB1))) > maxDrift32) continue;
            count++;
        }
        pairCount[a] = count;
        pairs += count;
    }
    for(int o = 16; o; o >>= 1) pairs += __shfl_xor_sync(0xffffffffu, pairs, o);
    if(lane == 0) job.pairEdges = pairs;
}

// One warp per read: the edges (createEdges), the out-edge lists (doneAddingEdges, src/CompactUndirectedGraph.hpp:537-583),
// findShortestPath (src/shortestPath.hpp:65-161) with the libstdc++ binary heap, and the decision
// (src/AssemblerAlign.cpp:741-766).
__global__ void palPathKernel(PalJob* __restrict__ jobs, uint32_t jobCount, const uint8_t* __restrict__ arena1,
                              uint8_t* __restrict__ arena2, Vertex* __restrict__ paths, uint32_t maxSkip32, uint32_t maxDrift32,
                              uint32_t deltaThreshold, double alignedFractionThreshold, double nearDiagonalFractionThreshold)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t j = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if(j >= jobCount) return;
    PalJob& job = jobs[j];
    const uint32_t n[2] = {job.n0, job.n1};
    const uint8_t* base = arena1 + job.off1;
    const uint32_t* corr[2]; corr[0] = reinterpret_cast<const uint32_t*>(base + align16(8ull * (n[0] + n[1]))); corr[1] = corr[0] + n[0];
    const Vertex* vert = reinterpret_cast<const Vertex*>(reinterpret_cast<const uint8_t*>(corr[0]) + align16(4ull * (n[0] + n[1])));
    uint32_t* pairCount = const_cast<uint32_t*>(reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(vert) + align16(8 * job.vCap)));
    const uint64_t V = job.V, P = job.pairEdges, E = P + 2 * V, N = V + 2;
    const uint32_t vStart = uint32_t(V), vFinish = uint32_t(V + 1);
    uint8_t* p = arena2 + job.off2;
    Edge* edges = reinterpret_cast<Edge*>(p);                    p += align16(16 * E);
    uint32_t* first = reinterpret_cast<uint32_t*>(p);            p += align16(4 * (N + 1));
    uint32_t* fill = reinterpret_cast<uint32_t*>(p);             p += align16(4 * (N + 1));
    uint32_t* lists = reinterpret_cast<uint32_t*>(p);            p += align16(8 * E);
    uint64_t* dist = reinterpret_cast<uint64_t*>(p);             p += align16(8 * N);
    uint32_t* pred = reinterpret_cast<uint32_t*>(p);             p += align16(4 * N);
    uint8_t* color = p;                                          p += align16(N);
    HeapItem* heap = reinterpret_cast<HeapItem*>(p);

    // Exclusive scan of the per-vertex pair-edge counts: vertex A's edges go to [offset(A), offset(A+1)), so the lanes
    // write the edge table in the reference's (A, B) loop order.
    if(lane == 0) { uint32_t s = 0; for(uint64_t a = 0; a < V; a++) { const uint32_t c = pairCount[a]; pairCount[a] = s; s += c; } }
    __syncwarp();
    const int maxSkip = int(maxSkip32);
    const bool driftTest = maxDrift32 < maxSkip32;
    for(uint64_t a = lane; a < V; a += 32) {
        const int cA0 = int(corr[0][vert[a].o0]), cA1 = int(corr[1][vert[a].o1]);
        uint64_t out = pairCount[a];
        for(uint64_t b = a + 1; b < V; b++) {
            const int cB0 = int(corr[0][vert[b].o0]);
            if(cB0 > cA0 + maxSkip) break;
            const int cB1 = int(corr[1][vert[b].o1]);
            if(cB1 < cA1) continue;
            if(uint32_t(abs(cB1 - cA1)) > maxSkip32) continue;
            if(driftTest && uint32_t(abs((cA0 - cA1) - (cB0 - cB1))) > maxDrift32) continue;
            edges[out++] = Edge{uint32_t(a), uint32_t(b), uint64_t(abs(cB0 - cA0 - 1) + abs(cB1 - cA1 - 1))};
        }
        const int c0 = cA0, c1 = cA1;
        edges[P + 2 * a] = Edge{uint32_t(a), vStart, uint64_t(abs(c0) + abs(c1))};
        edges[P + 2 * a + 1] = Edge{uint32_t(a), vFinish, uint64_t(abs(int(n[0]) - c0) + abs(int(n[1]) - c1))};
    }
    for(uint64_t v = lane; v < N + 1; v += 32) first[v] = 0;
    for(uint64_t v = lane; v < N; v += 32) { dist[v] = ~0ull; pred[v] = 0xffffffffu; color[v] = 0; }
    __syncwarp();
    if(lane != 0) return;

    // CSR with each vertex's out-edges in increasing edge index.
    for(uint64_t e = 0; e < E; e++) { first[edges[e].a + 1]++; first[edges[e].b + 1]++; }
    for(uint64_t v = 0; v < N; v++) first[v + 1] += first[v];
    for(uint64_t v = 0; v <= N; v++) fill[v] = first[v];
    for(uint64_t e = 0; e < E; e++) { lists[fill[edges[e].a]++] = uint32_t(e); lists[fill[edges[e].b]++] = uint32_t(e); }

    // findShortestPath(graph, vStart, vFinish): std::priority_queue ordered by distance only, lazy deletion.
    HeapLess less;
    pred[vStart] = vStart; dist[vStart] = 0;
    uint64_t q = 0, pushes = 1;
    heap[q++] = HeapItem{0, vStart};
    uint64_t pathCount = 0, nearCount = 0;
    bool found = false;
    while(q) {
        const HeapItem top = heap[0];
        if(q > 1) { const HeapItem value = heap[q - 1]; heap[q - 1] = heap[0]; adjustHeap(heap, int64_t(0), int64_t(q - 1), value, less); }
        q--;
        const uint32_t v0 = top.v;
        if(color[v0] == 1) continue;
        color[v0] = 1;
        if(v0 == vFinish) { found = true; break; }
        for(uint32_t i = first[v0]; i < first[v0 + 1]; i++) {
            const Edge e = edges[lists[i]];
            const uint32_t v1 = (e.a == v0) ? e.b : e.a;
            if(color[v1] == 1) continue;
            const uint64_t d1 = top.d + e.w;
            if(d1 < dist[v1]) {
                pushHeap(heap, int64_t(q), int64_t(0), HeapItem{d1, v1}, less);
                q++; pushes++;
                pred[v1] = v0; dist[v1] = d1;
            }
        }
    }
    if(found) {
        // The predecessor chain from vFinish, without vStart and vFinish, is the alignment (src/AlignmentGraph.cpp:119-128).
        for(uint32_t v = pred[vFinish]; v != vStart; v = pred[v]) {
            pathCount++;
            const uint32_t delta = uint32_t(abs(int32_t(vert[v].o0) - int32_t(vert[v].o1)));
            if(delta < deltaThreshold) nearCount++;
        }
        if(job.pathOff != ~0ull) {
            uint64_t i = pathCount;
            for(uint32_t v = pred[vFinish]; v != vStart; v = pred[v]) paths[job.pathOff + --i] = vert[v];
        }
    }
    const double alignedFraction = double(pathCount) / double(n[0]);
    const double nearDiagonalFraction = double(nearCount) / double(n[0]);
    job.flag = (!(alignedFraction < alignedFractionThreshold) && !(nearDiagonalFraction < nearDiagonalFractionThreshold)) ? 1 : 0;
    job.aligned = uint32_t(pathCount);
    job.nearDiagonal = uint32_t(nearCount);
    job.heapPushes = pushes;
}

struct ExactTotals { uint64_t vertices = 0, edges = 0, heapPushes = 0, fallbacks = 0; };

constexpr uint32_t kPalWarpsPerBlock = 4;

// Phase B for the given reads. Scratch is sized per read (the phase-1 arena from the marker counts, the phase-2 arena
// from the exact vertex and edge counts phase 1 returns) and the reads are taken in batches whose scratch fits the budget
// (SHB_PALINDROMIC_BUDGET_MB, default 4096). wantPaths: the path ordinals of every read are returned in paths.
void runExact(shb_context* c, const shb_palindromic_params& p, const std::vector<uint64_t>& readIds, std::vector<PalJob>& out,
              std::vector<std::vector<uint32_t>>* paths, ExactTotals& totals)
{
    cudaStream_t st = c->stream;
    const uint64_t budget = uint64_t(envCount("SHB_PALINDROMIC_BUDGET_MB", 4096)) << 20;
    out.assign(readIds.size(), PalJob{});
    if(paths) paths->assign(readIds.size(), {});
    DeviceBuffer<uint8_t> arena1, arena2;
    DeviceBuffer<PalJob> jobsDev;
    DeviceBuffer<Vertex> pathDev;
    for(uint64_t begin = 0; begin < readIds.size(); ) {
        // Batch by phase-1 scratch.
        uint64_t end = begin, bytes1 = 0;
        while(end < readIds.size()) {
            const uint64_t r = readIds[end];
            PalJob& J = out[end];
            J = PalJob{};
            J.readId = r;
            J.n0 = uint32_t(c->tocHost[2 * r + 1] - c->tocHost[2 * r]);
            J.n1 = uint32_t(c->tocHost[2 * r + 2] - c->tocHost[2 * r + 1]);
            const uint64_t lo = std::min(J.n0, J.n1), hi = std::max(J.n0, J.n1);
            J.vCap = lo * std::min<uint64_t>(p.maxMarkerFrequency, hi);
            const uint64_t b = arena1Bytes(uint64_t(J.n0) + J.n1, J.vCap);
            if(end > begin && bytes1 + b > budget) break;
            J.off1 = bytes1; J.pathOff = ~0ull;
            bytes1 += b;
            end++;
        }
        const uint32_t nb = uint32_t(end - begin);
        arena1.reserve(bytes1 + 16);
        jobsDev.reserve(nb);
        SHB_CUDA(cudaMemcpyAsync(jobsDev.get(), out.data() + begin, nb * sizeof(PalJob), cudaMemcpyHostToDevice, st));
        SHB_LAUNCH(palVerticesKernel, ceilDiv(nb, kPalWarpsPerBlock), kPalWarpsPerBlock * 32, 0, st, jobsDev.get(), nb, arena1.get(),
                   c->kmerIds, (const uint64_t*)c->toc.get(), p.maxSkip, p.maxDrift, p.maxMarkerFrequency);
        SHB_CUDA(cudaMemcpyAsync(out.data() + begin, jobsDev.get(), nb * sizeof(PalJob), cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        // Phase 2 in sub-batches by its own scratch.
        for(uint64_t b2 = begin; b2 < end; ) {
            uint64_t e2 = b2, bytes2 = 0, pathEntries = 0;
            while(e2 < end) {
                SHB_REQUIRE(out[e2].pairEdges + 2 * out[e2].V < (1ull << 31), SHB_ERR_INVALID,
                        "A palindromic-read alignment graph has more than 2^31 edges.");
            const uint64_t b = arena2Bytes(out[e2].V, out[e2].pairEdges);
                if(e2 > b2 && bytes2 + b > budget) break;
                out[e2].off2 = bytes2;
                bytes2 += b;
                if(paths) { out[e2].pathOff = pathEntries; pathEntries += out[e2].V; }
                e2++;
            }
            const uint32_t n2 = uint32_t(e2 - b2);
            arena2.reserve(bytes2 + 16);
            if(paths) pathDev.reserve(pathEntries + 1);
            SHB_CUDA(cudaMemcpyAsync(jobsDev.get(), out.data() + b2, n2 * sizeof(PalJob), cudaMemcpyHostToDevice, st));
            // The phase-1 arena offsets of this sub-batch are relative to the batch, which is still resident.
            SHB_LAUNCH(palPathKernel, ceilDiv(n2, kPalWarpsPerBlock), kPalWarpsPerBlock * 32, 0, st, jobsDev.get(), n2, arena1.get(),
                       arena2.get(), paths ? pathDev.get() : nullptr, p.maxSkip, p.maxDrift, p.deltaThreshold,
                       p.alignedFractionThreshold, p.nearDiagonalFractionThreshold);
            SHB_CUDA(cudaMemcpyAsync(out.data() + b2, jobsDev.get(), n2 * sizeof(PalJob), cudaMemcpyDeviceToHost, st));
            SHB_CUDA(cudaStreamSynchronize(st));
            if(paths) {
                std::vector<Vertex> h(pathEntries);
                if(pathEntries) SHB_CUDA(cudaMemcpy(h.data(), pathDev.get(), pathEntries * sizeof(Vertex), cudaMemcpyDeviceToHost));
                for(uint64_t i = b2; i < e2; i++) {
                    std::vector<uint32_t>& v = (*paths)[i];
                    v.resize(2ull * out[i].aligned);
                    for(uint32_t k = 0; k < out[i].aligned; k++) { v[2 * k] = h[out[i].pathOff + k].o0; v[2 * k + 1] = h[out[i].pathOff + k].o1; }
                }
            }
            b2 = e2;
        }
        for(uint64_t i = begin; i < end; i++) {
            totals.vertices += out[i].V; totals.edges += out[i].pairEdges + 2 * out[i].V;
            totals.heapPushes += out[i].heapPushes; totals.fallbacks += out[i].fallbacks;
        }
        begin = end;
    }
}

} // namespace

void flagPalindromicReads(shb_context* c, const shb_palindromic_params& p, uint8_t* flagsOut, uint32_t* alignedOut,
                          uint32_t* nearOut, shb_palindromic_result* result)
{
    SHB_CUDA(cudaSetDevice(c->device));
    requireWholeAssembly(c, "flagPalindromicReads");
    const uint64_t launches0 = g_launchCount;
    const auto t0 = std::chrono::steady_clock::now();
    cudaStream_t st = c->stream;
    const uint64_t R = c->readCountTotal;
    DeviceBuffer<unsigned long long> vBound, vNearBound;
    DeviceBuffer<uint8_t> survives;
    vBound.reserve(R + 1); vNearBound.reserve(R + 1); survives.reserve(R + 1);

    // Phase A, in chunks of whole reads (SHB_PALINDROMIC_SORT_CHUNK markers: test hook), so that strand 0 of each read is
    // merge-joined against strand 1 inside one chunk.
    const uint64_t chunkLimit = envCount("SHB_PALINDROMIC_SORT_CHUNK", 1u << 28);
    sortMarkersByKmer(c, 2, chunkLimit, 32, "A read has more than 2^32-1 markers.",
                      [&](const uint64_t* keys, const uint32_t* vals, uint32_t rowBegin, uint32_t rowEnd, uint64_t markerBegin, uint32_t) {
        const uint64_t readBegin = rowBegin / 2, readEnd = rowEnd / 2;
        SHB_LAUNCH(palPrefilterKernel, ceilDiv(readEnd - readBegin, 128), 128, 0, st, keys, vals, (const uint64_t*)c->toc.get(),
                   readBegin, readEnd, markerBegin, p.maxMarkerFrequency, p.deltaThreshold, p.alignedFractionThreshold,
                   p.nearDiagonalFractionThreshold, vBound.get(), vNearBound.get(), survives.get());
    });
    std::vector<uint64_t> vb(R), vnb(R);
    std::vector<uint8_t> sv(R);
    if(R) {
        SHB_CUDA(cudaMemcpyAsync(vb.data(), vBound.get(), 8 * R, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaMemcpyAsync(vnb.data(), vNearBound.get(), 8 * R, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaMemcpyAsync(sv.data(), survives.get(), R, cudaMemcpyDeviceToHost, st));
    }
    SHB_CUDA(cudaStreamSynchronize(st));

    // Phase B.
    const auto t1 = std::chrono::steady_clock::now();
    std::vector<uint64_t> exactReads;
    for(uint64_t r = 0; r < R; r++) if(sv[r]) exactReads.push_back(r);
    std::vector<PalJob> jobs;
    ExactTotals totals;
    runExact(c, p, exactReads, jobs, nullptr, totals);
    const double totalMs = msSince(t0), exactMs = msSince(t1);

    // Bit 0 of the flags: reset everywhere (src/AssemblerAlign.cpp:676-681), set on the reads phase B flags. Bits 1-7 are kept.
    uint64_t palindromic = 0;
    for(uint64_t r = 0; r < R; r++) c->readFlagsHost[r] &= uint8_t(~1u);
    for(const PalJob& J : jobs) if(J.flag) { c->readFlagsHost[J.readId] |= 1u; palindromic++; }
    if(R) SHB_CUDA(cudaMemcpyAsync(c->readFlags.get(), c->readFlagsHost.data(), R, cudaMemcpyHostToDevice, st));
    SHB_CUDA(cudaStreamSynchronize(st));
    if(flagsOut) for(uint64_t r = 0; r < R; r++) flagsOut[r] = uint8_t((flagsOut[r] & ~1u) | (c->readFlagsHost[r] & 1u));
    // Counts: the reads phase A decided carry their bounds V and V_near (saturated to 32 bits); phase-B reads carry the
    // reference's aligned and near-diagonal counts.
    if(alignedOut) for(uint64_t r = 0; r < R; r++) alignedOut[r] = uint32_t(std::min<uint64_t>(vb[r], 0xffffffffu));
    if(nearOut) for(uint64_t r = 0; r < R; r++) nearOut[r] = uint32_t(std::min<uint64_t>(vnb[r], 0xffffffffu));
    for(const PalJob& J : jobs) {
        if(alignedOut) alignedOut[J.readId] = J.aligned;
        if(nearOut) nearOut[J.readId] = J.nearDiagonal;
    }
    if(result) {
        memset(result, 0, sizeof(*result));
        result->readCount = R;
        result->palindromicReadCount = palindromic;
        result->exactReadCount = exactReads.size();
        result->vertexCount = totals.vertices;
        result->edgeCount = totals.edges;
        result->heapPushCount = totals.heapPushes;
        result->heapsortFallbackCount = totals.fallbacks;
        result->totalMs = totalMs;
        result->exactMs = exactMs;
        result->kernelLaunches = g_launchCount - launches0;
    }
}

void palindromicReadAlignment(shb_context* c, uint64_t readId, const shb_palindromic_params& p, uint32_t** ordinals, uint64_t* count)
{
    SHB_CUDA(cudaSetDevice(c->device));
    requireWholeAssembly(c, "flagPalindromicReads");
    SHB_REQUIRE(readId < c->readCountTotal, SHB_ERR_INVALID, "Read id out of range.");
    std::vector<PalJob> jobs;
    std::vector<std::vector<uint32_t>> paths;
    ExactTotals totals;
    runExact(c, p, std::vector<uint64_t>{readId}, jobs, &paths, totals);
    const std::vector<uint32_t>& path = paths[0];
    HostResult out(allocHostResult(4 * path.size() + 8));
    SHB_REQUIRE(out.p != nullptr, SHB_ERR_OOM, "Out of host memory for the alignment.");
    if(!path.empty()) memcpy(out.p, path.data(), 4 * path.size());
    *count = path.size() / 2;
    *ordinals = static_cast<uint32_t*>(out.take());
}

} // namespace shb
