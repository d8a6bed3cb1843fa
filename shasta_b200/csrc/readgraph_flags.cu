// Assembler::flagCrossStrandReadGraphEdges1 (src/AssemblerReadGraph.cpp:775-1041, ReadGraph.strandSeparationMethod 1) and
// Assembler::flagChimericReads (:355-583) on the GPU: the two steps every default assembly runs between the read graph and
// the marker graph vertices.
//
// Both are one bounded breadth-first search per read over the read graph. The device holds the graph as a CSR of
// neighbours: adj[p] = the other oriented read of edge connData[p] seen from the row's oriented read, with bit 31 set when
// the edge crossesStrands. One warp searches from one read:
//   * the reached oriented reads sit in an open-addressing table (keys, 2 * capacity slots, linear probing); verts[i] is
//     the table slot of the i-th reached vertex. The search is level-synchronous, so every level is a range of verts and
//     a vertex's distance is the level it falls in;
//   * the lanes spread over the adjacency rows of 32 frontier vertices at a time (an inclusive scan of the row lengths,
//     then each lane finds its row by a binary search over the shuffled scan);
//   * new vertices get their verts index from a ballot, so the count stays in a register and needs no atomic.
// The table lives in shared memory (capacity SHB_READGRAPH_FLAGS_TABLE_CAPACITY, default 1024). A read whose search
// reaches more vertices than that is marked as overflowed and is searched again by the same warp code with its table in
// global memory, in batches under SHB_READGRAPH_FLAGS_BUDGET_MB (default 2048; SHB_READGRAPH_FLAGS_BATCH caps the reads per
// batch, for tests), at 8x the capacity per round until the capacity holds every oriented read of the graph. So no answer
// is ever truncated. The overflow path keeps one warp per read: such reads are rare (none on the bench workload), and one
// code path for both tables keeps them exact by construction.
//
// Exactness.
//   Cross-strand, step 2: ReadGraph::computeShortPath(x-0, x-1, d) (src/ReadGraph.cpp:64-157) dequeues only vertices at
//   distance < d and reports a path as soon as x-1 is a neighbour of a dequeued vertex, so it finds one iff
//   dist(x-0, x-1) <= d. The search here expands levels 0 .. d-1 from x-0 and stops at the first edge into x-1: the same
//   predicate. Every crossesStrands flag is cleared before the searches, so no edge is skipped.
//   Cross-strand, step 3: the regions are the connected components of the edges whose two ends are near a strand jump: a
//   min-linking union-find on the device, whose partition does not depend on the order of the unions.
//   Cross-strand, step 4: on the host, over the regions, with the reference's gathering order and std::sort with the same
//   comparisons on the same element types (processRegion below): the same input and libstdc++ give the same permutation.
//   Chimeric: the search from x-0 skips crossesStrands edges and records every vertex at distance <= d; the components are
//   those of the recorded vertices other than x-0 and x-1 under the edges that do not cross strands and do not touch read
//   x; x is chimeric iff the recorded vertices at distance exactly d, other than x-1, fall into two or more components.
//   All of these are properties of sets, which the order of the search and of the unions does not change. The union-find
//   is over table slots, min-linking with atomicCAS.
#include "context.cuh"
#include "hostpool.cuh"

#include <algorithm>
#include <array>
#include <chrono>
#include <cstring>
#include <string>
#include <vector>

namespace shb {
namespace {

constexpr uint32_t kEmpty = 0xffffffffu;
constexpr uint32_t kCrossBit = 0x80000000u;
constexpr uint32_t kWarps = 4;                              // warps (reads) per block

// Result codes of one read's search.
constexpr uint8_t kNo = 0, kYes = 1, kOverflow = 2;

// One warp's table: keys[2 * capacity], verts[capacity], and for the chimeric test parent[2 * capacity].
struct Table {
    uint32_t* keys;
    uint32_t* verts;
    uint32_t* parent;
    uint32_t capacity;
};

__device__ __forceinline__ uint32_t hashSlot(uint32_t key, uint32_t mask) { return (key * 2654435761u) & mask; }

// Slot of key, or kEmpty when it is not in the table.
__device__ __forceinline__ uint32_t lookup(const Table& t, uint32_t key)
{
    const uint32_t mask = 2u * t.capacity - 1u;
    for(uint32_t s = hashSlot(key, mask);; s = (s + 1u) & mask) {
        const uint32_t k = ((volatile uint32_t*)t.keys)[s];
        if(k == key) return s;
        if(k == kEmpty) return kEmpty;
    }
}

// Inserts key; returns its slot and whether this call put it there.
__device__ __forceinline__ uint32_t insert(const Table& t, uint32_t key, bool& isNew)
{
    const uint32_t mask = 2u * t.capacity - 1u;
    for(uint32_t s = hashSlot(key, mask);; s = (s + 1u) & mask) {
        const uint32_t old = atomicCAS(t.keys + s, kEmpty, key);
        if(old == kEmpty) { isNew = true; return s; }
        if(old == key) { isNew = false; return s; }
    }
}

__device__ __forceinline__ uint32_t findRoot(const uint32_t* parent, uint32_t i)
{
    for(;;) {
        const uint32_t p = ((volatile const uint32_t*)parent)[i];
        if(p == i) return i;
        i = p;
    }
}

__device__ __forceinline__ void unite(uint32_t* parent, uint32_t a, uint32_t b)
{
    for(;;) {
        a = findRoot(parent, a);
        b = findRoot(parent, b);
        if(a == b) return;
        if(a < b) { const uint32_t t = a; a = b; b = t; }
        if(atomicCAS(parent + a, a, b) == a) return;    // link the larger root under the smaller
    }
}

// Calls f(vertex index, adjacency word, valid) on every lane for the adjacency entries of verts[begin, end), the lanes
// spread over the rows of 32 vertices at a time; lanes without an entry get valid = false (f may use warp collectives).
// f returns true, warp-uniformly, to stop; the return value says whether it did.
template<class F>
__device__ __forceinline__ bool forEachNeighbour(const Table& t, const uint32_t* __restrict__ toc, const uint32_t* __restrict__ adj,
                                                 uint32_t begin, uint32_t end, uint32_t lane, F&& f)
{
    for(uint32_t chunk = begin; chunk < end; chunk += 32u) {
        const uint32_t i = chunk + lane;
        uint32_t rowStart = 0, deg = 0;
        if(i < end) {
            const uint32_t v = t.keys[t.verts[i]];
            rowStart = toc[v];
            deg = toc[v + 1] - rowStart;
        }
        uint32_t incl = deg;
#pragma unroll
        for(uint32_t o = 1; o < 32u; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
            if(lane >= o) incl += y;
        }
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        for(uint32_t base = 0; base < total; base += 32u) {
            const uint32_t e = base + lane;
            uint32_t owner = 0;                     // the number of lanes whose inclusive sum is <= e
#pragma unroll
            for(uint32_t step = 16; step >= 1; step >>= 1) {
                const uint32_t probe = __shfl_sync(0xffffffffu, incl, owner + step - 1u);
                if(probe <= e) owner += step;
            }
            const uint32_t ownerIncl = __shfl_sync(0xffffffffu, incl, owner);
            const uint32_t ownerDeg = __shfl_sync(0xffffffffu, deg, owner);
            const uint32_t ownerStart = __shfl_sync(0xffffffffu, rowStart, owner);
            const bool valid = e < total;
            const uint32_t w = valid ? adj[ownerStart + e - (ownerIncl - ownerDeg)] : 0u;
            if(f(chunk + owner, w, valid)) return true;
        }
    }
    return false;
}

// The bounded search from `start`: levels 0 .. maxDistance-1 are expanded, so every vertex at distance <= maxDistance is
// reached. With target != kEmpty it stops at the first edge into target and returns kYes. Otherwise it returns kNo with
// [lastBegin, n) = the vertices at distance exactly maxDistance (empty when the ball ends earlier). kOverflow when the ball
// does not fit the table.
__device__ uint8_t boundedSearch(const Table& t, const uint32_t* __restrict__ toc, const uint32_t* __restrict__ adj, uint32_t start,
                                 uint32_t target, uint32_t maxDistance, bool skipCross, uint32_t lane, uint32_t& n, uint32_t& lastBegin)
{
    if(lane == 0) {
        bool isNew;
        t.verts[0] = insert(t, start, isNew);
    }
    __syncwarp();
    n = 1;
    uint32_t levelBegin = 0, levelEnd = 1, depth = 0;
    uint8_t outcome = kNo;
    while(depth < maxDistance && levelBegin < levelEnd) {
        const bool stopped = forEachNeighbour(t, toc, adj, levelBegin, levelEnd, lane, [&](uint32_t, uint32_t w, bool valid) -> bool {
            bool isNew = false, hit = false;
            uint32_t slot = 0;
            if(valid && !(skipCross && (w & kCrossBit))) {
                const uint32_t u = w & ~kCrossBit;
                if(u == target) hit = true;
                else slot = insert(t, u, isNew);
            }
            const uint32_t newMask = __ballot_sync(0xffffffffu, isNew);
            const uint32_t added = __popc(newMask);
            if(n + added > t.capacity) { outcome = kOverflow; return true; }
            if(isNew) t.verts[n + __popc(newMask & ((1u << lane) - 1u))] = slot;
            n += added;
            if(__any_sync(0xffffffffu, hit)) { outcome = kYes; return true; }
            return false;
        });
        __syncwarp();
        if(stopped) break;
        levelBegin = levelEnd;
        levelEnd = n;
        depth++;
    }
    lastBegin = (depth == maxDistance) ? levelBegin : n;
    return outcome;
}

// One warp per read. jobs (nullptr: read = job index) lists the reads; tables (nullptr: shared memory) holds one table of
// `words` words per job, cleared to kEmpty by the caller. out[read] = kYes / kNo; an overflowed read goes to overflowList.
// hist[k] counts the searches that reached [2^k, 2^(k+1)) vertices.
template<bool kChimeric>
__global__ void __launch_bounds__(kWarps * 32) searchKernel(const uint32_t* __restrict__ toc, const uint32_t* __restrict__ adj,
                                                            const uint32_t* __restrict__ jobs, uint32_t jobCount, uint32_t maxDistance,
                                                            uint32_t capacity, uint32_t* tables, uint8_t* __restrict__ out,
                                                            uint32_t* __restrict__ overflowList, uint32_t* __restrict__ overflowCount,
                                                            unsigned long long* __restrict__ hist)
{
    extern __shared__ uint32_t smem[];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t job = blockIdx.x * kWarps + warp;
    if(job >= jobCount) return;
    const uint32_t read = jobs ? jobs[job] : job;
    const uint64_t words = uint64_t(kChimeric ? 5u : 3u) * capacity;
    uint32_t* base = tables ? tables + uint64_t(job) * words : smem + warp * words;
    const Table t{base, base + 2ull * capacity, kChimeric ? base + 3ull * capacity : nullptr, capacity};
    if(!tables) {
        for(uint32_t s = lane; s < 2u * capacity; s += 32u) t.keys[s] = kEmpty;
        __syncwarp();
    }
    uint32_t n, lastBegin;
    uint8_t r = boundedSearch(t, toc, adj, 2u * read, kChimeric ? kEmpty : 2u * read + 1u, maxDistance, kChimeric, lane, n, lastBegin);
    if(kChimeric && r == kNo) {
        for(uint32_t i = lane; i < n; i += 32u) t.parent[t.verts[i]] = t.verts[i];
        __syncwarp();
        // Components of the ball without read x and without the edges that cross strands or touch read x.
        forEachNeighbour(t, toc, adj, 0u, n, lane, [&](uint32_t i, uint32_t w, bool valid) -> bool {
            if(valid && !(w & kCrossBit) && (w >> 1) != read) {
                const uint32_t sv = t.verts[i];
                if((t.keys[sv] >> 1) != read) {
                    const uint32_t su = lookup(t, w);
                    if(su != kEmpty) unite(t.parent, sv, su);
                }
            }
            return false;
        });
        __syncwarp();
        uint32_t lo = kEmpty, hi = 0;
        for(uint32_t i = lastBegin; i < n; i += 32u) {
            const uint32_t k = i + lane;
            if(k < n && (t.keys[t.verts[k]] >> 1) != read) {
                const uint32_t root = findRoot(t.parent, t.verts[k]);
                lo = min(lo, root);
                hi = max(hi, root);
            }
        }
#pragma unroll
        for(uint32_t o = 16; o >= 1; o >>= 1) {
            lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
        r = (lo != kEmpty && lo != hi) ? kYes : kNo;
    }
    if(lane == 0) {
        if(r == kOverflow) {
            overflowList[atomicAdd(overflowCount, 1u)] = read;
        } else {
            out[read] = r;
            atomicAdd(hist + (31 - __clz(n)), 1ull);
        }
    }
}

// adj[p] for every connectivity entry p of row `row` (one thread per entry, the row found by binary search in toc). An
// entry whose edge does not exist or does not touch its row counts in *bad (the reference's getOther asserts).
__global__ void adjacencyKernel(const uint32_t* __restrict__ toc, uint32_t rows, const uint32_t* __restrict__ data, uint32_t entries,
                                const uint32_t* __restrict__ edges, uint64_t edgeCount, bool keepCross, uint32_t* __restrict__ adj,
                                uint32_t* __restrict__ bad)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if(p >= entries) return;
    const uint32_t lo = rowOf(toc, 0u, rows, p);
    const uint32_t e = data[p];
    if(e >= edgeCount) { atomicAdd(bad, 1u); adj[p] = 0; return; }
    const uint32_t w0 = edges[4ull * e], w1 = edges[4ull * e + 1], flags = edges[4ull * e + 3];
    uint32_t other;
    if(w0 == lo) other = w1;
    else if(w1 == lo) other = w0;
    else { atomicAdd(bad, 1u); adj[p] = 0; return; }
    if(other >= rows) { atomicAdd(bad, 1u); adj[p] = 0; return; }
    adj[p] = other | ((keepCross && (flags & 0x40000000u)) ? kCrossBit : 0u);
}

// Regions: min-linking union-find over the edges whose two ends are near a strand jump (nearRead[v >> 1] == kYes).
__global__ void regionUnionKernel(const uint32_t* __restrict__ edges, uint64_t edgeCount, const uint8_t* __restrict__ nearRead,
                                  uint32_t* parent)
{
    const uint64_t e = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if(e >= edgeCount) return;
    const uint32_t v0 = edges[4 * e], v1 = edges[4 * e + 1];
    if(nearRead[v0 >> 1] == kYes && nearRead[v1 >> 1] == kYes) unite(parent, v0, v1);
}

__global__ void regionInitKernel(uint32_t* parent, uint32_t rows)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if(v < rows) parent[v] = v;
}

// root[v] = the smallest vertex of v's region for a vertex near a strand jump, kEmpty otherwise.
__global__ void regionRootKernel(uint32_t* parent, uint32_t rows, const uint8_t* __restrict__ nearRead, uint32_t* __restrict__ root)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if(v < rows) root[v] = nearRead[v >> 1] == kYes ? findRoot(parent, v) : kEmpty;
}

struct DeviceGraph {
    DeviceBuffer<uint32_t> toc, adj, edges, scratch;
};

constexpr uint32_t kAlignmentWords = 16;            // 64-byte AlignmentData
constexpr uint32_t kMarkerCountWord = 9;
constexpr uint32_t kInfoFlagsWord = 15;             // bit 0: AlignmentInfo::isInReadGraph

// Checks the shape of the read graph and builds the device CSR. keepCross: the adjacency words carry crossesStrands.
void buildGraph(shb_context* c, const uint32_t* edges, uint64_t edgeCount, const uint32_t* connToc, const uint32_t* connData,
                uint64_t readCount, bool keepCross, DeviceGraph& g, Footprint& fp)
{
    // Oriented read ids below 2^30 leave bit 31 of an adjacency word to crossesStrands, and a table that holds every oriented
    // read (2^30 entries, 2^31 hash slots) still indexes in 32 bits.
    SHB_REQUIRE(readCount < (1ull << 29), SHB_ERR_INVALID, "Too many reads for the read graph flags (limit 2^29-1).");
    SHB_REQUIRE(edgeCount < (1ull << 32), SHB_ERR_INVALID, "Too many read graph edges.");
    const uint64_t rows = 2 * readCount;
    SHB_REQUIRE(connToc[0] == 0, SHB_ERR_INVALID, "ReadGraphConnectivity does not start at 0.");
    for(uint64_t v = 0; v < rows; v++) {
        SHB_REQUIRE(connToc[v + 1] >= connToc[v], SHB_ERR_INVALID, "ReadGraphConnectivity is not monotone.");
    }
    for(uint64_t e = 0; e < edgeCount; e++) {
        SHB_REQUIRE(edges[4 * e] < rows && edges[4 * e + 1] < rows, SHB_ERR_INVALID,
                    "Read graph edge " + std::to_string(e) + " refers to an oriented read that does not exist.");
    }
    const uint32_t entries = connToc[rows];
    cudaStream_t st = c->stream;
    fp.add(g.toc, rows + 1); fp.add(g.adj, uint64_t(entries) + 1); fp.add(g.edges, 4 * edgeCount + 4); fp.add(g.scratch, uint64_t(entries) + 1);
    SHB_CUDA(cudaMemcpyAsync(g.toc.get(), connToc, 4 * (rows + 1), cudaMemcpyHostToDevice, st));
    if(edgeCount) SHB_CUDA(cudaMemcpyAsync(g.edges.get(), edges, 16 * edgeCount, cudaMemcpyHostToDevice, st));
    if(entries) {
        uint32_t* dData = g.scratch.get();
        SHB_CUDA(cudaMemcpyAsync(dData, connData, 4ull * entries, cudaMemcpyHostToDevice, st));
        uint32_t* bad = reinterpret_cast<uint32_t*>(c->scalar(kSlotBadConnectivity));
        SHB_CUDA(cudaMemsetAsync(bad, 0, 4, st));
        SHB_LAUNCH(adjacencyKernel, ceilDiv(entries, 256), 256, 0, st, (const uint32_t*)g.toc.get(), uint32_t(rows), (const uint32_t*)dData,
                   entries, (const uint32_t*)g.edges.get(), edgeCount, keepCross, g.adj.get(), bad);
        const uint32_t badHost = readBack(bad, st);
        SHB_REQUIRE(badHost == 0, SHB_ERR_INVALID, std::to_string(badHost) +
                    " ReadGraphConnectivity entries name an edge that does not exist or does not touch their oriented read.");
    }
}

uint32_t pow2AtLeast(uint64_t x)
{
    uint32_t p = 32;
    while(p < x && p < (1u << 31)) p <<= 1;
    return p;
}

// Every read's search: out[read] = kYes / kNo (host, readCount bytes). Overflowed reads are searched again with tables in
// global memory at 8x the capacity per round, in batches under the budget, until none is left.
template<bool kChimeric>
void runSearches(shb_context* c, DeviceGraph& g, uint64_t readCount, uint32_t maxDistance, uint8_t* outHost, uint64_t* overflowReads,
                 uint64_t* histOut, Footprint& fp)
{
    cudaStream_t st = c->stream;
    const uint32_t R = uint32_t(readCount);
    const uint32_t wordsPer = kChimeric ? 5u : 3u;
    uint32_t capacity = std::min<uint32_t>(pow2AtLeast(envCount("SHB_READGRAPH_FLAGS_TABLE_CAPACITY", 1024)), 2048);
    const uint64_t budget = uint64_t(envCount("SHB_READGRAPH_FLAGS_BUDGET_MB", 2048)) << 20;
    const uint32_t maxBatch = envCount("SHB_READGRAPH_FLAGS_BATCH", 1u << 30);
    DeviceBuffer<uint8_t> dOut;
    DeviceBuffer<uint32_t> dOverflow, dJobs, dTables;
    DeviceBuffer<unsigned long long> dHist;
    fp.add(dOut, R + 1); fp.add(dOverflow, R + 2); fp.add(dHist, 32);
    uint32_t* dCount = dOverflow.get() + R + 1;
    SHB_CUDA(cudaMemsetAsync(dHist.get(), 0, 32 * 8, st));
    SHB_CUDA(cudaMemsetAsync(dCount, 0, 4, st));
    const size_t smem = size_t(kWarps) * wordsPer * capacity * 4;
    SHB_CUDA(cudaFuncSetAttribute(searchKernel<kChimeric>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    SHB_LAUNCH(searchKernel<kChimeric>, ceilDiv(R, kWarps), kWarps * 32, smem, st, (const uint32_t*)g.toc.get(), (const uint32_t*)g.adj.get(),
               (const uint32_t*)nullptr, R, maxDistance, capacity, (uint32_t*)nullptr, dOut.get(), dOverflow.get(), dCount, dHist.get());
    std::vector<uint32_t> pending;
    auto collect = [&] {
        uint32_t k = 0;
        SHB_CUDA(cudaMemcpyAsync(&k, dCount, 4, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        pending.resize(k);
        if(k) SHB_CUDA(cudaMemcpyAsync(pending.data(), dOverflow.get(), 4ull * k, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaMemsetAsync(dCount, 0, 4, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        std::sort(pending.begin(), pending.end());      // batches do not depend on the order the warps finished in
    };
    collect();
    *overflowReads = pending.size();
    const uint64_t vertices = 2ull * readCount;
    while(!pending.empty()) {
        // A table of capacity >= 2 * readCount holds every oriented read: the last round cannot overflow.
        capacity = uint32_t(std::min<uint64_t>(uint64_t(capacity) * 8, pow2AtLeast(vertices)));
        const uint64_t perRead = uint64_t(wordsPer) * capacity * 4;
        const uint64_t batch = std::max<uint64_t>(1, std::min<uint64_t>({budget / perRead, pending.size(), maxBatch}));
        fp.add(dJobs, batch); fp.add(dTables, batch * wordsPer * capacity);
        const std::vector<uint32_t> round = std::move(pending);
        for(uint64_t b = 0; b < round.size(); b += batch) {
            const uint32_t jobs = uint32_t(std::min<uint64_t>(batch, round.size() - b));
            SHB_CUDA(cudaMemcpyAsync(dJobs.get(), round.data() + b, 4ull * jobs, cudaMemcpyHostToDevice, st));
            // only the keys (the first 2 * capacity words of each job's table) need clearing
            SHB_CUDA(cudaMemset2DAsync(dTables.get(), 4ull * wordsPer * capacity, 0xff, 8ull * capacity, jobs, st));
            SHB_LAUNCH(searchKernel<kChimeric>, ceilDiv(jobs, kWarps), kWarps * 32, 0, st, (const uint32_t*)g.toc.get(),
                       (const uint32_t*)g.adj.get(), (const uint32_t*)dJobs.get(), jobs, maxDistance, capacity, dTables.get(),
                       dOut.get(), dOverflow.get(), dCount, dHist.get());
        }
        collect();
        SHB_REQUIRE(pending.empty() || capacity < vertices, SHB_ERR_CUDA, "A read graph search overflowed a table that holds every read.");
    }
    SHB_CUDA(cudaMemcpyAsync(outHost, dOut.get(), R, cudaMemcpyDeviceToHost, st));
    unsigned long long hist[32];
    SHB_CUDA(cudaMemcpyAsync(hist, dHist.get(), sizeof(hist), cudaMemcpyDeviceToHost, st));
    SHB_CUDA(cudaStreamSynchronize(st));
    for(int k = 0; k < 32; k++) histOut[k] = hist[k];
}

struct HostUnionFind {
    std::vector<uint32_t> p;
    explicit HostUnionFind(uint32_t n) : p(n) { for(uint32_t i = 0; i < n; i++) p[i] = i; }
    uint32_t find(uint32_t i) { while(p[i] != i) { p[i] = p[p[i]]; i = p[i]; } return i; }
    void unite(uint32_t a, uint32_t b) { a = find(a); b = find(b); if(a != b) p[std::max(a, b)] = std::min(a, b); }
};

// Step 4 of flagCrossStrandReadGraphEdges1 for one strand jump region (src/AssemblerReadGraph.cpp:869-1010). vertices: the
// region's oriented reads in increasing order. Appends the edges it flags to `flagged`; a reference assertion throws
// SHB_ERR_INVALID (nothing is written before every region is processed).
void processRegion(const std::vector<uint32_t>& vertices, const uint32_t* edges, const uint32_t* connToc, const uint32_t* connData,
                   const uint32_t* rec, uint64_t alignmentCount, std::vector<uint32_t>& flagged)
{
    const size_t vertexCount = vertices.size();
    const std::string where = "The strand jump region that contains oriented read " + std::to_string(vertices.front());
    SHB_REQUIRE(vertexCount % 2 == 0, SHB_ERR_INVALID, where + " has an odd number of vertices.");
    for(size_t i = 0; i < vertexCount; i += 2) {
        SHB_REQUIRE((vertices[i] >> 1) == (vertices[i + 1] >> 1) && (vertices[i] & 1) == 0 && (vertices[i + 1] & 1) == 1, SHB_ERR_INVALID,
                    where + " is not made of the two strands of its reads.");
    }
    auto index = [&](uint32_t v) -> int64_t {
        const auto it = std::lower_bound(vertices.begin(), vertices.end(), v);
        return (it != vertices.end() && *it == v) ? int64_t(it - vertices.begin()) : -1;
    };
    // :897-914, in (vertex, connectivity row) order
    std::vector<std::pair<uint32_t, uint64_t>> edgeIds;
    for(const uint32_t v0 : vertices) {
        for(uint32_t p = connToc[v0]; p < connToc[v0 + 1]; p++) {
            const uint32_t e = connData[p];
            const uint32_t* w = edges + 4ull * e;
            const uint32_t v1 = (w[0] == v0) ? w[1] : w[0];
            if(index(v1) < 0) continue;
            if(w[0] == v0) edgeIds.push_back(std::make_pair(e, uint64_t(w[2]) | (uint64_t(w[3] & 0x3fffffffu) << 32)));
        }
    }
    SHB_REQUIRE(edgeIds.size() % 2 == 0, SHB_ERR_INVALID, where + " has an odd number of edges.");
    // :920-921, OrderPairsBySecondOnly (unstable)
    std::sort(edgeIds.begin(), edgeIds.end(), [](const std::pair<uint32_t, uint64_t>& x, const std::pair<uint32_t, uint64_t>& y) {
        return x.second < y.second;
    });
    std::vector<std::pair<std::array<uint32_t, 2>, uint32_t>> edgePairs;
    for(size_t i = 0; i < edgeIds.size(); i += 2) {
        const uint64_t alignmentId = edgeIds[i].second;
        SHB_REQUIRE(alignmentId == edgeIds[i + 1].second, SHB_ERR_INVALID,
                    where + " has edges " + std::to_string(edgeIds[i].first) + " and " + std::to_string(edgeIds[i + 1].first) +
                    " paired by alignment id order but with different alignment ids.");
        SHB_REQUIRE(alignmentId < alignmentCount, SHB_ERR_INVALID,
                    "Read graph edge " + std::to_string(edgeIds[i].first) + " refers to an alignment that does not exist.");
        const uint32_t markerCount = rec[kAlignmentWords * alignmentId + kMarkerCountWord];
        edgePairs.push_back(std::make_pair(std::array<uint32_t, 2>{edgeIds[i].first, edgeIds[i + 1].first}, markerCount));
    }
    // :937-938, OrderPairsBySecondOnlyGreater (unstable)
    std::sort(edgePairs.begin(), edgePairs.end(), [](const std::pair<std::array<uint32_t, 2>, uint32_t>& x,
                                                     const std::pair<std::array<uint32_t, 2>, uint32_t>& y) { return x.second > y.second; });
    HostUnionFind uf{uint32_t(vertexCount)};
    for(const auto& pr : edgePairs) {
        for(const uint32_t e : pr.first) {
            const uint32_t* w = edges + 4ull * e;
            const uint32_t i0 = uint32_t(index(w[0])), i1 = uint32_t(index(w[1]));
            const uint32_t i0rc = uint32_t(index(w[0] ^ 1u)), i1rc = uint32_t(index(w[1] ^ 1u));
            const uint32_t c0 = uf.find(i0), c1 = uf.find(i1), c0rc = uf.find(i0rc), c1rc = uf.find(i1rc);
            // The reference's SHASTA_ASSERT(component0 != component0rc). Every union joins (u, v) and (rc u, rc v) together,
            // so the components stay closed under reverse complement, and an edge that would join a vertex to its reverse
            // complement is flagged instead; the check cannot fail. It is kept as the reference keeps it.
            SHB_REQUIRE(c0 != c0rc && c1 != c1rc, SHB_ERR_INVALID,
                        where + ": an oriented read and its reverse complement are already joined when edge " + std::to_string(e) +
                        " is processed.");
            if(c0 == c1rc || c1 == c0rc) {
                flagged.push_back(e);
            } else {
                uf.unite(i0, i1);
                uf.unite(i0rc, i1rc);
            }
        }
    }
}

} // namespace

void flagCrossStrandReadGraphEdges1(shb_context* c, int64_t maxDistance, uint32_t* edges, uint64_t edgeCount, const uint32_t* connToc,
                                    const uint32_t* connData, uint64_t readCount, uint32_t* rec, uint64_t alignmentCount,
                                    shb_cross_strand_result* result)
{
    const auto t0 = std::chrono::steady_clock::now();
    shb_cross_strand_result res{};
    SHB_REQUIRE(maxDistance >= 0, SHB_ERR_INVALID, "flagCrossStrandReadGraphEdges1: maxDistance must not be negative.");
    SHB_CUDA(cudaSetDevice(c->device));
    const uint64_t rows = 2 * readCount;
    std::vector<uint32_t> flagged;
    std::vector<uint8_t> nearRead(readCount, 0);
    if(maxDistance > 0 && readCount) {
        const auto t1 = std::chrono::steady_clock::now();
        Footprint fp;
        DeviceGraph g;
        buildGraph(c, edges, edgeCount, connToc, connData, readCount, false, g, fp);
        runSearches<false>(c, g, readCount, uint32_t(std::min<uint64_t>(uint64_t(maxDistance), rows)), nearRead.data(),
                           &res.overflowReadCount, res.ballSizeHistogram, fp);
        // Regions (:830-863) on the device; the near flags are still there from the searches.
        cudaStream_t st = c->stream;
        DeviceBuffer<uint8_t> dNear;
        DeviceBuffer<uint32_t> dParent, dRoot;
        fp.add(dNear, readCount); fp.add(dParent, rows); fp.add(dRoot, rows);
        SHB_CUDA(cudaMemcpyAsync(dNear.get(), nearRead.data(), readCount, cudaMemcpyHostToDevice, st));
        SHB_LAUNCH(regionInitKernel, ceilDiv(rows, 256), 256, 0, st, dParent.get(), uint32_t(rows));
        if(edgeCount) SHB_LAUNCH(regionUnionKernel, ceilDiv(edgeCount, 256), 256, 0, st, (const uint32_t*)g.edges.get(), edgeCount,
                                 (const uint8_t*)dNear.get(), dParent.get());
        SHB_LAUNCH(regionRootKernel, ceilDiv(rows, 256), 256, 0, st, dParent.get(), uint32_t(rows), (const uint8_t*)dNear.get(), dRoot.get());
        std::vector<uint32_t> root(rows);
        SHB_CUDA(cudaMemcpyAsync(root.data(), dRoot.get(), 4 * rows, cudaMemcpyDeviceToHost, st));
        SHB_CUDA(cudaStreamSynchronize(st));
        res.deviceMs = msSince(t1);
        res.peakDeviceBytes = fp.peak;
        // Step 4 on the host. A region's root is its smallest vertex, so it is met first in increasing vertex order.
        const auto t2 = std::chrono::steady_clock::now();
        std::vector<uint32_t> regionOf(rows, kEmpty);
        std::vector<std::vector<uint32_t>> regions;
        for(uint64_t v = 0; v < rows; v++) {
            if(root[v] == kEmpty) continue;
            if(root[v] == v) { regionOf[v] = uint32_t(regions.size()); regions.emplace_back(); }
            regions[regionOf[root[v]]].push_back(uint32_t(v));
        }
        for(const auto& vertices : regions) {
            if(vertices.size() < 2) continue;
            res.regionCount++;
            processRegion(vertices, edges, connToc, connData, rec, alignmentCount, flagged);
        }
        res.hostMs = msSince(t2);
        for(uint64_t x = 0; x < readCount; x++) {
            if(nearRead[x] != kYes) continue;
            res.nearStrandJumpCount += 2;
            res.nearStrandJumpReportedCount += (2 * x < readCount) + (2 * x + 1 < readCount);      // isNearStrandJump[readId], readId < readCount (:820-824)
        }
    }
    // Nothing was written so far: apply (:796-799, :992-998).
    for(uint64_t e = 0; e < edgeCount; e++) edges[4 * e + 3] &= ~0x40000000u;
    for(const uint32_t e : flagged) {
        edges[4ull * e + 3] |= 0x40000000u;
        const uint64_t a = uint64_t(edges[4ull * e + 2]) | (uint64_t(edges[4ull * e + 3] & 0x3fffffffu) << 32);
        rec[kAlignmentWords * a + kInfoFlagsWord] &= ~1u;
    }
    res.crossStrandEdgeCount = flagged.size();
    res.totalMs = msSince(t0);
    if(result) *result = res;
}

void flagChimericReads(shb_context* c, uint64_t maxDistance, const uint32_t* edges, uint64_t edgeCount, const uint32_t* connToc,
                       const uint32_t* connData, uint64_t readCount, uint8_t* readFlags, uint32_t* rec, uint64_t alignmentCount,
                       shb_chimeric_result* result)
{
    const auto t0 = std::chrono::steady_clock::now();
    shb_chimeric_result res{};
    SHB_REQUIRE(maxDistance < 255, SHB_ERR_INVALID, "flagChimericReads: maxDistance must be less than 255.");
    SHB_CUDA(cudaSetDevice(c->device));
    std::vector<uint8_t> chimeric(readCount, 0);
    if(maxDistance > 0 && readCount) {
        for(uint64_t a = 0; a < alignmentCount; a++) {
            SHB_REQUIRE(rec[kAlignmentWords * a] < readCount && rec[kAlignmentWords * a + 1] < readCount, SHB_ERR_INVALID,
                        "Alignment " + std::to_string(a) + " refers to a read that does not exist.");
        }
        const auto t1 = std::chrono::steady_clock::now();
        Footprint fp;
        DeviceGraph g;
        buildGraph(c, edges, edgeCount, connToc, connData, readCount, true, g, fp);
        runSearches<true>(c, g, readCount, uint32_t(maxDistance), chimeric.data(), &res.overflowReadCount, res.ballSizeHistogram, fp);
        res.peakDeviceBytes = fp.peak;
        res.deviceMs = msSince(t1);
    }
    // Nothing was written so far: the isChimeric bit of every read (ReadFlags bit 1), then isInReadGraph of every alignment
    // of a chimeric read (alignmentTable[x-0] holds every alignment with readIds[0] == x or readIds[1] == x).
    for(uint64_t x = 0; x < readCount; x++) {
        readFlags[x] = uint8_t((readFlags[x] & ~2u) | (chimeric[x] ? 2u : 0u));
        res.chimericReadCount += chimeric[x];
    }
    if(res.chimericReadCount) {
        for(uint64_t a = 0; a < alignmentCount; a++) {
            uint32_t* r = rec + kAlignmentWords * a;
            if(chimeric[r[0]] || chimeric[r[1]]) r[kInfoFlagsWord] &= ~1u;
        }
    }
    res.totalMs = msSince(t0);
    if(result) *result = res;
}

} // namespace shb
