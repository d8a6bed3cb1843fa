// Host buffers handed to the caller (candidates, AlignmentData, compressed alignments, alignment table).
//
// Small buffers are plain malloc. Large ones (>= 8 MiB) are anonymous mappings, 2 MiB aligned with transparent huge pages
// requested, that can grow without copying what they hold (grow: mremap moves the pages). They are RECYCLED: shb_free puts
// them on a free list instead of returning them to the OS, so that a caller that runs the path repeatedly (the steady state
// bench.py measures) neither page-faults a fresh gigabyte per call nor munmaps one. A block that is reused is page-locked
// once (cudaHostRegister) and from then on filled by direct DMA instead of through the pinned staging ring (hostcopy.cuh).
// A one-shot caller never pays for page-locking. shb_trim_host_cache() returns the cached blocks to the OS.
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>
#include <vector>
#include <sys/mman.h>
#include <cuda_runtime.h>

namespace shb {

class HostPool {
public:
    static HostPool& instance()
    {
        static HostPool* pool = new HostPool();      // never destroyed: blocks may outlive the CUDA runtime at exit
        return *pool;
    }

    // Returns nullptr when out of memory.
    void* allocate(uint64_t bytes)
    {
        if(bytes < kLargeBytes) return malloc(bytes ? bytes : 1);
        std::lock_guard<std::mutex> lock(mutex_);
        // smallest cached block that fits without wasting more than 4x
        int best = -1;
        for(size_t k = 0; k < free_.size(); k++) {
            if(free_[k].capacity >= bytes && free_[k].capacity / 4 <= bytes && (best < 0 || free_[k].capacity < free_[size_t(best)].capacity)) best = int(k);
        }
        Block blk;
        if(best >= 0) {
            blk = free_[size_t(best)];
            free_.erase(free_.begin() + best);
            if(!blk.registered && !blk.registerFailed) {
                if(cudaHostRegister(blk.p, blk.capacity, cudaHostRegisterPortable) == cudaSuccess) blk.registered = true;
                else { cudaGetLastError(); blk.registerFailed = true; }
            }
        } else {
            const uint64_t slack = bytes + bytes / 8;                           // call-to-call size jitter still fits
            blk.capacity = (slack + kAlign - 1) & ~(kAlign - 1);
            blk.p = mapAligned(blk.capacity);
            if(!blk.p) return nullptr;
        }
        live_[blk.p] = blk;
        return blk.p;
    }

    // The block p (from allocate) must now hold `bytes`; its first `used` bytes are kept. Returns its address, which may have
    // changed, or nullptr when out of memory (p is then still valid). Nothing may write into p meanwhile, DMA included: a
    // page-locked block is unlocked first. A large block keeps its pages (mremap); only a small one is copied.
    void* grow(void* p, uint64_t used, uint64_t bytes)
    {
        std::unique_lock<std::mutex> lock(mutex_);
        auto it = live_.find(p);
        if(it == live_.end()) {             // small malloc block
            lock.unlock();
            void* q = allocate(bytes);
            if(q) { memcpy(q, p, used); free(p); }
            return q;
        }
        Block blk = it->second;
        if(blk.capacity >= bytes) return p;
        const uint64_t capacity = (bytes + bytes / 8 + kAlign - 1) & ~(kAlign - 1);
        void* q = mapAligned(capacity);
        if(!q) return nullptr;
        if(blk.registered && cudaHostUnregister(blk.p) != cudaSuccess) cudaGetLastError();
        it->second.registered = false;
        // onto the aligned range just mapped (MREMAP_FIXED replaces it), so that the grown block stays 2 MiB aligned
        if(mremap(blk.p, blk.capacity, capacity, MREMAP_MAYMOVE | MREMAP_FIXED, q) == MAP_FAILED) {
            munmap(q, capacity);
            return nullptr;
        }
        madvise(q, capacity, MADV_HUGEPAGE);
        live_.erase(it);
        blk.p = q; blk.capacity = capacity; blk.registered = false;
        live_[q] = blk;
        return q;
    }

    void release(void* p)
    {
        if(!p) return;
        std::lock_guard<std::mutex> lock(mutex_);
        auto it = live_.find(p);
        if(it == live_.end()) { free(p); return; }
        free_.push_back(it->second);
        live_.erase(it);
        while(free_.size() > kMaxCached) { destroy(free_.front()); free_.erase(free_.begin()); }    // oldest first
    }

    // True when device -> host copies into p can be plain asynchronous DMA.
    bool isPageLocked(const void* p)
    {
        std::lock_guard<std::mutex> lock(mutex_);
        auto it = live_.find(const_cast<void*>(p));
        return it != live_.end() && it->second.registered;
    }

    void trim()
    {
        std::lock_guard<std::mutex> lock(mutex_);
        for(Block& b : free_) destroy(b);
        free_.clear();
    }

private:
    struct Block { void* p = nullptr; uint64_t capacity = 0; bool registered = false, registerFailed = false; };
    static constexpr uint64_t kLargeBytes = 8ull << 20, kAlign = 2ull << 20;
    static constexpr size_t kMaxCached = 8;
    // An anonymous mapping of `bytes` (a multiple of kAlign) at a kAlign boundary; a page is only backed once touched.
    static void* mapAligned(uint64_t bytes)
    {
        void* raw = mmap(nullptr, bytes + kAlign, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if(raw == MAP_FAILED) return nullptr;
        const uintptr_t r = reinterpret_cast<uintptr_t>(raw), a = (r + kAlign - 1) & ~(kAlign - 1);
        if(a > r) munmap(raw, a - r);
        if(r + kAlign > a) munmap(reinterpret_cast<void*>(a + bytes), r + kAlign - a);
        madvise(reinterpret_cast<void*>(a), bytes, MADV_HUGEPAGE);
        return reinterpret_cast<void*>(a);
    }
    static void destroy(Block& b)
    {
        if(b.registered) { if(cudaHostUnregister(b.p) != cudaSuccess) cudaGetLastError(); }
        munmap(b.p, b.capacity);
    }
    std::mutex mutex_;
    std::vector<Block> free_;
    std::unordered_map<void*, Block> live_;
};

inline void* allocHostResult(uint64_t bytes) { return HostPool::instance().allocate(bytes); }

// Owns a host result block until it is handed to the caller: an exception on the way out releases it.
struct HostResult {
    void* p = nullptr;
    explicit HostResult(void* q = nullptr) : p(q) {}
    HostResult(const HostResult&) = delete;
    HostResult& operator=(const HostResult&) = delete;
    ~HostResult() { if(p) HostPool::instance().release(p); }
    void* take() { void* q = p; p = nullptr; return q; }
    void reset(void* q) { if(p) HostPool::instance().release(p); p = q; }
};

} // namespace shb
