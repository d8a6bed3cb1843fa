// Device -> host copies of results into host blocks from the pool (hostpool.cuh), queued while the GPU still works.
//
// A page-locked block is filled by plain DMA on the copy stream. A pageable one is filled through the context's ring of pinned
// staging chunks: DMA into a chunk on the copy stream, then a host memcpy from the chunk into the block, on one of a few
// long-lived threads of the copier. Those threads also take the first-touch page faults of the blocks. The thread that queues
// a copy never waits for them; finish() waits once, at the end of the call.
#pragma once
#include "context.cuh"
#include "hostpool.cuh"

#include <condition_variable>
#include <deque>
#include <exception>
#include <functional>
#include <mutex>
#include <shared_mutex>
#include <thread>
#include <vector>

namespace shb {

// A host result block that the copier may grow (data of unknown size): p and capacity change only under `resize`.
struct HostBlock {
    HostResult owner;
    uint64_t capacity = 0;
    bool pageLocked = false;
    std::shared_mutex resize;           // shared: a memcpy into the block; exclusive: growing it
    explicit HostBlock(uint64_t bytes) : owner(allocHostResult(bytes)), capacity(bytes)
    {
        SHB_REQUIRE(owner.p != nullptr, SHB_ERR_OOM, "Out of host memory for the results.");
        pageLocked = HostPool::instance().isPageLocked(owner.p);
    }
    uint8_t* data() const { return static_cast<uint8_t*>(owner.p); }
};

// The pinned chunks of the ring, allocated once per context: kStageSlots * kStageBytes.
inline void ensureStagingRing(shb_context* c)
{
    if(c->pinnedStage[0]) return;
    for(int i = 0; i < kStageSlots; i++) {
        SHB_CUDA(cudaHostAlloc(&c->pinnedStage[i], kStageBytes, cudaHostAllocDefault));
        SHB_CUDA(cudaEventCreateWithFlags(&c->stageEvent[i], cudaEventDisableTiming));
    }
}

class StagedCopier {
public:
    // threads <= kStageSlots / 2 (two chunks each). srcLock, when set, is held while a DMA is queued: the source
    // address is looked up under it (the device buffer may move between the queueing of a copy and its DMA).
    StagedCopier(shb_context* c, cudaStream_t stream, int threads, std::mutex* srcLock = nullptr)
        : c_(c), stream_(stream), srcLock_(srcLock)
    {
        SHB_REQUIRE(threads >= 1 && 2 * threads <= kStageSlots, SHB_ERR_INVALID, "Too many copier threads for the staging ring.");
        ensureStagingRing(c);
        for(int t = 0; t < threads; t++) threads_.emplace_back([this, t] { run(t); });
    }
    StagedCopier(const StagedCopier&) = delete;
    StagedCopier& operator=(const StagedCopier&) = delete;
    ~StagedCopier() { stop(); }

    // Copies `bytes` from src() (a device address, looked up when the DMA is queued) to dst at dstOffset, growing dst when it
    // is too small. Work queued on the copy stream before this call is ordered before the copy.
    void copy(HostBlock& dst, uint64_t dstOffset, std::function<const uint8_t*()> src, uint64_t bytes)
    {
        if(bytes == 0) return;
        std::lock_guard<std::mutex> lock(mutex_);
        for(uint64_t off = 0; off < bytes; off += kStageBytes) {
            const uint64_t n = std::min<uint64_t>(kStageBytes, bytes - off);
            pieces_.push_back(Piece{&dst, dstOffset + off, src, off, n});
        }
        ready_.notify_all();
    }

    // Waits until every queued copy has landed in its block; rethrows the first error of the copier threads.
    void finish()
    {
        stop();
        if(error_) std::rethrow_exception(error_);
    }

private:
    struct Piece { HostBlock* dst; uint64_t dstOffset; std::function<const uint8_t*()> src; uint64_t srcOffset, bytes; };

    void stop()
    {
        {
            std::lock_guard<std::mutex> lock(mutex_);
            done_ = true;
        }
        ready_.notify_all();
        for(std::thread& t : threads_) if(t.joinable()) t.join();
        threads_.clear();
    }

    // Next piece in queue order; false when the queue is drained and no more will come (or another thread failed). When
    // `wait` is false, returns false at once if nothing is queued.
    bool take(Piece& p, bool wait)
    {
        std::unique_lock<std::mutex> lock(mutex_);
        if(wait) ready_.wait(lock, [this] { return !pieces_.empty() || done_ || failed_; });
        if(pieces_.empty() || failed_) return false;
        p = std::move(pieces_.front());
        pieces_.pop_front();
        return true;
    }

    void issue(const Piece& p, int slot)
    {
        {
            std::unique_lock<std::mutex> lock;
            if(srcLock_) lock = std::unique_lock<std::mutex>(*srcLock_);
            SHB_CUDA(cudaMemcpyAsync(c_->pinnedStage[slot], p.src() + p.srcOffset, p.bytes, cudaMemcpyDeviceToHost, stream_));
        }
        SHB_CUDA(cudaEventRecord(c_->stageEvent[slot], stream_));
    }

    void drain(const Piece& p, int slot)
    {
        SHB_CUDA(cudaEventSynchronize(c_->stageEvent[slot]));
        HostBlock& b = *p.dst;
        const uint64_t end = p.dstOffset + p.bytes;
        std::shared_lock<std::shared_mutex> shared(b.resize);
        if(end > b.capacity) {
            shared.unlock();
            {
                std::unique_lock<std::shared_mutex> exclusive(b.resize);
                if(end > b.capacity) {      // every DMA into b was queued before this piece's: all have landed
                    const uint64_t capacity = std::max(end, b.capacity + b.capacity / 2);
                    void* q = HostPool::instance().grow(b.owner.p, b.capacity, capacity);
                    SHB_REQUIRE(q != nullptr, SHB_ERR_OOM, "Out of host memory for the results.");
                    b.owner.p = q; b.capacity = capacity; b.pageLocked = false;
                }
            }
            shared.lock();
        }
        memcpy(b.data() + p.dstOffset, c_->pinnedStage[slot], p.bytes);
    }

    // Thread t owns chunks 2t and 2t + 1: the DMA of its next piece runs while it copies the current one out.
    void run(int t)
    {
        try {
            SHB_CUDA(cudaSetDevice(c_->device));
            Piece cur, next;
            int k = 0;
            bool haveCur = take(cur, true);
            if(haveCur) issue(cur, 2 * t);
            while(haveCur) {
                const bool haveNext = take(next, false);
                if(haveNext) issue(next, 2 * t + ((k + 1) & 1));
                drain(cur, 2 * t + (k & 1));
                k++;
                if(haveNext) cur = std::move(next);
                else if((haveCur = take(cur, true))) issue(cur, 2 * t + (k & 1));
            }
        } catch(...) {
            std::lock_guard<std::mutex> lock(mutex_);
            if(!error_) error_ = std::current_exception();
            failed_ = true;
            ready_.notify_all();
        }
    }

    shb_context* c_;
    cudaStream_t stream_;
    std::mutex* srcLock_;
    std::mutex mutex_;
    std::condition_variable ready_;
    std::deque<Piece> pieces_;
    bool done_ = false, failed_ = false;
    std::exception_ptr error_;
    std::vector<std::thread> threads_;
};

// Copies bytes from a device address to dst at dstOffset after the work queued on the copy stream: direct DMA into a
// page-locked block that is large enough, through the copier otherwise.
inline void copyResult(StagedCopier& copier, cudaStream_t stream, HostBlock& dst, uint64_t dstOffset, const uint8_t* src, uint64_t bytes)
{
    if(bytes == 0) return;
    if(dst.pageLocked && dstOffset + bytes <= dst.capacity) {
        SHB_CUDA(cudaMemcpyAsync(dst.data() + dstOffset, src, bytes, cudaMemcpyDeviceToHost, stream));
    } else copier.copy(dst, dstOffset, [src] { return src; }, bytes);
}

} // namespace shb
