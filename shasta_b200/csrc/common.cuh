// Shared host-side helpers for the CUDA library: error propagation to the C ABI, RAII device
// buffers, launch accounting, read-backs and timers.
#pragma once

#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <utility>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>

#include "../../include/shasta_b200.h"

namespace shb {

struct Error : public std::runtime_error {
    shb_status status;
    Error(shb_status s, const std::string& what) : std::runtime_error(what), status(s) {}
};

void setLastError(const std::string& message);

#define SHB_CUDA(call)                                                                       \
    do {                                                                                     \
        cudaError_t shbErr_ = (call);                                                        \
        if(shbErr_ != cudaSuccess) {                                                         \
            throw ::shb::Error(shbErr_ == cudaErrorMemoryAllocation ? SHB_ERR_OOM : SHB_ERR_CUDA, \
                std::string(#call) + " failed at " + __FILE__ + ":" + std::to_string(__LINE__) + ": " + \
                cudaGetErrorString(shbErr_));                                                \
        }                                                                                    \
    } while(0)

#define SHB_CHECK_LAUNCH() SHB_CUDA(cudaGetLastError())

#define SHB_REQUIRE(cond, status, message)                                                   \
    do { if(!(cond)) throw ::shb::Error(status, message); } while(0)

// Counts kernels launched through SHB_LAUNCH (bench.py reports it as gpu_launches).
extern thread_local uint64_t g_launchCount;

#define SHB_LAUNCH(kernel, grid, block, smem, stream, ...)                                   \
    do {                                                                                     \
        kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);                          \
        SHB_CHECK_LAUNCH();                                                                  \
        ++::shb::g_launchCount;                                                              \
    } while(0)

// Grow-only typed device buffer.
template<class T> class DeviceBuffer {
public:
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    ~DeviceBuffer() { release(); }

    T* get() const { return ptr_; }
    uint64_t capacity() const { return capacity_; }

    // Ensure room for n elements. Contents are NOT preserved unless keep is true.
    void reserve(uint64_t n, bool keep = false, cudaStream_t stream = 0)
    {
        if(n <= capacity_) return;
        // Grow geometrically to amortise repeated appends.
        uint64_t newCap = n;
        if(keep && capacity_) newCap = (n > capacity_ + capacity_/2) ? n : capacity_ + capacity_/2;
        if(!keep) release();            // nothing to preserve: return the old block first (the buffers can be tens of GB)
        T* p = nullptr;
        SHB_CUDA(cudaMalloc(&p, (newCap ? newCap : 1) * sizeof(T)));
        if(keep && ptr_ && capacity_) {
            SHB_CUDA(cudaMemcpyAsync(p, ptr_, capacity_ * sizeof(T), cudaMemcpyDeviceToDevice, stream));
            SHB_CUDA(cudaStreamSynchronize(stream));
        }
        release();
        ptr_ = p;
        capacity_ = newCap;
    }
    void release()
    {
        if(ptr_) cudaFree(ptr_);
        ptr_ = nullptr;
        capacity_ = 0;
    }
    void swap(DeviceBuffer& o) { std::swap(ptr_, o.ptr_); std::swap(capacity_, o.capacity_); }

private:
    T* ptr_ = nullptr;
    uint64_t capacity_ = 0;
};

inline uint32_t ceilDiv(uint64_t a, uint64_t b) { return uint32_t((a + b - 1) / b); }

// Bits needed for every value in [0, maxValue]: at least 1. A sort over n rows takes bitsFor(n ? n - 1 : 0) row bits.
inline uint32_t bitsFor(uint64_t maxValue)
{
    uint32_t b = 0;
    while(b < 64 && (maxValue >> b)) b++;
    return b ? b : 1;
}

// One value copied back from the device, with one synchronisation of the stream.
template<class T> T readBack(const T* dev, cudaStream_t stream)
{
    T v;
    SHB_CUDA(cudaMemcpyAsync(&v, dev, sizeof(T), cudaMemcpyDeviceToHost, stream));
    SHB_CUDA(cudaStreamSynchronize(stream));
    return v;
}

// A start and a stop timing event. elapsedMs() needs the stop event to have completed: the caller synchronises.
struct EventTimer {
    cudaEvent_t startEvent = nullptr, stopEvent = nullptr;
    EventTimer()
    {
        SHB_CUDA(cudaEventCreate(&startEvent));
        const cudaError_t e = cudaEventCreate(&stopEvent);
        if(e != cudaSuccess) cudaEventDestroy(startEvent);
        SHB_CUDA(e);
    }
    EventTimer(const EventTimer&) = delete;
    EventTimer& operator=(const EventTimer&) = delete;
    ~EventTimer() { cudaEventDestroy(startEvent); cudaEventDestroy(stopEvent); }
    void start(cudaStream_t stream) { SHB_CUDA(cudaEventRecord(startEvent, stream)); }
    void stop(cudaStream_t stream) { SHB_CUDA(cudaEventRecord(stopEvent, stream)); }
    float elapsedMs() const
    {
        float ms = 0.f;
        SHB_CUDA(cudaEventElapsedTime(&ms, startEvent, stopEvent));
        return ms;
    }
};

// Wall-clock milliseconds since t0.
inline double msSince(std::chrono::steady_clock::time_point t0)
{
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

} // namespace shb
