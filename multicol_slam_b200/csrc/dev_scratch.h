// dev_scratch.h -- RAII device scratch for the stateless matcher / bag-of-words entry points.
// Those calls are made once per frame with a handful of small buffers each; a cudaMalloc + cudaFree pair per buffer costs
// more than the microsecond-scale kernels those buffers feed.  Freed blocks
// therefore go to a per-thread, per-device free list (best fit, at most 2x oversize, 1 GiB held at most) instead of back
// to the driver.  Every entry point synchronises before it returns, so a block is idle when its Dev dies.
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <cstddef>
#include <map>

namespace mcs {

class DevCache {
public:
    ~DevCache() { for (auto& e : free_) cudaFree(e.second.p); }
    cudaError_t take(size_t bytes, void** p, size_t* cap, int* dev) {
        cudaError_t e = cudaGetDevice(dev);
        if (e != cudaSuccess) return e;
        bytes = std::max<size_t>((bytes + 255) & ~(size_t)255, 256);
        for (auto it = free_.lower_bound(bytes); it != free_.end() && it->first <= 2 * bytes; ++it)
            if (it->second.dev == *dev) {
                *p = it->second.p; *cap = it->first; held_ -= it->first;
                free_.erase(it);
                return cudaSuccess;
            }
        e = cudaMalloc(p, bytes);
        if (e != cudaSuccess && !free_.empty()) {          // out of memory: give the cached blocks back and retry once
            cudaGetLastError();
            for (auto& b : free_) cudaFree(b.second.p);
            free_.clear(); held_ = 0;
            e = cudaMalloc(p, bytes);
        }
        *cap = bytes;
        return e;
    }
    void give(void* p, size_t cap, int dev) {
        if (held_ + cap > kMaxHeld) { cudaFree(p); return; }
        free_.emplace(cap, Block{p, dev});
        held_ += cap;
    }
    static DevCache& local() { static thread_local DevCache c; return c; }

private:
    struct Block { void* p; int dev; };
    static constexpr size_t kMaxHeld = (size_t)1 << 30;
    std::multimap<size_t, Block> free_;
    size_t held_ = 0;
};

struct Dev {   // RAII device scratch buffer
    void* p = nullptr;
    size_t cap = 0;
    int dev = 0;
    Dev() = default;
    Dev(const Dev&) = delete;
    Dev& operator=(const Dev&) = delete;
    ~Dev() { if (p) DevCache::local().give(p, cap, dev); }
    cudaError_t alloc(size_t bytes) {
        if (p) { DevCache::local().give(p, cap, dev); p = nullptr; }
        return DevCache::local().take(bytes, &p, &cap, &dev);
    }
    template <typename T> T* as() { return (T*)p; }
};

}  // namespace mcs
