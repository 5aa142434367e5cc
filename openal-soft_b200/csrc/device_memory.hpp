// device_memory.hpp — owners of the host library's CUDA resources.
//
// DevArray<T> (cudaMalloc), PinnedArray<T> (cudaMallocHost) and Event free what they hold when
// they are destroyed or reallocated; they move but do not copy.  Allocation returns the
// cudaError_t, so nothing throws across the C ABI.  An array converts to its pointer: a view,
// valid while the owner holds the allocation.
#pragma once

#include <cstddef>
#include <cstring>
#include <utility>
#include <vector>

#include <cuda_runtime.h>

namespace b200mix {

template<typename T, bool Pinned>
class CudaArray {
public:
    CudaArray() = default;
    CudaArray(CudaArray &&o) noexcept { *this = std::move(o); }
    CudaArray &operator=(CudaArray &&o) noexcept
    {
        if(this != &o) { reset(); p_ = std::exchange(o.p_, nullptr); n_ = std::exchange(o.n_, 0); }
        return *this;
    }
    ~CudaArray() { reset(); }

    // `count` uninitialised elements (none for 0) in place of what the array held
    cudaError_t alloc(size_t count)
    {
        reset();
        if(!count) return cudaSuccess;
        void *p = nullptr;
        const cudaError_t e = Pinned ? cudaMallocHost(&p, count*sizeof(T)) : cudaMalloc(&p, count*sizeof(T));
        if(e == cudaSuccess) { p_ = static_cast<T*>(p); n_ = count; }
        return e;
    }
    // `count` elements zeroed on `stream` (device arrays)
    cudaError_t alloc(size_t count, cudaStream_t stream)
    {
        const cudaError_t e = alloc(count);
        return e != cudaSuccess || !count ? e : cudaMemsetAsync(p_, 0, bytes(), stream);
    }
    void reset() { if(p_) { if(Pinned) cudaFreeHost(p_); else cudaFree(p_); } p_ = nullptr; n_ = 0; }
    T *get() const { return p_; }
    operator T*() const { return p_; }
    size_t size() const { return n_; }
    size_t bytes() const { return n_*sizeof(T); }

private:
    T *p_{nullptr};
    size_t n_{0};
};

template<typename T> using DevArray = CudaArray<T, false>;
template<typename T> using PinnedArray = CudaArray<T, true>;

class Event {
public:
    Event() = default;
    Event(Event &&o) noexcept : e_(std::exchange(o.e_, nullptr)) {}
    Event &operator=(Event &&o) noexcept { if(this != &o) { reset(); e_ = std::exchange(o.e_, nullptr); } return *this; }
    ~Event() { reset(); }

    cudaError_t create(unsigned flags = cudaEventDefault) { reset(); return cudaEventCreateWithFlags(&e_, flags); }
    void reset() { if(e_) cudaEventDestroy(e_); e_ = nullptr; }
    operator cudaEvent_t() const { return e_; }

private:
    cudaEvent_t e_{nullptr};
};

// Reallocates `a` to `count` elements once `stream` is idle: queued work may still read the old array.
template<typename T>
cudaError_t regrow(DevArray<T> &a, size_t count, cudaStream_t stream)
{
    const cudaError_t e = cudaStreamSynchronize(stream);
    return e != cudaSuccess ? e : a.alloc(count);
}

// Copies a host vector to the front of a device array, then synchronises the stream: the vector
// may be rebuilt (or go away) before an asynchronous copy would have read it.
template<typename T>
cudaError_t upload(DevArray<T> &dst, const std::vector<T> &src, cudaStream_t stream)
{
    if(!src.empty())
        if(const cudaError_t e = cudaMemcpyAsync(dst.get(), src.data(), src.size()*sizeof(T), cudaMemcpyHostToDevice,
            stream)) return e;
    return cudaStreamSynchronize(stream);
}

// A pinned block and a device block that one call packs its inputs into (16-byte aligned parts)
// and ships with ONE host-to-device copy.  The device block may be longer: what follows the
// packed parts is device-only scratch.
class UploadArena {
public:
    // Before the host block is overwritten: the last copy out of it has completed.
    cudaError_t wait() { return std::exchange(in_flight_, false) ? cudaEventSynchronize(done_) : cudaSuccess; }
    // Room for n units (whatever the caller counts) when the arena holds fewer: synchronises the
    // stream (the last update may still read the device block), then reallocates both blocks for
    // `cap` units, host_bytes pinned and dev_bytes on the device.
    cudaError_t reserve(size_t n, size_t cap, size_t host_bytes, size_t dev_bytes, cudaStream_t stream)
    {
        if(n <= cap_) return cudaSuccess;
        cap_ = 0;
        host_.reset();
        cudaError_t e = regrow(dev_, dev_bytes, stream);
        if(e == cudaSuccess) e = host_.alloc(host_bytes);
        if(e == cudaSuccess && !done_) e = done_.create(cudaEventDisableTiming);
        if(e != cudaSuccess) { host_.reset(); dev_.reset(); return e; }
        cap_ = cap;
        return cudaSuccess;
    }
    size_t capacity() const { return cap_; }
    void begin() { off_ = used_ = 0; }
    // The next part of the host block, for the caller to fill, and its device address.
    template<typename T>
    T *host_part(size_t count)
    { T *h = reinterpret_cast<T*>(host_.get() + off_); used_ = off_ + count*sizeof(T); off_ = align(used_); return h; }
    template<typename T>
    T *dev_of(const T *h) const { return reinterpret_cast<T*>(dev_ + (reinterpret_cast<const char*>(h) - host_)); }
    // Copies `count` elements into the next part; returns their device address.
    template<typename T>
    const T *pack(const T *src, size_t count) { T *h = host_part<T>(count); std::memcpy(h, src, count*sizeof(T)); return dev_of(h); }
    // The next part as device-only scratch (after every host part).
    template<typename T>
    T *carve(size_t count) { T *p = reinterpret_cast<T*>(dev_ + off_); off_ = align(off_ + count*sizeof(T)); return p; }
    // One asynchronous copy of the packed parts, then the event wait() waits on.
    cudaError_t ship(cudaStream_t stream)
    {
        cudaError_t e = cudaMemcpyAsync(dev_, host_, used_, cudaMemcpyHostToDevice, stream);
        if(e == cudaSuccess) e = cudaEventRecord(done_, stream);
        in_flight_ = e == cudaSuccess;
        return e;
    }
    static size_t align(size_t v) { return (v + 15u) & ~size_t(15); }

private:
    PinnedArray<char> host_;
    DevArray<char> dev_;
    Event done_;
    bool in_flight_{false};
    size_t cap_{0}, off_{0}, used_{0};
};

} // namespace b200mix
