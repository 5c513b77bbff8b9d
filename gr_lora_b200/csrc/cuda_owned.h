// cuda_owned.h -- owners of the device buffers, pinned buffers, streams and events of a decoder or a channelizer.  Only
// the owner knows whether its resource exists: a failed reserve() / ensure() leaves it empty, and the next call retries.
#pragma once
#include <cuda_runtime.h>

namespace lb {

// n elements of T from cudaMalloc, or cudaMallocHost when Pinned; converts to T *
template <class T, bool Pinned>
class CudaBuffer {
public:
    CudaBuffer() = default;
    CudaBuffer(CudaBuffer &&) = delete;          // neither copied nor moved
    ~CudaBuffer() { reset(); }
    // grows to at least n elements, without keeping the contents: the old buffer is freed first, so the peak is the
    // larger size alone, and the pointer and capacity are set only once the allocation has succeeded
    cudaError_t reserve(size_t n) {
        if (n <= cap_) return cudaSuccess;
        void *p = nullptr;
        cudaError_t e = reset();
        if (e == cudaSuccess) e = Pinned ? cudaMallocHost(&p, sizeof(T) * n) : cudaMalloc(&p, sizeof(T) * n);
        if (e == cudaSuccess) { p_ = static_cast<T *>(p); cap_ = n; }
        return e;
    }
    cudaError_t reset() {                        // frees the buffer
        T *p = p_;
        p_ = nullptr;
        cap_ = 0;
        return !p ? cudaSuccess : Pinned ? cudaFreeHost(p) : cudaFree(p);
    }
    size_t capacity() const { return cap_; }
    T *get() const { return p_; }
    operator T *() const { return p_; }

private:
    T *p_ = nullptr;
    size_t cap_ = 0;
};
template <class T> using DeviceBuffer = CudaBuffer<T, false>;
template <class T> using PinnedBuffer = CudaBuffer<T, true>;

// a stream or event handle, created by the first successful ensure(); converts to the handle (null before)
template <class H, cudaError_t (*Create)(H *), cudaError_t (*Destroy)(H)>
class CudaHandle {
public:
    CudaHandle() = default;
    CudaHandle(CudaHandle &&) = delete;          // neither copied nor moved
    ~CudaHandle() { if (h_) Destroy(h_); }
    cudaError_t ensure() {
        H h = nullptr;
        const cudaError_t e = h_ ? cudaSuccess : Create(&h);
        if (e == cudaSuccess && h) h_ = h;
        return e;
    }
    operator H() const { return h_; }

private:
    H h_ = nullptr;
};
inline cudaError_t stream_create(cudaStream_t *s) { return cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); }
inline cudaError_t event_create(cudaEvent_t *e) { return cudaEventCreateWithFlags(e, cudaEventDisableTiming); }
using CudaStream = CudaHandle<cudaStream_t, stream_create, cudaStreamDestroy>;
using CudaEvent = CudaHandle<cudaEvent_t, event_create, cudaEventDestroy>;

}  // namespace lb
