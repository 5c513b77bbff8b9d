// device_once.h -- per-device one-time set-up of a kernel (shared-memory opt-in, constant upload) that host threads
// creating decoders may race to do.
#pragma once
#include <cuda_runtime.h>

#include <mutex>
#include <set>
#include <utility>

namespace lb {

// once(device, fn) runs fn() -- which returns a cudaError_t -- for a device ordinal until one call has succeeded; later
// calls for that device return cudaSuccess without running it.  Concurrent callers wait for each other.
class DeviceOnce {
public:
    template <class F>
    cudaError_t operator()(int device, F fn) {
        std::lock_guard<std::mutex> lock(mu_);
        if (done_.count(device)) return cudaSuccess;
        const cudaError_t e = fn();
        if (e == cudaSuccess) done_.insert(device);
        return e;
    }

private:
    std::mutex mu_;
    std::set<int> done_;
};

// Raises the dynamic shared-memory limit of `kernel` on `device` (the current device) to `bytes`, until one call for that
// kernel and device has succeeded.  Keyed by the kernel's address: instantiations such as k1_fft_kernel<7, 8> and
// k1_fft_kernel<8, 8> share one function type, so a static per type would opt in only the first of them.
inline cudaError_t opt_in_smem(const void *kernel, int device, size_t bytes) {
    static std::mutex mu;
    static std::set<std::pair<const void *, int>> done;
    std::lock_guard<std::mutex> lock(mu);
    if (done.count({kernel, device})) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) done.insert({kernel, device});
    return e;
}

}  // namespace lb
