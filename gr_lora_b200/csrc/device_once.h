// device_once.h -- per-device one-time set-up of a kernel (shared-memory opt-in, constant upload) that host threads
// creating decoders may race to do.
#pragma once
#include <cuda_runtime.h>

#include <mutex>
#include <set>

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

}  // namespace lb
