// k1_launch.h -- the calling convention of the batch K1 launchers.  They live in three translation units (the complex
// product form is a per-unit definition, lora_common.cuh): k1_packed.cu (SF7 warp and SF9 group kernels), k1_rows.cu
// (SF11 / SF12 rows kernel) and lora_b200.cu (SF8 group, SF10 and the generic CTA-wide kernel); dispatch_k1_impl in
// lora_b200.cu picks one per SF.
#pragma once
#include "k1_fft.cuh"
#include "device_once.h"

#include <cstdio>

namespace lb {

struct K1Launch {
    K1Args a;                        // a.n_symbols > 0
    const float2 *tw_host;           // host copy of the a.tw table
    uint32_t *bins;
    float *mags;                     // may be null
    unsigned long long *packed;      // kernels that merge partial argmaxes: n_symbols zeroed keys, finalised by the caller
    int device, n_sms;
    cudaStream_t st;
    char *err;                       // message of a failure
    size_t err_cap;
};

// A launcher enqueues one kernel on k.st and returns 0, or a cudaError_t value with a message in k.err.
typedef int (*K1Launcher)(const K1Launch &k);

#define K1_CU(call)                                                                   \
    do {                                                                              \
        cudaError_t e_ = (call);                                                      \
        if (e_ != cudaSuccess) {                                                      \
            snprintf(k.err, k.err_cap, "%s: %s", #call, cudaGetErrorString(e_));      \
            return (int)e_;                                                           \
        }                                                                             \
    } while (0)

int k1_launch_warp7(const K1Launch &k);                  // k1_packed.cu
int k1_launch_group9(const K1Launch &k);                 // k1_packed.cu
template <int SF> int k1_launch_rows(const K1Launch &k); // k1_rows.cu, SF11 and SF12

}  // namespace lb
