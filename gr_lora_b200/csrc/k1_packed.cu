// k1_packed.cu -- the SF7 warp kernel and the SF9 group kernel compiled with the LB_PACKED_CMUL complex product
// (cmul / cfma as fma(b, a.x, (-b.y, b.x) * a.y), lora_common.cuh).  The product form decides the last bit of every
// dechirped sample, and the inline product is a per-translation-unit definition, so these two kernels live in their own unit.
#define LB_PACKED_CMUL 1
#include "k1_group.cuh"
#include "k1_packed.h"

#include <cstdio>

namespace lb {
namespace {

#define PCU(call)                                                                     \
    do {                                                                              \
        cudaError_t e_ = (call);                                                      \
        if (e_ != cudaSuccess) {                                                      \
            snprintf(err, err_cap, "%s: %s", #call, cudaGetErrorString(e_));          \
            return (int)e_;                                                           \
        }                                                                             \
    } while (0)

}  // namespace

int k1_packed_launch(int sf, int device, int n_sms, const float2 *iq, const float2 *chirp, const float2 *tw, size_t n_symbols,
                     uint32_t *bins, float *mags, cudaStream_t st, char *err, size_t err_cap) {
    K1Args a{iq, chirp, tw, n_symbols};
    if (n_symbols == 0) return 0;
    if (sf == 7) {
        constexpr int NW = 12, NS = 2;
        static bool attr_set[64] = {};
        const size_t smem = sizeof(W7Smem<NW, NS>);
        if (!attr_set[device & 63]) {
            PCU(cudaFuncSetAttribute(k1_sf7_warp_kernel<NW, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr_set[device & 63] = true;
        }
        const int grid = (int)(((n_symbols + NW - 1) / NW) < (size_t)n_sms ? ((n_symbols + NW - 1) / NW) : (size_t)n_sms);
        k1_sf7_warp_kernel<NW, NS><<<grid, NW * 32, smem, st>>>(a, bins, mags);
        PCU(cudaGetLastError());
        return 0;
    }
    if (sf == 9) {
        constexpr int NG = 3, NS = 2;
        static bool attr_set[64] = {};
        const size_t smem = sizeof(GSmem<9, NG, NS>);
        if (!attr_set[device & 63]) {
            PCU(cudaFuncSetAttribute(k1_group_kernel<9, NG, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr_set[device & 63] = true;
        }
        const int grid = (int)(((n_symbols + NG - 1) / NG) < (size_t)n_sms ? ((n_symbols + NG - 1) / NG) : (size_t)n_sms);
        k1_group_kernel<9, NG, NS><<<grid, NG * GCfg<9>::T, smem, st>>>(a, bins, mags);
        PCU(cudaGetLastError());
        return 0;
    }
    snprintf(err, err_cap, "k1_packed: SF7 / SF9 only");
    return (int)cudaErrorInvalidValue;
}

}  // namespace lb
