// k1_packed.cu -- the SF7 warp kernel and the SF9 group kernel compiled with the LB_PACKED_CMUL complex product
// (cmul / cfma as fma(b, a.x, (-b.y, b.x) * a.y), lora_common.cuh).  The product form decides the last bit of every
// dechirped sample, and the inline product is a per-translation-unit definition, so these two kernels live in their own unit.
#define LB_PACKED_CMUL 1
#include "k1_warp.cuh"
#include "k1_group.cuh"

namespace lb {

int k1_launch_warp7(const K1Launch &k) {
    constexpr int NW = 12, NS = 2;
    const size_t smem = sizeof(W7Smem<NW, NS>);
    K1_CU(opt_in_smem((const void *)k1_sf7_warp_kernel<NW, NS>, k.device, smem));
    const int grid = (int)std::min((k.a.n_symbols + NW - 1) / NW, (size_t)k.n_sms);
    k1_sf7_warp_kernel<NW, NS><<<grid, NW * 32, smem, k.st>>>(k.a, k.bins, k.mags);
    K1_CU(cudaGetLastError());
    return 0;
}

int k1_launch_group9(const K1Launch &k) { return k1_launch_group<9, 3, 2>(k); }

}  // namespace lb
