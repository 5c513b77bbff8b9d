// k1_rows.cu -- host side of the SF11 / SF12 rows kernel: shared-memory opt-in, per-q2 constants, the 2-D tensor map of
// the IQ batch (SF12) and the launch (SF12: clusters of two CTAs).
#define LB_PACKED_CMUL 1
#include "k1_rows.cuh"
#include "k1_launch.h"

#include <cstring>

namespace lb {
namespace {

typedef CUresult (*encode_tiled_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

encode_tiled_fn get_encoder() {
    static encode_tiled_fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (encode_tiled_fn)p;
    }
    return fn;
}

}  // namespace

// SF11 writes bins / mags directly; SF12 merges the two CTAs' argmax keys into k.packed
template <int SF>
int k1_launch_rows(const K1Launch &k) {
    using C = RCfg<SF>;
    static DeviceOnce once;
    const size_t smem = sizeof(RSmem<SF>);
    K1_CU(opt_in_smem((const void *)k1_rows_kernel<SF>, k.device, smem));
    K1_CU(once(k.device, [&] {      // the cluster opt-in, and the per-q2 constants from the host table
        const cudaError_t e = C::CL > 1 ? cudaFuncSetAttribute(k1_rows_kernel<SF>, cudaFuncAttributeNonPortableClusterSizeAllowed, 0) : cudaSuccess;
        if (e != cudaSuccess) return e;
        RConsts rc;
        r_build_consts<SF>(k.tw_host, rc);
        return cudaMemcpyToSymbol(r_consts_dev, &rc, sizeof rc, sizeof(RConsts) * (SF - 11));
    }));
    const size_t n_symbols = k.a.n_symbols;
    RParams P;
    memset(&P, 0, sizeof P);
    P.a = k.a;
    P.packed = k.packed; P.bins = k.bins; P.mags = k.mags;
    if (C::CL == 2) {
        encode_tiled_fn enc = get_encoder();
        if (!enc) { snprintf(k.err, k.err_cap, "cuTensorMapEncodeTiled is not available from this driver"); return (int)cudaErrorNotSupported; }
        // the batch as a 2-D float array: 16 floats (8 branches x re/im) per n1, n_symbols * L values of n1;
        // a box = 8 floats (this CTA's 4 branches) x 256 n1 = one row of 8 KiB, dense in shared memory
        const cuuint64_t dims[2] = {16, (cuuint64_t)n_symbols * C::L};
        const cuuint64_t strides[1] = {64};
        const cuuint32_t box[2] = {8, (cuuint32_t)C::A};
        const cuuint32_t estr[2] = {1, 1};
        const CUresult r = enc(&P.tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float2 *>(k.a.x), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { snprintf(k.err, k.err_cap, "cuTensorMapEncodeTiled failed (%d)", (int)r); return (int)cudaErrorInvalidValue; }
    }
    size_t units = (size_t)k.n_sms / C::CL;
    if (units > n_symbols) units = n_symbols;
    if (units == 0) return 0;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(units * C::CL));
    cfg.blockDim = dim3(C::T);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = k.st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = C::CL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    K1_CU(cudaLaunchKernelEx(&cfg, k1_rows_kernel<SF>, P));
#ifdef LB_ROWS_TIMING
    {   // diagnosis build: mean cycles per symbol and warp class spent in each wait
        K1_CU(cudaStreamSynchronize(k.st));
        static unsigned int h[160 * 16 * 8];
        K1_CU(cudaMemcpyFromSymbol(h, r_timing_dev, sizeof h));
        const char *names[6] = {"x_full", "x_free", "sym_full", "sym_late", "barrier", "-"};
        for (int rank = 0; rank < C::CL; rank++)
            for (int half = 0; half < 2; half++) {
                double acc[7] = {0, 0, 0, 0, 0, 0, 0}, nsym = 0;
                int cnt = 0;
                for (unsigned b = 0; b < cfg.gridDim.x; b++) {
                    if ((int)(b % C::CL) != rank) continue;
                    for (int w = 8 * half; w < 8 * half + 8; w++) {
                        const unsigned int *o = h + (b * 16 + w) * 8;
                        for (int i = 0; i < 7; i++) acc[i] += o[i];
                        nsym += o[7];
                        cnt++;
                    }
                }
                fprintf(stderr, "rows<%d> rank %d warps %d-%d: %.0f cycles/symbol;", SF, rank, 8 * half, 8 * half + 7, acc[6] / nsym);
                for (int i = 0; i < 5; i++) fprintf(stderr, " %s %.0f", names[i], acc[i] / nsym);
                fprintf(stderr, "\n");
            }
    }
#endif
    return 0;
}

template int k1_launch_rows<11>(const K1Launch &k);
template int k1_launch_rows<12>(const K1Launch &k);

}  // namespace lb
