// k1_llr.cuh -- the soft-output demodulator: K1's dechirp + pruned FFT with a max-log LLR epilogue.
//
// For a window's kept bins k = 0..N-1 with magnitudes |X_k| (K1's |tmp|, the tmp[N/2] quirk included) and w(k) the word the
// receive path makes of bin k (rx_fft_bin, then rx_demod_word: (k - 1) mod N, folded to N/4 bins for reduced-rate symbols,
// Gray), bit j of the demodulated word gets
//     LLR_j = max_{k: bit_j(w(k)) = 0} |X_k|  -  max_{k: bit_j(w(k)) = 1} |X_k|          (> 0: bit 0)
// for j < ppm (SF, or SF - 2 for reduced-rate symbols).  Max-log in magnitude units: the non-coherent metric log I0(.) is
// close to linear in |X| at the per-symbol SNRs the dechirp receiver works at, and one frame shares one noise level, so a
// maximum-likelihood decision over these LLRs needs no SNR scale.
//
// The phases are K1's own (k1_pass0, k1_pass, k1_combine_twiddles, the horner<D> / plus_quirk sum per kept bin, D = sps / N
// = 2, 8, 16 or 32), so the
// argmax key -- and the bin reported beside the LLRs -- is k1_fft_kernel's bit for bit.  The epilogue keeps 2 SF running
// maxima of |X|^2 per thread and takes square roots only at the end.  Where K1Cfg splits a symbol (S > 1) a CTA loops over the S sub-problems
// of its symbol (as RsDevOps::argmax does): each warp's maxima are kept in shared memory between them, and no merge pass
// over global memory follows.
#pragma once
#include "k1_fft.cuh"
#include "rx_stream.cuh"

namespace lb {

constexpr int LLR_MAX_PPM = 12;

// the demodulated word of kept bin k
LB_HD uint32_t llr_word(uint32_t k, uint32_t n_bins, bool reduced) {
    return rx_demod_word((uint32_t)rx_fft_bin(k, n_bins), reduced, n_bins >> 2);
}

// running maxima of |X|^2 per bit value (|X|^2 >= 0, so 0 is the identity), and the K1 argmax key
template <int SF>
struct LlrAcc {
    float m0[SF], m1[SF];
    unsigned long long key;
    LB_HD void init() {
#pragma unroll
        for (int j = 0; j < SF; j++) { m0[j] = 0.f; m1[j] = 0.f; }
        key = 0ull;
    }
    LB_HD void add(float m2, uint32_t w) {
#pragma unroll
        for (int j = 0; j < SF; j++) {
            if ((w >> j) & 1u) m1[j] = fmaxf(m1[j], m2);
            else m0[j] = fmaxf(m0[j], m2);
        }
    }
    LB_HD void merge(const LlrAcc &o) {
#pragma unroll
        for (int j = 0; j < SF; j++) { m0[j] = fmaxf(m0[j], o.m0[j]); m1[j] = fmaxf(m1[j], o.m1[j]); }
        key = o.key > key ? o.key : key;
    }
    LB_HD void store(int ppm, float *llr) const {
        for (int j = 0; j < ppm; j++) llr[j] = sqrtf(m0[j]) - sqrtf(m1[j]);
    }
};

// k1_combine's loop with the LLR epilogue: the thread's kept bins of sub-problem s into acc
template <int SF, int D = 8>
LB_HD void k1_llr_combine(const K1Args &a, int s, int tid, const float2 *buf, const float2 *wtab, bool reduced, LlrAcc<SF> &acc) {
    using C = K1Cfg<SF, D>;
    const int g = tid / C::TPS, lt = tid % C::TPS;
    const float2 *bs = buf + g * C::SYM_STRIDE;
#pragma unroll
    for (int i = 0; i < C::NP / C::TPS; i++) {
        const int p = lt + C::TPS * i;
        const int q = k1_pos_to_bin<SF, D>(p);
        const int qs = q < C::NP / 2 ? q : q - C::NP;
        const float2 w = wtab[i];
        const int pp = k1_pad(p);
        float2 gv[D];
#pragma unroll
        for (int r = 0; r < D; r++) gv[r] = bs[r * C::SB + pp];
        float2 v = horner<D>(gv, w);
        if (s == 0 && q == C::NP / 2) v = plus_quirk<D>(v, gv, w);
        const int kp = C::S * qs + s;
        const uint32_t idx = (uint32_t)(kp >= 0 ? kp : C::N + kp);
        const float m2 = cnorm2(v);
        const unsigned long long key = pack_key(m2, idx);
        acc.key = key > acc.key ? key : acc.key;
        acc.add(m2, llr_word(idx, (uint32_t)C::N, reduced));
    }
}

#ifdef __CUDACC__
LB_D float warp_max_nonneg(float v) { return __uint_as_float(__reduce_max_sync(0xffffffffu, __float_as_uint(v))); }
// ... of each aligned group of W lanes (W = 32: the warp)
template <int W>
LB_D float group_max_nonneg(float v) {
    if (W == 32) return warp_max_nonneg(v);
#pragma unroll
    for (int o = W / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// llrs[i * ppm + j] of symbol i, bins[i] its K1 argmax (may be NULL).  Persistent CTAs over batches of G symbols.
// A "warp" below is a reduction group of C::W lanes: the warp at D = 8, one symbol's TPS < 32 lanes at D = 2, SF7 / SF8.
template <int SF, int D = 8>
__global__ void __launch_bounds__(K1_THREADS, 2)
k1_llr_kernel(K1Args a, int reduced, float *__restrict__ llrs, uint32_t *__restrict__ bins) {
    using C = K1Cfg<SF, D>;
    constexpr int NW = K1_THREADS / C::W, WPS = C::TPS / C::W, W_LOG = k1_log2(C::W);   // groups, groups per symbol
    extern __shared__ float2 llr_smem[];
    __shared__ float wm[NW][2 * SF];
    __shared__ unsigned long long wkey[NW];
    float2 *buf = llr_smem;
    const int tid = threadIdx.x, lane = tid & (C::W - 1), warp = tid >> W_LOG, ppm = reduced ? SF - 2 : SF;
    const size_t n_batches = (a.n_symbols + C::G - 1) / C::G;
    float2 wtab[C::NP / C::TPS];
    k1_combine_twiddles<SF, D>(a, tid, wtab);
    for (size_t batch = blockIdx.x; batch < n_batches; batch += gridDim.x) {
#pragma unroll 1
        for (int s = 0; s < C::S; s++) {
            k1_pass0<SF, true, D>(a, batch, s, tid, buf);
            __syncthreads();
            k1_pass<SF, C::R1, C::SIG1, D>(a, tid, buf);
            __syncthreads();
            if (C::R2 > 1) {
                k1_pass<SF, (C::R2 > 1 ? C::R2 : 2), 1, D>(a, tid, buf);
                __syncthreads();
            }
            LlrAcc<SF> acc;
            acc.init();
            k1_llr_combine<SF, D>(a, s, tid, buf, wtab, reduced != 0, acc);
            // the group's maxima, kept over the sub-problems by its lane 0 (a group never spans two symbols)
            const unsigned long long key = group_max_key<C::W>(acc.key);
#pragma unroll
            for (int j = 0; j < SF; j++) {
                const float m0 = group_max_nonneg<C::W>(acc.m0[j]), m1 = group_max_nonneg<C::W>(acc.m1[j]);
                if (lane == 0) {
                    wm[warp][2 * j] = s ? fmaxf(wm[warp][2 * j], m0) : m0;
                    wm[warp][2 * j + 1] = s ? fmaxf(wm[warp][2 * j + 1], m1) : m1;
                }
            }
            if (lane == 0) wkey[warp] = s && wkey[warp] > key ? wkey[warp] : key;
            __syncthreads();                              // (the next pass 0 rewrites buf; wm is read below)
        }
        // across the warps of one symbol
        if (tid < C::G) {
            LlrAcc<SF> r;
            r.init();
            for (int k = 0; k < WPS; k++) {
                const int wi = tid * WPS + k;
#pragma unroll
                for (int j = 0; j < SF; j++) { r.m0[j] = fmaxf(r.m0[j], wm[wi][2 * j]); r.m1[j] = fmaxf(r.m1[j], wm[wi][2 * j + 1]); }
                r.key = wkey[wi] > r.key ? wkey[wi] : r.key;
            }
            const size_t sym = batch * C::G + tid;
            if (sym < a.n_symbols) {
                r.store(ppm, llrs + sym * ppm);
                if (bins) bins[sym] = key_idx(r.key);
            }
        }
        // wm and wkey are rewritten only after the next batch's passes and their __syncthreads
    }
}
#endif  // __CUDACC__

// ---- CPU emulation of the kernel (same phase functions, threads run one after another) ---
template <int SF, int D = 8>
inline void k1_llr_emulate(const K1Args &a, bool reduced, float *llrs, uint32_t *bins) {
    using C = K1Cfg<SF, D>;
    float2 *buf = new float2[C::SMEM_ELEMS];
    const size_t n_batches = (a.n_symbols + C::G - 1) / C::G;
    const int ppm = reduced ? SF - 2 : SF;
    for (size_t batch = 0; batch < n_batches; batch++) {
        LlrAcc<SF> acc[C::G];
        for (int g = 0; g < C::G; g++) acc[g].init();
        for (int s = 0; s < C::S; s++) {
            for (int i = 0; i < C::SMEM_ELEMS; i++) buf[i] = make_float2(NAN, NAN);   // catch unwritten reads
            for (int t = 0; t < K1_THREADS; t++) k1_pass0<SF, true, D>(a, batch, s, t, buf);
            for (int t = 0; t < K1_THREADS; t++) k1_pass<SF, C::R1, C::SIG1, D>(a, t, buf);
            if (C::R2 > 1)
                for (int t = 0; t < K1_THREADS; t++) k1_pass<SF, (C::R2 > 1 ? C::R2 : 2), 1, D>(a, t, buf);
            for (int t = 0; t < K1_THREADS; t++) {
                float2 wtab[C::NP / C::TPS];
                k1_combine_twiddles<SF, D>(a, t, wtab);
                LlrAcc<SF> r;
                r.init();
                k1_llr_combine<SF, D>(a, s, t, buf, wtab, reduced, r);
                acc[t / C::TPS].merge(r);
            }
        }
        for (int g = 0; g < C::G; g++) {
            const size_t sym = batch * C::G + g;
            if (sym >= a.n_symbols) break;
            acc[g].store(ppm, llrs + sym * ppm);
            if (bins) bins[sym] = key_idx(acc[g].key);
        }
    }
    delete[] buf;
}

}  // namespace lb
