// k1_fft.cuh -- K1: dechirp + pruned FFT + argmax (the north-star kernel).
//
// Computes, for each aligned symbol window x[0..sps), exactly what the reference's
// get_shift_fft does (lib/decoder_impl.cc:430-464):
//     m[n]   = x[n] * down[n]                                   (:436-438)
//     F      = forward sps-point DFT of m                        (:443)
//     tmp[k] = F[k] (k < N/2), F[sps - N + k] (k >= N/2), tmp[N/2] += F[N/2]   (:447-450)
//     bin    = first argmax |tmp|                                (:452-463)
// without ever forming the 7N unused bins:  with n = 8*n1 + r (sps = 8N at fs/bw = 8)
//     F[k'] = sum_r W_sps^{k' r} G_r[k' mod N],   G_r = N-point DFT over n1 of m[8 n1 + r]
// i.e. 8 N-point FFTs (one per polyphase branch) and one 8-term twiddled sum per kept bin.  The phase functions take the
// oversampling factor D = sps / N as a template argument (default 8); at fs/bw = 2, 16 and 32 the same sum has D branches
// (n = D n1 + r) and the split below starts at SF12 (D = 2: sub-problems of up to 2048 bins), SF10 (D = 16: 512) or SF9
// (D = 32: 256).  fs/bw = 4 has no kernels.
// For N > NP_MAX (SF11/12 at D = 8) a radix-S decimation-in-frequency step (S = 2 .. 16) is folded into
// the load:  F[S q + s] = DFT_{sps/S}( y_s )[q],  y_s[n] = W_sps^{s n} sum_j W_S^{s j} m[n + j sps/S],
// giving S independent sub-problems of N' = N/S = NP_MAX bins whose partial argmaxes are
// merged with a 64-bit atomicMax.
//
// Data flow per CTA (256 threads) and batch of G = 8192/(D N') symbols:
//   pass 0  coalesced float4 loads straight into registers (each thread: 16 rows x 2 branches),
//           dechirp, radix-16 DIF in registers, inter-pass twiddle, store to shared memory
//   pass i  in-place radix-8/16/4 passes in shared memory (padded, conflict-free layout)
//   combine Horner evaluation of the D-branch twiddled sum, |.|^2, argmax
// The phase functions are __host__ __device__ so tests/test_k1_emulation.py can run the
// very same index arithmetic on the CPU.
#pragma once
#include "lora_common.cuh"

namespace lb {

constexpr int K1_THREADS = 256;

LB_HD constexpr int k1_log2(int v) { return v > 1 ? 1 + k1_log2(v >> 1) : 0; }

// D = sps / N, the oversampling factor: D polyphase branches (8 at fs/bw = 8; 2, 16 and 32 at those rates).  Every CTA
// batch holds G * D * NP = 8192 samples whatever D is, so a symbol's share of the threads and of shared memory scales with
// D * NP, and a symbol is split into sub-problems of NP_MAX = min(2048, 8192 / D) bins.
template <int SF, int D = 8>
struct K1Cfg {
    static constexpr int N = 1 << SF;                 // bins
    static constexpr int SPS = D * N;                 // samples per symbol
    static constexpr int NP_MAX = 8192 / D < 2048 ? 8192 / D : 2048;   // the passes below cover sub-problems of up to 2048 bins
    static constexpr int S = N <= NP_MAX ? 1 : N / NP_MAX;   // DIF split factor
    static constexpr int NP = N / S;                  // bins per sub-problem (128..1024 at D = 8, ..2048 at 2, ..512 at 16, ..256 at 32)
    static constexpr int SPS_SUB = D * NP;
    static constexpr int HB = D / 2;                  // float4 loads (2 adjacent branches each) per row in pass 0
    static constexpr int G = 8192 / (D * NP);         // symbols per CTA batch
    static constexpr int M0 = NP / 16;                // columns after the radix-16 pass 0
    static constexpr int SB0 = NP + NP / 16;
    // branch stride: == 2 (mod 16) at D = 8; == 4 (mod 16) at D = 2, where a half-warp can span two symbols (M0 = 8) and
    // their strides must then fall 8 float2 apart; == 1 (mod 8) at D = 16 and 32, where a pass-0 half-warp stores 8 branch
    // pairs x 2 columns (D = 16: distinct banks) or 16 branch pairs of one column (D = 32: offsets 2 b SB, all of one parity,
    // so 2-way whatever SB is).  tests/test_rx_osr_high_host.py replays every phase's shared-memory indices.
    static constexpr int SB_MOD = D == 8 ? 2 : D == 2 ? 4 : 1;
    static constexpr int SB_M = D == 8 || D == 2 ? 16 : 8;
    static constexpr int SB = SB0 + ((SB_MOD - SB0 % SB_M) + SB_M) % SB_M;
    static constexpr int SYM_STRIDE = D * SB;
    static constexpr int SMEM_ELEMS = G * SYM_STRIDE; // float2 elements
    static constexpr int TPS = K1_THREADS / G;        // threads per symbol in the combine phase
    static constexpr int W = TPS < 32 ? TPS : 32;     // lanes of one argmax reduction group (one symbol's, or the warp)
    // passes after pass 0 on blocks of M0 points: (R1, SIG1) then (R2, 1)
    static constexpr int R1 = M0 == 8 ? 8 : M0 == 16 ? 16 : 8;
    static constexpr int SIG1 = M0 / R1;              // 1, 1, 4, 8 (16 for NP = 2048)
    static constexpr int R2 = SIG1;                   // 1 (none), 1, 4, 8 (16)
    static_assert(SF >= 7 && SF <= 12, "K1 supports SF7..SF12");
    static_assert(D == 2 || D == 8 || D == 16 || D == 32, "K1 runs at fs/bw = 2, 8, 16 or 32");
    static_assert(G * TPS == K1_THREADS && G * M0 * HB == K1_THREADS, "one thread per pass-0 column pair and combine slot");
    // the D = 2 and D = 8 configurations as they were before D = 16 and 32 were added (their kernels must not change)
    static_assert(D != 8 || (NP == (N < 1024 ? N : 1024) && S == N / NP && G == 1024 / NP && SB % 16 == 2 && TPS == 256 / G &&
                             W == (TPS < 32 ? TPS : 32)), "fs/bw = 8 layout");
    static_assert(D != 2 || (NP == (N < 2048 ? N : 2048) && S == N / NP && G == 4096 / NP && SB % 16 == 4 && TPS == 256 / G &&
                             W == (TPS < 32 ? TPS : 32)), "fs/bw = 2 layout");
    static_assert((D != 8 && D != 2) || (SB >= SB0 && SB < SB0 + 16), "fs/bw = 8 and 2: the least such branch stride");
    static_assert(D != 16 || (NP == (N < 512 ? N : 512) && S == N / NP && G == 512 / NP && SB == SB0 + 1), "fs/bw = 16 layout");
    static_assert(D != 32 || (NP == (N < 256 ? N : 256) && S == N / NP && G == 256 / NP && SB == SB0 + 1), "fs/bw = 32 layout");
};

LB_HD int k1_pad(int i) { return i + (i >> 4); }

struct K1Args {
    const float2 *x;        // n_symbols * SPS samples
    const float2 *chirp;    // down-chirp table, SPS entries
    const float2 *tw;       // W_sps^j = exp(-2 pi i j / sps), SPS entries
    size_t n_symbols;
};

// AL16: the window starts on a 16-byte boundary (batch path); the stream state machine
// hands windows at arbitrary sample offsets (8-byte aligned only)
template <bool AL16>
LB_HD float4 k1_ld_stream(const float2 *p) {
#ifdef __CUDA_ARCH__
    if (AL16) return __ldcs(reinterpret_cast<const float4 *>(p));
    const float2 a = __ldcs(p), b = __ldcs(p + 1);
    return make_float4(a.x, a.y, b.x, b.y);
#else
    return make_float4(p[0].x, p[0].y, p[1].x, p[1].y);
#endif
}
LB_HD float4 k1_ld_table4(const float2 *p) {
#ifdef __CUDA_ARCH__
    return __ldg(reinterpret_cast<const float4 *>(p));
#else
    return make_float4(p[0].x, p[0].y, p[1].x, p[1].y);
#endif
}
LB_HD float2 k1_ld_table(const float2 *p) {
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}

// Horner evaluation of the twiddled branch sum sum_r w^r g[r] over NB branches, g[NB-1] first
template <int NB>
LB_HD float2 horner(const float2 *g, float2 w) {
    float2 acc = g[NB - 1];
#pragma unroll
    for (int r = NB - 2; r >= 0; r--) acc = cfma(acc, w, g[r]);
    return acc;
}
// tmp[N/2] += F[N/2] (:450): bin N/2 is summed a second time with the conjugate twiddle, over gq (its branches, or what
// stands for them)
template <int NB>
LB_HD float2 plus_quirk(float2 acc, const float2 *gq, float2 w) { return cadd(acc, horner<NB>(gq, cconj(w))); }

// result of symbol i from its argmax key: the bin and, when asked for, the magnitude
LB_HD void k1_store(uint32_t *bins, float *mags, size_t i, unsigned long long key) {
    bins[i] = key_idx(key);
    if (mags) mags[i] = sqrtf(key_mag2(key));
}

// ---- pass 0: global -> registers -> radix-16 -> shared ---------------------------------
// Thread (g, m, b) of symbol g holds branches 2b and 2b + 1 of column m: HB = D / 2 threads per column
template <int SF, bool AL16 = true, int D = 8>
LB_HD void k1_pass0(const K1Args &a, size_t batch, int s, int tid, float2 *buf) {
    using C = K1Cfg<SF, D>;
    constexpr int HB_LOG = k1_log2(C::HB);
    const int g = tid / (C::HB * C::M0);
    const int rem = tid % (C::HB * C::M0);
    const int m = rem >> HB_LOG, b = rem & (C::HB - 1);
    const size_t sym = batch * C::G + g;
    const bool valid = sym < a.n_symbols;
    const float2 *xs = a.x + (valid ? sym : 0) * (size_t)C::SPS;
    float2 v0[16], v1[16];
#pragma unroll
    for (int c = 0; c < 16; c++) {
        const int n = D * (c * C::M0 + m) + 2 * b;       // index inside the sub-problem
        if (C::S == 1) {
            const float4 xv = k1_ld_stream<AL16>(xs + n);
            const float4 dv = k1_ld_table4(a.chirp + n);
            v0[c] = cmul(make_float2(xv.x, xv.y), make_float2(dv.x, dv.y));
            v1[c] = cmul(make_float2(xv.z, xv.w), make_float2(dv.z, dv.w));
        } else {
            float2 acc0 = make_float2(0.f, 0.f), acc1 = make_float2(0.f, 0.f);
#pragma unroll
            for (int j = 0; j < C::S; j++) {
                const int nf = n + j * C::SPS_SUB;
                const float4 xv = k1_ld_stream<AL16>(xs + nf);
                const float4 dv = k1_ld_table4(a.chirp + nf);
                const float2 w = k1_ld_table(a.tw + ((s * j * (C::SPS / C::S)) & (C::SPS - 1)));   // W_S^{s j}
                acc0 = cfma(cmul(make_float2(xv.x, xv.y), make_float2(dv.x, dv.y)), w, acc0);
                acc1 = cfma(cmul(make_float2(xv.z, xv.w), make_float2(dv.z, dv.w)), w, acc1);
            }
            v0[c] = cmul(acc0, k1_ld_table(a.tw + s * n));          // W_sps^{s n}
            v1[c] = cmul(acc1, k1_ld_table(a.tw + s * (n + 1)));
        }
        if (!valid) { v0[c] = make_float2(0.f, 0.f); v1[c] = make_float2(0.f, 0.f); }
    }
    dft_dif<16>(v0);
    dft_dif<16>(v1);
    float2 *b0 = buf + g * C::SYM_STRIDE + (2 * b) * C::SB;
    float2 *b1 = b0 + C::SB;
    // inter-pass twiddle W_{N'}^{m kc} = u^kc with the lane-invariant base u = W_{N'}^m: one table
    // load and a running product instead of 15 scattered loads (they were half of the L1 wavefronts
    // in the first profile).  15 fp32 products in a row: relative error < 2e-6.
    const float2 u = k1_ld_table(a.tw + m * D * C::S);
    float2 t = make_float2(1.0f, 0.0f);
#pragma unroll
    for (int kc = 0; kc < 16; kc++) {
        const int br = bitrev<16>(kc);
        const int pos = k1_pad(kc * C::M0 + m);
        if (kc == 0) {
            b0[pos] = v0[br];
            b1[pos] = v1[br];
        } else {
            t = kc == 1 ? u : cmul(t, u);
            b0[pos] = cmul(v0[br], t);
            b1[pos] = cmul(v1[br], t);
        }
    }
}

// ---- in-place shared-memory pass of radix R, stride SIG (in n1 units) -------------------
template <int SF, int R, int SIG, int D = 8>
LB_HD void k1_pass(const K1Args &a, int tid, float2 *buf) {
    using C = K1Cfg<SF, D>;
    constexpr int PER_BRANCH = C::NP / R;
    constexpr int ITEMS = C::G * D * PER_BRANCH;
    for (int it = tid; it < ITEMS; it += K1_THREADS) {
        const int j = it % PER_BRANCH;
        const int gr = it / PER_BRANCH;                  // g * D + r
        const int lo = j % SIG;
        const int base = (j / SIG) * (R * SIG) + lo;
        float2 *p = buf + gr * C::SB;
        float2 v[R];
#pragma unroll
        for (int c = 0; c < R; c++) v[c] = p[k1_pad(base + SIG * c)];
        dft_dif<R>(v);
        float2 u = make_float2(1.0f, 0.0f), t = u;
        if (SIG > 1) u = k1_ld_table(a.tw + lo * (C::SPS / (R * SIG)));      // W_{R SIG}^{lo}; t runs through its powers
#pragma unroll
        for (int kc = 0; kc < R; kc++) {
            float2 o = v[bitrev<R>(kc)];
            if (SIG > 1 && kc > 0) {
                t = kc == 1 ? u : cmul(t, u);
                o = cmul(o, t);
            }
            p[k1_pad(base + SIG * kc)] = o;
        }
    }
}

// position p (inside one branch) -> sub-problem bin q held there after all passes
template <int SF, int D = 8>
LB_HD int k1_pos_to_bin(int p) {
    using C = K1Cfg<SF, D>;
    const int d0 = p / C::M0, dr = p % C::M0;
    int rest;
    if (C::SIG1 == 1) rest = dr;                          // one more pass: digit d1 = dr
    else rest = (dr / C::SIG1) + C::R1 * (dr % C::SIG1);  // d1 + R1 * d2
    return d0 + 16 * rest;
}

// ---- combine: D-branch twiddled sum, |.|^2, per-thread argmax over its NP/TPS positions ---
// (4 positions at D = 8, 16 at D = 2).  At signed bin -N/2 the sum is F[sps - N/2] (tmp[N/2], :447) and plus_quirk adds
// F[N/2] with the conjugate twiddle (:450): two distinct bins for any D > 1.
// lane-invariant combine twiddles W_{sps'}^{qs} for the thread's NP/TPS positions (hoisted out of
// the persistent loop: they were 4 scattered loads per thread and batch)
template <int SF, int D = 8>
LB_HD void k1_combine_twiddles(const K1Args &a, int tid, float2 *w) {
    using C = K1Cfg<SF, D>;
    const int lt = tid % C::TPS;
    for (int i = 0; i < C::NP / C::TPS; i++) {
        const int q = k1_pos_to_bin<SF, D>(lt + C::TPS * i);
        const int qs = q < C::NP / 2 ? q : q - C::NP;
        w[i] = k1_ld_table(a.tw + ((qs * C::S) & (C::SPS - 1)));
    }
}

template <int SF, int D = 8>
LB_HD unsigned long long k1_combine(const K1Args &a, int s, int tid, const float2 *buf, const float2 *wtab) {
    using C = K1Cfg<SF, D>;
    const int g = tid / C::TPS, lt = tid % C::TPS;
    const float2 *bs = buf + g * C::SYM_STRIDE;
    unsigned long long best = 0ull;
#pragma unroll
    for (int i = 0; i < C::NP / C::TPS; i++) {
        const int p = lt + C::TPS * i;
        const int q = k1_pos_to_bin<SF, D>(p);
        const int qs = q < C::NP / 2 ? q : q - C::NP;      // signed bin of the sub-problem
        const float2 w = wtab[i];                          // W_{sps'}^{qs}
        const int pp = k1_pad(p);
        float2 gv[D];
#pragma unroll
        for (int r = 0; r < D; r++) gv[r] = bs[r * C::SB + pp];
        float2 acc = horner<D>(gv, w);
        if (s == 0 && q == C::NP / 2) acc = plus_quirk<D>(acc, gv, w);
        const int kp = C::S * qs + s;
        const uint32_t idx = (uint32_t)(kp >= 0 ? kp : C::N + kp);
        const unsigned long long key = pack_key(cnorm2(acc), idx);
        best = key > best ? key : best;
    }
    return best;
}

// ---- several antennas: the combined spectrum P[k] = sum_a |tmp_a[k]|^2 of M windows ------------------------------------------
// The combine phase of each antenna's window adds |.|^2 at the thread's NP/TPS positions into pw -- k1_combine's sum, the
// same branch sums and quirk -- and once every antenna of sub-problem s is in, k1_power_key gives the first argmax of the
// summed powers.  (k1_combine keeps its own copy of the sum: the single-antenna kernels compile exactly as before.)
template <int SF, int D = 8>
LB_HD void k1_combine_power(int s, int tid, const float2 *buf, const float2 *wtab, float *pw) {
    using C = K1Cfg<SF, D>;
    const int g = tid / C::TPS, lt = tid % C::TPS;
    const float2 *bs = buf + g * C::SYM_STRIDE;
#pragma unroll
    for (int i = 0; i < C::NP / C::TPS; i++) {
        const int p = lt + C::TPS * i;
        const int q = k1_pos_to_bin<SF, D>(p);
        const int pp = k1_pad(p);
        float2 gv[D];
#pragma unroll
        for (int r = 0; r < D; r++) gv[r] = bs[r * C::SB + pp];
        float2 acc = horner<D>(gv, wtab[i]);
        if (s == 0 && q == C::NP / 2) acc = plus_quirk<D>(acc, gv, wtab[i]);
        pw[i] += cnorm2(acc);
    }
}
template <int SF, int D = 8>
LB_HD unsigned long long k1_power_key(int s, int tid, const float *pw) {
    using C = K1Cfg<SF, D>;
    const int lt = tid % C::TPS;
    unsigned long long best = 0ull;
#pragma unroll
    for (int i = 0; i < C::NP / C::TPS; i++) {
        const int q = k1_pos_to_bin<SF, D>(lt + C::TPS * i);
        const int kp = C::S * (q < C::NP / 2 ? q : q - C::NP) + s;
        const unsigned long long key = pack_key(pw[i], (uint32_t)(kp >= 0 ? kp : C::N + kp));
        best = key > best ? key : best;
    }
    return best;
}

#ifdef __CUDACC__
// several antennas, one work item (group g, batch of G window positions) per CTA turn: for each sub-problem s the M windows
// of every position go through pass 0 .. combine in turn and sum their |.|^2 per kept bin before the argmax.  bins / mags of
// group g, position j at out[g * out_stride + j]; sqrt(P[bin]) is the magnitude.
template <int SF, int D = 8>
__global__ void __launch_bounds__(K1_THREADS, 2)
k1_antennas_kernel(K1Args a /* x: group 0, antenna 0, position 0; n_symbols: positions per row */, size_t row_stride, uint32_t m,
                   uint32_t n_groups, size_t out_stride, uint32_t *__restrict__ bins, float *__restrict__ mags) {
    using C = K1Cfg<SF, D>;
    constexpr int W_LOG = k1_log2(C::W);
    extern __shared__ float2 k1_smem[];
    __shared__ unsigned long long warp_best[K1_THREADS / C::W];
    float2 *buf = k1_smem;
    const int tid = threadIdx.x;
    const size_t n_batches = (a.n_symbols + C::G - 1) / C::G;
    const size_t n_work = n_batches * n_groups;
    float2 wtab[C::NP / C::TPS];
    k1_combine_twiddles<SF, D>(a, tid, wtab);
    for (size_t w = blockIdx.x; w < n_work; w += gridDim.x) {
        const size_t g = w / n_batches, batch = w % n_batches;
        unsigned long long best = 0ull;
        for (int s = 0; s < C::S; s++) {
            float pw[C::NP / C::TPS];
#pragma unroll
            for (int i = 0; i < C::NP / C::TPS; i++) pw[i] = 0.f;
            for (uint32_t ant = 0; ant < m; ant++) {
                K1Args aa = a;
                aa.x = a.x + (g * m + ant) * row_stride;
                k1_pass0<SF, true, D>(aa, batch, s, tid, buf);
                __syncthreads();
                k1_pass<SF, C::R1, C::SIG1, D>(aa, tid, buf);
                __syncthreads();
                if (C::R2 > 1) {
                    k1_pass<SF, (C::R2 > 1 ? C::R2 : 2), 1, D>(aa, tid, buf);
                    __syncthreads();
                }
                k1_combine_power<SF, D>(s, tid, buf, wtab, pw);
                __syncthreads();
            }
            const unsigned long long k = k1_power_key<SF, D>(s, tid, pw);
            best = k > best ? k : best;
        }
        best = group_max_key<C::W>(best);
        if ((tid & (C::W - 1)) == 0) warp_best[tid >> W_LOG] = best;
        __syncthreads();
        if (tid < C::G) {
            constexpr int WPS = C::TPS / C::W;
            unsigned long long bb = 0ull;
#pragma unroll
            for (int k = 0; k < WPS; k++) {
                const unsigned long long o = warp_best[tid * WPS + k];
                bb = o > bb ? o : bb;
            }
            const size_t sym = batch * C::G + tid;
            if (sym < a.n_symbols) k1_store(bins, mags, g * out_stride + sym, bb);
        }
        // warp_best is rewritten only after the next work item's passes and their __syncthreads
    }
}
#endif  // __CUDACC__

#ifdef __CUDACC__
// ---- the kernel: persistent CTAs over (batch, s) work items ------------------------------
// D = 8: fs/bw = 8; D = 2: fs/bw = 2, where one symbol's combine spans fewer than 32 lanes at SF7 and SF8 and each group
// of W = TPS lanes reduces on its own
template <int SF, int D = 8>
__global__ void __launch_bounds__(K1_THREADS, 2)
k1_fft_kernel(K1Args a, uint32_t *__restrict__ bins, float *__restrict__ mags,
              unsigned long long *__restrict__ packed /* S > 1 only */) {
    using C = K1Cfg<SF, D>;
    constexpr int W_LOG = k1_log2(C::W);
    extern __shared__ float2 k1_smem[];
    __shared__ unsigned long long warp_best[K1_THREADS / C::W];
    float2 *buf = k1_smem;
    const int tid = threadIdx.x;
    const size_t n_batches = (a.n_symbols + C::G - 1) / C::G;
    const size_t n_work = n_batches * C::S;
    float2 wtab[C::NP / C::TPS];
    k1_combine_twiddles<SF, D>(a, tid, wtab);
    for (size_t w = blockIdx.x; w < n_work; w += gridDim.x) {
        const size_t batch = w / C::S;
        const int s = (int)(w % C::S);
        k1_pass0<SF, true, D>(a, batch, s, tid, buf);
        __syncthreads();
        k1_pass<SF, C::R1, C::SIG1, D>(a, tid, buf);
        __syncthreads();
        if (C::R2 > 1) {
            k1_pass<SF, (C::R2 > 1 ? C::R2 : 2), 1, D>(a, tid, buf);
            __syncthreads();
        }
        unsigned long long best = k1_combine<SF, D>(a, s, tid, buf, wtab);
        // group argmax (the warp, or one symbol's lanes), then across the groups of one symbol
        best = group_max_key<C::W>(best);
        if ((tid & (C::W - 1)) == 0) warp_best[tid >> W_LOG] = best;
        __syncthreads();
        if (tid < C::G) {
            constexpr int WPS = C::TPS / C::W;            // groups per symbol
            unsigned long long bb = 0ull;
#pragma unroll
            for (int k = 0; k < WPS; k++) {
                const unsigned long long o = warp_best[tid * WPS + k];
                bb = o > bb ? o : bb;
            }
            const size_t sym = batch * C::G + tid;
            if (sym < a.n_symbols) {
                if (C::S == 1) k1_store(bins, mags, sym, bb);
                else atomicMax(packed + sym, bb);
            }
        }
        // warp_best and buf are rewritten only after the next pass0 + __syncthreads
    }
}
#endif  // __CUDACC__

// ---- CPU emulation of the kernel (same phase functions, threads run one after another) ---
template <int SF, int D = 8>
inline void k1_emulate(const K1Args &a, uint32_t *bins, float *mags) {
    using C = K1Cfg<SF, D>;
    float2 *buf = new float2[C::SMEM_ELEMS];
    const size_t n_batches = (a.n_symbols + C::G - 1) / C::G;
    unsigned long long *packed = new unsigned long long[n_batches * C::G]();
    for (size_t batch = 0; batch < n_batches; batch++) {
        for (int s = 0; s < C::S; s++) {
            for (int i = 0; i < C::SMEM_ELEMS; i++) buf[i] = make_float2(NAN, NAN);   // catch unwritten reads
            for (int t = 0; t < K1_THREADS; t++) k1_pass0<SF, true, D>(a, batch, s, t, buf);
            for (int t = 0; t < K1_THREADS; t++) k1_pass<SF, C::R1, C::SIG1, D>(a, t, buf);
            if (C::R2 > 1)
                for (int t = 0; t < K1_THREADS; t++) k1_pass<SF, (C::R2 > 1 ? C::R2 : 2), 1, D>(a, t, buf);
            for (int t = 0; t < K1_THREADS; t++) {
                float2 wtab[C::NP / C::TPS];
                k1_combine_twiddles<SF, D>(a, t, wtab);
                const unsigned long long k = k1_combine<SF, D>(a, s, t, buf, wtab);
                const size_t sym = batch * C::G + t / C::TPS;
                if (k > packed[sym]) packed[sym] = k;
            }
        }
    }
    for (size_t i = 0; i < a.n_symbols; i++) k1_store(bins, mags, i, packed[i]);
    delete[] buf;
    delete[] packed;
}

// ... and of k1_antennas_kernel: M rows of n_symbols windows each, row_stride apart, into bins / mags[n_symbols]
template <int SF, int D = 8>
inline void k1_antennas_emulate(const K1Args &a, size_t row_stride, uint32_t m, uint32_t *bins, float *mags) {
    using C = K1Cfg<SF, D>;
    constexpr int NPT = C::NP / C::TPS;
    float2 *buf = new float2[C::SMEM_ELEMS];
    float *pw = new float[K1_THREADS * NPT];
    const size_t n_batches = (a.n_symbols + C::G - 1) / C::G;
    unsigned long long *packed = new unsigned long long[n_batches * C::G]();
    for (size_t batch = 0; batch < n_batches; batch++) {
        for (int s = 0; s < C::S; s++) {
            for (int i = 0; i < K1_THREADS * NPT; i++) pw[i] = 0.f;
            for (uint32_t ant = 0; ant < m; ant++) {
                K1Args aa = a;
                aa.x = a.x + ant * row_stride;
                for (int i = 0; i < C::SMEM_ELEMS; i++) buf[i] = make_float2(NAN, NAN);
                for (int t = 0; t < K1_THREADS; t++) k1_pass0<SF, true, D>(aa, batch, s, t, buf);
                for (int t = 0; t < K1_THREADS; t++) k1_pass<SF, C::R1, C::SIG1, D>(aa, t, buf);
                if (C::R2 > 1)
                    for (int t = 0; t < K1_THREADS; t++) k1_pass<SF, (C::R2 > 1 ? C::R2 : 2), 1, D>(aa, t, buf);
                for (int t = 0; t < K1_THREADS; t++) {
                    float2 wtab[NPT];
                    k1_combine_twiddles<SF, D>(aa, t, wtab);
                    k1_combine_power<SF, D>(s, t, buf, wtab, pw + t * NPT);
                }
            }
            for (int t = 0; t < K1_THREADS; t++) {
                const unsigned long long k = k1_power_key<SF, D>(s, t, pw + t * NPT);
                const size_t sym = batch * C::G + t / C::TPS;
                if (k > packed[sym]) packed[sym] = k;
            }
        }
    }
    for (size_t i = 0; i < a.n_symbols; i++) k1_store(bins, mags, i, packed[i]);
    delete[] buf;
    delete[] pw;
    delete[] packed;
}

}  // namespace lb
