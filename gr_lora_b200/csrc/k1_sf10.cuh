// k1_sf10.cuh -- K1 for SF10: one CTA-wide group of 256 threads per symbol, two radix-32 passes.
//
// N = 1024 = 32 x 32.  Same pipeline as k1_group.cuh (TMA-fed ring of 64 KiB symbols, two swizzled
// exchanges, lane-invariant twiddles) but every thread carries ONE polyphase
// branch: pass 0 is a radix-32 over the 32 rows of column a = t >> 3, branch r = t & 7 (64-bit accesses,
// sample n = 256 c + t), pass 1 a radix-32 over the 32 columns of output column kc.  The inter-pass
// twiddle W_N^{a kc} (31 values per lane) is formed from two short lane-invariant tables,
// W^{a (kc & 3)} and W^{a (kc & ~3)}.
// The 32 down-chirp samples a thread multiplies with are the same for every symbol; the CTA keeps the chirp as a
// 64 KiB shared-memory table next to a ring of two TMA slots (64 + 2 x 64 KiB).
#pragma once
#include "k1_ring.cuh"

namespace lb {

constexpr int S10_T = 256, S10_N = 1024, S10_SPS = 8192;
constexpr int S10_SLOT_F2 = 8192;                    // float2 per slot

struct S10Consts {
    float2 tl[4];            // W_N^{a j},   j = 0..3
    float2 th[8];            // W_N^{a 4j},  j = 0..7
    float2 wq[4];            // W_sps^{q'}, q = t + 256 i
};

LB_HD void s10_consts(int t, const float2 *tw, S10Consts &c) {
    const int a = t >> 3;
    for (int j = 0; j < 4; j++) c.tl[j] = k1_ld_table(tw + ((a * j * 8) & (S10_SPS - 1)));
    for (int j = 0; j < 8; j++) c.th[j] = k1_ld_table(tw + ((a * 4 * j * 8) & (S10_SPS - 1)));
    for (int i = 0; i < 4; i++) {
        const int q = t + S10_T * i;
        c.wq[i] = k1_ld_table(tw + ((q < S10_N / 2 ? q : q - S10_N) & (S10_SPS - 1)));
    }
}

LB_HD void s10_pass0_fft(const S10Consts &c, float2 *v);
LB_HD void s10_pass0(int t, const float2 *slot, const float2 *chirp, const S10Consts &c, float2 *v) {
#pragma unroll
    for (int r = 0; r < 32; r++) v[r] = cmul(slot[r * S10_T + t], chirp[r * S10_T + t]);
    s10_pass0_fft(c, v);
}
LB_HD void s10_pass0_fft(const S10Consts &c, float2 *v) {
    dft_dif<32>(v);
#pragma unroll
    for (int kc = 1; kc < 32; kc++) {
        const int br = bitrev<32>(kc);
        float2 w;
        if ((kc & 3) == 0) w = c.th[kc >> 2];
        else if ((kc >> 2) == 0) w = c.tl[kc & 3];
        else w = cmul(c.th[kc >> 2], c.tl[kc & 3]);
        v[br] = cmul(v[br], w);
    }
}

// exchange 1: [kc][(a*8 + r) ^ ((kc & 1) << 3)]
LB_HD void s10_store1(int t, float2 *slot, const float2 *v) {
#pragma unroll
    for (int kc = 0; kc < 32; kc++) slot[kc * S10_T + (t ^ ((kc & 1) << 3))] = v[bitrev<32>(kc)];
}

LB_HD void s10_pass1(int t, const float2 *slot, float2 *g) {
    const int kc = t >> 3, r = t & 7;
    const int sw = (kc & 1) << 3;
#pragma unroll
    for (int a = 0; a < 32; a++) g[a] = slot[kc * S10_T + ((a * 8 + r) ^ sw)];
    dft_dif<32>(g);
}

// exchange 2: [q][r] with the 16-byte unit of the row XOR-swizzled by (q >> 1) & 3
LB_HD int s10_pos2(int q, int r) { return q * 8 + ((((r >> 1) ^ ((q >> 1) & 3)) << 1) | (r & 1)); }

LB_HD void s10_store2(int t, float2 *slot, const float2 *g) {
    const int kc = t >> 3, r = t & 7;
#pragma unroll
    for (int ka = 0; ka < 32; ka++) slot[s10_pos2(kc + 32 * ka, r)] = g[bitrev<32>(ka)];
}

LB_HD unsigned long long s10_combine(int t, const float2 *slot, const S10Consts &c) {
    unsigned long long best = 0ull;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int q = t + S10_T * i;
        float2 gv[8];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const float4 v = *reinterpret_cast<const float4 *>(slot + q * 8 + ((u ^ ((q >> 1) & 3)) << 1));
            gv[2 * u] = make_float2(v.x, v.y);
            gv[2 * u + 1] = make_float2(v.z, v.w);
        }
        float2 acc = horner<8>(gv, c.wq[i]);
        if (q == S10_N / 2) acc = plus_quirk<8>(acc, gv, c.wq[i]);
        const unsigned long long key = pack_key(cnorm2(acc), (uint32_t)q);
        best = key > best ? key : best;
    }
    return best;
}

#ifdef __CUDACC__
template <int NSLOT>
struct S10Smem {
    float2 chirp[S10_SLOT_F2];
    float2 slots[NSLOT][S10_SLOT_F2];
    uint64_t bars[NSLOT];
    unsigned long long keys[S10_T / 32];
};

template <int NSLOT>
__global__ void __launch_bounds__(S10_T, 1)
k1_sf10_kernel(K1Args a, uint32_t *__restrict__ bins, float *__restrict__ mags) {
    extern __shared__ __align__(128) unsigned char s10_raw[];
    S10Smem<NSLOT> &sm = *reinterpret_cast<S10Smem<NSLOT> *>(s10_raw);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const size_t g0 = blockIdx.x, g_total = gridDim.x;
    const SymbolRing<float2, S10_SLOT_F2, NSLOT> ring{sm.slots, sm.bars, a.x, g0, g_total, a.n_symbols};
    if (t == 0) ring.init();
    for (int i = t; i < S10_SLOT_F2; i += S10_T) sm.chirp[i] = k1_ld_table(a.chirp + i);
    __syncthreads();
    if (t == 0) ring.fill();
    S10Consts c;
    s10_consts(t, a.tw, c);
    uint32_t it = 0;
    for (size_t sym = g0; sym < a.n_symbols; sym += g_total, it++) {
        float2 *slot = ring.wait(it);
        float2 v[32];
        s10_pass0(t, slot, sm.chirp, c, v);
        __syncthreads();
        s10_store1(t, slot, v);
        __syncthreads();
        s10_pass1(t, slot, v);
        __syncthreads();
        s10_store2(t, slot, v);
        __syncthreads();
        unsigned long long best = s10_combine(t, slot, c);
        best = warp_max_key(best);
        if (lane == 0) sm.keys[warp] = best;
        __syncthreads();
        if (t == 0) {
            ring.refill(it, sym);
            unsigned long long bb = sm.keys[0];
#pragma unroll
            for (int k = 1; k < S10_T / 32; k++) bb = sm.keys[k] > bb ? sm.keys[k] : bb;
            k1_store(bins, mags, sym, bb);
        }
    }
}
#endif

inline void s10_emulate(const K1Args &a, uint32_t *bins, float *mags) {
    float2 *slot = new float2[S10_SLOT_F2];
    S10Consts *c = new S10Consts[S10_T];
    auto v = new float2[S10_T][32];
    for (int t = 0; t < S10_T; t++) s10_consts(t, a.tw, c[t]);
    for (size_t sym = 0; sym < a.n_symbols; sym++) {
        const float2 *x = a.x + sym * S10_SPS;
        for (int i = 0; i < S10_SLOT_F2; i++) slot[i] = x[i];
        for (int t = 0; t < S10_T; t++) s10_pass0(t, slot, a.chirp, c[t], v[t]);
        for (int i = 0; i < S10_SLOT_F2; i++) slot[i] = make_float2(NAN, NAN);
        for (int t = 0; t < S10_T; t++) s10_store1(t, slot, v[t]);
        for (int t = 0; t < S10_T; t++) s10_pass1(t, slot, v[t]);
        for (int i = 0; i < S10_SLOT_F2; i++) slot[i] = make_float2(NAN, NAN);
        for (int t = 0; t < S10_T; t++) s10_store2(t, slot, v[t]);
        unsigned long long best = 0ull;
        for (int t = 0; t < S10_T; t++) {
            const unsigned long long k = s10_combine(t, slot, c[t]);
            best = k > best ? k : best;
        }
        k1_store(bins, mags, sym, best);
    }
    delete[] slot; delete[] c; delete[] v;
}

}  // namespace lb
