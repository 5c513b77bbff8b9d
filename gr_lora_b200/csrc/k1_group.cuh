// k1_group.cuh -- K1 for SF8 / SF9: a GROUP of W = 2^(SF-7) warps per symbol.
//
// The SF7 warp kernel (k1_warp.cuh) generalised: the T = 32 W threads of a group own a ring of TMA-fed
// shared-memory slots (one symbol = 8*sps bytes each) and run, per symbol,
//   pass 0   float4 #t of each of the 16 rows -> dechirp -> two radix-16 DIF FFTs in registers,
//            inter-pass twiddle u^kc (u = W_N^a lane invariant, powers kept in registers)
//   exch 1   XOR-swizzled 128-bit exchange through the consumed slot: thread (kc, h) receives its
//            NR = 4/W polyphase branches of output column kc, all M0 = 8 W points
//   pass 1   NR radix-M0 FFTs in registers (radix 16 at SF8, radix 32 at SF9), branch pairs combined
//   exch 2   second swizzled exchange ([bin][branch pair]) so that each thread holds all 4 pair sums of 4 bins
//   combine  Horner over the 4 pairs with ONE lane-invariant twiddle per bin, |.|^2, group argmax
// Same arithmetic as get_shift_fft (lib/decoder_impl.cc:430-464); see k1_fft.cuh for the derivation.
// Shared-memory traffic per symbol: 6 x 8*sps bytes (slot read, chirp read, two exchanges).  The down-chirp is one
// shared-memory table per CTA, read by every group (the samples a thread multiplies with are symbol-invariant).
#pragma once
#include "k1_ring.cuh"
#include "k1_group_consts.h"
#include "k1_launch.h"

#include <algorithm>

namespace lb {

template <int SF>
struct GCfg {
    static constexpr int W = 1 << (SF - 7);          // warps per group
    static constexpr int T = 32 * W;                 // threads per group
    static constexpr int N = 1 << SF, SPS = 8 * N;
    static constexpr int M0 = 8 * W;                 // points of the second FFT (columns)
    static constexpr int NR = 4 / W;                 // branches per thread in pass 1: 2, 1
    static constexpr int LPK = 2 * W;                // lanes per output column kc
    static constexpr int SLOT_F4 = 16 * T;           // float4 per slot
    static_assert(SF == 8 || SF == 9, "group kernel: SF8, SF9");
};

LB_HD int g_swz1(int kc) { return (kc & 1) << 2; }
template <int SF> LB_HD int g_signed_bin(int q) { return q < GCfg<SF>::N / 2 ? q : q - GCfg<SF>::N; }

template <int SF>
struct GConsts {
    float2 twk[16];          // W_N^{a kc}, a = t >> 2 (pass-0 output twiddle), twk[0] = 1
    float2 wq2[4];           // wq^2 (Horner over branch PAIRS)
    float2 wb;               // pair-twiddle base of this lane: W_sps^{kc} (times the upper-half factor at SF9)
};

template <int SF>
LB_HD void g_consts(int t, const float2 *tw, GConsts<SF> &c) {
    using C = GCfg<SF>;
    const int a = t >> 2;
    for (int kc = 0; kc < 16; kc++) c.twk[kc] = k1_ld_table(tw + ((a * kc * 8) & (C::SPS - 1)));     // W_N = W_sps^8
    for (int i = 0; i < 4; i++) c.wq2[i] = k1_ld_table(tw + ((2 * g_signed_bin<SF>(t + C::T * i)) & (C::SPS - 1)));
    {   // w[ka] = W_sps^{q'} with q = kc + 16 ka = wb * g_cc[ka]; at SF9 the odd lane of a pair owns ka >= M0/2:
        // g_cc[ka] = g_cc[ka - M0/2] * W_sps^{16 M0/2 - N}, folded into its wb
        const int kc = t / C::LPK, h = t % C::LPK;
        int e = kc;
        if (C::NR == 1 && (h & 1)) e += 16 * (C::M0 / 2) - C::N;
        c.wb = k1_ld_table(tw + (e & (C::SPS - 1)));
    }
}

template <int SF>
LB_HD float2 g_cc(int ka) {
#ifdef __CUDA_ARCH__
    return SF == 8 ? g_cc8_dev[ka & 15] : g_cc9_dev[ka & 31];
#else
    return SF == 8 ? g_cc8_host[ka & 15] : g_cc9_host[ka & 31];
#endif
}

// pass 0 + exchange-1 write.  slot/chirp: natural sample order as float4 pairs.
template <int SF>
LB_HD void g_pass0(int t, const float4 *slot, const float4 *chirp, const GConsts<SF> &c, float2 *v0, float2 *v1) {
    using C = GCfg<SF>;
#pragma unroll
    for (int r = 0; r < 16; r++) {
        const float4 xv = slot[r * C::T + t];
        const float4 dv = chirp[r * C::T + t];
        v0[r] = cmul(make_float2(xv.x, xv.y), make_float2(dv.x, dv.y));
        v1[r] = cmul(make_float2(xv.z, xv.w), make_float2(dv.z, dv.w));
    }
    dft_dif<16>(v0);
    dft_dif<16>(v1);
#pragma unroll
    for (int kc = 1; kc < 16; kc++) {
        const int br = bitrev<16>(kc);
        v0[br] = cmul(v0[br], c.twk[kc]);
        v1[br] = cmul(v1[br], c.twk[kc]);
    }
}

template <int SF>
LB_HD void g_store1(int t, float4 *slot, const float2 *v0, const float2 *v1) {
    using C = GCfg<SF>;
#pragma unroll
    for (int kc = 0; kc < 16; kc++) {
        const int br = bitrev<16>(kc);
        slot[kc * C::T + (t ^ g_swz1(kc))] = make_float4(v0[br].x, v0[br].y, v1[br].x, v1[br].y);
    }
}

// pass 1: thread (kc = t / LPK, h = t % LPK) loads branches r = h*NR .. h*NR+NR-1, all M0 columns,
// and runs NR radix-M0 FFTs.  g[i][bitrev(ka)] = G_{h NR + i}[kc + 16 ka].
template <int SF>
LB_HD void g_pass1(int t, const float4 *slot, float2 (*g)[GCfg<SF>::M0]) {
    using C = GCfg<SF>;
    const int kc = t / C::LPK, h = t % C::LPK;
    const int sw = g_swz1(kc);
    const float4 *row = slot + kc * C::T;
#pragma unroll
    for (int a = 0; a < C::M0; a++) {
        if constexpr (C::NR == 2) {
            const float4 u = row[(4 * a + h) ^ sw];
            g[0][a] = make_float2(u.x, u.y);
            g[C::NR - 1][a] = make_float2(u.z, u.w);
        } else {
            const float2 *p2 = reinterpret_cast<const float2 *>(row + ((4 * a + (h >> 1)) ^ sw));
            g[0][a] = p2[h & 1];
        }
    }
#pragma unroll
    for (int i = 0; i < C::NR; i++) dft_dif<C::M0>(g[i]);
}

// ---- combine branch pairs BEFORE the second exchange ----------------------------------------------
// P_pr[q] = G_{2pr}[q] + w[q] G_{2pr+1}[q].  SF8 (NR = 2): both branches are in the thread.  SF9 (NR = 1):
// the partner lane t^1 holds the other branch; the even lane finishes ka < M0/2, the odd lane ka >= M0/2
// (own = this lane's G, bit-reversed; other = what the partner sent for this lane's half).
// Returns NP = M0 (SF8) or M0/2 (SF9) values P[j] for ka = j (+ M0/2 on odd SF9 lanes).
// Pq = the same with the conjugate twiddle for the quirk bin q = N/2 (kc = 0, ka = M0/2), else 0.
template <int SF> struct GPair { static constexpr int NP = GCfg<SF>::NR == 2 ? GCfg<SF>::M0 : GCfg<SF>::M0 / 2; };

template <int SF>
LB_HD void g_pair_sf8(int t, float2 (*g)[GCfg<SF>::M0], const GConsts<SF> &c, float2 *P, float2 &Pq) {
    using C = GCfg<SF>;
    const int kc = t / C::LPK;
    Pq = make_float2(0.f, 0.f);
#pragma unroll
    for (int ka = 0; ka < C::M0; ka++) {
        const int br = bitrev<C::M0>(ka);
        const float2 od = cmul(g[C::NR - 1][br], g_cc<SF>(ka));
        P[ka] = cfma(od, c.wb, g[0][br]);
        if (ka == C::M0 / 2 && kc == 0) Pq = cfma(cmul(g[C::NR - 1][br], cconj(g_cc<SF>(ka))), cconj(c.wb), g[0][br]);
    }
}

// SF9: keep[j]/other[j] for ka = j + (odd ? M0/2 : 0); even_part/odd_part by lane parity
template <int SF>
LB_HD void g_pair_sf9(int t, const float2 *keep, const float2 *recv, const GConsts<SF> &c, float2 *P, float2 &Pq) {
    using C = GCfg<SF>;
    const int kc = t / C::LPK, odd = t & 1;
    Pq = make_float2(0.f, 0.f);
#pragma unroll
    for (int j = 0; j < C::M0 / 2; j++) {
        const float2 ev = odd ? recv[j] : keep[j];
        const float2 od = odd ? keep[j] : recv[j];
        const float2 odc = cmul(od, g_cc<SF>(j));
        P[j] = cfma(odc, c.wb, ev);
        if (j == 0 && kc == 0 && odd) Pq = cfma(cmul(od, cconj(g_cc<SF>(j))), cconj(c.wb), ev);   // ka = M0/2
    }
}

// exchange 2 (pair variant): [bin q][pair pr] float2, 4 pairs = 32 B per bin, 16-byte unit XOR (q >> 2) & 1
// (rows of the upper half, written by the odd lanes at SF9, take the other 64-byte half of the bank window)
LB_HD int g_row2p(int q) { return q ^ (((q >> 8) & 1) << 1); }
LB_HD int g_pos2p(int q, int pr) { return g_row2p(q) * 4 + ((((pr >> 1) ^ ((q >> 2) & 1)) << 1) | (pr & 1)); }

template <int SF>
LB_HD void g_store2p(int t, float2 *slot2, const float2 *P, float2 Pq, float2 *quirk) {
    using C = GCfg<SF>;
    const int kc = t / C::LPK, h = t % C::LPK;
    const int pr = C::NR == 2 ? h : (h >> 1);
    const int ka0 = (C::NR == 1 && (h & 1)) ? C::M0 / 2 : 0;
#pragma unroll
    for (int j = 0; j < GPair<SF>::NP; j++) slot2[g_pos2p(kc + 16 * (ka0 + j), pr)] = P[j];
    if (kc == 0 && (C::NR == 2 || (h & 1))) quirk[pr] = Pq;
}

template <int SF>
LB_HD unsigned long long g_combine_p(int t, const float2 *slot2, const float2 *quirk, const GConsts<SF> &c) {
    using C = GCfg<SF>;
    unsigned long long best = 0ull;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int q = t + C::T * i;
        float2 pv[4];
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const float4 v = *reinterpret_cast<const float4 *>(slot2 + g_row2p(q) * 4 + ((u ^ ((q >> 2) & 1)) << 1));
            pv[2 * u] = make_float2(v.x, v.y);
            pv[2 * u + 1] = make_float2(v.z, v.w);
        }
        float2 acc = horner<4>(pv, c.wq2[i]);
        if (q == C::N / 2) acc = plus_quirk<4>(acc, quirk, c.wq2[i]);
        const unsigned long long key = pack_key(cnorm2(acc), (uint32_t)q);
        best = key > best ? key : best;
    }
    return best;
}

#ifdef __CUDACC__
template <int SF, int NGROUPS, int NSLOT>
struct GSmem {
    float4 chirp[GCfg<SF>::SLOT_F4];
    float4 slots[NGROUPS][NSLOT][GCfg<SF>::SLOT_F4];
    uint64_t bars[NGROUPS][NSLOT];
    unsigned long long keys[NGROUPS][GCfg<SF>::W];
    float2 quirk[NGROUPS][4];
};

LB_D void group_bar(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

template <int SF, int NGROUPS, int NSLOT>
__global__ void __launch_bounds__(NGROUPS * GCfg<SF>::T, 1)
k1_group_kernel(K1Args a, uint32_t *__restrict__ bins, float *__restrict__ mags) {
    using C = GCfg<SF>;
    extern __shared__ __align__(128) unsigned char g_raw[];
    GSmem<SF, NGROUPS, NSLOT> &sm = *reinterpret_cast<GSmem<SF, NGROUPS, NSLOT> *>(g_raw);
    const int grp = threadIdx.x / C::T, t = threadIdx.x % C::T;
    const int lane = t & 31, wig = t >> 5;              // warp in group
    const int bar_id = 1 + grp;                         // named barrier of this group (0 = __syncthreads)
    const size_t gg = (size_t)blockIdx.x * NGROUPS + grp, g_total = (size_t)gridDim.x * NGROUPS;

    const SymbolRing<float4, C::SLOT_F4, NSLOT> ring{sm.slots[grp], sm.bars[grp], a.x, gg, g_total, a.n_symbols};

    if (t == 0) ring.init();
    for (int i = threadIdx.x; i < C::SLOT_F4; i += NGROUPS * C::T) sm.chirp[i] = k1_ld_table4(a.chirp + 2 * i);
    __syncthreads();
    if (t == 0) ring.fill();
    GConsts<SF> c;
    g_consts<SF>(t, a.tw, c);

    uint32_t it = 0;
    for (size_t sym = gg; sym < a.n_symbols; sym += g_total, it++) {
        float4 *slot = ring.wait(it);
        {
            float2 v0[16], v1[16];
            g_pass0<SF>(t, slot, sm.chirp, c, v0, v1);
            group_bar(bar_id, C::T);                    // everyone has read the slot
            g_store1<SF>(t, slot, v0, v1);
        }
        group_bar(bar_id, C::T);
        float2 g[C::NR][C::M0];
        g_pass1<SF>(t, slot, g);
        float2 P[GPair<SF>::NP], Pq;
        if constexpr (C::NR == 2) {
            g_pair_sf8<SF>(t, g, c, P, Pq);
        } else {
            const int odd = t & 1;
            float2 keep[C::M0 / 2], recv[C::M0 / 2];
#pragma unroll
            for (int j = 0; j < C::M0 / 2; j++) {
                const float2 lo = g[0][bitrev<C::M0>(j)], hi = g[0][bitrev<C::M0>(j + C::M0 / 2)];
                keep[j] = odd ? hi : lo;
                const float2 send = odd ? lo : hi;
                recv[j].x = __shfl_xor_sync(0xffffffffu, send.x, 1);
                recv[j].y = __shfl_xor_sync(0xffffffffu, send.y, 1);
            }
            g_pair_sf9<SF>(t, keep, recv, c, P, Pq);
        }
        group_bar(bar_id, C::T);                        // exchange-1 reads done
        g_store2p<SF>(t, reinterpret_cast<float2 *>(slot), P, Pq, sm.quirk[grp]);
        group_bar(bar_id, C::T);
        unsigned long long best = g_combine_p<SF>(t, reinterpret_cast<const float2 *>(slot), sm.quirk[grp], c);
        best = warp_max_key(best);
        if (lane == 0) sm.keys[grp][wig] = best;
        group_bar(bar_id, C::T);                        // exchange-2 reads done + keys visible
        if (t == 0) {
            ring.refill(it, sym);
            unsigned long long bb = sm.keys[grp][0];
#pragma unroll
            for (int k = 1; k < C::W; k++) bb = sm.keys[grp][k] > bb ? sm.keys[grp][k] : bb;
            k1_store(bins, mags, sym, bb);
        }
        // keys[] is rewritten only after four more group barriers: no hazard with thread 0's read
    }
}

// instantiated in the translation unit that owns the SF's kernel: SF8 lora_b200.cu, SF9 k1_packed.cu
template <int SF, int NGROUPS, int NSLOT>
int k1_launch_group(const K1Launch &k) {
    const size_t smem = sizeof(GSmem<SF, NGROUPS, NSLOT>);
    K1_CU(opt_in_smem((const void *)k1_group_kernel<SF, NGROUPS, NSLOT>, k.device, smem));
    const int grid = (int)std::min((k.a.n_symbols + NGROUPS - 1) / NGROUPS, (size_t)k.n_sms);
    k1_group_kernel<SF, NGROUPS, NSLOT><<<grid, NGROUPS * GCfg<SF>::T, smem, k.st>>>(k.a, k.bins, k.mags);
    K1_CU(cudaGetLastError());
    return 0;
}
#endif  // __CUDACC__

// ---- CPU emulation ---------------------------------------------------------------------------
template <int SF>
inline void g_emulate(const K1Args &a, uint32_t *bins, float *mags) {
    using C = GCfg<SF>;
    float4 *slot = new float4[C::SLOT_F4];
    float4 *chirp = new float4[C::SLOT_F4];
    GConsts<SF> *c = new GConsts<SF>[C::T];
    for (int t = 0; t < C::T; t++) g_consts<SF>(t, a.tw, c[t]);
    for (int i = 0; i < C::SLOT_F4; i++) chirp[i] = make_float4(a.chirp[2 * i].x, a.chirp[2 * i].y, a.chirp[2 * i + 1].x, a.chirp[2 * i + 1].y);
    auto v0 = new float2[C::T][16];
    auto v1 = new float2[C::T][16];
    auto g = new float2[C::T][C::NR][C::M0];
    for (size_t sym = 0; sym < a.n_symbols; sym++) {
        const float2 *x = a.x + sym * C::SPS;
        for (int i = 0; i < C::SLOT_F4; i++) slot[i] = make_float4(x[2 * i].x, x[2 * i].y, x[2 * i + 1].x, x[2 * i + 1].y);
        for (int t = 0; t < C::T; t++) g_pass0<SF>(t, slot, chirp, c[t], v0[t], v1[t]);
        for (int i = 0; i < C::SLOT_F4; i++) slot[i] = make_float4(NAN, NAN, NAN, NAN);
        for (int t = 0; t < C::T; t++) g_store1<SF>(t, slot, v0[t], v1[t]);
        for (int t = 0; t < C::T; t++) g_pass1<SF>(t, slot, g[t]);
        for (int i = 0; i < C::SLOT_F4; i++) slot[i] = make_float4(NAN, NAN, NAN, NAN);
        float2 quirk[4] = {};
        float2 *slot2 = reinterpret_cast<float2 *>(slot);
        for (int t = 0; t < C::T; t++) {
            float2 P[GPair<SF>::NP], Pq;
            if constexpr (C::NR == 2) {
                g_pair_sf8<SF>(t, g[t], c[t], P, Pq);
            } else {
                const int odd = t & 1;
                float2 keep[C::M0 / 2], recv[C::M0 / 2];
                for (int j = 0; j < C::M0 / 2; j++) {
                    const int mine = bitrev<C::M0>(j + (odd ? C::M0 / 2 : 0));
                    keep[j] = g[t][0][mine];
                    recv[j] = g[t ^ 1][0][mine];          // what the partner sends: its value at MY ka
                }
                g_pair_sf9<SF>(t, keep, recv, c[t], P, Pq);
            }
            g_store2p<SF>(t, slot2, P, Pq, quirk);
        }
        unsigned long long best = 0ull;
        for (int t = 0; t < C::T; t++) {
            const unsigned long long k = g_combine_p<SF>(t, slot2, quirk, c[t]);
            best = k > best ? k : best;
        }
        k1_store(bins, mags, sym, best);
    }
    delete[] slot; delete[] chirp; delete[] c; delete[] v0; delete[] v1; delete[] g;
}

}  // namespace lb
