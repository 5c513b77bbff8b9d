// k1_warp.cuh -- K1 for SF7, one WARP per symbol (the headline configuration of BASELINE.json).
//
// Same arithmetic as k1_fft.cuh (get_shift_fft, lib/decoder_impl.cc:430-464: dechirp, pruned
// 8x128-point FFT, 8-branch twiddled sum, first argmax) but organised around what the first
// ncu capture of the CTA-wide kernel showed: the L1/LSU data
// pipe was the limiter (78 %), half of it scattered twiddle loads, and long-scoreboard stalls
// dominated because all warps of a CTA loaded in lock step.
//
//   * each warp owns a ring of NSLOT 8 KB shared-memory slots filled by TMA bulk copies
//     (cp.async.bulk + mbarrier complete_tx): loads are asynchronous, cost no registers and no
//     LSU wavefronts, and the warps drift out of phase (no CTA barrier in the steady state);
//   * lane l reads float4 #l of each of the 16 rows (conflict free), dechirps against the chirp
//     table kept in shared memory, runs two radix-16 DIF FFTs in registers;
//   * one XOR-swizzled 128-bit exchange through the (now consumed) slot re-distributes the data so
//     that lane (kc, h) holds branches 4h..4h+3 of output column kc;
//   * every twiddle a lane needs is lane-invariant and lives in registers for the whole kernel;
//   * four radix-8 FFTs, a Horner evaluation of the branch sum, one shuffle exchange with the
//     partner lane, |.|^2, warp argmax.
// Shared-memory traffic per symbol: 4 x 8 KB (read data, read chirp, exchange write + read).
#pragma once
#include "k1_ring.cuh"

namespace lb {

constexpr int W7_N = 128, W7_SPS = 1024;
constexpr int W7_SLOT_F4 = 512;          // float4 per 8 KB slot

struct W7Consts {                        // lane-invariant twiddles
    float2 tw1[8];                       // W_128^{a*kc}, a = 0..7          (inter-pass twiddle)
    float2 wq[8];                        // W_1024^{q'}, q = kc + 16*ka      (branch-sum twiddle)
    float2 w4[4];                        // wq^4 for the lane's own 4 ka
};

LB_HD int w7_swz(int kc) { return (kc & 1) | ((kc & 2) << 1); }
LB_HD int w7_signed_bin(int q) { return q < 64 ? q : q - 128; }

LB_HD void w7_consts(int lane, const float2 *tw, W7Consts &c) {
    const int kc = lane >> 1, h = lane & 1;
    for (int a = 0; a < 8; a++) c.tw1[a] = k1_ld_table(tw + ((a * kc * 8) & 1023));
    for (int ka = 0; ka < 8; ka++) c.wq[ka] = k1_ld_table(tw + (w7_signed_bin(kc + 16 * ka) & 1023));
    for (int j = 0; j < 4; j++) c.w4[j] = k1_ld_table(tw + ((4 * w7_signed_bin(kc + 16 * (4 * h + j))) & 1023));
}

// pass 0: slot (natural sample order) -> dechirp -> 2 x radix-16 -> v0 (r = 2b), v1 (r = 2b+1), bit-reversed
LB_HD void w7_pass0(int lane, const float4 *slot, const float4 *chirp, float2 *v0, float2 *v1) {
#pragma unroll
    for (int c = 0; c < 16; c++) {
        const float4 xv = slot[c * 32 + lane];
        const float4 dv = chirp[c * 32 + lane];
        v0[c] = cmul(make_float2(xv.x, xv.y), make_float2(dv.x, dv.y));
        v1[c] = cmul(make_float2(xv.z, xv.w), make_float2(dv.z, dv.w));
    }
    dft_dif<16>(v0);
    dft_dif<16>(v1);
}

// exchange write: unit (kc, lane ^ swz(kc)) holds (X_{2b}[a][kc], X_{2b+1}[a][kc])
LB_HD void w7_store(int lane, float4 *slot, const float2 *v0, const float2 *v1) {
#pragma unroll
    for (int kc = 0; kc < 16; kc++) {
        const int br = bitrev<16>(kc);
        slot[kc * 32 + (lane ^ w7_swz(kc))] = make_float4(v0[br].x, v0[br].y, v1[br].x, v1[br].y);
    }
}

// pass 1 for lane (kc, h): load branches 4h..4h+3, twiddle, 4 x radix-8, Horner over the 4 branches.
// P[ka] = sum_{i<4} wq[ka]^i * G_{4h+i}[kc + 16 ka];  Pq = the same with conj(wq) for the N/2 quirk bin.
LB_HD void w7_pass1(int lane, const float4 *slot, const W7Consts &c, float2 *P, float2 &Pq) {
    const int kc = lane >> 1, h = lane & 1;
    const int sw = w7_swz(kc);
    float2 g[4][8];
#pragma unroll
    for (int a = 0; a < 8; a++) {
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const float4 u = slot[kc * 32 + ((4 * a + 2 * h + e) ^ sw)];
            g[2 * e][a] = make_float2(u.x, u.y);
            g[2 * e + 1][a] = make_float2(u.z, u.w);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
#pragma unroll
        for (int a = 1; a < 8; a++) g[i][a] = cmul(g[i][a], c.tw1[a]);
        dft_dif<8>(g[i]);
    }
#pragma unroll
    for (int ka = 0; ka < 8; ka++) {
        const int br = bitrev<8>(ka);
        const float2 gv[4] = {g[0][br], g[1][br], g[2][br], g[3][br]};
        P[ka] = horner<4>(gv, c.wq[ka]);
    }
    Pq = make_float2(0.f, 0.f);
    if (kc == 0) {                                   // bin q = 64: tmp[N/2] += F[N/2] (:450)
        const int br = bitrev<8>(4);
        const float2 gv[4] = {g[0][br], g[1][br], g[2][br], g[3][br]};
        Pq = horner<4>(gv, cconj(c.wq[4]));
    }
}

// final: lane (kc, h) finishes ka = 4h + j, j = 0..3.  own[] = this lane's P for those ka,
// other[] = the partner's.  F = P_0 + wq^4 * P_1.
LB_HD unsigned long long w7_final(int lane, const W7Consts &c, const float2 *own, const float2 *other,
                                  float2 own_q, float2 other_q) {
    const int kc = lane >> 1, h = lane & 1;
    unsigned long long best = 0ull;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int ka = 4 * h + j;
        const float2 p0 = h ? other[j] : own[j];
        const float2 p1 = h ? own[j] : other[j];
        float2 f = cfma(p1, c.w4[j], p0);
        const int q = kc + 16 * ka;
        if (q == 64) {                               // only lane 1 (kc = 0, h = 1), j = 0
            const float2 q0 = h ? other_q : own_q, q1 = h ? own_q : other_q;
            f = cadd(f, cfma(q1, cconj(c.w4[j]), q0));
        }
        const unsigned long long key = pack_key(cnorm2(f), (uint32_t)q);   // tmp index == q for both halves
        best = key > best ? key : best;
    }
    return best;
}

#ifdef __CUDACC__
// the end of a symbol: lane h of each pair keeps ka = 4h..4h+3 of P and sends the other half to its partner, w7_final, and
// the warp's argmax key in every lane
LB_D unsigned long long w7_reduce(int lane, const W7Consts &c, const float2 *P, float2 Pq) {
    const int h = lane & 1;
    float2 own[4], other[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const float2 send = h ? P[j] : P[4 + j];
        own[j] = h ? P[4 + j] : P[j];
        other[j].x = __shfl_xor_sync(0xffffffffu, send.x, 1);
        other[j].y = __shfl_xor_sync(0xffffffffu, send.y, 1);
    }
    float2 other_q;
    other_q.x = __shfl_xor_sync(0xffffffffu, Pq.x, 1);
    other_q.y = __shfl_xor_sync(0xffffffffu, Pq.y, 1);
    return warp_max_key(w7_final(lane, c, own, other, Pq, other_q));
}

template <int NWARPS, int NSLOT>
struct W7Smem {
    float4 chirp[W7_SLOT_F4];
    float4 slots[NWARPS][NSLOT][W7_SLOT_F4];
    uint64_t bars[NWARPS][NSLOT];
};

template <int NWARPS, int NSLOT>
__global__ void __launch_bounds__(NWARPS * 32, 1)
k1_sf7_warp_kernel(K1Args a, uint32_t *__restrict__ bins, float *__restrict__ mags) {
    extern __shared__ __align__(128) unsigned char w7_raw[];
    W7Smem<NWARPS, NSLOT> &sm = *reinterpret_cast<W7Smem<NWARPS, NSLOT> *>(w7_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t gw = (size_t)blockIdx.x * NWARPS + warp, tw_total = (size_t)gridDim.x * NWARPS;

    const SymbolRing<float4, W7_SLOT_F4, NSLOT> ring{sm.slots[warp], sm.bars[warp], a.x, gw, tw_total, a.n_symbols};

    if (lane == 0) ring.init();
    for (int i = threadIdx.x; i < W7_SLOT_F4; i += NWARPS * 32) sm.chirp[i] = k1_ld_table4(a.chirp + 2 * i);
    __syncthreads();
    if (lane == 0) ring.fill();
    W7Consts c;
    w7_consts(lane, a.tw, c);

    uint32_t it = 0;
    for (size_t sym = gw; sym < a.n_symbols; sym += tw_total, it++) {
        float4 *slot = ring.wait(it);
        float2 v0[16], v1[16];
        w7_pass0(lane, slot, sm.chirp, v0, v1);
        __syncwarp();                                   // every lane has read the slot
        w7_store(lane, slot, v0, v1);
        __syncwarp();
        float2 P[8], Pq;
        w7_pass1(lane, slot, c, P, Pq);
        __syncwarp();                                   // exchange reads done: the slot can be refilled
        if (lane == 0) ring.refill(it, sym);
        const unsigned long long best = w7_reduce(lane, c, P, Pq);
        if (lane == 0) k1_store(bins, mags, sym, best);
    }
}
#endif  // __CUDACC__

// ---- CPU emulation (lanes run one after another; shuffles become array reads) ------------------
inline void w7_emulate(const K1Args &a, uint32_t *bins, float *mags) {
    float4 *slot = new float4[W7_SLOT_F4];
    float4 *chirp = new float4[W7_SLOT_F4];
    for (int i = 0; i < W7_SLOT_F4; i++) chirp[i] = make_float4(a.chirp[2 * i].x, a.chirp[2 * i].y, a.chirp[2 * i + 1].x, a.chirp[2 * i + 1].y);
    for (size_t sym = 0; sym < a.n_symbols; sym++) {
        const float2 *x = a.x + sym * W7_SPS;
        for (int i = 0; i < W7_SLOT_F4; i++) slot[i] = make_float4(x[2 * i].x, x[2 * i].y, x[2 * i + 1].x, x[2 * i + 1].y);
        float2 v0[32][16], v1[32][16];
        for (int l = 0; l < 32; l++) w7_pass0(l, slot, chirp, v0[l], v1[l]);
        for (int i = 0; i < W7_SLOT_F4; i++) slot[i] = make_float4(NAN, NAN, NAN, NAN);
        for (int l = 0; l < 32; l++) w7_store(l, slot, v0[l], v1[l]);
        float2 P[32][8], Pq[32];
        W7Consts c[32];
        for (int l = 0; l < 32; l++) { w7_consts(l, a.tw, c[l]); w7_pass1(l, slot, c[l], P[l], Pq[l]); }
        unsigned long long best = 0ull;
        for (int l = 0; l < 32; l++) {
            const int h = l & 1;
            float2 own[4], other[4];
            for (int j = 0; j < 4; j++) {
                own[j] = h ? P[l][4 + j] : P[l][j];
                other[j] = h ? P[l ^ 1][4 + j] : P[l ^ 1][j];      // what the partner sends: its half for MY ka range
            }
            const unsigned long long k = w7_final(l, c[l], own, other, Pq[l], Pq[l ^ 1]);
            best = k > best ? k : best;
        }
        k1_store(bins, mags, sym, best);
    }
    delete[] slot;
    delete[] chirp;
}

}  // namespace lb
