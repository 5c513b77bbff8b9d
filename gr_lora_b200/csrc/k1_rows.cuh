// k1_rows.cuh -- K1 (dechirp + pruned FFT + argmax, lib/decoder_impl.cc:430-464) for SF11 and SF12.
//
// What bounds the large spreading factors (measured in round 1 and re-derived from the microarchitecture notes): one
// symbol is 128 / 256 KiB, every organisation that moves intermediate data BETWEEN SMs pays for it -- the exchange through
// L2 triples the L2 traffic and the L2 slices deliver only about one HBM bandwidth in total (k1_xchg, k1_ab: <= 1/3),
// DSMEM moves ~20 B/clk per SM (k1_cluster, k1_big), and splitting the DFT by output residue re-reads the input.  This
// kernel keeps every sample of a symbol inside ONE SM from its TMA load to the argmax:
//
//   * the 8 polyphase branches (n = 8 n1 + r) are independent L-point FFTs (L = N = 2^SF).  SF11: one CTA per symbol, all 8
//     branches (8 x 2048 points = 128 KiB).  SF12: a cluster of two CTAs per symbol, CTA c takes branches 4c .. 4c+3 (4 x 4096
//     points = 128 KiB, the 32-byte halves of every 64-byte group of samples, fetched with a 2-D tensor-map TMA so that L2
//     delivers every sector once); the only data that crosses SMs is one partial sum per output bin (16 KiB per symbol
//     and direction, st.async into the peer's shared memory) -- 1/16 of the symbol; the receiving warp keeps its own
//     half in registers and completes the sums one symbol later.
//   * a symbol is 16 ROWS of 8 KiB (row j = n1 in [j L/16, (j+1) L/16), all local branches).  Rows live in a pool of
//     28 (SF12: 24) shared-memory slots of 8 KiB that rotates: global row g of this CTA's symbol sequence sits in slot g mod P.
//     16 slots hold the symbol being transformed, the others receive the next rows by TMA while it is; a slot is
//     re-armed by the warp that finished with it.  All three FFT passes are IN PLACE, so shared-memory traffic is
//     6 x 8 B per sample (TMA write, three read-modify passes): 48 B against the 128 B/clk crossbar = 0.8 of the HBM
//     roofline; there is no room (and no need) for a second copy of anything.
//   * the dechirp table (128 KiB per CTA) and the inter-pass twiddles do not fit in shared memory next to that; they are
//     read per symbol from global memory, where every CTA reads the same few hundred KiB, so they stay in L2.
//   * pass structure per symbol (512 threads = 16 warps, ONE CTA barrier per symbol):
//       pass 0  warp a1, lane (a0, p): float4 #(a, p) of each of the 16 rows -> dechirp -> two radix-16 DIFs over the rows
//               -> twiddle W_L^{a kc} -> written back to row kc (in place; 16-byte units XOR-swizzled by a1 & 7 inside
//               the warp's own 512-byte block, so no other warp's data is touched)                       __syncthreads
//       pass 1  warp kc, lane (a0, p): radix-16 over a1 inside row kc -> twiddle W_{L/16}^{a0 kb} -> in place    __syncwarp
//       pass 2  warp kc, lane (kb, h): radix-(L/256) over a0 for half of the local branches -> Horner over the branches with
//               W_sps^{k'} -> lane-pair exchange -> [SF12: partial sums to / from the peer CTA] -> |.|^2 -> argmax
//               -> the warp re-arms its slot with the row that maps to it P rows later.
//     bin k = kc + 16 kb + 256 q2.  Same arithmetic as get_shift_fft including tmp[N/2] += F[N/2] and the first-maximum
//     tie break; bins are bit-equal to the oracle's on the parity inputs, magnitudes within fp32 rounding.
// The index arithmetic and the butterflies are __host__ __device__ (r_emulate below runs them on the CPU for the
// non-GPU tests, with shared memory and the peer exchange modelled as plain arrays).
#pragma once
#include "k1_ring.cuh"
#ifdef __CUDACC__
#include <cuda.h>      // CUtensorMap (type only; the encoder is fetched through cudaGetDriverEntryPoint)
#endif

namespace lb {

template <int SF>
struct RCfg {
    static constexpr int N = 1 << SF, SPS = 8 * N, L = N;
    static constexpr int CL = SF == 12 ? 2 : 1;          // CTAs per symbol
    static constexpr int NB = 8 / CL;                    // branches per CTA
    static constexpr int A = L / 16;                     // n1 values per row: 128 / 256
    static constexpr int A0 = L / 256;                   // points of the last pass: 8 / 16
    static constexpr int CPA = NB / 2;                   // 16-byte units (branch pairs) per n1: 4 / 2
    static constexpr int ROW_F4 = A * CPA;               // 512 float4 = 8 KiB
    static constexpr uint32_t ROW_BYTES = 8192u;
    static constexpr int NSLOT = SF == 12 ? 24 : 28;     // slot pool, a multiple of 4 rows (SF12 gives 16 KiB to the peer-exchange buffer)
    static constexpr int T = 512, NW = 16;
    static constexpr int HB = NB / 2;                    // branches per lane in pass 2: 4 / 2
    static_assert(SF == 11 || SF == 12, "rows kernel: SF11, SF12");
    static_assert(A0 * CPA == 32, "one warp = one a1 block of every row");
};

constexpr int R_NSYM_BAR = 4;                            // symbol barriers in rotation (<= 2.75 symbols in flight)
// Rows of the next symbol that have to wait for slots of the current one are always its LAST ones (NSLOT - 16 rows are
// prefetched into free slots).  They get their own barrier: pass 0 loads and dechirps the early rows first and only then
// waits for the late ones (second capture: 8.8 % of all samples sat in the single wait at the top of the loop).
template <int SF> struct RLate { static constexpr int EARLY = RCfg<SF>::NSLOT - 16; };      // 12 (SF11) / 8 (SF12) early rows

// ---- index arithmetic --------------------------------------------------------------------------------------------------
template <int SF> LB_HD int r_a0(int lane) { return lane / RCfg<SF>::CPA; }
template <int SF> LB_HD int r_p(int lane) { return lane % RCfg<SF>::CPA; }
// sample index of the first of the two samples (branches 2p, 2p+1 of this CTA) a pass-0 thread reads from row j
template <int SF> LB_HD int r_sample(int rank, int warp, int lane, int j) {
    using C = RCfg<SF>;
    const int a = warp * C::A0 + r_a0<SF>(lane);
    return 8 * (j * C::A + a) + rank * C::NB + 2 * r_p<SF>(lane);
}
// Swizzle of the 16-byte units inside a 512-byte block.  128-bit shared-memory accesses are served a quarter warp (8 lanes)
// at a time; in pass 2 those 8 lanes are 4 consecutive blocks x the lane pair h, and h toggles unit bit 1 (SF11) / bit 0
// (SF12), so the block number must toggle the other two of the low three bits.  (The first version XORed block & 7: two
// lanes of every quarter met in one bank group, ncu: 2x the ideal wavefronts on the pass-2 loads.)
template <int SF> LB_HD int r_swz(int block) { return SF == 11 ? ((block & 1) | ((block & 2) << 1)) : ((block & 3) << 1); }
template <int SF> LB_HD int r_unit(int block, int within) { return block * 32 + (within ^ r_swz<SF>(block)); }   // float4 index in a row
// exponent (mod sps) of the per-q2 factor of W_sps^{e k'}: k' = kc + 16 kb + 256 q2 - (q2 >= A0/2 ? L : 0)
template <int SF> LB_HD int r_cq_exp(int e, int q2) {
    using C = RCfg<SF>;
    const int d = 256 * q2 - (q2 >= C::A0 / 2 ? C::L : 0);
    return (e * d) & (C::SPS - 1);
}

struct RConsts {            // per-q2 factors, [e index][q2]; SF11: e = 1, 4; SF12: e = 1, 2, 4, 6
    float2 cq[4][16];
};
template <int SF> LB_HD int r_e_of(int i) { return SF == 11 ? (i == 0 ? 1 : 4) : (i == 0 ? 1 : 2 * i); }
template <int SF>
inline void r_build_consts(const float2 *tw_host, RConsts &c) {
    for (int i = 0; i < 4; i++)
        for (int q2 = 0; q2 < 16; q2++) c.cq[i][q2] = tw_host[r_cq_exp<SF>(r_e_of<SF>(i), q2 % RCfg<SF>::A0)];
}

// ---- pass 0 / pass 1 arithmetic on registers -----------------------------------------------------------------------------
// v0 / v1: the two branches of the thread's float4 column, 16 points each; tw[kc - 1] the output twiddles
LB_HD void r_dif16(float2 *v0, float2 *v1) {
    dft_dif<16>(v0);
    dft_dif<16>(v1);
}
LB_HD void r_twiddle16(float2 *v0, float2 *v1, const float2 *tw) {
#pragma unroll
    for (int k = 1; k < 16; k++) {
        const int br = bitrev<16>(k);
        v0[br] = cmul(v0[br], tw[k - 1]);
        v1[br] = cmul(v1[br], tw[k - 1]);
    }
}

// ---- pass 2 arithmetic ----------------------------------------------------------------------------------------------------
// g[b][.]: A0 points of local branch (HB h + b); after r_pass2_dft g[b][bitrev(q2)] = G_r[kc + 16 kb + 256 q2].
// r_pass2_term returns this lane's share t(q2) of the sum over the branches, already multiplied by the power of w that places
// it:  t(q2) = w^{E} * sum_b w^b g[b][q2],  E = global index of the lane's first branch,  w = W_sps^{k'(q2)}.
// wb1 = W_sps^{kc + 16 kb}, wbE = W_sps^{E (kc + 16 kb)};  cq1 / cqE the per-q2 factors (RConsts rows).
template <int SF>
LB_HD void r_pass2_dft(float2 (*g)[RCfg<SF>::A0]) {
#pragma unroll
    for (int b = 0; b < RCfg<SF>::HB; b++) dft_dif<RCfg<SF>::A0>(g[b]);
}
template <int SF>
LB_HD float2 r_pass2_term(float2 (*g)[RCfg<SF>::A0], int q2, int E, float2 wb1, float2 wbE, const float2 *cq1, const float2 *cqE) {
    using C = RCfg<SF>;
    const int br = bitrev<C::A0>(q2);
    const float2 w = cmul(wb1, cq1[q2]);
    float2 acc = g[C::HB - 1][br];
#pragma unroll
    for (int b = C::HB - 2; b >= 0; b--) acc = cfma(acc, w, g[b][br]);
    return E ? cmul(acc, cmul(wbE, cqE[q2])) : acc;
}
// the second evaluation of bin N/2 (tmp[N/2] += F[N/2], :450): same G values, conjugate twiddles (W_sps^{+N/2 r})
template <int SF>
LB_HD float2 r_pass2_quirk(float2 (*g)[RCfg<SF>::A0], int E, float2 wb1, float2 wbE, const float2 *cq1, const float2 *cqE) {
    using C = RCfg<SF>;
    const int q2 = C::A0 / 2, br = bitrev<C::A0>(q2);
    const float2 w = cconj(cmul(wb1, cq1[q2]));
    float2 acc = g[C::HB - 1][br];
#pragma unroll
    for (int b = C::HB - 2; b >= 0; b--) acc = cfma(acc, w, g[b][br]);
    return E ? cmul(acc, cconj(cmul(wbE, cqE[q2]))) : acc;
}

#ifdef __CUDACC__
LB_D float4 lds128(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}
LB_D void sts128(uint32_t addr, float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ---- cluster helpers (SF12) -----------------------------------------------------------------------------------------------
LB_D uint32_t cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
LB_D uint32_t map_to_peer(uint32_t local_smem_addr, uint32_t peer) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(peer));
    return r;
}
LB_D void mbar_arrive_peer_relaxed(uint32_t peer_bar_addr) {
    asm volatile("mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%0];" ::"r"(peer_bar_addr) : "memory");
}
// 16 bytes from registers into the peer CTA's shared memory through the async proxy; counted on the PEER's mbarrier
LB_D void st_async_peer_f4(uint32_t peer_dst, float4 v, uint32_t peer_bar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];"
                 ::"r"(peer_dst), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"(peer_bar) : "memory");
}
LB_D void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// 2-D tensor-map TMA: box {8 floats (the CTA's 4 branches of one n1), 256 n1} -> 8 KiB, dense in shared memory
LB_D void tma_rows_2d(void *dst_smem, const void *tmap, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst_smem)), "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

// Diagnosis build (-DLB_ROWS_TIMING, tools only): cycles every warp spends in each kind of wait, read back by the launcher.
#ifdef LB_ROWS_TIMING
__device__ unsigned int r_timing_dev[160 * 16 * 8];
#define RT_DECL unsigned int rt_acc[6] = {0, 0, 0, 0, 0, 0}; const unsigned int rt_start = (unsigned int)clock();
#define RT(i, stmt) do { const unsigned int rt_t0 = (unsigned int)clock(); stmt; rt_acc[i] += (unsigned int)clock() - rt_t0; } while (0)
#define RT_FLUSH do { if (lane == 0) { unsigned int *o = r_timing_dev + (blockIdx.x * 16 + warp) * 8; for (int i = 0; i < 6; i++) o[i] = rt_acc[i]; \
                                    o[6] = (unsigned int)clock() - rt_start; o[7] = (unsigned int)n_mine; } } while (0)
#else
#define RT_DECL
#define RT(i, stmt) stmt
#define RT_FLUSH
#endif

template <int SF>
struct RSmem {
    float4 slots[RCfg<SF>::NSLOT][RCfg<SF>::ROW_F4];
    // SF12 only: the peer's partial sums of the bins THIS CTA finishes, written by the peer's st.async.  Two buffers (symbol
    // parity) of one 2 KiB block per warp pair, a block = 128 float4 = [i][lane] (i = 0..3: the lane's bins 2i, 2i+1), lane-major
    // inside each i so that the 128-bit reads of a quarter warp fall into 8 different bank groups
    float2 recv[RCfg<SF>::CL == 2 ? 2 * 8 * 256 : 2];
    unsigned long long keys[2][RCfg<SF>::NW];
    uint64_t sym_full[R_NSYM_BAR];                        // early rows of a symbol
    uint64_t sym_late[R_NSYM_BAR];                        // its last 16 - EARLY rows
    uint64_t x_full[16], x_free[16];                      // SF12: per buffer and receiving / sending warp pair, index 8 b + i
};

struct alignas(64) RParams {
    CUtensorMap tmap;                  // SF12: 2-D view of the IQ batch {16 floats per n1, n_symbols * L}, box {8, 256}
    K1Args a;
    unsigned long long *packed;        // SF12: per-symbol argmax keys merged by atomicMax (finalised by k1_finalize_kernel)
    uint32_t *bins;                    // SF11: written directly
    float *mags;
};

static __device__ __constant__ RConsts r_consts_dev[2];          // [SF - 11]

template <int SF>
__global__ void __launch_bounds__(RCfg<SF>::T, 1)
k1_rows_kernel(const __grid_constant__ RParams P) {
    using C = RCfg<SF>;
    extern __shared__ __align__(1024) unsigned char r_raw[];
    RSmem<SF> &sm = *reinterpret_cast<RSmem<SF> *>(r_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t rank = C::CL == 2 ? cluster_rank() : 0u, peer = rank ^ 1u;
    const size_t unit = blockIdx.x / C::CL, n_units = gridDim.x / C::CL;        // symbol sequence of this CTA (cluster)
    const K1Args &a = P.a;
    const size_t n_mine = unit < a.n_symbols ? (a.n_symbols - unit + n_units - 1) / n_units : 0;
    const RConsts &rc = r_consts_dev[SF - 11];

    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < R_NSYM_BAR; i++) { mbar_init(&sm.sym_full[i], RLate<SF>::EARLY); mbar_init(&sm.sym_late[i], 16 - RLate<SF>::EARLY); }
#pragma unroll
        for (int i = 0; i < 16; i++) { mbar_init(&sm.x_full[i], 1); mbar_init(&sm.x_free[i], 32); }     // full: one expect_tx + the stores' bytes; free: every lane
        if (C::CL == 2 && n_mine > 0)
#pragma unroll
            for (int i = 0; i < 16; i++)
                if (i < 8 || n_mine > 1) mbar_expect_tx(&sm.x_full[i], 2048u);          // phase 0 of the receive barriers (symbols 0 and 1)
        fence_mbar_init();
    }
    // issue of global row g of this CTA's sequence (symbol g / 16, row g % 16) into slot g % NSLOT
    auto issue_row = [&](size_t g) {
        const size_t s = g >> 4;
        if (s >= n_mine) return;
        const int j = (int)(g & 15);
        const size_t sym = unit + s * n_units;
        uint64_t *bar = j < RLate<SF>::EARLY ? &sm.sym_full[s % R_NSYM_BAR] : &sm.sym_late[s % R_NSYM_BAR];
        float4 *dst = sm.slots[g % C::NSLOT];
        mbar_expect_tx(bar, C::ROW_BYTES);
        if (C::CL == 1) bulk_g2s(dst, a.x + sym * C::SPS + (size_t)j * (C::SPS / 16), C::ROW_BYTES, bar);
        else tma_rows_2d(dst, &P.tmap, (int)(rank * 8u), (int)(sym * C::L + (size_t)j * C::A), bar);
    };
    if (tid == 0)
        for (int g = 0; g < C::NSLOT; g++) issue_row((size_t)g);

    // thread-invariant table offsets: pass-0 twiddles W_L^{a kc} = W_sps^{8 a kc}, pass-1 twiddles W_{L/16}^{a0 kb} = W_sps^{128 a0 kb}
    const int tw0_step = 8 * (warp * C::A0 + r_a0<SF>(lane)), tw1_step = 128 * r_a0<SF>(lane);
    // pass-2 lane constants: kc = warp, kb = lane >> 1, h = lane & 1; E = global index of the lane's first branch
    const int kb2 = lane >> 1, h2 = lane & 1;
    const int E2 = (int)rank * C::NB + h2 * C::HB;
    const int e_idx = SF == 11 ? (E2 ? 1 : 0) : (E2 >> 1);            // row of RConsts::cq for w^E (unused when E == 0)
    const float2 wb1 = k1_ld_table(a.tw + ((warp + 16 * kb2) & (C::SPS - 1)));
    const float2 wbE = k1_ld_table(a.tw + ((E2 * (warp + 16 * kb2)) & (C::SPS - 1)));
    if (C::CL == 2) cluster_sync_all(); else __syncthreads();     // barriers are initialised (the peer's too)

    // ---- shared-memory addressing (32-bit shared addresses; every per-access term below is an immediate) -------------------
    // rows of the current symbol sit in slots (base + j) mod NSLOT, base = 16 s mod NSLOT; NSLOT and 16 are multiples of 4, so
    // the four rows of a group 4q .. 4q+3 are consecutive slots: one byte offset per group and symbol
    const uint32_t slots0 = smem_u32(&sm.slots[0][0]);
    const uint32_t ld0 = slots0 + (uint32_t)(warp * 32 + lane) * 16u;                     // pass-0 loads: natural order
    const uint32_t st0 = slots0 + (uint32_t)r_unit<SF>(warp, lane) * 16u;                 // pass-0 stores: swizzled
    uint32_t lane_sw[4];                                                                   // pass 1: (lane ^ swizzle) * 16, 4 swizzle values
#pragma unroll
    for (int c = 0; c < 4; c++) lane_sw[c] = (uint32_t)(lane ^ r_swz<SF>(c)) * 16u;
    // pass 2: unit = K ^ m with K = (a0, e) a compile-time number and m = (the lane pair's bit) ^ swizzle(kb) a lane constant;
    // only the low three unit bits meet m, so 4 XORed addresses per symbol cover all 16 loads
    const uint32_t m2 = (uint32_t)((SF == 11 ? 2 * (lane & 1) : (lane & 1)) ^ r_swz<SF>(lane >> 1)) * 16u + (uint32_t)(lane >> 1) * 512u;
    RT_DECL
    // SF12 exchange roles: warp pair x_i; this CTA finishes the bins of rows kc with (kc >> 3) == rank
    const int x_i = warp & 7;
    const bool x_mine = C::CL == 2 && (uint32_t)(warp >> 3) == rank;
    float2 stash[8];                               // SF12 receiver warps: own partial sums of the previous symbol
    auto finalize_prev = [&](size_t sp) {          // receiver warps: own sums (stash) + the peer's (recv) of symbol sp -> argmax
        const int xb = (int)(sp & 1) * 8 + x_i;
        RT(0, mbar_wait(&sm.x_full[xb], (uint32_t)((sp >> 1) & 1)));
        const float2 *o = stash;
        const float4 *rblk = reinterpret_cast<const float4 *>(&sm.recv[xb * 256]);
        float4 u[4];
#pragma unroll
        for (int i = 0; i < 4; i++) u[i] = rblk[i * 32 + lane];
        uint32_t dep = 0;
        unsigned long long bk = 0ull;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const float2 fa = cadd(o[2 * i], make_float2(u[i].x, u[i].y));
            const float2 fb = cadd(o[2 * i + 1], make_float2(u[i].z, u[i].w));
            dep |= __float_as_uint(u[i].w);
            const int q0 = 2 * i + (lane & 1) * (C::A0 / 2);
            const unsigned long long ka = pack_key(cnorm2(fa), (uint32_t)(warp + 16 * (lane >> 1) + 256 * q0));
            const unsigned long long kb = pack_key(cnorm2(fb), (uint32_t)(warp + 16 * (lane >> 1) + 256 * (q0 + 1)));
            bk = ka > bk ? ka : bk;
            bk = kb > bk ? kb : bk;
        }
        bk = warp_max_key(bk);
        if (lane == 0) {
            atomicMax(P.packed + unit + sp * n_units, bk);
            if (sp + 2 < n_mine) mbar_expect_tx(&sm.x_full[xb], 2048u);     // arm the buffer's next phase (this one has completed)
        }
        // tell the peer the block has been read: the arrive carries no data (relaxed), but it must not be issued before this
        // lane's loads have returned, so its address depends on them
        asm volatile("and.b32 %0, %0, 0;" : "+r"(dep));
        mbar_arrive_peer_relaxed(map_to_peer(smem_u32(&sm.x_free[xb]), peer) + dep);
    };
    int base = 0;
    for (size_t s = 0; s < n_mine; s++, base = base + 16 >= C::NSLOT ? base + 16 - C::NSLOT : base + 16) {
        const size_t g0 = s * 16;
        uint32_t gb[4];
        {
            int t = base;
#pragma unroll
            for (int q = 0; q < 4; q++) { gb[q] = (uint32_t)t * C::ROW_BYTES; t += 4; if (t >= C::NSLOT) t -= C::NSLOT; }
        }
        uint32_t rowaddr;
        { int t = base + warp; if (t >= C::NSLOT) t -= C::NSLOT; rowaddr = slots0 + (uint32_t)t * C::ROW_BYTES; }
        RT(2, mbar_wait(&sm.sym_full[s % R_NSYM_BAR], (uint32_t)((s / R_NSYM_BAR) & 1)));

        // ---- pass 0: radix 16 over the rows, warp = a1 block -----------------------------------------------------------
        {
            float2 v0[16], v1[16], tw[16];
#pragma unroll
            for (int q = 0; q < 4; q++) {
                if (4 * q == RLate<SF>::EARLY) RT(3, mbar_wait(&sm.sym_late[s % R_NSYM_BAR], (uint32_t)((s / R_NSYM_BAR) & 1)));
                float4 ch[4];
#pragma unroll
                for (int jj = 0; jj < 4; jj++) ch[jj] = k1_ld_table4(a.chirp + r_sample<SF>((int)rank, warp, lane, 4 * q + jj));
                float4 xv[4];
                const uint32_t ga = ld0 + gb[q];
#pragma unroll
                for (int jj = 0; jj < 4; jj++) xv[jj] = lds128(ga + (uint32_t)jj * C::ROW_BYTES);
#pragma unroll
                for (int jj = 0; jj < 4; jj++) {
                    v0[4 * q + jj] = cmul(make_float2(xv[jj].x, xv[jj].y), make_float2(ch[jj].x, ch[jj].y));
                    v1[4 * q + jj] = cmul(make_float2(xv[jj].z, xv[jj].w), make_float2(ch[jj].z, ch[jj].w));
                }
            }
            r_dif16(v0, v1);
#pragma unroll
            for (int kc = 1; kc < 16; kc++) tw[kc - 1] = k1_ld_table(a.tw + ((tw0_step * kc) & (C::SPS - 1)));
            r_twiddle16(v0, v1, tw);
            __syncwarp();      // the loads read the TMA's linear layout, the stores write the swizzled one: inside the warp's own
                               // block, but lanes swap units -- every lane's loads before any lane's stores
#pragma unroll
            for (int kc = 0; kc < 16; kc++) {
                const int br = bitrev<16>(kc);
                sts128(st0 + gb[kc >> 2] + (uint32_t)(kc & 3) * C::ROW_BYTES, make_float4(v0[br].x, v0[br].y, v1[br].x, v1[br].y));
            }
        }
        RT(4, __syncthreads());
        // result of the previous symbol (its keys were complete before this barrier)
        if (C::CL == 1 && s > 0 && warp == 0) {
            unsigned long long k = lane < C::NW ? sm.keys[(s - 1) & 1][lane] : 0ull;
            k = warp_max_key(k);      // lanes >= NW hold 0
            if (lane == 0) {
                const size_t psym = unit + (s - 1) * n_units;
                if (C::CL == 2) atomicMax(P.packed + psym, k);
                else { P.bins[psym] = key_idx(k); if (P.mags) P.mags[psym] = sqrtf(key_mag2(k)); }
            }
        }
        // ---- pass 1: radix 16 over a1 inside row kc = warp -------------------------------------------------------------
        {
            float2 v0[16], v1[16], tw[16];
            uint32_t ra[4];
#pragma unroll
            for (int c = 0; c < 4; c++) ra[c] = rowaddr + lane_sw[c];
#pragma unroll
            for (int a1 = 0; a1 < 16; a1++) {
                const float4 u = lds128(ra[a1 & 3] + (uint32_t)a1 * 512u);
                v0[a1] = make_float2(u.x, u.y);
                v1[a1] = make_float2(u.z, u.w);
            }
            r_dif16(v0, v1);
#pragma unroll
            for (int kb = 1; kb < 16; kb++) tw[kb - 1] = k1_ld_table(a.tw + ((tw1_step * kb) & (C::SPS - 1)));
            r_twiddle16(v0, v1, tw);
#pragma unroll
            for (int kb = 0; kb < 16; kb++) {
                const int br = bitrev<16>(kb);
                sts128(ra[kb & 3] + (uint32_t)kb * 512u, make_float4(v0[br].x, v0[br].y, v1[br].x, v1[br].y));
            }
        }
        __syncwarp();
        // ---- pass 2: radix A0 over a0, branch sum, argmax ---------------------------------------------------------------
        // SF12: the sums of the PREVIOUS symbol are completed first (the peer's half has had a symbol time to arrive).
        // Measured alternatives (tools/k1_ab.py, LB_ROWS_TIMING build): merging the same symbol's sums at the end of pass 2
        // 0.43 (9 % of samples in the wait); this 0.46 although the receivers still wait ~4 300 of 12 750 cycles for the 128
        // remote st.async transactions of a block; one cp.async.bulk per block instead (no wait, but 32 KiB for send + receive
        // buffers) 0.42; this merge moved behind the pass-2 arithmetic 0.41.  The last two remove the wait and lose: with it the
        // receiving half of the warps runs a third of a symbol behind the sending half, so the TMA refills and the FMA-heavy
        // and LSU-heavy phases of the two halves interleave instead of colliding; what bounds SF12 is the refill of the last 8
        // rows (sym_late: 2 100 - 3 300 cycles per symbol in every variant), i.e. 24 slots = 1.5 symbols of shared memory.
        if (C::CL == 2 && x_mine && s > 0) finalize_prev(s - 1);
        unsigned long long best = 0ull;
        {
            float2 g[C::HB][C::A0];
            {
                const uint32_t qm = rowaddr + m2;
                uint32_t pa[4];
                if (SF == 11) {
                    // K = a0 * 4 + e: unit bits 0 (e) and 2 (a0 & 1) meet m; (a0 >> 1) * 128 bytes stays an immediate
#pragma unroll
                    for (int c = 0; c < 4; c++) pa[c] = qm ^ (uint32_t)(((c >> 1) * 4 + (c & 1)) * 16);
#pragma unroll
                    for (int a0 = 0; a0 < C::A0; a0++)
#pragma unroll
                        for (int e = 0; e < 2; e++) {
                            const float4 u = lds128(pa[(a0 & 1) * 2 + e] + (uint32_t)(a0 >> 1) * 128u);
                            g[2 * e][a0] = make_float2(u.x, u.y);
                            g[(2 * e + 1) % C::HB][a0] = make_float2(u.z, u.w);
                        }
                } else {
                    // K = a0 * 2: unit bits 1, 2 (a0 & 3) meet m; (a0 >> 2) * 128 bytes stays an immediate
#pragma unroll
                    for (int c = 0; c < 4; c++) pa[c] = qm ^ (uint32_t)(c * 2 * 16);
#pragma unroll
                    for (int a0 = 0; a0 < C::A0; a0++) {
                        const float4 u = lds128(pa[a0 & 3] + (uint32_t)(a0 >> 2) * 128u);
                        g[0][a0] = make_float2(u.x, u.y);
                        g[C::HB - 1][a0] = make_float2(u.z, u.w);
                    }
                }
            }
            r_pass2_dft<SF>(g);
            // the row has been read (the DFT above consumed every loaded register of this lane, the warp barrier covers the
            // others): re-arm its slot NOW, so that the TMA of the row that lands here NSLOT rows later runs under the rest
            // of pass 2 -- the rows of the next symbol that wait for slots of this one are its last ones, and their
            // latency would otherwise be exposed at the top of the loop (first capture: 15 % of all samples there)
            __syncwarp();
            if (lane == 0) {
                fence_proxy_async();
                issue_row(g0 + (size_t)warp + (size_t)C::NSLOT);
            }
            // the products of the lane's twiddle bases with the per-q2 constants are loop invariant; hoisted out of the
            // symbol loop they would occupy (and spill) 64 registers, so the bases are made opaque here
            float2 wb1s = wb1, wbEs = wbE;
            asm volatile("" : "+f"(wb1s.x), "+f"(wb1s.y), "+f"(wbEs.x), "+f"(wbEs.y));
            const bool quirk_warp = warp == 0;                       // bin N/2 = (kc 0, kb 0, q2 A0/2): lanes 0 and 1 of warp 0
            float2 tq = make_float2(0.f, 0.f);
            if (quirk_warp && kb2 == 0) tq = r_pass2_quirk<SF>(g, E2, wb1s, wbEs, rc.cq[0], rc.cq[e_idx]);
            // lane pair: h = 0 keeps q2 < A0/2, h = 1 keeps q2 >= A0/2; each sends the other half
            float2 f[C::A0 / 2];
#pragma unroll
            for (int i = 0; i < C::A0 / 2; i++) {
                const float2 tlo = r_pass2_term<SF>(g, i, E2, wb1s, wbEs, rc.cq[0], rc.cq[e_idx]);
                const float2 thi = r_pass2_term<SF>(g, i + C::A0 / 2, E2, wb1s, wbEs, rc.cq[0], rc.cq[e_idx]);
                const float2 give = h2 ? tlo : thi;
                const float2 keep = h2 ? thi : tlo;
                float2 got;
                got.x = __shfl_xor_sync(0xffffffffu, give.x, 1);
                got.y = __shfl_xor_sync(0xffffffffu, give.y, 1);
                f[i] = cadd(keep, got);
            }
            if (quirk_warp) {                                          // both halves of the conjugate evaluation end up in lane 1
                float2 got;
                got.x = __shfl_xor_sync(0xffffffffu, tq.x, 1);
                got.y = __shfl_xor_sync(0xffffffffu, tq.y, 1);
                tq = cadd(tq, got);
            }
            if (C::CL == 2) {
                // bins of rows kc < 8 are finished by CTA 0, kc >= 8 by CTA 1.  The other CTA sends its partial sums straight
                // from registers through the async proxy (st.async ... mbarrier::complete_tx on the peer's barrier): no staging
                // buffer (its 16 KiB are the second receive buffer), no cluster-scope fence or acquire (the first version's
                // DSMEM stores + fence.acq_rel.cluster + try_wait.acquire.cluster compiled to MEMBAR.ALL.GPU + ERRBAR +
                // CCTL.IVALL: 30 % of all stall samples).  The 128 remote transactions per block take ~4 000 cycles to land
                // (LB_ROWS_TIMING build), which the one-symbol deferral of the merge hides.
                if (quirk_warp && lane == 1) f[0] = cadd(f[0], tq);      // both evaluations of bin N/2 are additive
                if (!x_mine) {
                    const int xb = (int)(s & 1) * 8 + x_i;
                    if (s > 1) RT(1, mbar_wait(&sm.x_free[xb], (uint32_t)(((s >> 1) - 1) & 1)));     // the peer has consumed symbol s - 2 (a symbol time ago)
                    const uint32_t dst = map_to_peer(smem_u32(&sm.recv[xb * 256]), peer) + (uint32_t)lane * 16u;
                    const uint32_t bar = map_to_peer(smem_u32(&sm.x_full[xb]), peer);
#pragma unroll
                    for (int i = 0; i < 4; i++) st_async_peer_f4(dst + (uint32_t)i * 512u, make_float4(f[2 * i].x, f[2 * i].y, f[2 * i + 1].x, f[2 * i + 1].y), bar);
                } else {
                    // own half: kept until the next pass 2 (finalize_prev)
#pragma unroll
                    for (int i = 0; i < 8; i++) stash[i] = f[i];
                }
            } else {
                if (quirk_warp && lane == 1) f[0] = cadd(f[0], tq);
#pragma unroll
                for (int i = 0; i < C::A0 / 2; i++) {
                    const int q2 = i + h2 * (C::A0 / 2);
                    const unsigned long long key = pack_key(cnorm2(f[i]), (uint32_t)(warp + 16 * kb2 + 256 * q2));
                    best = key > best ? key : best;
                }
            }
        }
        best = warp_max_key(best);
        if (C::CL == 1 && lane == 0) sm.keys[s & 1][warp] = best;
    }
    if (C::CL == 2 && x_mine && n_mine > 0) finalize_prev(n_mine - 1);
    RT_FLUSH;
    __syncthreads();
    if (C::CL == 1 && n_mine > 0 && warp == 0) {
        unsigned long long k = lane < C::NW ? sm.keys[(n_mine - 1) & 1][lane] : 0ull;
        k = warp_max_key(k);      // lanes >= NW hold 0
        if (lane == 0) {
            const size_t psym = unit + (n_mine - 1) * n_units;
            if (C::CL == 2) atomicMax(P.packed + psym, k);
            else { P.bins[psym] = key_idx(k); if (P.mags) P.mags[psym] = sqrtf(key_mag2(k)); }
        }
    }
    if (C::CL == 2) cluster_sync_all();           // no CTA of the pair exits while the other may still store into it
}
#endif  // __CUDACC__

// ---- CPU emulation of the same index arithmetic (tests/test_host_emulation.py) ---------------------------------------------------
// Shared memory slots and the peer exchange are plain arrays; the threads of a pass run one after
// the other (legal: a pass only reads what the previous barrier made visible, and its in-place writes stay inside the
// thread's own units -- the emulation asserts that by poisoning).
template <int SF>
inline void r_emulate(const K1Args &a, uint32_t *bins, float *mags) {
    using C = RCfg<SF>;
    RConsts rc;
    r_build_consts<SF>(a.tw, rc);
    const int NSL = C::NSLOT;
    float4 *slots[2];
    float2 *part[2];
    for (int c = 0; c < C::CL; c++) { slots[c] = new float4[(size_t)NSL * C::ROW_F4]; part[c] = new float2[C::L + 1]; }
    unsigned long long *keys = new unsigned long long[C::CL * C::NW];
    for (size_t s = 0; s < a.n_symbols; s++) {
        const float2 *x = a.x + s * C::SPS;
        const size_t g0 = s * 16;
        for (int c = 0; c < C::CL; c++) {
            float4 *sl = slots[c];
            auto slot = [&](size_t g) { return sl + (g % NSL) * C::ROW_F4; };
            for (int j = 0; j < 16; j++)                         // TMA: row j, natural order
                for (int aa = 0; aa < C::A; aa++)
                    for (int p = 0; p < C::CPA; p++) {
                        const int n = 8 * (j * C::A + aa) + c * C::NB + 2 * p;
                        slot(g0 + j)[aa * C::CPA + p] = make_float4(x[n].x, x[n].y, x[n + 1].x, x[n + 1].y);
                    }
            for (int warp = 0; warp < C::NW; warp++) {           // pass 0 (a warp's reads all precede its writes)
                float2 v0[32][16], v1[32][16];
                for (int lane = 0; lane < 32; lane++) {
                    float2 tw[16];
                    const int a_idx = warp * C::A0 + r_a0<SF>(lane);
                    for (int kc = 1; kc < 16; kc++) tw[kc - 1] = a.tw[(8 * a_idx * kc) & (C::SPS - 1)];
                    for (int j = 0; j < 16; j++) {
                        const float4 xv = slot(g0 + j)[warp * 32 + lane];
                        const int n = r_sample<SF>(c, warp, lane, j);
                        v0[lane][j] = cmul(make_float2(xv.x, xv.y), a.chirp[n]);
                        v1[lane][j] = cmul(make_float2(xv.z, xv.w), a.chirp[n + 1]);
                    }
                    r_dif16(v0[lane], v1[lane]);
                    r_twiddle16(v0[lane], v1[lane], tw);
                }
                for (int lane = 0; lane < 32; lane++)
                    for (int kc = 0; kc < 16; kc++) {
                        const int br = bitrev<16>(kc);
                        slot(g0 + kc)[r_unit<SF>(warp, lane)] = make_float4(v0[lane][br].x, v0[lane][br].y, v1[lane][br].x, v1[lane][br].y);
                    }
            }
            for (int warp = 0; warp < C::NW; warp++) {           // pass 1 + pass 2 of row kc = warp
                float4 *row = slot(g0 + warp);
                float2 v0[32][16], v1[32][16];
                for (int lane = 0; lane < 32; lane++) {
                    float2 tw[16];
                    for (int kb = 1; kb < 16; kb++) tw[kb - 1] = a.tw[(128 * r_a0<SF>(lane) * kb) & (C::SPS - 1)];
                    for (int a1 = 0; a1 < 16; a1++) {
                        const float4 u = row[r_unit<SF>(a1, lane)];
                        v0[lane][a1] = make_float2(u.x, u.y);
                        v1[lane][a1] = make_float2(u.z, u.w);
                    }
                    r_dif16(v0[lane], v1[lane]);
                    r_twiddle16(v0[lane], v1[lane], tw);
                }
                for (int lane = 0; lane < 32; lane++)
                    for (int kb = 0; kb < 16; kb++) {
                        const int br = bitrev<16>(kb);
                        row[r_unit<SF>(kb, lane)] = make_float4(v0[lane][br].x, v0[lane][br].y, v1[lane][br].x, v1[lane][br].y);
                    }
                float2 t[32][C::A0], tq[32];
                for (int lane = 0; lane < 32; lane++) {
                    const int kb2 = lane >> 1, h2 = lane & 1;
                    const int E2 = c * C::NB + h2 * C::HB;
                    const int e_idx = SF == 11 ? (E2 ? 1 : 0) : (E2 >> 1);
                    const float2 wb1 = a.tw[(warp + 16 * kb2) & (C::SPS - 1)];
                    const float2 wbE = a.tw[(E2 * (warp + 16 * kb2)) & (C::SPS - 1)];
                    float2 g[C::HB][C::A0];
                    for (int a0 = 0; a0 < C::A0; a0++) {
                        if (SF == 11) {
                            for (int e = 0; e < 2; e++) {
                                const float4 u = row[r_unit<SF>(kb2, a0 * 4 + 2 * h2 + e)];
                                g[2 * e][a0] = make_float2(u.x, u.y);
                                g[(2 * e + 1) % C::HB][a0] = make_float2(u.z, u.w);
                            }
                        } else {
                            const float4 u = row[r_unit<SF>(kb2, a0 * 2 + h2)];
                            g[0][a0] = make_float2(u.x, u.y);
                            g[C::HB - 1][a0] = make_float2(u.z, u.w);
                        }
                    }
                    tq[lane] = make_float2(0.f, 0.f);
                    r_pass2_dft<SF>(g);
                    if (warp == 0 && kb2 == 0) tq[lane] = r_pass2_quirk<SF>(g, E2, wb1, wbE, rc.cq[0], rc.cq[e_idx]);
                    for (int q2 = 0; q2 < C::A0; q2++) t[lane][q2] = r_pass2_term<SF>(g, q2, E2, wb1, wbE, rc.cq[0], rc.cq[e_idx]);
                }
                for (int lane = 0; lane < 32; lane++) {          // lane-pair exchange -> this CTA's partial sum per bin
                    const int kb2 = lane >> 1, h2 = lane & 1;
                    for (int i = 0; i < C::A0 / 2; i++) {
                        const int q2 = i + h2 * (C::A0 / 2);
                        part[c][warp + 16 * kb2 + 256 * q2] = cadd(t[lane][q2], t[lane ^ 1][q2]);
                    }
                }
                if (warp == 0) part[c][C::L] = cadd(tq[0], tq[1]);
            }
        }
        unsigned long long best = 0ull;
        for (int k = 0; k < C::L; k++) {
            float2 f = part[0][k];
            if (C::CL == 2) f = cadd(f, part[1][k]);
            if (k == C::L / 2) {
                float2 q = part[0][C::L];
                if (C::CL == 2) q = cadd(q, part[1][C::L]);
                f = cadd(f, q);
            }
            const unsigned long long key = pack_key(cnorm2(f), (uint32_t)k);
            best = key > best ? key : best;
        }
        k1_store(bins, mags, s, best);
    }
    for (int c = 0; c < C::CL; c++) { delete[] slots[c]; delete[] part[c]; }
    delete[] keys;
}

}  // namespace lb
