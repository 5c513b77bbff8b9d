// rx_sync.cuh -- the dechirp-synchronised receive path (lora_b200_receive): frames below the noise floor.
//
// The stream state machine (rx_stream.cuh, rx_warp.cuh) gates on per-sample statistics -- an autocorrelation and a Pearson
// correlation of instantaneous frequency -- which gain nothing from the spreading factor.  This path gates on dechirped
// windows instead, whose peak carries the full sps-fold processing gain:
//   screen      K1 (dechirp + FFT + argmax) on every window of every stream, at hops of sps in two phases sps/2 apart
//   detect      runs of >= min_preamble windows of one phase whose bins agree within +-1: one candidate per preamble
//   synchronise one CTA per candidate: SFD bin (up-chirp dechirp) -> integer CFO and timing, fractional CFO from the phase
//               advance of the preamble peak, timing to the sample by the summed energy of the frame's known symbols,
//               sync-word check
//   assemble    each frame's data windows, de-rotated by its CFO, contiguous -> K1 batch kernels -> bins
//   decode      rx_symbol_commit / rx_frame_record of rx_stream.cuh over the bins, header checksum, then K8
// With soft decisions the assemble stage runs the LLR demodulator (k1_llr.cuh) instead of K1, and each interleaver block's
// code words are decoded to their maximum-likelihood nibbles and re-encoded into corrected bins (rs_soft_* below); decode
// then runs unchanged on those bins.
// A window at p dechirped with the down-chirp sees an up-chirp that started tau samples before p at bin tau / decim + F, and
// dechirped with the up-chirp sees a down-chirp at bin -tau / decim + F (F = CFO in bins, modulo N): the preamble bin A and
// the SFD bin B give 2F = A + B and 2 tau / decim = A - B, the N/2 ambiguity resolved by |F| <= N/4.
// Wider offsets (rx_params.wide_cfo) search hypotheses c = -C..C of a coarse offset c N/2 bins: the screen runs once per
// hypothesis with the shifted tables down_c[n] = down[n] e^{-j pi c n / D} (rs_shift_tables), whose windows see the preamble at
// tau / decim + F - c N/2, and the synchroniser resolves the ambiguity F = c N/2 + smod(A + B, N) / 2 + k N/2 by scoring the
// branches k = -1, 0, 1 (rs_synchronise).  C = 0 (|F| <= N/4) is the procedure above.
// Everything a kernel decides is in the __host__ __device__ functions below, which host_emul.cu runs on the CPU.
#pragma once
#include "int_chain.cuh"
#include "k1_fft.cuh"
#include "k1_llr.cuh"
#include "lora_crc.h"
#include "rx_stream.cuh"
#include "tx_encode.cuh"

#include <cmath>

namespace lb {

struct RsParams {
    uint32_t sps, n_bins, decim;
    float sfo_ppm;                     // clock offset of every frame, in ppm (0: none)
    uint32_t min_preamble;             // windows of one phase
    uint32_t sw[2];                    // sync-word bins, ((sw >> 4) & 15) * 8 and (sw & 15) * 8 (tx.modulate_frame)
    float max_cfo_bins;                // |CFO| accepted, in bins (<= N / 4 unless wide_cfo)
    float ppm_per_bin;                 // clock offset per bin of CFO: 1e6 * bin_hz / carrier_hz (0: no carrier given)
    int32_t hyp;                       // C: coarse-offset hypotheses c = -C..C (rs_hypotheses; 0: the one screen of c = 0)
};

// coarse-offset hypotheses: the largest |c| the screen needs so that every |F| <= max_cfo_bins lies within N/4 of some c N/2.
// At fs / bw = D the sampled band, |F| <= (D - 1) N / 2, needs C <= D - 1 (7 at 8, 15 at 16, 31 at 32; 1 at 2), that is
// 2 (2 C + 1) screens: 30, 62, 126.
constexpr int rs_max_hyp(int D) { return D - 1; }
constexpr int rs_max_screens(int D) { return 2 * (2 * rs_max_hyp(D) + 1); }
constexpr int RS_MAX_HYP = rs_max_hyp(8);          // (fs - BW) / 2 at fs / bw = 8: 3.5 N bins
constexpr int RS_MAX_SCREENS = rs_max_screens(8);
inline int rs_hypotheses(float max_cfo_bins, uint32_t N) {
    const double c = std::ceil(((double)max_cfo_bins - 0.25 * N) / (0.5 * N));
    return c > 0.0 ? (int)c : 0;
}

// the shifted dechirp tables of hypotheses c = -C..C, out[((c + C) * 2 + up) * sps + n] = table[n] e^{-j pi c n / D}, table the
// down- (up = 0) or up-chirp (up = 1); the phase is reduced exactly, (c n) mod 2D, and the product is formed in double.
// (2 C + 1) 2 sps float2 in all, on the host and on the device: 7.9 MB at SF12, fs/bw = 8, C = 7, and 132 MB at SF12,
// fs/bw = 32, C = 31 (the whole band of a 4 MS/s capture at 125 kHz)
inline void rs_shift_tables(const float2 *down, const float2 *up, uint32_t sps, uint32_t D, int C, float2 *out) {
    for (int c = -C; c <= C; c++)
        for (int u = 0; u < 2; u++) {
            const float2 *t = u ? up : down;
            float2 *o = out + ((size_t)(c + C) * 2 + u) * sps;
            for (uint32_t n = 0; n < sps; n++) {
                const long long r = (((long long)c * n) % (2 * (long long)D) + 2 * (long long)D) % (2 * (long long)D);
                const double a = -M_PI * (double)r / (double)D, cs = std::cos(a), sn = std::sin(a);
                o[n] = make_float2((float)(t[n].x * cs - t[n].y * sn), (float)(t[n].x * sn + t[n].y * cs));
            }
        }
}

struct RsCand {                        // one preamble run of the screen
    long long p_last;                  // first sample of the run's last window
    uint32_t bin;                      // its bin
    uint32_t run;                      // windows in the run
    float mag;                         // mean peak magnitude of the run
    int32_t hyp;                       // the coarse-offset hypothesis c of its screen
};

enum RsStatus { RS_OK = 0, RS_INCOMPLETE = 1, RS_REJECT = 2 };

struct RsFrame {                       // a synchronised frame
    long long start;                   // first preamble sample (in the row)
    uint32_t stream;
    float cfo_bins;                    // CFO in bins (BW / N Hz)
    float snr_db;                      // estimated SNR in the LoRa bandwidth
    int32_t status;                    // RsStatus
    int32_t n_payload;                 // after the header round: payload symbols, -1 = header checksum failed
    float sfo_ppm;                     // the clock offset its windows are placed with
};

// ---- clock offset ----------------------------------------------------------------------------------------------------------
// delta = ppm * 1e-6.  delta > 0: the transmitter's clock is fast against the receiver's, and receiver sample n holds
// transmitter time u = (n - start) (1 + delta) samples (tests/conftest.py::make_capture(sfo_ppm=...)); one crystal makes its
// carrier high by delta * carrier_hz as well, a positive CFO.  A frame's delta is sfo_ppm * 1e-6 + cfo_hz / carrier_hz (the
// second term 0 without a carrier frequency).  TX symbol position j counts from the frame start: 0..7 preamble, 8, 9 sync
// word, 10..12.25 SFD, 12.25 + k data symbol k.  It starts at receiver sample start + llround(j sps / (1 + delta)), which is
// exactly start + j sps at delta = 0.  Every window of a frame is placed by this rule, each at its own rounded start.
LB_HD long long rs_sym(long long start, double j, uint32_t sps, float ppm) {
    const double u = j * (double)sps;                 // (exact: j is a multiple of 1/4 and sps of 4)
    return start + (ppm == 0.f ? (long long)u : llround(u / (1.0 + 1e-6 * (double)ppm)));   // (no division at delta = 0)
}

// TX symbol position of data symbol k: 8 preamble up-chirps, 2 sync symbols, 2.25 down-chirps come first
LB_HD double rs_data_j(long long k) { return 12.25 + (double)k; }

// the clock offset (ppm) of a hypothesis with CFO F bins
LB_HD float rs_ppm(const RsParams &p, float F) { return p.sfo_ppm + F * p.ppm_per_bin; }

// whether a call places windows with a clock offset at all; without one the synchroniser is instantiated with DRIFT = false
// and does no drift arithmetic (rs_pos = start + j sps, the clock offset 0)
LB_HD bool rs_drift(const RsParams &p) { return p.sfo_ppm != 0.f || p.ppm_per_bin != 0.f; }
template <bool DRIFT> LB_HD float rs_ppm_of(const RsParams &p, float F) { return DRIFT ? rs_ppm(p, F) : 0.f; }
template <bool DRIFT> LB_HD long long rs_pos(long long start, int j, uint32_t sps, float ppm) {
    return DRIFT ? rs_sym(start, j, sps, ppm) : start + (long long)j * sps;
}

LB_HD int rs_smod(int v, int n) {      // v mod n in [-n/2, n/2)
    v %= n;
    if (v < 0) v += n;
    return v >= n / 2 ? v - n : v;
}

// ---- detect: one stream's screen -> candidates --------------------------------------------------------------------------
// The screens are s = 0 .. 2 (2 C + 1) - 1 (C = p.hyp): phase ph = s % 2 of hypothesis c = s / 2 - C.  bins/mags[s] hold the
// windows of screen s, window j at j * sps + ph * sps / 2, n[ph] of them.  Windows are visited in order of position; a run of
// one screen grows while consecutive bins agree within +-1.  Runs of any screens that end within two symbols of each other
// describe the same preamble: the one with the larger mean peak (the better aligned, in the better hypothesis) is kept.
// Writes at most cap candidates, returns how many there were (more than cap: the caller holds back from the first extra).
// S_MAX bounds the screens (2: the one hypothesis c = 0).
template <int S_MAX>
LB_HD uint32_t rs_detect_stream(const uint32_t *const *bins, const float *const *mags, const uint32_t n[2], const RsParams &p,
                                RsCand *out, uint32_t cap, long long *first_dropped) {
    const int N = (int)p.n_bins, ns = 2 * (2 * p.hyp + 1) < S_MAX ? 2 * (2 * p.hyp + 1) : S_MAX;
    uint32_t run[S_MAX], last[S_MAX];
    float msum[S_MAX];
    for (int s = 0; s < S_MAX; s++) { run[s] = 0; last[s] = 0; msum[s] = 0.f; }
    RsCand pend = {0, 0, 0, 0.f, 0};
    bool have = false;
    uint32_t cnt = 0;
    *first_dropped = -1;
    auto emit = [&](const RsCand &c) {
        if (cnt < cap) out[cnt] = c;
        else if (cnt == cap) *first_dropped = c.p_last - (long long)c.run * p.sps;
        cnt++;
    };
    auto close = [&](int s, uint32_t j_end) {      // run of screen s whose last window is j_end - 1
        if (run[s] >= p.min_preamble) {
            RsCand c;
            c.p_last = (long long)(j_end - 1) * p.sps + (s & 1) * (p.sps / 2);
            c.bin = last[s]; c.run = run[s]; c.mag = msum[s] / (float)run[s]; c.hyp = s / 2 - p.hyp;
            if (have && c.p_last - pend.p_last < 2ll * p.sps && pend.p_last - c.p_last < 2ll * p.sps) {
                if (c.mag > pend.mag) pend = c;
            } else {
                if (have) emit(pend);
                pend = c;
                have = true;
            }
        }
        run[s] = 0; msum[s] = 0.f;
    };
    const uint32_t jmax = n[0] > n[1] ? n[0] : n[1];
    for (uint32_t j = 0; j < jmax; j++) {
#pragma unroll
        for (int s = 0; s < S_MAX; s++) {
            if (s >= ns || j >= n[s & 1]) continue;
            const uint32_t b = bins[s][j];
            if (run[s] && (rs_smod((int)b - (int)last[s], N) < -1 || rs_smod((int)b - (int)last[s], N) > 1)) close(s, j);
            run[s]++;
            msum[s] += mags[s][j];
            last[s] = b;
        }
    }
#pragma unroll
    for (int s = 0; s < S_MAX; s++)
        if (s < ns) close(s, n[s & 1]);
    if (have) emit(pend);
    return cnt;
}

// ---- synchronise ---------------------------------------------------------------------------------------------------------
// Ops gives the procedure its windows (block-collective on the device, plain loops on the host).  A receiver may have
// several antennas (rows) sharing one timing and CFO; Ops::M is how many values binvals writes (1 for one row; with
// fewer antennas than M the rest are 0):
//   bool in_range(long long pos)                       window [pos, pos + sps) inside the row
//   unsigned long long argmax(long long pos, bool up, int c)  K1 argmax key of the raw window, dechirped with the down (up)
//                                                      chirp of hypothesis c (rs_shift_tables; c = 0: the plain tables);
//                                                      over several antennas the key of the summed |tmp_a|^2
//   void binvals(long long pos, float F, bool up, int bin, float2 *v)   v[a]: bin `bin` (signed, -N/2..N/2) of antenna a's
//                                                      window de-rotated by F bins
//   float energy(long long pos)                        sum |x|^2 over the window (of every antenna)
// The dechirp tables are (1 + 1j) e^{+-j phase}: |table|^2 = 2.
constexpr int RS_MAX_ANTENNAS = 4;

LB_HD float rs_phase_rev(float2 z) { return atan2f(z.y, z.x) * 0.15915494309189535f; }   // arg / 2 pi

// score of a hypothesis (start rs_sym(t, m), CFO F bins, windows placed with its clock offset): energy at the expected bins
// of the preamble, the sync word and the SFD.  The windows are placed from t, so that hypotheses a symbol apart (m = -1, 0,
// 1) score the very same windows, whatever the clock offset.
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <bool DRIFT, class Ops>
LB_HD float rs_score(Ops &ops, const RsParams &p, long long t, int m, float F) {
    const int N = (int)p.n_bins;
    const float ppm = rs_ppm_of<DRIFT>(p, F);
    float s = 0.f;
    for (int i = 0; i < 12; i++) {
        const long long pos = rs_pos<DRIFT>(t, i + m, p.sps, ppm);
        if (pos < 0 || !ops.in_range(pos)) continue;
        const int bin = i == 8 ? rs_smod((int)p.sw[0], N) : i == 9 ? rs_smod((int)p.sw[1], N) : 0;
        float2 v[Ops::M];
        ops.binvals(pos, F, i >= 10, bin, v);
        for (int a = 0; a < Ops::M; a++) s += cnorm2(v[a]);
    }
    return s;
}

#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
// The candidate's hypothesis c: its windows saw the preamble at A = tau / decim + F - c N/2 and the SFD, dechirped with up_c, at
// B = -tau / decim + F - c N/2 (mod N), so F = c N/2 + smod(A + B, N) / 2 + k N/2.  Each branch k (k = 0 only while
// max_cfo_bins <= N/4, where |F| <= N/4 decides it) gets its own timing, which moves by sps/2 per k, and its own fractional
// CFO, and all branches' hypotheses compete in one score.
template <bool DRIFT, class Ops>
LB_HD RsFrame rs_synchronise(Ops &ops, const RsCand &c, const RsParams &p, uint32_t stream) {
    const long long sps = p.sps;
    const int N = (int)p.n_bins;
    const float decim = (float)p.decim;
    RsFrame r;
    r.start = c.p_last - (long long)c.run * sps; r.stream = stream; r.cfo_bins = 0.f; r.snr_db = 0.f;
    r.status = RS_REJECT; r.n_payload = 0; r.sfo_ppm = 0.f;
    // SFD: the window 2..6 symbols after the run's last one with the strongest up-chirp dechirp.  A preamble tone often
    // shows as strongly in two neighbouring hypotheses while the SFD's tone lies outside one of their bands, so the SFD is
    // taken over hypotheses c - 1 .. c + 1 (those searched), and its bin moved into c's: B_c = B_c' + (c' - c) N/2
    unsigned long long best = 0ull;
    int kbest = -1, cbest = c.hyp;
    const int c0 = c.hyp > -p.hyp ? c.hyp - 1 : c.hyp, c1 = c.hyp < p.hyp ? c.hyp + 1 : c.hyp;
    for (int k = 2; k <= 6; k++) {
        const long long pos = c.p_last + k * sps;
        if (!ops.in_range(pos)) { r.status = RS_INCOMPLETE; return r; }
        for (int h = c0; h <= c1; h++) {
            const unsigned long long key = ops.argmax(pos, true, h);
            if (key > best) { best = key; kbest = k; cbest = h; }
        }
    }
    const int A = (int)c.bin, B = (int)key_idx(best) + (cbest - c.hyp) * (N / 2);
    const float Fh = (float)c.hyp * (float)(N / 2);
    const int kmax = p.max_cfo_bins > 0.25f * (float)N ? 1 : 0;
    float best_s = -1.f, Fb = 0.f;
    long long tb = 0;
    for (int kb = -kmax; kb <= kmax; kb++) {
        const float Fr = 0.5f * (float)rs_smod(A + B, N) + (float)(kb * (N / 2)), Fc = Fh + Fr;
        if (fabsf(Fc) > p.max_cfo_bins + 1.0f) continue;
        float tau = fmodf((float)A - Fr, (float)N);
        if (tau < 0.f) tau += (float)N;
        // frame start if the SFD window (kbest symbols after the run's last window) lies in the first down-chirp, TX symbol
        // position 10: the run's last window, whose bin gave tau, then lies in preamble symbol 10 - kbest
        const float rc = rs_ppm_of<DRIFT>(p, Fc);
        const long long t0 = DRIFT ? c.p_last - (long long)lrintf(tau * decim) - rs_pos<DRIFT>(0, 10 - kbest, p.sps, rc)
                                   : c.p_last + kbest * sps - (long long)lrintf(tau * decim) - 10 * sps;
        // fractional CFO: phase advance of the preamble peak from symbol to symbol (its residual modulo one bin)
        float2 z = make_float2(0.f, 0.f), prev[Ops::M];
        for (int a = 0; a < Ops::M; a++) prev[a] = make_float2(0.f, 0.f);
        for (int i = 1; i <= 6; i++) {
            const long long pos = rs_pos<DRIFT>(t0, i, p.sps, rc);
            if (pos < 0 || !ops.in_range(pos)) continue;
            float2 x[Ops::M];
            ops.binvals(pos, Fc, false, 0, x);
            for (int a = 0; a < Ops::M; a++) {
                if (i > 1) z = cadd(z, cmul(x[a], cconj(prev[a])));
                prev[a] = x[a];
            }
        }
        const float eps = rs_phase_rev(z);
        for (int j = -1; j <= 1; j++) {
            const float F = Fc + eps + (float)j;
            if (fabsf(F) > p.max_cfo_bins + 0.5f) continue;
            const long long tj = t0 + (long long)lrintf((F - Fc) * decim);   // timing follows the CFO: tau = (A - F) decim
            for (int m = -1; m <= 1; m++) {
                const float s = DRIFT ? rs_score<DRIFT>(ops, p, tj, m, F) : rs_score<DRIFT>(ops, p, tj + m * sps, 0, F);
                if (s > best_s) { best_s = s; Fb = F; tb = rs_pos<DRIFT>(tj, m, p.sps, rs_ppm_of<DRIFT>(p, F)); }
            }
        }
    }
    if (best_s < 0.f) return r;
    // timing to the sample: +-decim/2 around the best hypothesis
    long long tf = tb;
    for (int d = -(int)p.decim / 2; d <= (int)p.decim / 2; d++) {
        if (d == 0) continue;
        const float s = rs_score<DRIFT>(ops, p, tb + d, 0, Fb);
        if (s > best_s) { best_s = s; tf = tb + d; }
    }
    // the residual CFO at the final timing
    float2 z = make_float2(0.f, 0.f), prev[Ops::M];
    float pk = 0.f, en = 0.f;
    int npk = 0;
    const float rb = rs_ppm_of<DRIFT>(p, Fb);
    for (int i = 0; i < 8; i++) {
        const long long pos = rs_pos<DRIFT>(tf, i, p.sps, rb);
        if (pos < 0 || !ops.in_range(pos)) continue;
        float2 x[Ops::M];
        ops.binvals(pos, Fb, false, 0, x);
        for (int a = 0; a < Ops::M; a++) {
            if (npk) z = cadd(z, cmul(x[a], cconj(prev[a])));
            prev[a] = x[a];
        }
        if (i >= 1 && i <= 6) {
            for (int a = 0; a < Ops::M; a++) pk += cnorm2(x[a]);
            en += ops.energy(pos);
        }
        npk++;
    }
    const float F = Fb + rs_phase_rev(z);
    // sync word: the argmax of both sync symbols (raw windows, so shifted by the CFO) within one bin of the expected one,
    // dechirped with the hypothesis c' whose c' N/2 lies nearest F
    const int Fi = (int)lrintf(F);
    int cs = (int)lrintf(F / (float)(N / 2));
    cs = cs < -p.hyp ? -p.hyp : cs > p.hyp ? p.hyp : cs;
    const float rf = rs_ppm_of<DRIFT>(p, F);
    for (int i = 0; i < 2; i++) {
        const long long pos = rs_pos<DRIFT>(tf, 8 + i, p.sps, rf);
        if (pos < 0 || !ops.in_range(pos)) return r;
        const int b = (int)key_idx(ops.argmax(pos, false, cs));
        const int dv = rs_smod(b - (Fi - cs * (N / 2)) - (int)p.sw[i], N);
        if (dv < -1 || dv > 1) return r;
    }
    if (fabsf(F) > p.max_cfo_bins) return r;
    // SNR: |X|^2 / (2 sps) = sps S + s2, window energy = sps (S + s2)  (S: signal power, s2: noise power per sample)
    const float px = pk / 12.0f / (float)sps, e = en / 6.0f;       // 6 windows, |table|^2 = 2
    const float s2 = fmaxf((e - px) / (float)(sps - 1), 1e-30f);
    const float S = fmaxf((px - s2) / (float)sps, 1e-30f);
    r.start = tf; r.cfo_bins = F; r.snr_db = 10.0f * log10f(S / s2 * decim); r.sfo_ppm = rs_ppm_of<DRIFT>(p, F);
    r.status = RS_OK;
    return r;
}

// ---- several antennas: channel estimates and maximum-ratio combining weights ------------------------------------------------
// At a synchronised frame's final timing and CFO, per antenna a of the m = Ops::M-or-fewer rows (energies(pos, e): e[a] =
// sum |x_a|^2 over the window):
//   h[a]  = the mean of its de-rotated preamble peaks binval_a(i, F, 0) over windows 1..6, over (1 + j) sps: the amplitude
//           per sample, with a phase whose reference is common to the frame's antennas
//   s2[a] = its noise power per sample, from window energy minus peak as rs_synchronise's SNR estimate (floored at 60 dB
//           below the strongest antenna's energy, so that noiseless rows keep finite weights)
//   w[a]  = conj(h[a]) / s2[a], scaled to sum |w|^2 = 1: y = sum_a w[a] x_a has the noise power of one antenna when all
//           are alike, and the scale of one frame's y does not move any decision of the decoder
// Returns the combined (post-MRC) SNR in dB in the LoRa bandwidth: the sum of the antennas' SNRs.
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <bool DRIFT, class Ops>
LB_HD float rs_channels(Ops &ops, const RsParams &p, const RsFrame &r, uint32_t m, float2 *h, float2 *w) {
    const float sps = (float)p.sps;
    float2 acc[Ops::M];
    float pk[Ops::M], en[Ops::M];
    for (int a = 0; a < Ops::M; a++) { acc[a] = make_float2(0.f, 0.f); pk[a] = 0.f; en[a] = 0.f; }
    int nw = 0;
    for (int i = 1; i <= 6; i++) {
        const long long pos = rs_pos<DRIFT>(r.start, i, p.sps, r.sfo_ppm);
        if (pos < 0 || !ops.in_range(pos)) continue;
        float2 x[Ops::M];
        float e[Ops::M];
        ops.binvals(pos, r.cfo_bins, false, 0, x);
        ops.energies(pos, e);
        for (int a = 0; a < Ops::M; a++) { acc[a] = cadd(acc[a], x[a]); pk[a] += cnorm2(x[a]); en[a] += e[a]; }
        nw++;
    }
    const float nwf = nw ? (float)nw : 1.f;
    float s2[Ops::M], emax = 0.f, snr = 0.f;
    for (int a = 0; a < (int)m; a++) emax = fmaxf(emax, en[a] / nwf / sps);
    for (int a = 0; a < (int)m; a++) {
        const float px = pk[a] / (2.0f * nwf) / sps, e = en[a] / nwf;          // |table|^2 = 2
        s2[a] = fmaxf(fmaxf((e - px) / (sps - 1.0f), 1e-6f * emax), 1e-30f);
        const float S = fmaxf((px - s2[a]) / sps, 1e-30f);
        snr += S / s2[a];
        // mean peak / ((1 + j) sps) = mean peak (1 - j) / (2 sps)
        const float2 c = make_float2(acc[a].x / nwf, acc[a].y / nwf);
        h[a] = make_float2((c.x + c.y) / (2.0f * sps), (c.y - c.x) / (2.0f * sps));
    }
    float s2min = s2[0];
    for (int a = 1; a < (int)m; a++) s2min = fminf(s2min, s2[a]);
    float norm = 0.f;
    for (int a = 0; a < (int)m; a++) {
        w[a] = make_float2(h[a].x * (s2min / s2[a]), -h[a].y * (s2min / s2[a]));
        norm += cnorm2(w[a]);
    }
    const float k = norm > 0.f ? 1.0f / sqrtf(norm) : 0.f;
    for (int a = 0; a < (int)m; a++) w[a] = norm > 0.f ? make_float2(w[a].x * k, w[a].y * k) : make_float2(a == 0 ? 1.f : 0.f, 0.f);
    for (int a = (int)m; a < Ops::M; a++) { h[a] = make_float2(0.f, 0.f); w[a] = make_float2(0.f, 0.f); }
    return 10.0f * log10f(snr * (float)p.decim);
}

// ---- fine time of arrival (rx_params.fine_toa) --------------------------------------------------------------------------
// A synchronised frame (start t, CFO F bins, clock offset delta = r.sfo_ppm 1e-6) whose transmitter time 0 lands at row position
// t + eps.  Its window j lies at pos_j = rs_pos(t, j) = t + j sps / (1 + delta) + r_j (r_j: that window's own rounding), so the
// symbol started tau_j = r_j - eps samples before it.  Dechirped, preamble window j (down-chirp) shows its tone at
// F + tau_j / decim + delta N / 2 and SFD window j (up-chirp) at F - tau_j / decim - delta N / 2: the chirps are stretched by
// the transmitter's clock, which moves the tone at a window's centre by +-delta N / 2.  Each window is evaluated at its own
// frequency F + nu + r_j / decim (preamble) or F + nu - r_j / decim (SFD), so that all of them peak at one nu:
//   P_up(nu) = sum_{j = 1..6} sum_a |binval_a(pos_j, F + nu + r_j / decim, down, 0)|^2   peaks at nu_A = -eps / decim + delta N / 2
//   P_dn(nu) = sum_{j = 10, 11} sum_a |binval_a(pos_j, F + nu - r_j / decim, up, 0)|^2    peaks at nu_B = +eps / decim - delta N / 2
// eps = decim (nu_B - nu_A) / 2 + delta sps / 2; F's own error moves both peaks alike and cancels.  Peak search, the same for
// nu_A and nu_B: the grid of RS_TOA_GRID points over +-W, W = (decim / 2 + 1) / decim + 1/4 bins (the timing refinement's
// residual of at most decim / 2 + 1 samples, and a quarter bin for F), step h = 2 W / (RS_TOA_GRID - 1) <= 1/4 bin (inside the
// main lobe of the peak, whose first nulls lie +-1 bin out); the first maximum, moved to the vertex of the parabola through it
// and its neighbours; then RS_TOA_ROUNDS times: h /= 4 and the vertex of the parabola through nu - h, nu, nu + h.  A vertex is
// taken only where the three values are concave, and clamped to +-h.  Windows outside the row are left out; a frame without
// a preamble or an SFD window inside the row gets toa = NaN.  Ops::tones<K>(pos, org, f0, df, up, p) gives
// p[k] = sum_a |binval_a(pos, f0 + k df, up, 0)|^2 for k < K in one pass over the window, its de-rotation phase counted from
// row position org = t instead of 0 (a phase common to the window, which |.|^2 drops): the same frame re-presented at another
// row offset gives the same sums, bit for bit, from the same t, F and clock offset.
constexpr int RS_TOA_GRID = 11;
constexpr int RS_TOA_ROUNDS = 2;
constexpr int RS_TOA_WINDOWS = 8;
LB_HD int rs_toa_j(int i) { return i < 6 ? i + 1 : i + 4; }      // windows 1..6 (preamble), 10, 11 (SFD)

struct RsToa {
    float nu_a, nu_b;                  // the peaks of P_up and P_dn, in bins from F
    double toa;                        // t + eps, in the row's samples
};

LB_HD float rs_toa_vertex(float ym, float y0, float yp, float h) {
    const float den = ym - 2.0f * y0 + yp;
    if (!(den < 0.0f)) return 0.0f;
    const float d = 0.5f * h * (ym - yp) / den;
    return d < -h ? -h : d > h ? h : d;
}

#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <bool DRIFT, class Ops>
LB_HD RsToa rs_toa(Ops &ops, const RsParams &p, const RsFrame &r) {
    const float decim = (float)p.decim, W = (0.5f * decim + 1.0f) / decim + 0.25f;
    const double rate = 1.0 + 1e-6 * (double)r.sfo_ppm;
    long long pos[RS_TOA_WINDOWS];
    float off[RS_TOA_WINDOWS];         // the frequency window i is evaluated at, minus F + nu: +-r_j / decim
    bool in[RS_TOA_WINDOWS], have_a = false, have_b = false;
    for (int i = 0; i < RS_TOA_WINDOWS; i++) {
        const int j = rs_toa_j(i);
        pos[i] = rs_pos<DRIFT>(r.start, j, p.sps, r.sfo_ppm);
        const double rj = DRIFT ? (double)(pos[i] - r.start) - (double)j * (double)p.sps / rate : 0.0;
        off[i] = (float)(i < 6 ? rj / (double)p.decim : -rj / (double)p.decim);
        in[i] = pos[i] >= 0 && ops.in_range(pos[i]);
        if (in[i]) { if (i < 6) have_a = true; else have_b = true; }
    }
    RsToa out;
    if (!have_a || !have_b) {
        out.nu_a = out.nu_b = 0.0f;
        out.toa = (double)NAN;
        return out;
    }
    // the grid
    float h = 2.0f * W / (float)(RS_TOA_GRID - 1);
    float pa[RS_TOA_GRID], pb[RS_TOA_GRID];
    for (int k = 0; k < RS_TOA_GRID; k++) { pa[k] = 0.0f; pb[k] = 0.0f; }
    for (int i = 0; i < RS_TOA_WINDOWS; i++) {
        if (!in[i]) continue;
        float t[RS_TOA_GRID];
        ops.template tones<RS_TOA_GRID>(pos[i], r.start, r.cfo_bins + off[i] - W, h, i >= 6, t);
        for (int k = 0; k < RS_TOA_GRID; k++) { if (i < 6) pa[k] += t[k]; else pb[k] += t[k]; }
    }
    float nu[2];
    for (int s = 0; s < 2; s++) {
        const float *q = s ? pb : pa;
        int kb = 0;
        for (int k = 1; k < RS_TOA_GRID; k++) if (q[k] > q[kb]) kb = k;
        nu[s] = -W + (float)kb * h;
        if (kb > 0 && kb < RS_TOA_GRID - 1) nu[s] += rs_toa_vertex(q[kb - 1], q[kb], q[kb + 1], h);
    }
    // the refinements
    for (int round = 0; round < RS_TOA_ROUNDS; round++) {
        h *= 0.25f;
        float qa[3] = {0.0f, 0.0f, 0.0f}, qb[3] = {0.0f, 0.0f, 0.0f};
        for (int i = 0; i < RS_TOA_WINDOWS; i++) {
            if (!in[i]) continue;
            float t[3];
            ops.template tones<3>(pos[i], r.start, r.cfo_bins + off[i] + nu[i >= 6] - h, h, i >= 6, t);
            for (int k = 0; k < 3; k++) { if (i < 6) qa[k] += t[k]; else qb[k] += t[k]; }
        }
        nu[0] += rs_toa_vertex(qa[0], qa[1], qa[2], h);
        nu[1] += rs_toa_vertex(qb[0], qb[1], qb[2], h);
    }
    out.nu_a = nu[0];
    out.nu_b = nu[1];
    const double delta = DRIFT ? 1e-6 * (double)r.sfo_ppm : 0.0;
    out.toa = (double)r.start + 0.5 * (double)p.decim * ((double)nu[1] - (double)nu[0]) + 0.5 * delta * (double)p.sps;
    return out;
}

// ---- the integer chain of one frame -------------------------------------------------------------------------------------
// FFT demodulator's bin -> rx_symbol_commit (rx_stream.cuh) for the 8 header-block symbols.  Returns the payload symbols
// to read, or -1 when the explicit header's checksum (or coding rate) is wrong.  implicit_len: payload bytes of an
// implicit-header frame.
LB_HD int32_t rs_header(RxStreamState *st, const RxParams &p, uint8_t phdr1, const uint32_t *bins, uint32_t implicit_len) {
    rx_state_init(st, phdr1);
    for (int k = 0; k < 8; k++) {
        if (rx_symbol_commit(st, p, true, true, rx_fft_bin(bins[k], p.n_bins)) == RX_HEADER_DONE) break;
    }
    if (p.implicit) {                                 // as many payload blocks as the code words of implicit_len bytes need
        const TxCode c{p.sf, (uint32_t)(phdr1 >> 5), 0u, (phdr1 >> 4) & 1u, p.reduced_rate ? 1u : 0u};
        st->payload_length = implicit_len;
        st->payload_symbols = (int32_t)(tx_payload_blocks(c, implicit_len) * (c.cr + 4u));
        return st->payload_symbols;
    }
    const uint32_t len = st->hdr_print[0], cr = st->hdr_print[1] >> 5, crc = (st->hdr_print[1] >> 4) & 1u;
    const uint32_t chk = ((st->hdr_print[1] & 1u) << 4) | (st->hdr_print[2] >> 4);
    if (cr < 1u || cr > 4u || header_checksum(len, cr, crc) != chk) return -1;
    return st->payload_symbols;
}

// ... and the payload symbols after it; fills the frame record K8 decodes
LB_HD void rs_frame(RxStreamState *st, const RxParams &p, const uint32_t *bins, int32_t n_payload, RxFrameRec *fr,
                    uint32_t stream, uint32_t seq, float snr_lin) {
    RxParams q = p;
    q.implicit = 0;                                   // count the payload down for an implicit header too
    for (int32_t k = 0; k < n_payload; k++) {
        if (rx_symbol_commit(st, q, false, true, rx_fft_bin(bins[k], p.n_bins)) == RX_FRAME_DONE) break;
    }
    st->frame_seq = seq;
    st->snr = snr_lin;
    rx_frame_record(fr, st, stream, p.implicit);
    for (uint32_t k = 0; k < st->n_demod; k++) fr->cw[k] = st->demodulated[k];
}

// ---- soft decisions --------------------------------------------------------------------------------------------------------
// llr[i * ppm + j]: the LLR of bit j of word i of one interleaver block (k1_llr.cuh, > 0: bit 0).  Code word x's bit i is
// bit (x - i) mod ppm of word i (the inverse of deinterleave_block), so candidate code word c at slot x scores
// sum_i (1 - 2 bit_i(c)) llr[i][(x - i) mod ppm] over the block's n_words words.  The candidates cw(s), s = 0..15, are the
// code words the encoder emits at that slot (tx_encode.cuh); the best score wins, the lowest s on ties (hamming84_decode's
// rule).  Returns the nibble.
template <class CW>
LB_HD uint32_t rs_soft_nibble(const CW &cw, const float *llr, uint32_t n_words, uint32_t ppm, uint32_t x) {
    float best = 0.f;
    uint32_t bs = 0;
    for (uint32_t s = 0; s < 16u; s++) {
        const uint32_t c = cw(s);
        float m = 0.f;
        for (uint32_t i = 0; i < n_words; i++) {
            const float l = llr[i * ppm + (x + 8u * ppm - i) % ppm];     // (i < 8)
            m += (c >> i) & 1u ? -l : l;
        }
        if (s == 0u || m > best) { best = m; bs = s; }
    }
    return bs;
}

// the code a frame is sent with as the receiver is configured: sf, the configured cr and CRC flag (phdr1), the header mode
LB_HD TxCode rs_code(const RxParams &p, uint8_t phdr1) {
    return TxCode{p.sf, (uint32_t)(phdr1 >> 5), p.implicit ? 0u : 1u, (phdr1 >> 4) & 1u, p.reduced_rate ? 1u : 0u};
}

// the header block (8 words, ppm = sf - 2, llr[8][sf - 2]).  An explicit header's 5 slots come first: their header gives the
// frame's cr, clamped to 4 as rx_symbol_commit clamps it, which whitens the remaining slots (the payload nibbles of the
// header block).  Writes the block's 8 corrected bins (the encoder's shifts of the chosen code words) and, when nib is
// given, its sf - 2 nibbles; returns c with the frame's cr.
LB_HD TxCode rs_soft_header(TxCode c, const float *llr, uint32_t *bins, uint32_t *nib_out) {
    const uint32_t ppm = c.sf - 2u;
    uint32_t nib[LLR_MAX_PPM];
    uint32_t x = 0;
    if (c.explicit_hdr) {
        for (; x < 5u; x++) nib[x] = rs_soft_nibble([&](uint32_t s) { return tx_header_cw(c, s, x); }, llr, 8u, ppm, x);
        c.cr = nib[2] >> 1 > 4u ? 4u : nib[2] >> 1;
    }
    for (; x < ppm; x++) nib[x] = rs_soft_nibble([&](uint32_t s) { return tx_header_cw(c, s, x); }, llr, 8u, ppm, x);
    for (uint32_t i = 0; i < 8u; i++) bins[i] = tx_block_shift([&](uint32_t y) { return tx_header_cw(c, nib[y], y); }, i, ppm, true, 1u << c.sf);
    if (nib_out)
        for (uint32_t k = 0; k < ppm; k++) nib_out[k] = nib[k];
    return c;
}

// payload block b of a frame sent with code c (c.cr the frame's): llr[4 + cr][tx_ppm(c)] -> its 4 + cr corrected bins and,
// when nib is given, its tx_ppm(c) nibbles
LB_HD void rs_soft_block(const TxCode &c, uint32_t b, const float *llr, uint32_t *bins, uint32_t *nib_out) {
    const uint32_t spb = c.cr + 4u, ppm = tx_ppm(c), p0 = tx_spare(c) + b * ppm;
    uint32_t nib[LLR_MAX_PPM];
    for (uint32_t x = 0; x < ppm; x++) nib[x] = rs_soft_nibble([&](uint32_t s) { return tx_payload_cw(c, s, p0 + x, spb); }, llr, spb, ppm, x);
    for (uint32_t j = 0; j < spb; j++)
        bins[j] = tx_block_shift([&](uint32_t y) { return tx_payload_cw(c, nib[y], p0 + y, spb); }, j, ppm, c.reduced_rate != 0u, 1u << c.sf);
    if (nib_out)
        for (uint32_t k = 0; k < ppm; k++) nib_out[k] = nib[k];
}

// the payload of one frame: its cr from its (corrected) header bins, replayed through rs_header as rs_frame_kernel does,
// then n_payload / (4 + cr) blocks of llr -> bins
LB_HD void rs_soft_payload(const RxParams &p, uint8_t phdr1, const uint32_t *hdr_bins, int32_t n_payload, uint32_t implicit_len,
                           const float *llr, uint32_t *bins) {
    RxStreamState st;
    rs_header(&st, p, phdr1, hdr_bins, implicit_len);
    TxCode c = rs_code(p, phdr1);
    c.cr = st.phdr[1] >> 5;
    const uint32_t spb = c.cr + 4u, ppm = tx_ppm(c);
    for (uint32_t b = 0; b < (uint32_t)n_payload / spb; b++) rs_soft_block(c, b, llr + (size_t)b * spb * ppm, bins + (size_t)b * spb, nullptr);
}

// ---- CRC-aided list decoding (rx_params.crc_list) ---------------------------------------------------------------------------
// A soft-decoded frame whose payload CRC (lora_crc.h) fails is given a second chance: of its code words that carry nibbles of
// the CRC's message (rs_crc_candidate), the K least reliable (smallest gap between the best and the runner-up metric, ties to the lowest nibble index)
// may each be replaced by its runner-up.  The CRC (initial value 0) and the whitening XOR are linear, so replacing nibble p's
// s1 by s2 moves the syndrome by a fixed delta; of the 2^K subsets, those whose deltas sum to the syndrome satisfy the CRC,
// and the one of least summed gap (the lowest subset mask on ties) is taken.  Its blocks are re-encoded into corrected bins,
// so that decoding runs unchanged.  A frame whose real errors lie outside the list passes some subset with probability about
// (2^K - 1) / 2^16: the price of the option, which is why K is at most RS_CRC_MAX_LIST and off by default.
constexpr uint32_t RS_CRC_MAX_LIST = 12;
constexpr uint32_t RS_CRC_MAX_SLOTS = 576;   // code words of one frame: sf - 2 in the header block, <= 2 (255 + 2) + sf in payload

struct RsSoftPick {
    uint32_t s1, s2;                   // the best nibble (rs_soft_nibble's) and the runner-up (the lowest on ties)
    float gap;                         // their metric difference, >= 0
};

// rs_soft_nibble's candidates and metrics, keeping the runner-up as well
template <class CW>
LB_HD RsSoftPick rs_soft_pick(const CW &cw, const float *llr, uint32_t n_words, uint32_t ppm, uint32_t x) {
    float m1 = 0.f, m2 = 0.f;
    uint32_t s1 = 0, s2 = 0;
    for (uint32_t s = 0; s < 16u; s++) {
        const uint32_t c = cw(s);
        float m = 0.f;
        for (uint32_t i = 0; i < n_words; i++) {
            const float l = llr[i * ppm + (x + 8u * ppm - i) % ppm];
            m += (c >> i) & 1u ? -l : l;
        }
        if (s == 0u) { m1 = m; s1 = 0; }
        else if (m > m1) { m2 = m1; s2 = s1; m1 = m; s1 = s; }
        else if (s == 1u || m > m2) { m2 = m; s2 = s; }
    }
    return RsSoftPick{s1, s2, m1 - m2};
}

// one published frame as the list decoder sees it.  Its code words ("slots") q: the header block's sf - 2, then ppm per
// payload block; slot q >= h carries payload nibble p = q - h (h = 5 header nibbles when explicit).
struct RsCrcFrame {
    TxCode c;                          // c.cr the frame's
    uint32_t L;                        // payload bytes without the CRC; 0: no CRC to check
    uint32_t hppm, ppm, spb, h, n_slots;
};

// the frame's header replayed from its corrected bins, as rs_frame_kernel does
LB_HD RsCrcFrame rs_crc_frame(const RxParams &p, uint8_t phdr1, const uint32_t *hdr_bins, int32_t n_payload, uint32_t implicit_len) {
    RxStreamState st;
    rs_header(&st, p, phdr1, hdr_bins, implicit_len);
    RsCrcFrame f;
    f.c = rs_code(p, phdr1);
    f.c.cr = st.phdr[1] >> 5;
    f.L = ((st.phdr[1] >> 4) & 1u) && st.payload_length >= 4u ? st.payload_length - 2u : 0u;
    f.hppm = p.sf - 2u; f.ppm = tx_ppm(f.c); f.spb = f.c.cr + 4u; f.h = f.c.explicit_hdr ? 5u : 0u;
    f.n_slots = f.hppm + (uint32_t)(n_payload > 0 ? n_payload : 0) / f.spb * f.ppm;
    return f;
}

// whether slot q is a list candidate: it carries a nibble of payload[0 .. L-2), the CRC's message.  The last two payload bytes
// and the two CRC bytes are XORed into the check as they are, so an error of v in payload[L-1] and the same v in c0 (and in
// payload[L-2] and c1) cancel: flipping one of them to "fix" an error in its partner satisfies the CRC and publishes a wrong
// payload.  The interleaver makes such equal errors common (one bad symbol hits the same bit of neighbouring nibbles), so
// these four bytes are never flipped: an error there leaves a syndrome that flips elsewhere only match by chance.
LB_HD bool rs_crc_candidate(const RsCrcFrame &f, uint32_t q) { return q >= f.h && q - f.h < 2u * (f.L - 2u); }

// slot q's pick from the header block's LLRs hllr[8][sf - 2] or the payload blocks' llr[][ppm]
LB_HD RsSoftPick rs_crc_pick(const RsCrcFrame &f, const float *hllr, const float *llr, uint32_t q) {
    if (q < f.hppm) return rs_soft_pick([&](uint32_t s) { return tx_header_cw(f.c, s, q); }, hllr, 8u, f.hppm, q);
    const uint32_t b = (q - f.hppm) / f.ppm, x = (q - f.hppm) % f.ppm, p0 = tx_spare(f.c) + b * f.ppm;
    return rs_soft_pick([&](uint32_t s) { return tx_payload_cw(f.c, s, p0 + x, f.spb); }, llr + (size_t)b * f.spb * f.ppm, f.spb, f.ppm, x);
}

// the syndrome of the published bytes that nibbles nib[q] (all slots) make: 0 iff the frame checks
LB_HD uint32_t rs_crc_syndrome(const RsCrcFrame &f, const uint8_t *nib) {
    auto byte = [&](uint32_t i) { return (uint32_t)nib[f.h + 2u * i] | ((uint32_t)nib[f.h + 2u * i + 1u] << 4); };
    uint32_t crc = 0;
    for (uint32_t i = 0; i + 2u < f.L; i++) crc = lb_crc16_byte(crc, byte(i));
    return crc ^ byte(f.L - 1u) ^ (byte(f.L - 2u) << 8) ^ byte(f.L) ^ (byte(f.L + 1u) << 8) ^ lb_crc_whitening(f.c.cr, f.L);
}

// how the syndrome moves when payload nibble p (a candidate: in the CRC's message) is XORed with v: the CRC of e at byte p / 2
// followed by the L - 3 - p / 2 bytes after it
LB_HD uint32_t rs_crc_delta(uint32_t L, uint32_t p, uint32_t v) {
    uint32_t c = lb_crc16_byte(0, v << (4u * (p & 1u)));
    for (uint32_t k = (p >> 1) + 3u; k < L; k++) c = lb_crc16_byte(c, 0);
    return c;
}

// the summed gap of subset `mask` of the list gap[0 .. K), in list order
LB_HD float rs_crc_cost(const float *gap, uint32_t mask) {
    float c = 0.f;
    for (uint32_t j = 0; mask; j++, mask >>= 1)
        if (mask & 1u) c += gap[j];
    return c;
}

LB_HD unsigned long long rs_crc_key(float v, uint32_t idx) {      // (v >= 0, idx) ordered lexicographically, smallest first
    union { float f; uint32_t u; } c;
    c.f = v;
    return ((unsigned long long)c.u << 32) | idx;
}

// number of bins of slot q's block, and bin i of it re-encoded from the frame's nibbles nib[q] (all slots); the header
// block's bins are hdr[0 .. 8), payload block b's are pay[b spb ..]
LB_HD uint32_t rs_crc_block_bins(const RsCrcFrame &f, uint32_t q) { return q < f.hppm ? 8u : f.spb; }
LB_HD uint32_t *rs_crc_block_out(const RsCrcFrame &f, uint32_t q, uint32_t *hdr, uint32_t *pay) {
    return q < f.hppm ? hdr : pay + (size_t)((q - f.hppm) / f.ppm) * f.spb;
}
LB_HD uint32_t rs_crc_block_bin(const RsCrcFrame &f, const uint8_t *nib, uint32_t q, uint32_t i) {
    if (q < f.hppm) return tx_block_shift([&](uint32_t y) { return tx_header_cw(f.c, nib[y], y); }, i, f.hppm, true, 1u << f.c.sf);
    const uint32_t b = (q - f.hppm) / f.ppm, q0 = f.hppm + b * f.ppm, p0 = tx_spare(f.c) + b * f.ppm;
    return tx_block_shift([&](uint32_t y) { return tx_payload_cw(f.c, nib[q0 + y], p0 + y, f.spb); }, i, f.ppm, f.c.reduced_rate != 0u,
                          1u << f.c.sf);
}

#ifdef __CUDACC__
// ---- kernels ---------------------------------------------------------------------------------------------------------------
// detect: one thread per stream.  The screen's windows of row s are the K1 results starting at s * stride / sps (stride a
// multiple of sps) in each phase array, those of hypothesis c at (c + hyp) * hyp_stride further.  S_MAX bounds the screens
// (2 without wide_cfo, with it rs_max_screens(D) of the rate: RS_MAX_SCREENS up to fs/bw = 8, 62 at 16, 126 at 32).
template <int S_MAX>
__global__ void rs_detect_kernel(const uint32_t *__restrict__ bins0, const float *__restrict__ mags0, const uint32_t *__restrict__ bins1,
                                 const float *__restrict__ mags1, size_t hyp_stride, size_t stride, size_t n_items, uint32_t n_streams,
                                 RsParams p, RsCand *__restrict__ cands, uint32_t cap, uint32_t *__restrict__ n_cands,
                                 long long *__restrict__ dropped) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_streams) return;
    const size_t base = s * (stride / p.sps);
    const uint32_t *b[S_MAX];
    const float *m[S_MAX];
#pragma unroll
    for (int k = 0; k < S_MAX; k++) {
        const size_t o = base + (size_t)(k >> 1) * hyp_stride;
        b[k] = (k & 1 ? bins1 : bins0) + o;
        m[k] = (k & 1 ? mags1 : mags0) + o;
    }
    const uint32_t n[2] = {(uint32_t)(n_items / p.sps), (uint32_t)(n_items >= p.sps + p.sps / 2 ? (n_items - p.sps / 2) / p.sps : 0)};
    n_cands[s] = rs_detect_stream<S_MAX>(b, m, n, p, cands + (size_t)s * cap, cap, dropped + s);
}

// sum of NV values over the CTA through red[RX_WARPS * NV] (shared), in a fixed order; result valid in every thread
template <int NV>
LB_D void rs_block_sums(float (&v)[NV], float *red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; k++) {
        const float s = warp_sum(v[k]);
        if (lane == 0) red[warp * NV + k] = s;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < NV; k++) {
        float t = 0.f;
        for (int w = 0; w < RX_WARPS; w++) t += red[w * NV + k];
        v[k] = t;
    }
    __syncthreads();
}

// the window sums of rs_toa: sample n's chirp product, de-rotated by f0 (phase counted from org), is formed once and stepped through the K frequencies
// f0 + k df by w = e^{-2 pi j df n / sps} (the phase e^{-2 pi j k df pos / sps} common to the window drops out of |.|^2); the
// 2 K M sums of M rows reduce through red (RX_WARPS * 2 K M floats of shared memory)
template <int K, int M>
LB_D void rs_tones(const float2 *x, size_t stride, uint32_t m, long long pos, long long org, const float2 *ch, uint32_t sps, float f0,
                   float df, float *red, float *pw) {
    double base = (double)f0 * (double)(pos - org) / (double)sps;
    base -= floor(base);
    const float fb = (float)base, fr = f0 / (float)sps, fd = df / (float)sps;
    float s[2 * K * M];
#pragma unroll
    for (int k = 0; k < 2 * K * M; k++) s[k] = 0.f;
    for (uint32_t n = threadIdx.x; n < sps; n += RX_THREADS) {
        float t = fmaf(fr, (float)n, fb);
        t -= floorf(t);
        float u = fd * (float)n;
        u -= floorf(u);
        float sn, cs, sw, cw;
        sincospif(-2.0f * t, &sn, &cs);
        sincospif(-2.0f * u, &sw, &cw);
        const float2 q = cmul(__ldg(ch + n), make_float2(cs, sn)), w = make_float2(cw, sw);
#pragma unroll
        for (int a = 0; a < M; a++) {
            if (a < (int)m) {
                float2 y = cmul(x[(size_t)a * stride + pos + n], q);
#pragma unroll
                for (int k = 0; k < K; k++) {
                    s[2 * (a * K + k)] += y.x; s[2 * (a * K + k) + 1] += y.y;
                    y = cmul(y, w);
                }
            }
        }
    }
    rs_block_sums<2 * K * M>(s, red);
#pragma unroll
    for (int k = 0; k < K; k++) {
        float p = 0.f;
#pragma unroll
        for (int a = 0; a < M; a++) p += s[2 * (a * K + k)] * s[2 * (a * K + k)] + s[2 * (a * K + k) + 1] * s[2 * (a * K + k) + 1];
        pw[k] = p;
    }
}

// the windows of one candidate, block-collective (all threads call every member with the same arguments); D = sps / N is
// argmax's only use of the sample rate (binval and energy take sps at run time)
template <int SF, int D = 8>
struct RsDevOps {
    static constexpr int M = 1;
    const float2 *x;                   // the row
    long long n_items;
    const float2 *down, *up, *tw;
    uint32_t sps;
    float2 *smem;
    RxShared *sh;
    const float2 *shift;               // the shifted tables of hypotheses -hyp..hyp (rs_shift_tables; NULL when hyp = 0)
    int hyp;
    LB_D bool in_range(long long pos) const { return pos >= 0 && pos + (long long)sps <= n_items; }
    LB_D const float2 *chirp(bool use_up, int c) const {
        return c == 0 ? (use_up ? up : down) : shift + ((size_t)(c + hyp) * 2 + (use_up ? 1 : 0)) * sps;
    }
    LB_D unsigned long long argmax(long long pos, bool use_up, int c) {
        using C = K1Cfg<SF, D>;
        const int tid = threadIdx.x;
        K1Args a{x + pos, chirp(use_up, c), tw, 1};
        unsigned long long best = 0ull;
        float2 wtab[C::NP / C::TPS];
        k1_combine_twiddles<SF, D>(a, tid, wtab);
        for (int s = 0; s < C::S; s++) {
            k1_pass0<SF, false, D>(a, 0, s, tid, smem);
            __syncthreads();
            k1_pass<SF, C::R1, C::SIG1, D>(a, tid, smem);
            __syncthreads();
            if (C::R2 > 1) { k1_pass<SF, (C::R2 > 1 ? C::R2 : 2), 1, D>(a, tid, smem); __syncthreads(); }
            const unsigned long long k = tid < C::TPS ? k1_combine<SF, D>(a, s, tid, smem, wtab) : 0ull;
            best = k > best ? k : best;
            __syncthreads();
        }
        return block_max_key(best, *sh);
    }
    LB_D float2 binval(long long pos, float F, bool use_up, int bin) {
        const float2 *ch = use_up ? up : down;
        double base = (double)F * (double)pos / (double)sps;     // de-rotation phase (revolutions) at the window's first sample
        base -= floor(base);
        const float fb = (float)base, fr = F / (float)sps;
        const uint32_t kb = (uint32_t)((bin % (int)sps) + (int)sps) % sps;
        float v[2] = {0.f, 0.f};
        for (uint32_t n = threadIdx.x; n < sps; n += RX_THREADS) {
            float t = fmaf(fr, (float)n, fb);
            t -= floorf(t);
            float sn, cs;
            sincospif(-2.0f * t, &sn, &cs);
            float2 m = cmul(cmul(x[pos + n], __ldg(ch + n)), make_float2(cs, sn));
            if (kb) m = cmul(m, __ldg(tw + (size_t)((unsigned long long)kb * n % sps)));
            v[0] += m.x; v[1] += m.y;
        }
        block_sum<2>(v, *sh);
        return make_float2(v[0], v[1]);
    }
    LB_D void binvals(long long pos, float F, bool use_up, int bin, float2 *v) { v[0] = binval(pos, F, use_up, bin); }
    // (rs_toa: smem holds RX_WARPS * 2 K floats)
    template <int K> LB_D void tones(long long pos, long long org, float f0, float df, bool use_up, float *p) {
        rs_tones<K, 1>(x, 0, 1, pos, org, use_up ? up : down, sps, f0, df, (float *)smem, p);
    }
    LB_D float energy(long long pos) {
        float v[1] = {0.f};
        for (uint32_t n = threadIdx.x; n < sps; n += RX_THREADS) { const float2 a = x[pos + n]; v[0] += a.x * a.x + a.y * a.y; }
        block_sum<1>(v, *sh);
        return v[0];
    }
};

// the windows of one candidate of a receiver with m <= RS_MAX_ANTENNAS antennas, rows one.x + a * stride: argmax of the
// combined spectrum (the phase functions of k1_antennas_kernel on one window position), binval and energy per antenna
template <int SF, int D = 8>
struct RsAntOps {
    static constexpr int M = RS_MAX_ANTENNAS;
    RsDevOps<SF, D> one;               // antenna 0
    size_t stride;
    uint32_t m;
    LB_D bool in_range(long long pos) const { return one.in_range(pos); }
    static_assert(M == 4, "binvals reduces 2 M sums as two block_sum<4>");
    LB_D unsigned long long argmax(long long pos, bool use_up, int c) {
        using C = K1Cfg<SF, D>;
        const int tid = threadIdx.x;
        K1Args a{one.x + pos, one.chirp(use_up, c), one.tw, 1};
        unsigned long long best = 0ull;
        float2 wtab[C::NP / C::TPS];
        k1_combine_twiddles<SF, D>(a, tid, wtab);
        for (int s = 0; s < C::S; s++) {
            float pw[C::NP / C::TPS];
            for (int i = 0; i < C::NP / C::TPS; i++) pw[i] = 0.f;
            for (uint32_t ant = 0; ant < m; ant++) {
                K1Args aa = a;
                aa.x = a.x + ant * stride;
                k1_pass0<SF, false, D>(aa, 0, s, tid, one.smem);
                __syncthreads();
                k1_pass<SF, C::R1, C::SIG1, D>(aa, tid, one.smem);
                __syncthreads();
                if (C::R2 > 1) { k1_pass<SF, (C::R2 > 1 ? C::R2 : 2), 1, D>(aa, tid, one.smem); __syncthreads(); }
                if (tid < C::TPS) k1_combine_power<SF, D>(s, tid, one.smem, wtab, pw);
                __syncthreads();
            }
            const unsigned long long k = tid < C::TPS ? k1_power_key<SF, D>(s, tid, pw) : 0ull;
            best = k > best ? k : best;
        }
        return block_max_key(best, *one.sh);
    }
    // every antenna's bin in one pass over the window: the de-rotation and bin twiddle of sample n are formed once and
    // applied to the m rows, and the 2m sums go through block_sum four at a time (one reduction for m <= 2, two for m > 2)
    LB_D void binvals(long long pos, float F, bool use_up, int bin, float2 *v) {
        const uint32_t sps = one.sps;
        const float2 *ch = use_up ? one.up : one.down;
        double base = (double)F * (double)pos / (double)sps;
        base -= floor(base);
        const float fb = (float)base, fr = F / (float)sps;
        const uint32_t kb = (uint32_t)((bin % (int)sps) + (int)sps) % sps;
        float s[2 * M];
#pragma unroll
        for (int k = 0; k < 2 * M; k++) s[k] = 0.f;
        for (uint32_t n = threadIdx.x; n < sps; n += RX_THREADS) {
            float t = fmaf(fr, (float)n, fb);
            t -= floorf(t);
            float sn, cs;
            sincospif(-2.0f * t, &sn, &cs);
            float2 q = cmul(__ldg(ch + n), make_float2(cs, sn));
            if (kb) q = cmul(q, __ldg(one.tw + (size_t)((unsigned long long)kb * n % sps)));
#pragma unroll
            for (int a = 0; a < M; a++) {
                if (a < (int)m) {
                    const float2 y = cmul(one.x[(size_t)a * stride + pos + n], q);
                    s[2 * a] += y.x; s[2 * a + 1] += y.y;
                }
            }
        }
        float r[4] = {s[0], s[1], s[2], s[3]};
        block_sum<4>(r, *one.sh);
        v[0] = make_float2(r[0], r[1]); v[1] = make_float2(r[2], r[3]);
        if (m > 2) {
            float r2[4] = {s[4], s[5], s[6], s[7]};
            block_sum<4>(r2, *one.sh);
            v[2] = make_float2(r2[0], r2[1]); v[3] = make_float2(r2[2], r2[3]);
        } else {
            v[2] = v[3] = make_float2(0.f, 0.f);
        }
    }
    LB_D void energies(long long pos, float *e) {
        float s[4] = {0.f, 0.f, 0.f, 0.f};
        for (uint32_t n = threadIdx.x; n < one.sps; n += RX_THREADS) {
#pragma unroll
            for (int a = 0; a < M; a++) {
                if (a < (int)m) { const float2 x = one.x[(size_t)a * stride + pos + n]; s[a] += x.x * x.x + x.y * x.y; }
            }
        }
        block_sum<4>(s, *one.sh);
        for (int a = 0; a < M; a++) e[a] = s[a];
    }
    LB_D float energy(long long pos) {
        float e[M], s = 0.f;
        energies(pos, e);
        for (int a = 0; a < M; a++) s += e[a];
        return s;
    }
    // (rs_toa: one.smem holds RX_WARPS * 2 K M floats)
    template <int K> LB_D void tones(long long pos, long long org, float f0, float df, bool use_up, float *p) {
        rs_tones<K, M>(one.x, stride, m, pos, org, use_up ? one.up : one.down, one.sps, f0, df, (float *)one.smem, p);
    }
};

// fine time of arrival: one CTA per frame k, frames[pub[k]] (pub NULL: frames[k]) on receiver group frames[..].stream, rows
// stream * m + a, `stride` apart (m = 1: RsDevOps, as rs_sync_kernel; m >= 2: RsAntOps, as rs_sync_antennas_kernel): rs_toa
// into toa[k] and, when given, (nu_A, nu_B) into nu[k]
template <int SF, int D, bool DRIFT>
__global__ void __launch_bounds__(RX_THREADS)
rs_toa_kernel(const float2 *__restrict__ iq, size_t stride, size_t n_items, uint32_t m, const float2 *down, const float2 *up,
              const float2 *tw, RsParams p, const RsFrame *__restrict__ frames, const uint32_t *__restrict__ pub, double *__restrict__ toa,
              float2 *__restrict__ nu) {
    __shared__ float2 red[RX_WARPS * RS_TOA_GRID * RS_MAX_ANTENNAS];
    __shared__ RxShared sh;
    const RsFrame r = frames[pub ? pub[blockIdx.x] : blockIdx.x];
    const float2 *x = iq + (size_t)r.stream * m * stride;
    RsToa t;
    if (m == 1) {
        RsDevOps<SF, D> ops{x, (long long)n_items, down, up, tw, p.sps, red, &sh, nullptr, 0};
        t = rs_toa<DRIFT>(ops, p, r);
    } else {
        RsAntOps<SF, D> ops{{x, (long long)n_items, down, up, tw, p.sps, red, &sh, nullptr, 0}, stride, m};
        t = rs_toa<DRIFT>(ops, p, r);
    }
    if (threadIdx.x == 0) {
        toa[blockIdx.x] = t.toa;
        if (nu) nu[blockIdx.x] = make_float2(t.nu_a, t.nu_b);
    }
}

// synchronise: one CTA per candidate slot (stream = slot / cap); synchronised frames are appended to `frames`
template <int SF, int D, bool DRIFT>
__global__ void __launch_bounds__(RX_THREADS)
rs_sync_kernel(const float2 *__restrict__ iq, size_t stride, size_t n_items, const float2 *down, const float2 *up, const float2 *tw,
               const float2 *shift, RsParams p, const RsCand *__restrict__ cands, const uint32_t *__restrict__ n_cands, uint32_t cap,
               RsFrame *__restrict__ frames, uint32_t *__restrict__ n_frames, uint32_t frame_cap,
               unsigned long long *__restrict__ hold) {
    extern __shared__ float2 rs_dyn_smem[];
    __shared__ RxShared sh;
    const uint32_t s = blockIdx.x / cap, i = blockIdx.x % cap;
    const uint32_t nc = n_cands[s];
    if (i >= (nc < cap ? nc : cap)) return;
    RsDevOps<SF, D> ops{iq + (size_t)s * stride, (long long)n_items, down, up, tw, p.sps, rs_dyn_smem, &sh, shift, p.hyp};
    const RsFrame r = rs_synchronise<DRIFT>(ops, cands[(size_t)s * cap + i], p, s);
    if (threadIdx.x == 0) {
        if (r.status == RS_INCOMPLETE) atomicMin(hold + s, (unsigned long long)(r.start > 0 ? r.start : 0));
        if (r.status == RS_OK) {
            const uint32_t slot = atomicAdd(n_frames, 1u);
            if (slot < frame_cap) frames[slot] = r;
        }
    }
}

// ... of receivers with m antennas each (group s: rows s * m .. s * m + m - 1): the same procedure over RsAntOps, then the
// channel estimates and combining weights (rs_channels) of every synchronised frame into chan[slot][0..4) (h) and
// chan[slot][4..8) (w); snr_db is the combined SNR
template <int SF, int D, bool DRIFT>
__global__ void __launch_bounds__(RX_THREADS)
rs_sync_antennas_kernel(const float2 *__restrict__ iq, size_t stride, size_t n_items, uint32_t m, const float2 *down, const float2 *up,
                        const float2 *tw, const float2 *shift, RsParams p, const RsCand *__restrict__ cands, const uint32_t *__restrict__ n_cands, uint32_t cap,
                        RsFrame *__restrict__ frames, uint32_t *__restrict__ n_frames, uint32_t frame_cap,
                        unsigned long long *__restrict__ hold, float2 *__restrict__ chan) {
    extern __shared__ float2 rs_dyn_smem[];
    __shared__ RxShared sh;
    const uint32_t s = blockIdx.x / cap, i = blockIdx.x % cap;
    const uint32_t nc = n_cands[s];
    if (i >= (nc < cap ? nc : cap)) return;
    RsAntOps<SF, D> ops{{iq + (size_t)s * m * stride, (long long)n_items, down, up, tw, p.sps, rs_dyn_smem, &sh, shift, p.hyp}, stride, m};
    RsFrame r = rs_synchronise<DRIFT>(ops, cands[(size_t)s * cap + i], p, s);
    float2 h[RS_MAX_ANTENNAS], w[RS_MAX_ANTENNAS];
    if (r.status == RS_OK) r.snr_db = rs_channels<DRIFT>(ops, p, r, m, h, w);
    if (threadIdx.x == 0) {
        if (r.status == RS_INCOMPLETE) atomicMin(hold + s, (unsigned long long)(r.start > 0 ? r.start : 0));
        if (r.status == RS_OK) {
            const uint32_t slot = atomicAdd(n_frames, 1u);
            if (slot < frame_cap) {
                frames[slot] = r;
                for (int a = 0; a < RS_MAX_ANTENNAS; a++) {
                    chan[(size_t)slot * 2 * RS_MAX_ANTENNAS + a] = h[a];
                    chan[(size_t)slot * 2 * RS_MAX_ANTENNAS + RS_MAX_ANTENNAS + a] = w[a];
                }
            }
        }
    }
}

// the synchroniser's window sums on their own (lora_b200_rs_window_dev), so that they can be held to a float64 reference:
// one CTA per query on a group of m rows `stride` apart, with the Ops the synchronise kernels run -- RsDevOps (m = 1,
// rs_sync_kernel) or RsAntOps (m >= 2, rs_sync_antennas_kernel): each antenna's binval and energy of the window at pos,
// and the argmax key of the (combined) spectrum there, dechirped with the chirp of the query
struct RsWindowQuery {
    long long pos;
    float cfo_bins;
    int32_t up, bin, pad;
};

template <int SF, int D>
__global__ void __launch_bounds__(RX_THREADS)
rs_window_kernel(const float2 *__restrict__ x, size_t stride, long long n_items, uint32_t m, const float2 *down, const float2 *up,
                 const float2 *tw, uint32_t sps, const RsWindowQuery *__restrict__ q, float2 *__restrict__ out, float *__restrict__ energy,
                 unsigned long long *__restrict__ key) {
    extern __shared__ float2 rs_dyn_smem[];
    __shared__ RxShared sh;
    const RsWindowQuery w = q[blockIdx.x];
    float2 v[RS_MAX_ANTENNAS];
    float e[RS_MAX_ANTENNAS];
    unsigned long long k;
    if (m == 1) {
        RsDevOps<SF, D> ops{x, n_items, down, up, tw, sps, rs_dyn_smem, &sh, nullptr, 0};
        ops.binvals(w.pos, w.cfo_bins, w.up != 0, w.bin, v);
        e[0] = ops.energy(w.pos);
        k = ops.argmax(w.pos, w.up != 0, 0);
    } else {
        RsAntOps<SF, D> ops{{x, n_items, down, up, tw, sps, rs_dyn_smem, &sh, nullptr, 0}, stride, m};
        ops.binvals(w.pos, w.cfo_bins, w.up != 0, w.bin, v);
        ops.energies(w.pos, e);
        k = ops.argmax(w.pos, w.up != 0, 0);
    }
    if (threadIdx.x == 0) {
        for (uint32_t a = 0; a < m; a++) {
            out[(size_t)blockIdx.x * m + a] = v[a];
            if (energy) energy[(size_t)blockIdx.x * m + a] = e[a];
        }
        key[blockIdx.x] = k;
    }
}

// the channel estimates and weights of given frames on their own (lora_b200_rs_frame_dev): one CTA per frame (group
// frames[f].stream, rows stream * m + a), rs_channels over RsAntOps as rs_sync_antennas_kernel runs it after synchronising,
// into chan[f][0..4) (h), chan[f][4..8) (w) and snr_db[f]
template <int SF, int D, bool DRIFT>
__global__ void __launch_bounds__(RX_THREADS)
rs_channels_kernel(const float2 *__restrict__ iq, size_t stride, size_t n_items, uint32_t m, const float2 *down, const float2 *up,
                   const float2 *tw, RsParams p, const RsFrame *__restrict__ frames, float2 *__restrict__ chan, float *__restrict__ snr_db) {
    __shared__ RxShared sh;
    const RsFrame r = frames[blockIdx.x];
    RsAntOps<SF, D> ops{{iq + (size_t)r.stream * m * stride, (long long)n_items, down, up, tw, p.sps, nullptr, &sh, nullptr, 0}, stride, m};
    float2 h[RS_MAX_ANTENNAS], w[RS_MAX_ANTENNAS];   // (rs_channels takes no argmax: no dynamic shared memory)
    const float s = rs_channels<DRIFT>(ops, p, r, m, h, w);
    if (threadIdx.x == 0) {
        for (int a = 0; a < RS_MAX_ANTENNAS; a++) {
            chan[(size_t)blockIdx.x * 2 * RS_MAX_ANTENNAS + a] = h[a];
            chan[(size_t)blockIdx.x * 2 * RS_MAX_ANTENNAS + RS_MAX_ANTENNAS + a] = w[a];
        }
        snr_db[blockIdx.x] = s;
    }
}

// assemble: frame f's windows k = 0 .. cnt-1 (first data symbol `first` + k) de-rotated by its CFO into
// out[(off_f + k) * sps ..]; off_f = f * 8 and cnt = 8 without tables (the header round).  One CTA per frame.
// With idx, frame f is frames[idx[f]] and its windows go to (offs[f] - off_base) * sps.  Each window is read from its own
// start (rs_sym, the frame's clock offset); samples past n_items read 0.
__global__ void rs_assemble_kernel(const float2 *__restrict__ iq, size_t stride, long long n_items, const RsFrame *__restrict__ frames, uint32_t n_frames,
                                   const uint32_t *__restrict__ idx, uint32_t first, const uint32_t *__restrict__ offs, uint32_t off_base,
                                   const uint32_t *__restrict__ cnts, uint32_t sps, float2 *__restrict__ out) {
    for (uint32_t f = blockIdx.x; f < n_frames; f += gridDim.x) {
        const RsFrame fr = frames[idx ? idx[f] : f];
        const uint32_t off = offs ? offs[f] - off_base : f * 8u, cnt = cnts ? cnts[f] : 8u;
        const float2 *x = iq + (size_t)fr.stream * stride;
        const double rev = (double)fr.cfo_bins / (double)sps;     // revolutions per sample (cfo / fs)
        for (uint32_t k = 0; k < cnt; k++) {
            const long long w = rs_sym(fr.start, rs_data_j((long long)first + k), sps, fr.sfo_ppm);
            float2 *o = out + ((size_t)off + k) * sps;
            for (uint32_t r = threadIdx.x; r < sps; r += blockDim.x) {
                const long long n = w + (long long)r;
                double t = rev * (double)n;                        // phase reduced in double, as tx_channel.cuh
                t -= floor(t);
                float sn, cs;
                sincospif(-2.0f * (float)t, &sn, &cs);
                o[r] = n < n_items ? cmul(x[n], make_float2(cs, sn)) : make_float2(0.f, 0.f);
            }
        }
    }
}

// ... of receivers with m antennas: window sample n of frame f (slot frames[idx[f]], or f) is
// sum_a w_a x_a[n] de-rotated by the frame's CFO, rows fr.stream * m + a, w_a = chan[slot][4 + a] (rs_sync_antennas_kernel)
__global__ void rs_assemble_antennas_kernel(const float2 *__restrict__ iq, size_t stride, long long n_items, uint32_t m,
                                            const RsFrame *__restrict__ frames, const float2 *__restrict__ chan, uint32_t n_frames,
                                            const uint32_t *__restrict__ idx, uint32_t first, const uint32_t *__restrict__ offs,
                                            uint32_t off_base, const uint32_t *__restrict__ cnts, uint32_t sps, float2 *__restrict__ out) {
    for (uint32_t f = blockIdx.x; f < n_frames; f += gridDim.x) {
        const uint32_t slot = idx ? idx[f] : f;
        const RsFrame fr = frames[slot];
        const uint32_t off = offs ? offs[f] - off_base : f * 8u, cnt = cnts ? cnts[f] : 8u;
        const float2 *x = iq + (size_t)fr.stream * m * stride;
        float2 w[RS_MAX_ANTENNAS];
        for (int a = 0; a < RS_MAX_ANTENNAS; a++) w[a] = chan[(size_t)slot * 2 * RS_MAX_ANTENNAS + RS_MAX_ANTENNAS + a];
        const double rev = (double)fr.cfo_bins / (double)sps;
        for (uint32_t k = 0; k < cnt; k++) {
            const long long ws = rs_sym(fr.start, rs_data_j((long long)first + k), sps, fr.sfo_ppm);
            float2 *o = out + ((size_t)off + k) * sps;
            for (uint32_t r = threadIdx.x; r < sps; r += blockDim.x) {
                const long long n = ws + (long long)r;
                if (n >= n_items) { o[r] = make_float2(0.f, 0.f); continue; }
                double t = rev * (double)n;
                t -= floor(t);
                float sn, cs;
                sincospif(-2.0f * (float)t, &sn, &cs);
                float2 y = make_float2(0.f, 0.f);
#pragma unroll
                for (int a = 0; a < RS_MAX_ANTENNAS; a++)
                    if (a < (int)m) y = cfma(w[a], x[(size_t)a * stride + n], y);
                o[r] = cmul(y, make_float2(cs, sn));
            }
        }
    }
}

// header round: one thread per frame
__global__ void rs_header_kernel(RsFrame *__restrict__ frames, const uint32_t *__restrict__ n_frames, uint32_t cap, RxParams p,
                                 uint8_t phdr1, const uint32_t *__restrict__ bins, uint32_t implicit_len) {
    uint32_t n = *n_frames;
    if (n > cap) n = cap;
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    RxStreamState st;
    frames[f].n_payload = rs_header(&st, p, phdr1, bins + (size_t)f * 8, implicit_len);
}

// payload round: one thread per published frame (index list `pub`), the header replayed from its bins
__global__ void rs_frame_kernel(const RsFrame *__restrict__ frames, const uint32_t *__restrict__ pub, const uint32_t *__restrict__ seq,
                                uint32_t n_pub, RxParams p, uint8_t phdr1, const uint32_t *__restrict__ hdr_bins,
                                const uint32_t *__restrict__ bins, const uint32_t *__restrict__ offs, uint32_t implicit_len,
                                RxFrameRec *__restrict__ recs) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_pub) return;
    const uint32_t f = pub[k];
    const RsFrame fr = frames[f];
    RxStreamState st;
    rs_header(&st, p, phdr1, hdr_bins + (size_t)f * 8, implicit_len);
    const float snr = exp10f(fr.snr_db / 10.0f);          // loratap's SNR byte: the estimate in dB
    rs_frame(&st, p, bins + offs[k], fr.n_payload, recs + k, fr.stream, seq[k], snr > 1e-30f ? snr : 1e-30f);
}

// soft decisions of the header round: one thread per frame, llr[f][8][sf - 2] -> corrected bins[f][8]
__global__ void rs_soft_header_kernel(uint32_t n, RxParams p, uint8_t phdr1, const float *__restrict__ llr, uint32_t *__restrict__ bins) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    rs_soft_header(rs_code(p, phdr1), llr + (size_t)f * 8 * (p.sf - 2u), bins + (size_t)f * 8, nullptr);
}

// soft decisions of the payload round: one thread per published frame (index list `pub`), its windows at offs[k] of
// llr (tx_ppm values each) and bins
__global__ void rs_soft_payload_kernel(const RsFrame *__restrict__ frames, const uint32_t *__restrict__ pub, uint32_t n_pub, RxParams p,
                                       uint8_t phdr1, const uint32_t *__restrict__ hdr_bins, const uint32_t *__restrict__ offs,
                                       uint32_t implicit_len, const float *__restrict__ llr, uint32_t *__restrict__ bins) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_pub) return;
    const uint32_t f = pub[k];
    rs_soft_payload(p, phdr1, hdr_bins + (size_t)f * 8, frames[f].n_payload, implicit_len,
                    llr + (size_t)offs[k] * tx_ppm(rs_code(p, phdr1)), bins + offs[k]);
}

// CRC-aided list decoding of the payload round: one warp per published frame (index list `pub`), after
// rs_soft_payload_kernel.  hllr: the header round's LLRs (frame f at f * 8 * (sf - 2)), llr / bins / offs as
// rs_soft_payload_kernel.  A recovered frame's changed blocks are re-encoded into hdr_bins and bins; recovered[k] = 1 then,
// else 0.  Lane l picks slots l, l + 32, ...; the list is chosen in K rounds of a warp-wide minimum; the 2^K subsets are
// split into 32 runs of consecutive Gray-code indices, one XOR per step.
constexpr int RS_CRC_WARPS = 4;

LB_D unsigned long long rs_warp_min(unsigned long long v) {
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w < v ? w : v;
    }
    return v;
}

__global__ void __launch_bounds__(32 * RS_CRC_WARPS)
rs_crc_list_kernel(const RsFrame *__restrict__ frames, const uint32_t *__restrict__ pub, uint32_t n_pub, RxParams p, uint8_t phdr1,
                   uint32_t K, uint32_t *__restrict__ hdr_bins, const uint32_t *__restrict__ offs, uint32_t implicit_len,
                   const float *__restrict__ hllr, const float *__restrict__ llr, uint32_t *__restrict__ bins,
                   uint8_t *__restrict__ recovered) {
    __shared__ uint8_t s_nib[RS_CRC_WARPS][RS_CRC_MAX_SLOTS], s_alt[RS_CRC_WARPS][RS_CRC_MAX_SLOTS];
    __shared__ float s_gap[RS_CRC_WARPS][RS_CRC_MAX_SLOTS];
    __shared__ uint32_t s_q[RS_CRC_WARPS][RS_CRC_MAX_LIST], s_delta[RS_CRC_WARPS][RS_CRC_MAX_LIST];
    __shared__ float s_lgap[RS_CRC_WARPS][RS_CRC_MAX_LIST];
    const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31u, k = blockIdx.x * RS_CRC_WARPS + w;
    if (k >= n_pub) return;                           // (whole warps)
    const uint32_t f = pub[k];
    const RsCrcFrame cf = rs_crc_frame(p, phdr1, hdr_bins + (size_t)f * 8, frames[f].n_payload, implicit_len);
    uint8_t *nib = s_nib[w], *alt = s_alt[w];
    float *gap = s_gap[w];
    if (cf.L == 0u || cf.n_slots > RS_CRC_MAX_SLOTS || cf.h + 2u * (cf.L + 2u) > cf.n_slots) {
        if (lane == 0) recovered[k] = 0;
        return;
    }
    // metrics of every slot: the soft decoder's nibble, the runner-up, the gap
    const float *hl = hllr + (size_t)f * 8 * cf.hppm, *pl = llr + (size_t)offs[k] * cf.ppm;
    for (uint32_t q = lane; q < cf.n_slots; q += 32u) {
        const RsSoftPick r = rs_crc_pick(cf, hl, pl, q);
        nib[q] = (uint8_t)r.s1; alt[q] = (uint8_t)r.s2; gap[q] = r.gap;
    }
    __syncwarp();
    const uint32_t S0 = rs_crc_syndrome(cf, nib);
    if (S0 == 0u) {
        if (lane == 0) recovered[k] = 0;
        return;
    }
    // the list: the K candidates of least gap, the lowest slot (= nibble index) on ties
    const uint32_t q0 = cf.h, q1 = cf.h + 2u * (cf.L - 2u);          // (rs_crc_candidate)
    uint32_t n = 0;
    for (; n < K; n++) {
        unsigned long long key = ~0ull;
        for (uint32_t q = q0 + lane; q < q1; q += 32u)
            if (!(alt[q] & 0x80u)) { const unsigned long long c = rs_crc_key(gap[q], q); key = c < key ? c : key; }
        key = rs_warp_min(key);
        if (key == ~0ull) break;
        const uint32_t q = (uint32_t)key;
        if (lane == 0) { alt[q] |= 0x80u; s_q[w][n] = q; s_lgap[w][n] = gap[q]; }
        __syncwarp();
    }
    if (lane < n) {
        const uint32_t q = s_q[w][lane];
        s_delta[w][lane] = rs_crc_delta(cf.L, q - cf.h, nib[q] ^ (alt[q] & 15u));
    }
    __syncwarp();
    // the subsets: lane l walks Gray-code indices [l per, (l + 1) per)
    const uint32_t total = 1u << n, per = total > 32u ? total >> 5 : 1u, g0 = lane * per;
    unsigned long long best = ~0ull;
    if (g0 < total) {
        uint32_t mask = g0 ^ (g0 >> 1), syn = 0;
        for (uint32_t j = 0; j < n; j++)
            if (mask >> j & 1u) syn ^= s_delta[w][j];
        for (uint32_t t = 0; t < per; t++) {
            if (t) {
                const uint32_t b = (uint32_t)(__ffs((int)(g0 + t)) - 1);
                mask ^= 1u << b;
                syn ^= s_delta[w][b];
            }
            if (syn == S0) {
                const unsigned long long c = rs_crc_key(rs_crc_cost(s_lgap[w], mask), mask);
                best = c < best ? c : best;
            }
        }
    }
    best = rs_warp_min(best);
    if (best == ~0ull) {
        if (lane == 0) recovered[k] = 0;
        return;
    }
    const uint32_t mask = (uint32_t)best;
    if (lane < n && (mask >> lane & 1u)) { const uint32_t q = s_q[w][lane]; nib[q] = alt[q] & 15u; }
    __syncwarp();
    uint32_t *hb = hdr_bins + (size_t)f * 8, *pb = bins + offs[k];
    for (uint32_t j = 0; j < n; j++) {
        if (!(mask >> j & 1u)) continue;
        const uint32_t q = s_q[w][j];
        if (lane < rs_crc_block_bins(cf, q)) rs_crc_block_out(cf, q, hb, pb)[lane] = rs_crc_block_bin(cf, nib, q, lane);
    }
    if (lane == 0) recovered[k] = 1;
}
#endif  // __CUDACC__

}  // namespace lb
