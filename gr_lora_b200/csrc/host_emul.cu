// host_emul.cu -- CPU entry points for the __host__ __device__ phase functions (tests only).
// Lets the non-GPU test-suite run the kernels' index arithmetic, twiddles and integer chain
// on the host and compare them with the oracle, and drive the owning buffer type of
// cuda_owned.h.  Not part of liblora_b200.so.
#include "cuda_owned.h"
#include "dispatch.h"
#include "k1_fft.cuh"
#include "k1_llr.cuh"
#include "k1_warp.cuh"
#include "k1_group.cuh"
#include "k1_sf10.cuh"
#include "k1_rows.cuh"
#include "int_chain.cuh"
#include "rx_stream.cuh"
#include "rx_sync.cuh"
#include "tx_channel.cuh"
#include "tx_encode.cuh"

#include <algorithm>
#include <cstring>
#include <vector>

extern "C" {

// k1_fft_kernel<SF, D> on the host, D = osr = sps / N (8, 2, 16 or 32); -1 for another SF or D
int lb_k1_emulate_osr(int sf, int osr, const float2 *x, size_t n_symbols, const float2 *chirp, const float2 *tw, uint32_t *bins,
                      float *mags) {
    const lb::K1Args a{x, chirp, tw, n_symbols};
    return lb::with_sf_osr(sf, osr, [] { return -1; }, [&](auto SF, auto D) { lb::k1_emulate<SF, D>(a, bins, mags); return 0; });
}

// k1_antennas_kernel<SF, D> on the host for one group: m rows of n_symbols windows, row_stride samples apart -> the argmax
// of the combined spectrum sum_a |tmp_a|^2 and its sqrt; -1 for another SF or D
int lb_k1_antennas_emulate_osr(int sf, int osr, const float2 *x, size_t row_stride, uint32_t m, size_t n_symbols, const float2 *chirp,
                               const float2 *tw, uint32_t *bins, float *mags) {
    const lb::K1Args a{x, chirp, tw, n_symbols};
    return lb::with_sf_osr(sf, osr, [] { return -1; }, [&](auto SF, auto D) {
        lb::k1_antennas_emulate<SF, D>(a, row_stride, m, bins, mags);
        return 0;
    });
}

int lb_k1_emulate(int sf, const float2 *x, size_t n_symbols, const float2 *chirp, const float2 *tw,
                  uint32_t *bins, float *mags) {
    return lb_k1_emulate_osr(sf, 8, x, n_symbols, chirp, tw, bins, mags);
}

// the LLR demodulator k1_llr_kernel<SF, D> (k1_llr.cuh) on the host, D = osr: llrs[i * ppm ..], bins may be NULL
int lb_k1_llr_emulate_osr(int sf, int osr, const float2 *x, size_t n_symbols, const float2 *chirp, const float2 *tw, int reduced,
                          float *llrs, uint32_t *bins) {
    const lb::K1Args a{x, chirp, tw, n_symbols};
    return lb::with_sf_osr(sf, osr, [] { return -1; }, [&](auto SF, auto D) {
        lb::k1_llr_emulate<SF, D>(a, reduced != 0, llrs, bins);
        return 0;
    });
}

// ... at fs/bw = 8
int lb_k1_llr_emulate(int sf, const float2 *x, size_t n_symbols, const float2 *chirp, const float2 *tw, int reduced, float *llrs,
                      uint32_t *bins) {
    return lb_k1_llr_emulate_osr(sf, 8, x, n_symbols, chirp, tw, reduced, llrs, bins);
}

int lb_k1_emulate_warp_sf7(const float2 *x, size_t n_symbols, const float2 *chirp, const float2 *tw, uint32_t *bins, float *mags) {
    lb::K1Args a{x, chirp, tw, n_symbols};
    lb::w7_emulate(a, bins, mags);
    return 0;
}

int lb_k1_emulate_group(int sf, const float2 *x, size_t n_symbols, const float2 *chirp, const float2 *tw, uint32_t *bins, float *mags) {
    lb::K1Args a{x, chirp, tw, n_symbols};
    switch (sf) {
    case 8: lb::g_emulate<8>(a, bins, mags); break;
    case 9: lb::g_emulate<9>(a, bins, mags); break;
    case 10: lb::s10_emulate(a, bins, mags); break;
    default: return -1;
    }
    return 0;
}

int lb_k1_emulate_rows(int sf, const float2 *x, size_t n_symbols, const float2 *chirp, const float2 *tw, uint32_t *bins, float *mags) {
    lb::K1Args a{x, chirp, tw, n_symbols};
    if (sf == 11) lb::r_emulate<11>(a, bins, mags);
    else if (sf == 12) lb::r_emulate<12>(a, bins, mags);
    else return -1;
    return 0;
}


// the counter-based generator of the transmitter / channel kernels (tx_channel.cuh), on the host
void lb_emul_philox4x32_10(const uint32_t *ctr, const uint32_t *key, uint32_t *out) {
    uint32_t c[4] = {ctr[0], ctr[1], ctr[2], ctr[3]};
    lb::philox4x32_10(c, key[0], key[1]);
    for (int i = 0; i < 4; i++) out[i] = c[i];
}

// the stream kernels' arg() (lora_common.cuh), on the host
void lb_emul_atan2f(const float *y, const float *x, float *out, size_t n) {
    for (size_t i = 0; i < n; i++) out[i] = lb::lb_atan2f(y[i], x[i]);
}

uint32_t lb_emul_decode(const uint8_t *cw, uint32_t n_cw, int is_header, uint32_t cr, uint8_t *out, uint32_t cap) {
    uint32_t n = lb::decode_len_bytes(lb::decode_len_words(n_cw, is_header), cr);
    if (n > cap) n = cap;
    for (uint32_t i = 0; i < n; i++) out[i] = lb::decode_byte(cw, n_cw, is_header, cr, i);
    return n;
}
void lb_emul_deinterleave(const uint32_t *words, uint32_t n_words, uint32_t ppm, uint8_t *out) { lb::deinterleave_block(words, n_words, ppm, out); }
uint32_t lb_emul_reduce_bin(uint32_t bin, uint32_t n_hdr) { return lb::reduce_bin(bin, n_hdr); }
uint32_t lb_emul_gray(uint32_t bin) { return lb::gray_encode(bin); }
uint8_t lb_emul_hamming84_decode(uint8_t cw) { return lb::hamming84_decode(cw); }
uint8_t lb_emul_hamming84_encode(uint8_t v) { return lb::hamming84_encode(v); }
uint8_t lb_emul_deshuffle(uint8_t v) { return lb::deshuffle_byte(v); }
int32_t lb_emul_payload_symbols(uint32_t len, uint32_t cr, uint32_t sf, int rr) { return lb::payload_symbols(len, cr, sf, rr); }

// the frame encoder of tx_encode_kernel (tx_encode.cuh), one frame on the host: writes its data symbols' chirp shifts and
// returns their number, 0 for a length the encoder refuses or more than cap symbols
uint32_t lb_emul_tx_encode(const uint8_t *payload, uint32_t len, uint32_t sf, uint32_t cr, int implicit, int crc, int reduced_rate,
                           uint32_t *shifts, uint32_t cap) {
    const lb::TxCode c{sf, cr, implicit ? 0u : 1u, crc ? 1u : 0u, reduced_rate ? 1u : 0u};
    if (!lb::tx_length_ok(c, len)) return 0;
    const uint32_t n = lb::tx_data_symbols(c, len);
    if (n > cap) return 0;
    for (uint32_t i = 0; i < n; i++) shifts[i] = lb::tx_symbol_shift(c, payload, len, i);
    return n;
}
// the soft block decoder of the dechirp receiver (rx_sync.cuh) on given LLRs.  Header block: llr[8][sf - 2] -> 8 corrected
// bins and sf - 2 nibbles (nib may be NULL); returns the frame's coding rate (from the header when explicit).  Payload block
// b of a frame with coding rate cr: llr[4 + cr][ppm] -> 4 + cr corrected bins and ppm nibbles.
uint32_t lb_emul_soft_header(uint32_t sf, uint32_t cr, int implicit, int crc, int reduced_rate, const float *llr, uint32_t *bins,
                             uint32_t *nib) {
    const lb::TxCode c{sf, cr, implicit ? 0u : 1u, crc ? 1u : 0u, reduced_rate ? 1u : 0u};
    return lb::rs_soft_header(c, llr, bins, nib).cr;
}
void lb_emul_soft_block(uint32_t sf, uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t b, const float *llr, uint32_t *bins,
                        uint32_t *nib) {
    const lb::TxCode c{sf, cr, implicit ? 0u : 1u, crc ? 1u : 0u, reduced_rate ? 1u : 0u};
    lb::rs_soft_block(c, b, llr, bins, nib);
}
uint32_t lb_emul_header_checksum(uint32_t length, uint32_t cr, uint32_t crc) { return lb::header_checksum(length, cr, crc); }

// the stream kernels' per-step bookkeeping (rx_stream.cuh) over a recorded step sequence: state at the start of step i,
// its metric (DETECT: autocorrelation, FIND_SFD: downchirp correlation) and its bin (-1: not demodulated).  next[i] gets
// the state step i leads to (-1 for SYNC, PAUSE and STOP steps, which need no bookkeeping), frames the queued records
// with their code words; returns the number of frames (at most cap are written)
uint32_t lb_emul_rx_replay(const int32_t *states, const float *metrics, const int32_t *bins, size_t n_steps, uint32_t sf,
                           int implicit, uint32_t cr, int crc, int reduced_rate, int32_t *next, lb::RxFrameRec *frames, uint32_t cap) {
    lb::RxParams p;
    memset(&p, 0, sizeof p);
    p.sf = sf; p.n_bins_hdr = 1u << (sf - 2); p.implicit = implicit; p.reduced_rate = reduced_rate;
    lb::RxStreamState st;
    lb::rx_state_init(&st, (uint8_t)(((cr & 7u) << 5) | (crc ? 1u << 4 : 0u)));
    uint32_t n_frames = 0;
    for (size_t i = 0; i < n_steps; i++) {
        const int s = states[i];
        next[i] = -1;
        if (s == LORA_B200_DETECT) next[i] = lb::rx_detect_commit(&st, 1.0f, 1.0f, 1u, metrics[i]);   // (no energies recorded)
        else if (s == LORA_B200_FIND_SFD) next[i] = lb::rx_sfd_commit(&st, metrics[i]);
        else if (s == LORA_B200_DECODE_HEADER || s == LORA_B200_DECODE_PAYLOAD) {
            const lb::RxSymbolResult r = lb::rx_symbol_commit(&st, p, s == LORA_B200_DECODE_HEADER, bins[i] >= 0, bins[i]);
            next[i] = r == lb::RX_HEADER_DONE ? LORA_B200_DECODE_PAYLOAD : r == lb::RX_FRAME_DONE ? LORA_B200_DETECT : s;
            if (r == lb::RX_FRAME_DONE) {
                if (n_frames < cap) {
                    lb::RxFrameRec *fr = frames + n_frames;
                    memcpy(fr->cw, st.demodulated, st.n_demod);
                    lb::rx_frame_record(fr, &st, 0, implicit);
                }
                n_frames++;
                lb::rx_frame_reset(&st);
            }
        }
    }
    return n_frames;
}
uint32_t lb_emul_rx_frame_rec_size(void) { return (uint32_t)sizeof(lb::RxFrameRec); }

}  // extern "C"

namespace {

// the windows of rs_synchronise on the host: K1 through its CPU emulation, the bin sums as plain loops in double
struct RsHostOps {
    static constexpr int M = 1;
    const float2 *x;
    long long n_items;
    const float2 *down, *up, *tw;
    uint32_t sps, sf, osr;
    const float2 *shift;               // the shifted tables of hypotheses -hyp..hyp (rs_shift_tables)
    int hyp;
    bool in_range(long long pos) const { return pos >= 0 && pos + (long long)sps <= n_items; }
    void binvals(long long pos, float F, bool use_up, int bin, float2 *v) { v[0] = binval(pos, F, use_up, bin); }
    const float2 *chirp(bool use_up, int c) const {
        return c == 0 ? (use_up ? up : down) : shift + ((size_t)(c + hyp) * 2 + (use_up ? 1 : 0)) * sps;
    }
    unsigned long long argmax(long long pos, bool use_up, int c) {
        uint32_t b;
        float m;
        lb_k1_emulate_osr((int)sf, (int)osr, x + pos, 1, chirp(use_up, c), tw, &b, &m);
        return lb::pack_key(m * m, b);
    }
    float2 binval(long long pos, float F, bool use_up, int bin) {
        const float2 *ch = use_up ? up : down;
        double re = 0.0, im = 0.0;
        for (uint32_t n = 0; n < sps; n++) {
            const double a = -2.0 * M_PI * ((double)F * (double)(pos + n) / sps + (double)bin * n / sps);
            const float2 v = lb::cmul(x[pos + n], ch[n]);
            re += v.x * cos(a) - v.y * sin(a);
            im += v.x * sin(a) + v.y * cos(a);
        }
        return make_float2((float)re, (float)im);
    }
    float energy(long long pos) {
        double e = 0.0;
        for (uint32_t n = 0; n < sps; n++) e += (double)x[pos + n].x * x[pos + n].x + (double)x[pos + n].y * x[pos + n].y;
        return (float)e;
    }
    // rs_toa's window powers: |binval(pos, f0 + k df, use_up, 0)|^2, each frequency formed in double, the phase counted from org
    template <int K> void tones(long long pos, long long org, float f0, float df, bool use_up, float *p) {
        const float2 *ch = use_up ? up : down;
        for (int k = 0; k < K; k++) {
            const double f = (double)f0 + (double)k * (double)df;
            double re = 0.0, im = 0.0;
            for (uint32_t n = 0; n < sps; n++) {
                const double a = -2.0 * M_PI * f * (double)(pos - org + n) / sps;
                const float2 v = lb::cmul(x[pos + n], ch[n]);
                re += v.x * cos(a) - v.y * sin(a);
                im += v.x * sin(a) + v.y * cos(a);
            }
            p[k] = (float)(re * re + im * im);
        }
    }
};

// ... of a receiver with m antennas, rows one.x + a * one.n_items: the combined K1 argmax through k1_antennas_emulate
struct RsHostAntOps {
    static constexpr int M = lb::RS_MAX_ANTENNAS;
    RsHostOps one;
    uint32_t m;
    bool in_range(long long pos) const { return one.in_range(pos); }
    RsHostOps row(uint32_t a) const { RsHostOps o = one; o.x = one.x + (size_t)a * one.n_items; return o; }
    unsigned long long argmax(long long pos, bool use_up, int c) {
        uint32_t b;
        float mg;
        lb_k1_antennas_emulate_osr((int)one.sf, (int)one.osr, one.x + pos, (size_t)one.n_items, m, 1, one.chirp(use_up, c), one.tw, &b, &mg);
        return lb::pack_key(mg * mg, b);
    }
    void binvals(long long pos, float F, bool use_up, int bin, float2 *v) {
        for (uint32_t a = 0; a < (uint32_t)M; a++) v[a] = a < m ? row(a).binval(pos, F, use_up, bin) : make_float2(0.f, 0.f);
    }
    void energies(long long pos, float *e) {
        for (uint32_t a = 0; a < (uint32_t)M; a++) e[a] = a < m ? row(a).energy(pos) : 0.f;
    }
    float energy(long long pos) {
        float e[M], s = 0.f;
        energies(pos, e);
        for (int a = 0; a < M; a++) s += e[a];
        return s;
    }
    template <int K> void tones(long long pos, long long org, float f0, float df, bool use_up, float *p) {
        for (int k = 0; k < K; k++) p[k] = 0.f;
        for (uint32_t a = 0; a < m; a++) {
            float q[K];
            row(a).tones<K>(pos, org, f0, df, use_up, q);
            for (int k = 0; k < K; k++) p[k] += q[k];
        }
    }
};

// data windows first .. first + cnt - 1 of frame r (each from its own start, rs_sym), de-rotated by its CFO
std::vector<float2> rs_host_windows(const RsHostOps &o, const lb::RsFrame &r, uint32_t first, uint32_t cnt) {
    std::vector<float2> w((size_t)cnt * o.sps);
    for (uint32_t k = 0; k < cnt; k++) {
        const long long s0 = lb::rs_sym(r.start, lb::rs_data_j((long long)first + k), o.sps, r.sfo_ppm);
        for (uint32_t i = 0; i < o.sps; i++) {
            const long long n = s0 + i;
            const double a = -2.0 * M_PI * (double)r.cfo_bins * (double)n / o.sps;
            const float2 v = o.x[n];
            w[(size_t)k * o.sps + i] = make_float2((float)(v.x * cos(a) - v.y * sin(a)), (float)(v.x * sin(a) + v.y * cos(a)));
        }
    }
    return w;
}

// ... through K1
void rs_host_bins(const RsHostOps &o, const lb::RsFrame &r, uint32_t first, uint32_t cnt, std::vector<uint32_t> &bins) {
    const std::vector<float2> w = rs_host_windows(o, r, first, cnt);
    bins.resize(cnt);
    std::vector<float> mags(cnt);
    lb_k1_emulate_osr((int)o.sf, (int)o.osr, w.data(), cnt, o.down, o.tw, bins.data(), mags.data());
}

// ... through the LLR demodulator
void rs_host_llrs(const RsHostOps &o, const lb::RsFrame &r, uint32_t first, uint32_t cnt, bool reduced, std::vector<float> &llr) {
    const std::vector<float2> w = rs_host_windows(o, r, first, cnt);
    llr.resize((size_t)cnt * (reduced ? o.sf - 2 : o.sf));
    lb_k1_llr_emulate_osr((int)o.sf, (int)o.osr, w.data(), cnt, o.down, o.tw, reduced, llr.data(), nullptr);
}

// rs_crc_list_kernel's procedure as plain loops: the whole list sorted, every subset in turn.  Corrects hb[8] and pb[n_payload]
// in place; returns 1 when the frame was recovered.
int rs_host_crc_list(const lb::RxParams &rp, uint8_t phdr1, uint32_t implicit_len, uint32_t K, int32_t n_payload, const float *hllr,
                     const float *llr, uint32_t *hb, uint32_t *pb) {
    const lb::RsCrcFrame cf = lb::rs_crc_frame(rp, phdr1, hb, n_payload, implicit_len);
    if (cf.L == 0u || cf.n_slots > lb::RS_CRC_MAX_SLOTS || cf.h + 2u * (cf.L + 2u) > cf.n_slots) return 0;
    std::vector<uint8_t> nib(cf.n_slots), alt(cf.n_slots);
    std::vector<float> gap(cf.n_slots);
    for (uint32_t q = 0; q < cf.n_slots; q++) {
        const lb::RsSoftPick r = lb::rs_crc_pick(cf, hllr, llr, q);
        nib[q] = (uint8_t)r.s1; alt[q] = (uint8_t)r.s2; gap[q] = r.gap;
    }
    const uint32_t S0 = lb::rs_crc_syndrome(cf, nib.data());
    if (S0 == 0u) return 0;
    std::vector<unsigned long long> cand;
    for (uint32_t q = 0; q < cf.n_slots; q++)
        if (lb::rs_crc_candidate(cf, q)) cand.push_back(lb::rs_crc_key(gap[q], q));
    std::sort(cand.begin(), cand.end());
    const uint32_t n = std::min<uint32_t>(K, (uint32_t)cand.size());
    uint32_t lq[lb::RS_CRC_MAX_LIST], delta[lb::RS_CRC_MAX_LIST];
    float lgap[lb::RS_CRC_MAX_LIST];
    for (uint32_t j = 0; j < n; j++) {
        lq[j] = (uint32_t)cand[j];
        lgap[j] = gap[lq[j]];
        delta[j] = lb::rs_crc_delta(cf.L, lq[j] - cf.h, nib[lq[j]] ^ alt[lq[j]]);
    }
    unsigned long long best = ~0ull;
    for (uint32_t mask = 1; mask < (1u << n); mask++) {
        uint32_t syn = 0;
        for (uint32_t j = 0; j < n; j++)
            if (mask >> j & 1u) syn ^= delta[j];
        if (syn == S0) best = std::min(best, lb::rs_crc_key(lb::rs_crc_cost(lgap, mask), mask));
    }
    if (best == ~0ull) return 0;
    const uint32_t mask = (uint32_t)best;
    for (uint32_t j = 0; j < n; j++)
        if (mask >> j & 1u) nib[lq[j]] = alt[lq[j]];
    for (uint32_t j = 0; j < n; j++) {
        if (!(mask >> j & 1u)) continue;
        uint32_t *out = lb::rs_crc_block_out(cf, lq[j], hb, pb);
        for (uint32_t i = 0; i < lb::rs_crc_block_bins(cf, lq[j]); i++) out[i] = lb::rs_crc_block_bin(cf, nib.data(), lq[j], i);
    }
    return 1;
}

// the rates the receiver runs at: those of the K1 kernels
bool rs_host_osr(uint32_t osr) {
    return lb::with_osr((int)osr, [] { return false; }, [](auto) { return true; });
}

// the receive path of lb_emul_rx_receive_osr (m = 1) and lb_emul_rx_receive_antennas (m rows of n_items each, x[a * n_items
// ..]); with several antennas chan[f * m ..] gets each synchronised frame's channel estimates h (may be NULL).  max_cfo_bins
// > 0: the coarse-offset search of rx_params.wide_cfo up to that CFO; else |CFO| <= N / 4 without it.
uint32_t rs_host_receive(const float2 *x, size_t n_items, uint32_t m, const float2 *down, const float2 *up, const float2 *tw, uint32_t sf,
                         uint32_t osr, uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t sync_word, uint32_t implicit_len,
                         uint32_t min_preamble, float sfo_ppm, double carrier_hz, int soft, long long *start, float *cfo_bins,
                         float *snr_db, int32_t *status, float *sfo, uint8_t *payload, uint32_t *len, float2 *chan, uint32_t cap,
                         uint32_t crc_list = 0, uint8_t *crc_status = nullptr, float max_cfo_bins = 0.f, double *toa = nullptr) {
    if (!rs_host_osr(osr)) return 0;
    const uint32_t N = 1u << sf, sps = osr * N;
    const double bin_hz = 125e3 / N;
    lb::RsParams p{sps, N, osr, sfo_ppm, min_preamble ? min_preamble : 5u, {((sync_word >> 4) & 15u) * 8u % N, (sync_word & 15u) * 8u % N},
                   max_cfo_bins > 0.f ? max_cfo_bins : (float)N / 4.0f, carrier_hz > 0.0 ? (float)(1e6 * bin_hz / carrier_hz) : 0.0f, 0};
    p.hyp = lb::rs_hypotheses(p.max_cfo_bins, N);
    if (p.hyp > lb::rs_max_hyp((int)osr)) return 0;
    std::vector<float2> shift((size_t)(2 * p.hyp + 1) * 2 * sps);
    lb::rs_shift_tables(down, up, sps, osr, p.hyp, shift.data());
    RsHostOps o{x, (long long)n_items, down, up, tw, sps, sf, osr, shift.data(), p.hyp};
    RsHostAntOps oa{o, m};
    // screen: both phases of every hypothesis, screen s = 2 (c + hyp) + ph (c = 0 with the plain down-chirp)
    const int ns = 2 * (2 * p.hyp + 1);
    std::vector<std::vector<uint32_t>> bins(ns);
    std::vector<std::vector<float>> mags(ns);
    std::vector<const uint32_t *> bp(ns);
    std::vector<const float *> mp(ns);
    uint32_t n[2];
    for (int ph = 0; ph < 2; ph++) n[ph] = n_items >= sps + ph * sps / 2 ? (uint32_t)((n_items - ph * sps / 2) / sps) : 0u;
    for (int s = 0; s < ns; s++) {
        const int ph = s & 1;
        const float2 *ch = o.chirp(false, s / 2 - p.hyp);
        bins[s].resize(n[ph] + 1);
        mags[s].resize(n[ph] + 1);
        if (n[ph] && m == 1) lb_k1_emulate_osr((int)sf, (int)osr, x + ph * sps / 2, n[ph], ch, tw, bins[s].data(), mags[s].data());
        else if (n[ph]) lb_k1_antennas_emulate_osr((int)sf, (int)osr, x + ph * sps / 2, n_items, m, n[ph], ch, tw, bins[s].data(), mags[s].data());
        bp[s] = bins[s].data();
        mp[s] = mags[s].data();
    }
    std::vector<lb::RsCand> cands(64);
    long long dropped;
    const uint32_t nc = std::min<uint32_t>(lb::rs_detect_stream<lb::rs_max_screens(32)>(bp.data(), mp.data(), n, p, cands.data(), 64, &dropped), 64u);
    lb::RxParams rp;
    memset(&rp, 0, sizeof rp);
    rp.sf = sf; rp.n_bins = N; rp.n_bins_hdr = N / 4; rp.sps = sps; rp.decim = osr; rp.implicit = implicit; rp.reduced_rate = reduced_rate;
    const uint8_t phdr1 = (uint8_t)(((cr & 7u) << 5) | (crc ? 1u << 4 : 0u));
    uint32_t nf = 0;
    std::vector<float2> y;                            // several antennas: the combined row sum_a w_a x_a of one frame
    for (uint32_t c = 0; c < nc && nf < cap; c++) {
        const bool drift = lb::rs_drift(p);
        lb::RsFrame r = m == 1 ? (drift ? lb::rs_synchronise<true>(o, cands[c], p, 0) : lb::rs_synchronise<false>(o, cands[c], p, 0))
                               : (drift ? lb::rs_synchronise<true>(oa, cands[c], p, 0) : lb::rs_synchronise<false>(oa, cands[c], p, 0));
        if (r.status == lb::RS_REJECT) continue;
        RsHostOps od = o;                             // the row the data windows are read from
        if (m > 1 && r.status == lb::RS_OK) {
            float2 h[lb::RS_MAX_ANTENNAS], w[lb::RS_MAX_ANTENNAS];
            r.snr_db = drift ? lb::rs_channels<true>(oa, p, r, m, h, w) : lb::rs_channels<false>(oa, p, r, m, h, w);
            if (chan)
                for (uint32_t a = 0; a < m; a++) chan[(size_t)nf * m + a] = h[a];
            y.assign(n_items, make_float2(0.f, 0.f));
            for (size_t i = 0; i < n_items; i++)
                for (uint32_t a = 0; a < m; a++) y[i] = lb::cfma(w[a], x[(size_t)a * n_items + i], y[i]);
            od.x = y.data();
        }
        start[nf] = r.start; cfo_bins[nf] = r.cfo_bins; snr_db[nf] = r.snr_db; status[nf] = 2; len[nf] = 0;
        if (toa) {
            toa[nf] = NAN;
            if (r.status == lb::RS_OK) {
                const lb::RsToa t = m == 1 ? (drift ? lb::rs_toa<true>(o, p, r) : lb::rs_toa<false>(o, p, r))
                                           : (drift ? lb::rs_toa<true>(oa, p, r) : lb::rs_toa<false>(oa, p, r));
                toa[nf] = t.toa;
            }
        }
        if (crc_status) crc_status[nf] = LORA_CRC_NONE;
        if (sfo) sfo[nf] = r.sfo_ppm;
        // end of the window of data symbol n - 1
        auto data_end = [&](long long n) { return lb::rs_sym(r.start, lb::rs_data_j(n - 1), sps, r.sfo_ppm) + (long long)sps; };
        if (r.status == lb::RS_OK && data_end(8) <= (long long)n_items) {
            std::vector<uint32_t> hb, pb;
            std::vector<float> llr, hllr;
            if (soft) {
                hb.resize(8);
                rs_host_llrs(od, r, 0, 8, true, hllr);
                lb::rs_soft_header(lb::rs_code(rp, phdr1), hllr.data(), hb.data(), nullptr);
            } else {
                rs_host_bins(od, r, 0, 8, hb);
            }
            lb::RxStreamState st;
            const int32_t np = lb::rs_header(&st, rp, phdr1, hb.data(), implicit_len);
            if (np < 0) status[nf] = 1;
            else if (data_end(8ll + np) <= (long long)n_items) {
                int recovered = 0;
                if (soft) {
                    pb.resize((size_t)np);
                    rs_host_llrs(od, r, 8, (uint32_t)np, reduced_rate != 0, llr);
                    lb::rs_soft_payload(rp, phdr1, hb.data(), np, implicit_len, llr.data(), pb.data());
                    if (crc_list) recovered = rs_host_crc_list(rp, phdr1, implicit_len, crc_list, np, hllr.data(), llr.data(), hb.data(), pb.data());
                } else {
                    rs_host_bins(od, r, 8, (uint32_t)np, pb);
                }
                lb::RxFrameRec fr;
                lb::rs_frame(&st, rp, pb.data(), np, &fr, 0, nf, 1.0f);
                const uint32_t nd = lb::decode_len_bytes(lb::decode_len_words(fr.n_cw, 0), fr.cr);
                std::vector<uint8_t> bytes(fr.payload_length);
                for (uint32_t i = 0; i < fr.payload_length; i++) bytes[i] = i < nd ? lb::decode_byte(fr.cw, fr.n_cw, 0, fr.cr, i) : 0;
                len[nf] = std::min<uint32_t>(fr.payload_length, 256u);
                std::copy(bytes.begin(), bytes.begin() + len[nf], payload + (size_t)nf * 256);
                status[nf] = 0;
                if (crc_status) {
                    const uint32_t c = lb::lb_crc_check(bytes.data(), fr.payload_length, fr.cr, (fr.phdr[1] >> 4) & 1u);
                    crc_status[nf] = (uint8_t)(c == LORA_CRC_OK && recovered ? LORA_CRC_RECOVERED : c);
                }
            }
        }
        nf++;
    }
    return nf;
}

}  // namespace

extern "C" {

// The whole dechirp-synchronised receive path (rx_sync.cuh) of one row on the host (BW = 125 kHz, fs = osr x BW with
// osr = 8, 2, 16 or 32, the decoder's sps / N; other values return 0 frames): screen,
// detect, synchronise, header and payload rounds, integer chain.  sfo_ppm and carrier_hz as in lora_b200_rx_params.  Per
// synchronised frame f (at most cap): start[f], cfo_bins[f], snr_db[f], status[f] (0 published, 1 header checksum failed,
// 2 incomplete), the clock offset its windows were placed with sfo[f] (may be NULL) and, when published, its payload in
// payload[f * 256 ..] with length len[f].  Returns the number of synchronised frames.
// soft != 0: soft decisions, as lora_b200_rx_params.soft (the LLR demodulator's emulation and the soft block decoder).
uint32_t lb_emul_rx_receive_osr(const float2 *x, size_t n_items, const float2 *down, const float2 *up, const float2 *tw, uint32_t sf,
                                uint32_t osr, uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t sync_word,
                                uint32_t implicit_len, uint32_t min_preamble, float sfo_ppm, double carrier_hz, int soft,
                                long long *start, float *cfo_bins, float *snr_db, int32_t *status, float *sfo, uint8_t *payload,
                                uint32_t *len, uint32_t cap) {
    return rs_host_receive(x, n_items, 1, down, up, tw, sf, osr, cr, implicit, crc, reduced_rate, sync_word, implicit_len, min_preamble,
                           sfo_ppm, carrier_hz, soft, start, cfo_bins, snr_db, status, sfo, payload, len, nullptr, cap);
}

// ... of one receiver with m (1..4) antennas, x[a * n_items ..] antenna a's row (lora_b200_receive_antennas): the combined
// screen, the synchroniser over all antennas, each frame's data windows sum_a w_a x_a (rs_channels); snr_db the combined
// SNR, chan[f * m ..] (may be NULL) the channel estimates h of synchronised frame f.  m = 1 is lb_emul_rx_receive_osr;
// another m returns 0 frames.
uint32_t lb_emul_rx_receive_antennas(const float2 *x, size_t n_items, uint32_t m, const float2 *down, const float2 *up, const float2 *tw,
                                     uint32_t sf, uint32_t osr, uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t sync_word,
                                     uint32_t implicit_len, uint32_t min_preamble, float sfo_ppm, double carrier_hz, int soft,
                                     long long *start, float *cfo_bins, float *snr_db, int32_t *status, float *sfo, uint8_t *payload,
                                     uint32_t *len, float *chan, uint32_t cap) {
    if (m < 1 || m > (uint32_t)lb::RS_MAX_ANTENNAS) return 0;
    return rs_host_receive(x, n_items, m, down, up, tw, sf, osr, cr, implicit, crc, reduced_rate, sync_word, implicit_len, min_preamble,
                           sfo_ppm, carrier_hz, soft, start, cfo_bins, snr_db, status, sfo, payload, len, (float2 *)chan, cap);
}

// lb_emul_rx_receive_antennas with CRC-aided list decoding (crc_list = K as lora_b200_rx_params.crc_list; 0 = off, any K
// needs soft) and each synchronised frame's payload CRC status in crc_status[f] (LORA_B200_CRC_*; NONE when not published).
uint32_t lb_emul_rx_receive_crc(const float2 *x, size_t n_items, uint32_t m, const float2 *down, const float2 *up, const float2 *tw,
                                uint32_t sf, uint32_t osr, uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t sync_word,
                                uint32_t implicit_len, uint32_t min_preamble, float sfo_ppm, double carrier_hz, int soft, uint32_t crc_list,
                                long long *start, float *cfo_bins, float *snr_db, int32_t *status, float *sfo, uint8_t *payload,
                                uint32_t *len, uint8_t *crc_status, uint32_t cap) {
    if (m < 1 || m > (uint32_t)lb::RS_MAX_ANTENNAS || crc_list > lb::RS_CRC_MAX_LIST || (crc_list && !soft)) return 0;
    return rs_host_receive(x, n_items, m, down, up, tw, sf, osr, cr, implicit, crc, reduced_rate, sync_word, implicit_len, min_preamble,
                           sfo_ppm, carrier_hz, soft, start, cfo_bins, snr_db, status, sfo, payload, len, nullptr, cap, crc_list, crc_status);
}

// rs_crc_list_kernel on one frame's given LLRs (header block hllr[8][sf - 2], payload blocks llr[n_payload][ppm]) and corrected
// bins (hbins[8], pbins[n_payload], as the soft decoder left them; corrected in place): 1 when the frame was recovered
int lb_emul_rx_crc_list(uint32_t sf, uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t implicit_len, uint32_t crc_list,
                        int32_t n_payload, const float *hllr, const float *llr, uint32_t *hbins, uint32_t *pbins) {
    lb::RxParams rp;
    memset(&rp, 0, sizeof rp);
    rp.sf = sf; rp.n_bins = 1u << sf; rp.n_bins_hdr = rp.n_bins / 4; rp.sps = 8u << sf; rp.decim = 8; rp.implicit = implicit;
    rp.reduced_rate = reduced_rate;
    const uint8_t phdr1 = (uint8_t)(((cr & 7u) << 5) | (crc ? 1u << 4 : 0u));
    return rs_host_crc_list(rp, phdr1, implicit_len, std::min<uint32_t>(crc_list, lb::RS_CRC_MAX_LIST), n_payload, hllr, llr, hbins, pbins);
}

// the payload CRC status (LORA_B200_CRC_NONE / _OK / _BAD) of a published record (lora_crc.h)
uint32_t lb_emul_crc_record_status(const uint8_t *rec, uint32_t len) { return lb::lb_crc_record_status(rec, len); }
uint32_t lb_emul_crc16(const uint8_t *b, uint32_t n) { return lb::lb_crc16(b, n); }

// lb_emul_rx_receive_crc with the coarse-offset search of lora_b200_rx_params.wide_cfo: |CFO| up to max_cfo_bins bins (> 0,
// at most (osr - 1) N / 2, the sampled band's limit; else 0 frames), as lora_b200_receive_antennas with wide_cfo = 1 and
// max_cfo_hz = max_cfo_bins * BW / N
uint32_t lb_emul_rx_receive_wide(const float2 *x, size_t n_items, uint32_t m, const float2 *down, const float2 *up, const float2 *tw,
                                 uint32_t sf, uint32_t osr, uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t sync_word,
                                 uint32_t implicit_len, uint32_t min_preamble, float sfo_ppm, double carrier_hz, int soft, float max_cfo_bins,
                                 long long *start, float *cfo_bins, float *snr_db, int32_t *status, float *sfo, uint8_t *payload,
                                 uint32_t *len, uint32_t cap) {
    if (m < 1 || m > (uint32_t)lb::RS_MAX_ANTENNAS || !(max_cfo_bins > 0.f) || max_cfo_bins > (float)((osr - 1u) << sf) / 2.0f) return 0;
    return rs_host_receive(x, n_items, m, down, up, tw, sf, osr, cr, implicit, crc, reduced_rate, sync_word, implicit_len, min_preamble,
                           sfo_ppm, carrier_hz, soft, start, cfo_bins, snr_db, status, sfo, payload, len, nullptr, cap, 0, nullptr,
                           max_cfo_bins);
}

// lb_emul_rx_receive_wide (max_cfo_bins 0: |CFO| <= N / 4 without the search) with the fine time of arrival of
// lora_b200_rx_params.fine_toa: toa[f] of every synchronised frame (rs_toa at its final synchronisation; NaN unless it
// synchronised, status 0 or 1)
uint32_t lb_emul_rx_receive_toa(const float2 *x, size_t n_items, uint32_t m, const float2 *down, const float2 *up, const float2 *tw,
                                uint32_t sf, uint32_t osr, uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t sync_word,
                                uint32_t implicit_len, uint32_t min_preamble, float sfo_ppm, double carrier_hz, int soft, float max_cfo_bins,
                                long long *start, float *cfo_bins, float *snr_db, int32_t *status, float *sfo, uint8_t *payload,
                                uint32_t *len, double *toa, uint32_t cap) {
    if (m < 1 || m > (uint32_t)lb::RS_MAX_ANTENNAS || max_cfo_bins < 0.f || max_cfo_bins > (float)((osr - 1u) << sf) / 2.0f) return 0;
    return rs_host_receive(x, n_items, m, down, up, tw, sf, osr, cr, implicit, crc, reduced_rate, sync_word, implicit_len, min_preamble,
                           sfo_ppm, carrier_hz, soft, start, cfo_bins, snr_db, status, sfo, payload, len, nullptr, cap, 0, nullptr,
                           max_cfo_bins, toa);
}

// rs_toa on given frames (lora_b200_rs_toa_dev on the host): frame i at start[i] with cfo_bins[i] and sfo_ppm[i] on the m rows
// x[a * n_items ..] (fs = osr x 125 kHz) -> nu_a[i], nu_b[i], toa[i]; -1 for another osr or m
int lb_emul_rs_toa(const float2 *x, size_t n_items, uint32_t m, const float2 *down, const float2 *up, const float2 *tw, uint32_t sf,
                   uint32_t osr, size_t n, const long long *start, const float *cfo_bins, const float *sfo_ppm, float *nu_a, float *nu_b,
                   double *toa) {
    if (!rs_host_osr(osr) || m < 1 || m > (uint32_t)lb::RS_MAX_ANTENNAS) return -1;
    const uint32_t N = 1u << sf, sps = osr * N;
    lb::RsParams p{sps, N, osr, 0.f, 5u, {0u, 0u}, (float)N / 4.0f, 0.f, 0};
    RsHostOps o{x, (long long)n_items, down, up, tw, sps, sf, osr, nullptr, 0};
    RsHostAntOps oa{o, m};
    for (size_t i = 0; i < n; i++) {
        const lb::RsFrame r{start[i], 0u, cfo_bins[i], 0.f, lb::RS_OK, 0, sfo_ppm[i]};
        const lb::RsToa t = m == 1 ? (sfo_ppm[i] != 0.f ? lb::rs_toa<true>(o, p, r) : lb::rs_toa<false>(o, p, r))
                                   : (sfo_ppm[i] != 0.f ? lb::rs_toa<true>(oa, p, r) : lb::rs_toa<false>(oa, p, r));
        nu_a[i] = t.nu_a; nu_b[i] = t.nu_b; toa[i] = t.toa;
    }
    return 0;
}

// lb_emul_rx_receive_osr at fs/bw = 8 (fs = 1 MHz)
uint32_t lb_emul_rx_receive_soft(const float2 *x, size_t n_items, const float2 *down, const float2 *up, const float2 *tw, uint32_t sf,
                                 uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t sync_word, uint32_t implicit_len,
                                 uint32_t min_preamble, float sfo_ppm, double carrier_hz, int soft, long long *start, float *cfo_bins,
                                 float *snr_db, int32_t *status, float *sfo, uint8_t *payload, uint32_t *len, uint32_t cap) {
    return lb_emul_rx_receive_osr(x, n_items, down, up, tw, sf, 8u, cr, implicit, crc, reduced_rate, sync_word, implicit_len,
                                  min_preamble, sfo_ppm, carrier_hz, soft, start, cfo_bins, snr_db, status, sfo, payload, len, cap);
}

// the header and payload rounds of one frame whose n_windows data windows are given (no synchronisation): as bins
// (llr NULL), or as LLRs -- the header block's llr[8][sf - 2] (reduced) first, then the payload windows' llr[][ppm].
// Writes the payload to payload[0 .. 256) and returns its length; -1: the explicit header's checksum failed, -2: the frame
// needs more than n_windows windows.
int32_t lb_emul_rx_decode(uint32_t sf, uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t implicit_len, const uint32_t *bins,
                          const float *llr, uint32_t n_windows, uint8_t *payload) {
    lb::RxParams rp;
    memset(&rp, 0, sizeof rp);
    rp.sf = sf; rp.n_bins = 1u << sf; rp.n_bins_hdr = rp.n_bins / 4; rp.sps = 8u << sf; rp.decim = 8; rp.implicit = implicit;
    rp.reduced_rate = reduced_rate;
    const uint8_t phdr1 = (uint8_t)(((cr & 7u) << 5) | (crc ? 1u << 4 : 0u));
    if (n_windows < 8u) return -2;
    std::vector<uint32_t> hb(8), pb;
    if (llr) lb::rs_soft_header(lb::rs_code(rp, phdr1), llr, hb.data(), nullptr);
    else std::copy(bins, bins + 8, hb.begin());
    lb::RxStreamState st;
    const int32_t np = lb::rs_header(&st, rp, phdr1, hb.data(), implicit_len);
    if (np < 0) return -1;
    if (8u + (uint32_t)np > n_windows) return -2;
    if (llr) {
        pb.resize((size_t)np);
        lb::rs_soft_payload(rp, phdr1, hb.data(), np, implicit_len, llr + 8 * (sf - 2), pb.data());
    } else {
        pb.assign(bins + 8, bins + 8 + np);
    }
    lb::RxFrameRec fr;
    lb::rs_frame(&st, rp, pb.data(), np, &fr, 0, 0, 1.0f);
    const uint32_t nd = lb::decode_len_bytes(lb::decode_len_words(fr.n_cw, 0), fr.cr), len = std::min<uint32_t>(fr.payload_length, 256u);
    for (uint32_t i = 0; i < len; i++) payload[i] = i < nd ? lb::decode_byte(fr.cw, fr.n_cw, 0, fr.cr, i) : 0;
    return (int32_t)len;
}

// lb_emul_rx_receive_soft with hard decisions
uint32_t lb_emul_rx_receive_sfo(const float2 *x, size_t n_items, const float2 *down, const float2 *up, const float2 *tw, uint32_t sf,
                                uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t sync_word, uint32_t implicit_len,
                                uint32_t min_preamble, float sfo_ppm, double carrier_hz, long long *start, float *cfo_bins,
                                float *snr_db, int32_t *status, float *sfo, uint8_t *payload, uint32_t *len, uint32_t cap) {
    return lb_emul_rx_receive_soft(x, n_items, down, up, tw, sf, cr, implicit, crc, reduced_rate, sync_word, implicit_len, min_preamble,
                                   sfo_ppm, carrier_hz, 0, start, cfo_bins, snr_db, status, sfo, payload, len, cap);
}

// lb_emul_rx_receive_sfo without a clock offset
uint32_t lb_emul_rx_receive(const float2 *x, size_t n_items, const float2 *down, const float2 *up, const float2 *tw, uint32_t sf,
                            uint32_t cr, int implicit, int crc, int reduced_rate, uint32_t sync_word, uint32_t implicit_len,
                            uint32_t min_preamble, long long *start, float *cfo_bins, float *snr_db, int32_t *status,
                            uint8_t *payload, uint32_t *len, uint32_t cap) {
    return lb_emul_rx_receive_sfo(x, n_items, down, up, tw, sf, cr, implicit, crc, reduced_rate, sync_word, implicit_len, min_preamble,
                                  0.0f, 0.0, start, cfo_bins, snr_db, status, nullptr, payload, len, cap);
}

// reserve(bytes[i]) in turn on one DeviceBuffer (cuda_owned.h): the cudaError_t, pointer and capacity after each
void lb_emul_buffer_reserve(const size_t *bytes, size_t n, int *rc, void **ptr, size_t *cap) {
    lb::DeviceBuffer<uint8_t> b;
    for (size_t i = 0; i < n; i++) { rc[i] = (int)b.reserve(bytes[i]); ptr[i] = b.get(); cap[i] = b.capacity(); }
}

}

namespace {
// The shared-memory indices (float2 units) of k1_fft_kernel<SF, D>'s phases over one batch, as k1_pass0, k1_pass and
// k1_combine form them from the thread index: instruction after instruction, the index of each of the K1_THREADS threads
// (-1: idle), and the phase (0 pass-0 stores, 1 and 2 the k1_pass loads -- its stores touch the same indices --, 3 the
// combine loads).
template <int SF, int D>
void k1_smem_indices(std::vector<int32_t> &idx, std::vector<int32_t> &phase) {
    using C = lb::K1Cfg<SF, D>;
    constexpr int T = lb::K1_THREADS, HB_LOG = lb::k1_log2(C::HB);
    auto instr = [&](int ph, auto at) {
        for (int t = 0; t < T; t++) idx.push_back(at(t));
        phase.push_back(ph);
    };
    for (int kc = 0; kc < 16; kc++)                   // thread (g, m, b): row kc of branches 2b, 2b + 1 of column m
        for (int br = 0; br < 2; br++)
            instr(0, [&](int tid) {
                const int g = tid / (C::HB * C::M0), rem = tid % (C::HB * C::M0), m = rem >> HB_LOG, b = rem & (C::HB - 1);
                return g * C::SYM_STRIDE + (2 * b + br) * C::SB + lb::k1_pad(kc * C::M0 + m);
            });
    auto pass = [&](int ph, int R, int SIG) {
        const int per = C::NP / R, items = C::G * D * per;
        for (int it0 = 0; it0 < items; it0 += T)
            for (int c = 0; c < R; c++)
                instr(ph, [&](int tid) {
                    const int it = it0 + tid;
                    if (it >= items) return -1;
                    const int j = it % per, gr = it / per, lo = j % SIG;
                    return gr * C::SB + lb::k1_pad((j / SIG) * (R * SIG) + lo + SIG * c);
                });
    };
    pass(1, C::R1, C::SIG1);
    if (C::R2 > 1) pass(2, C::R2, 1);
    for (int i = 0; i < C::NP / C::TPS; i++)
        for (int r = 0; r < D; r++)
            instr(3, [&](int tid) { return (tid / C::TPS) * C::SYM_STRIDE + r * C::SB + lb::k1_pad(tid % C::TPS + C::TPS * i); });
}
}  // namespace

extern "C" {
// k1_smem_indices of k1_fft_kernel<sf, osr>: returns the number of indices n (a multiple of K1_THREADS; -1 for another SF or
// osr) and, when cap >= n, writes them to idx[n] and the phase of each instruction to phase[n / K1_THREADS]
long lb_k1_smem_replay(int sf, int osr, int32_t *idx, int32_t *phase, long cap) {
    std::vector<int32_t> v, ph;
    if (lb::with_sf_osr(sf, osr, [] { return -1; }, [&](auto SF, auto D) { k1_smem_indices<SF, D>(v, ph); return 0; })) return -1;
    if (idx && phase && cap >= (long)v.size()) {
        std::copy(v.begin(), v.end(), idx);
        std::copy(ph.begin(), ph.end(), phase);
    }
    return (long)v.size();
}
}
