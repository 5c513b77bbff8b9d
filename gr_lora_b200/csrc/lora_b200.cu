// lora_b200.cu -- C-ABI implementation of liblora_b200.so (see include/lora_b200.h).
// Host side: parameter derivation and table construction exactly as the reference's
// constructor does them (lib/decoder_impl.cc:49-122,141-175), device memory, streams,
// pinned staging and kernel launches.  There is no CPU compute path in this file.
#include "../../include/lora_b200.h"
#include "cuda_owned.h"
#include "k1_fft.cuh"
#include "k1_group.cuh"
#include "k1_sf10.cuh"
#include "k1_launch.h"
#include "dispatch.h"
#include "rx_stream.cuh"
#include "rx_sync.cuh"
#include "rx_warp.cuh"
#include "tx_channel.cuh"
#include "tx_encode.cuh"

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

using namespace lb;

namespace {

thread_local std::string g_err;

int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CU(call)                                                                                  \
    do {                                                                                          \
        cudaError_t e_ = (call);                                                                  \
        if (e_ != cudaSuccess) return fail(LORA_B200_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

struct Tables {          // offsets (bytes) inside the device blob, see lora_b200_tables_bytes
    size_t down, up, down_ifreq, up_ifreq, up_ifreq_v, tw, total;
};

struct A1Params {        // what both a decoder and lora_b200_tables_build_host derive from a configuration
    uint32_t samples_per_second, sps, n_bins;
    double dt, symbols_per_second;
};

A1Params a1_params(const lora_b200_config &cfg) {     // A1, decoder_impl.cc:74-85 (same types)
    const uint32_t fs = (uint32_t)cfg.samp_rate;                          // :74 (uint32_t member)
    const double symbols_per_second = (double)cfg.bandwidth / (1u << cfg.sf);    // :80
    // sps :83, n_bins :85, dt :77 (a float divide kept in a double)
    return {fs, (uint32_t)(fs / symbols_per_second), 1u << cfg.sf, 1.0f / fs, symbols_per_second};
}

// Scratch of one K1 launch in flight: the 64-bit argmax keys that the split kernels merge with atomicMax.  A launch
// zeroes it on its stream first, so two launches that share one K1Scratch must not overlap: slot 0
// (lora_b200_demod_fft_dev) is ordered across user streams by `done`, and every slot of the host pipeline
// (lora_b200_demod_fft_host) owns its own.
struct K1Scratch {
    DeviceBuffer<unsigned long long> packed;
    CudaEvent done;
    cudaStream_t last = nullptr;          // the stream `done` was last recorded on
};

constexpr uint32_t MAX_STAGE_GROUPS = 8;     // staging groups of one work_batch call

}  // namespace

// Every device buffer, pinned buffer, stream and event below is owned by its member (cuda_owned.h).
struct lora_b200_decoder : A1Params {
    lora_b200_config cfg;
    // derived, decoder_impl.cc:69-91 (A1Params and these)
    uint32_t n_bins_hdr, decim;
    double bits_per_second, bits_per_symbol;
    int k1_osr;                           // the K1 kernels' D = fs/bw with SF7..12: 8 (every K1 kernel), 2, 16 or 32 (the
                                          // generic K1 and LLR kernels), or 0 (none)
    int device, n_sms;
    Tables toff;
    DeviceBuffer<uint8_t> d_tables;
    std::vector<uint8_t> h_tables;
    float down_ifreq_avg = 0.f, down_ifreq_sd = 0.f;
    // K1
    K1Scratch k1s[3];                     // [0] device entry point, [1], [2] host pipeline slots
    DeviceBuffer<float> d_k2_scratch;
    int k2_grid = 0;
    // e2e host path
    CudaStream copy_streams[2];
    DeviceBuffer<float2> d_chunk[2];
    DeviceBuffer<short2> d_chunk16[2];
    PinnedBuffer<float2> h_chunk[2];      // bounce buffers for pageable input
    DeviceBuffer<uint32_t> d_chunk_bins[2];
    DeviceBuffer<float> d_chunk_mags[2];
    // stream path
    CudaStream rx_stream, rx_stream2;
    CudaEvent rx2_done, rx_begin_ev;
    DeviceBuffer<RxStreamState> d_states;
    uint8_t phdr1_init = 0;
    DeviceBuffer<float> d_scratch;
    DeviceBuffer<unsigned long long> d_consumed;
    DeviceBuffer<RxFrameRec> d_frames;
    DeviceBuffer<RxFrameOut> d_frames_out;
    DeviceBuffer<uint32_t> d_n_frames;
    uint32_t frame_cap = 0;
    DeviceBuffer<lora_b200_step> d_trace;
    DeviceBuffer<uint32_t> d_trace_n;
    DeviceBuffer<float2> d_stage;         // [n_streams][max_items]
    DeviceBuffer<short2> d_stage16;       // same shape, int16 / int8 I/Q ingest (lora_b200_work_batch_sc16 / _sc8)
    PinnedBuffer<float2> h_stage;         // same shape
    CudaEvent stage_events[MAX_STAGE_GROUPS];
    std::vector<unsigned long long> h_consumed;
    PinnedBuffer<RxFrameOut> h_frames;    // frame_cap records
    std::vector<RxFrameOut> h_sorted;
    std::vector<std::string> stdout_last;
    uint64_t launches = 0;
    bool cfo_estimate = false;            // lora_b200_set_cfo_estimate
    // per-frame tables of lora_b200_tx_encode_dev / lora_b200_tx_frames_dev, uploaded on the caller's stream; `tx_done`
    // marks the end of the last launch that reads them, so the next upload waits for it on the host
    DeviceBuffer<uint8_t> d_tx;
    CudaEvent tx_done;
    // lora_b200_receive (rx_sync.cuh), all on rx_stream
    DeviceBuffer<float2> d_rs_stage, d_rs_win;
    DeviceBuffer<uint32_t> d_rs_bins[2], d_rs_hbins, d_rs_pbins, d_rs_ncand, d_rs_nframes, d_rs_tab;
    DeviceBuffer<float> d_rs_mags[2], d_rs_llr;
    DeviceBuffer<float> d_rs_hllr;        // the header round's LLRs, kept for list decoding (rx_params.crc_list)
    DeviceBuffer<uint8_t> d_rs_recovered; // per published frame: recovered by rs_crc_list_kernel
    DeviceBuffer<RsCand> d_rs_cands;
    DeviceBuffer<long long> d_rs_dropped;
    DeviceBuffer<unsigned long long> d_rs_hold;
    DeviceBuffer<RsFrame> d_rs_frames;
    DeviceBuffer<RxFrameRec> d_rs_recs;
    DeviceBuffer<RxFrameOut> d_rs_out;
    std::vector<lora_b200_rx_info> rs_info;
    uint32_t rs_hdr_drops = 0;
    // lora_b200_receive_antennas with several antennas: per synchronised frame h[4] | w[4] (rs_sync_antennas_kernel), and
    // the published frames' h (rs_chan_m per frame) for lora_b200_rx_channels_last
    DeviceBuffer<float2> d_rs_chan;
    std::vector<float2> rs_chan;
    uint32_t rs_chan_m = 1;
    // lora_b200_frames_crc_last: the frames of the last call that list decoding recovered (empty: none), and the statuses
    std::vector<uint8_t> rs_recovered, crc_status;
    // rx_params.wide_cfo: the shifted dechirp tables of hypotheses c = -rs_shift_hyp..rs_shift_hyp (rs_shift_tables), built
    // once for the widest search asked so far
    DeviceBuffer<float2> d_rs_shift;
    std::vector<float2> h_rs_shift;
    int rs_shift_hyp = 0;
    // rx_params.fine_toa: per published frame, its time of arrival (rs_toa_kernel), for lora_b200_rx_toa_last
    DeviceBuffer<double> d_rs_toa;
    std::vector<double> rs_toa;
};

namespace {

// ---- table construction (host, float phase + sincosf exactly like gr_expj) ---------------
void ifreq_host(const float2 *in, float *out, uint32_t window) {     // decoder_impl.cc:224-244
    for (uint32_t i = 1u; i < window; i++) {
        const float p1 = atan2f(in[i - 1].y, in[i - 1].x);
        float p2 = atan2f(in[i].y, in[i].x);
        while ((p2 - p1) > M_PI) p2 = (float)(p2 - 2.0f * M_PI);
        while ((p2 - p1) < -M_PI) p2 = (float)(p2 + 2.0f * M_PI);
        out[i - 1] = p2 - p1;
    }
    out[window - 1] = out[window - 2];
}

// the table blob of one configuration into h; returns its layout
Tables build_tables(const A1Params &p, uint32_t bandwidth, std::vector<uint8_t> &h) {
    const uint32_t sps = p.sps;
    Tables t;
    size_t o = 0;
    t.down = o; o += sizeof(float2) * sps;
    t.up = o; o += sizeof(float2) * sps;
    t.down_ifreq = o; o += sizeof(float) * sps;
    t.up_ifreq = o; o += sizeof(float) * sps;
    t.up_ifreq_v = o; o += sizeof(float) * sps * 3;
    t.tw = o; o += sizeof(float2) * sps;
    t.total = (o + 255) & ~(size_t)255;
    h.assign(t.total, 0);
    float2 *down = (float2 *)(h.data() + t.down);
    float2 *up = (float2 *)(h.data() + t.up);
    float *dif = (float *)(h.data() + t.down_ifreq);
    float *uif = (float *)(h.data() + t.up_ifreq);
    float *uifv = (float *)(h.data() + t.up_ifreq_v);
    float2 *tw = (float2 *)(h.data() + t.tw);

    const double T = -0.5 * bandwidth * p.symbols_per_second;            // :149
    const double f0 = bandwidth / 2.0;                                   // :150
    const double pre_dir = 2.0 * M_PI;
    for (uint32_t i = 0; i < sps; i++) {
        const double tt = p.dt * i;                                      // :158
        const float ph_d = (float)(pre_dir * tt * (f0 + T * tt));        // gr_expj(float), :159
        const float ph_u = (float)(pre_dir * tt * (f0 + T * tt) * -1.0f);    // :160
        const float cd = cosf(ph_d), sd = sinf(ph_d), cu = cosf(ph_u), su = sinf(ph_u);
        down[i] = make_float2(cd - sd, sd + cd);                         // (1+1j) * e^{j phase}
        up[i] = make_float2(cu - su, su + cu);
    }
    ifreq_host(down, dif, sps);                                          // :164
    ifreq_host(up, uif, sps);                                            // :165
    std::vector<float2> tmp(3 * (size_t)sps);
    for (int k = 0; k < 3; k++) memcpy(tmp.data() + (size_t)k * sps, up, sizeof(float2) * sps);   // :171-173
    ifreq_host(tmp.data(), uifv, 3 * sps);                               // :174
    for (uint32_t j = 0; j < sps; j++) {                                 // forward DFT twiddles W_sps^j
        const double a = -2.0 * M_PI * (double)j / (double)sps;
        tw[j] = make_float2((float)cos(a), (float)sin(a));
    }
    return t;
}

// chirp_avg and stddev of the ideal down-chirp's instantaneous frequency `dif`, :287-289
void table_stats(const float *dif, uint32_t sps, float *avg_out, float *sd_out) {
    const uint32_t to_idx = sps - 1u;
    float acc = 0.0f;
    for (uint32_t i = 0; i < to_idx; i++) acc += dif[i];
    const float avg = acc / (float)to_idx;
    float var = 0.0f;
    for (uint32_t i = 0; i < to_idx; i++) { const float t = dif[i] - avg; var += t * t; }
    var /= (float)to_idx;
    *avg_out = avg;
    *sd_out = sqrtf(var);
}
void table_stats(lora_b200_decoder *d) { table_stats((const float *)(d->h_tables.data() + d->toff.down_ifreq), d->sps, &d->down_ifreq_avg, &d->down_ifreq_sd); }

template <typename T>
const T *tab(const lora_b200_decoder *d, size_t off) { return (const T *)(d->d_tables + off); }

int launched(lora_b200_decoder *d) { d->launches++; CU(cudaGetLastError()); return LORA_B200_OK; }

// LORA_B200_OK when the K1 kernels serve this decoder's configuration, else the error that `what` needs them
int need_k1(const lora_b200_decoder *d, const char *what) {
    if (d->k1_osr) return LORA_B200_OK;
    return fail(LORA_B200_EUNSUPPORTED, "%s needs samp_rate/bandwidth == 8, 2, 16 or 32 and SF7..SF12", what);
}

// the `otherwise` of a dispatch on the decoder's SF
auto unsupported_sf(const lora_b200_decoder *d) {
    return [d] { return fail(LORA_B200_EUNSUPPORTED, "unsupported SF %u", d->cfg.sf); };
}

// ---- K1 launch -----------------------------------------------------------------------------
template <int SF, int D>
int k1_launch_generic(const K1Launch &k) {
    using C = K1Cfg<SF, D>;
    const size_t smem = sizeof(float2) * C::SMEM_ELEMS;
    K1_CU(opt_in_smem((const void *)k1_fft_kernel<SF, D>, k.device, smem));
    const size_t n_work = ((k.a.n_symbols + C::G - 1) / C::G) * C::S;
    const int grid = (int)std::min<size_t>(n_work, (size_t)k.n_sms * 2);
    k1_fft_kernel<SF, D><<<grid, K1_THREADS, smem, k.st>>>(k.a, k.bins, k.mags, k.packed);
    K1_CU(cudaGetLastError());
    return 0;
}

// SF10: one 256-thread group per symbol, two radix-32 passes (k1_sf10.cuh)
int k1_launch_sf10(const K1Launch &k) {
    const size_t smem = sizeof(S10Smem<2>);
    K1_CU(opt_in_smem((const void *)k1_sf10_kernel<2>, k.device, smem));
    const int grid = (int)std::min<size_t>(k.a.n_symbols, (size_t)k.n_sms);
    k1_sf10_kernel<2><<<grid, S10_T, smem, k.st>>>(k.a, k.bins, k.mags);
    K1_CU(cudaGetLastError());
    return 0;
}

__global__ void k1_finalize_kernel(const unsigned long long *__restrict__ packed, size_t n, uint32_t *__restrict__ bins,
                                   float *__restrict__ mags) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < n) k1_store(bins, mags, i, packed[i]);
}

// LORA_B200_K1=generic selects k1_fft_kernel (the CTA-wide kernel the stream state machine also uses) for every SF;
// LORA_B200_K1_ROWS=0 does the same for SF11 / SF12 only.  Both exist for A/B runs (tools/k1_ab.py); the defaults are the
// measured best per SF (DESIGN.md 5).
bool k1_generic() {
    static int v = -1;
    if (v < 0) { const char *e = getenv("LORA_B200_K1"); v = e && !strcmp(e, "generic") ? 1 : 0; }
    return v == 1;
}

// fs/bw = 8: each SF's own kernel, each one a separate measured choice (DESIGN.md 5)
K1Launcher k1_launcher(int sf) {
    switch (sf) {
    case 7: return k1_launch_warp7;                  // k1_packed.cu
    case 8: return k1_launch_group<8, 6, 2>;         // a group of 2 warps per symbol (k1_group.cuh)
    case 9: return k1_launch_group9;                 // k1_packed.cu
    case 10: return k1_launch_sf10;
    case 11: return k1_launch_rows<11>;              // every sample stays inside one SM (k1_rows.cuh, k1_rows.cu)
    case 12: return k1_launch_rows<12>;              // a cluster of two CTAs per symbol
    }
    return nullptr;
}

// the generic kernel k1_fft_kernel<SF, D>: every SF at fs/bw = 2, 16 and 32 (where it splits a symbol from SF12, SF10 and SF9
// on), and at fs/bw = 8 when `generic` is set
K1Launcher k1_launcher_generic(int sf, int osr) {
    static_assert(K1Cfg<11, 2>::S == 1 && K1Cfg<12, 2>::S == 2, "k1_fft_kernel<SF, 2> splits SF12 only");
    static_assert(K1Cfg<9, 16>::S == 1 && K1Cfg<10, 16>::S == 2 && K1Cfg<12, 16>::S == 8, "k1_fft_kernel<SF, 16> splits SF10..12");
    static_assert(K1Cfg<8, 32>::S == 1 && K1Cfg<9, 32>::S == 2 && K1Cfg<12, 32>::S == 16, "k1_fft_kernel<SF, 32> splits SF9..12");
    return with_sf_osr(sf, osr, [] { return K1Launcher(); }, [](auto SF, auto D) -> K1Launcher { return k1_launch_generic<SF, D>; });
}

// whether k1_fft_kernel<sf, osr> splits a symbol into sub-problems (K1Cfg::S > 1)
bool k1_generic_splits(int sf, int osr) {
    return with_sf_osr(sf, osr, [] { return false; }, [](auto SF, auto D) { return K1Cfg<SF, D>::S > 1; });
}

int dispatch_k1_impl(lora_b200_decoder *d, K1Scratch &ks, const float2 *iq, size_t n, uint32_t *bins, float *mags, cudaStream_t st,
                     const float2 *chirp) {
    if (int rc = need_k1(d, "FFT demodulator")) return rc;
    if (n == 0) return LORA_B200_OK;
    static const char *rows = getenv("LORA_B200_K1_ROWS");
    const int sf = (int)d->cfg.sf;
    const bool generic = k1_generic() || (sf >= 11 && rows && rows[0] == '0');
    const bool tuned = d->k1_osr == 8 && !generic;
    const K1Launcher launch = tuned ? k1_launcher(sf) : k1_launcher_generic(sf, d->k1_osr);
    if (!launch) return fail(LORA_B200_EUNSUPPORTED, "unsupported SF %u", d->cfg.sf);
    // the kernels that split a symbol merge partial argmax keys in ks.packed: of the fs/bw = 8 kernels the SF12 one (a cluster
    // of two CTAs per symbol), of the generic ones those whose K1Cfg has S > 1
    const bool split = tuned ? sf == 12 : k1_generic_splits(sf, d->k1_osr);
    if (split) {
        CU(ks.packed.reserve(n));
        CU(cudaMemsetAsync(ks.packed, 0, sizeof(unsigned long long) * n, st));
    }
    char err[256] = {0};
    const K1Launch k{K1Args{iq, chirp ? chirp : tab<float2>(d, d->toff.down), tab<float2>(d, d->toff.tw), n},
                     (const float2 *)(d->h_tables.data() + d->toff.tw), bins, mags, split ? ks.packed.get() : nullptr,
                     d->device, d->n_sms, st, err, sizeof err};
    if (launch(k)) return fail(LORA_B200_ECUDA, "K1: %s", err);
    d->launches++;
    if (split) {
        k1_finalize_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ks.packed, n, bins, mags);
        if (int rc = launched(d)) return rc;
    }
    return LORA_B200_OK;
}

// K1 on stream `st` with scratch `ks`: a launch that follows one on ANOTHER stream with the same scratch waits for it
// (the memset of the keys / flags at the head of a launch must not run under the previous kernel; a wait on `done`
// before its first record is a no-op).  chirp: the dechirp table (NULL: the decoder's down-chirp).
int dispatch_k1(lora_b200_decoder *d, K1Scratch &ks, const float2 *iq, size_t n, uint32_t *bins, float *mags, cudaStream_t st,
                const float2 *chirp = nullptr) {
    CU(ks.done.ensure());
    if (ks.last != st) CU(cudaStreamWaitEvent(st, ks.done, 0));
    const int rc = dispatch_k1_impl(d, ks, iq, n, bins, mags, st, chirp);
    if (rc) return rc;
    CU(cudaEventRecord(ks.done, st));
    ks.last = st;
    return LORA_B200_OK;
}

// ---- the LLR demodulator (k1_llr.cuh) ----------------------------------------------------------
template <int SF, int D>
int llr_launch(lora_b200_decoder *d, const float2 *iq, size_t n, bool reduced, float *llrs, uint32_t *bins, cudaStream_t st) {
    using C = K1Cfg<SF, D>;
    const size_t smem = sizeof(float2) * C::SMEM_ELEMS;
    CU(opt_in_smem((const void *)k1_llr_kernel<SF, D>, d->device, smem));
    const size_t n_batches = (n + C::G - 1) / C::G;
    const int grid = (int)std::min<size_t>(n_batches, (size_t)d->n_sms * 2);
    k1_llr_kernel<SF, D><<<grid, K1_THREADS, smem, st>>>(K1Args{iq, tab<float2>(d, d->toff.down), tab<float2>(d, d->toff.tw), n},
                                                         reduced ? 1 : 0, llrs, bins);
    return launched(d);
}

int dispatch_llr(lora_b200_decoder *d, const float2 *iq, size_t n, bool reduced, float *llrs, uint32_t *bins, cudaStream_t st) {
    if (int rc = need_k1(d, "the LLR demodulator")) return rc;
    if (n == 0) return LORA_B200_OK;
    return with_sf_osr(d->cfg.sf, d->k1_osr, unsupported_sf(d),
                       [&](auto SF, auto D) { return llr_launch<SF, D>(d, iq, n, reduced, llrs, bins, st); });
}

// ---- stream-path launch -----------------------------------------------------------------------
template <int SF, bool FFT>
int launch_rx_t(lora_b200_decoder *d, const RxParams &p, int grid, cudaStream_t st) {
    size_t smem = 0;
    if (FFT) {
        smem = sizeof(float2) * K1Cfg<SF>::SMEM_ELEMS;
        CU(opt_in_smem((const void *)rx_stream_kernel<SF, FFT>, d->device, smem));
    }
    rx_stream_kernel<SF, FFT><<<grid, RX_THREADS, smem, st>>>(p);
    return launched(d);
}

// SF7 at fs / bw = 8 runs rx_warp_kernel (one warp per stream); every other configuration rx_stream_kernel (one CTA per stream)
bool rx_warp_path(const lora_b200_decoder *d) { return d->cfg.sf == 7 && d->sps == (uint32_t)RW_SPS && d->n_bins == (uint32_t)RW_N; }

template <bool FFT>
int launch_rx_warp(lora_b200_decoder *d, const RxParams &p, int n_streams, cudaStream_t st) {
    const size_t smem = sizeof(RWSmem);
    CU(opt_in_smem((const void *)rx_warp_kernel<FFT>, d->device, smem));
    rx_warp_kernel<FFT><<<(n_streams + RW_WARPS - 1) / RW_WARPS, RW_WARPS * 32, smem, st>>>(p);
    return launched(d);
}

int launch_rx(lora_b200_decoder *d, const RxParams &p, int grid, cudaStream_t st) {
    const bool fft = d->cfg.demod == LORA_B200_DEMOD_FFT;
    if (rx_warp_path(d)) return fft ? launch_rx_warp<true>(d, p, grid, st) : launch_rx_warp<false>(d, p, grid, st);
    if (!fft) return launch_rx_t<7, false>(d, p, grid, st);       // SF is a run-time value on the gradient path
    // the FFT demodulator at SF7 always has sps = RW_SPS, so rx_stream_kernel<7, true> is not built
    return with_sf<8, 12>(d->cfg.sf, unsupported_sf(d), [&](auto SF) { return launch_rx_t<SF, true>(d, p, grid, st); });
}

void append_hex(std::string &s, const uint8_t *v, size_t n, bool endline, bool ascii) {   // print_vector_hex, utilities.h:351-368
    static const char digits[] = "0123456789abcdef";
    // (one snprintf per byte was 20 ms per call at 16 384 frames: more than the state machine of the last staging group)
    const size_t at = s.size();
    s.resize(at + 3 * n);
    char *o = &s[at];
    for (size_t i = 0; i < n; i++) { *o++ = ' '; *o++ = digits[v[i] >> 4]; *o++ = digits[v[i] & 15]; }
    if (ascii) {
        s += " (";
        for (size_t i = 0; i < n; i++)
            if (v[i] >= ' ' && v[i] <= '~') s.push_back((char)v[i]);
        s += ")";
    }
    if (endline) s += "\n";
}

int rx_begin(lora_b200_decoder *d) {
    CU(cudaMemsetAsync(d->d_n_frames, 0, sizeof(uint32_t), d->rx_stream));
    return LORA_B200_OK;
}

// the state machine for streams [stream_base, stream_base + n_launch) over staged IQ (one CTA per stream), async on rx_stream
int rx_launch(lora_b200_decoder *d, const float2 *d_iq, size_t stride_items, size_t n_items, uint32_t stream_base, uint32_t n_launch,
              cudaStream_t st = nullptr) {
    RxParams p;
    memset(&p, 0, sizeof p);
    p.iq = d_iq; p.stride_items = stride_items; p.n_items = n_items; p.stream_base = stream_base; p.n_launch = n_launch;
    p.down = tab<float2>(d, d->toff.down);
    p.down_ifreq = tab<float>(d, d->toff.down_ifreq);
    p.up_ifreq = tab<float>(d, d->toff.up_ifreq);
    p.up_ifreq_v = tab<float>(d, d->toff.up_ifreq_v);
    p.tw = tab<float2>(d, d->toff.tw);
    p.down_ifreq_avg = d->down_ifreq_avg; p.down_ifreq_sd = d->down_ifreq_sd;
    p.sps = d->sps; p.n_bins = d->n_bins; p.n_bins_hdr = d->n_bins_hdr; p.decim = d->decim; p.sf = d->cfg.sf;
    p.implicit = d->cfg.implicit; p.reduced_rate = d->cfg.reduced_rate; p.enable_fine_sync = !d->cfg.disable_drift_correction;
    p.cfo_estimate = d->cfo_estimate ? 1 : 0; p.samples_per_second = (float)d->samples_per_second;
    p.states = d->d_states; p.scratch = d->d_scratch; p.consumed = d->d_consumed;
    p.frames = d->d_frames; p.n_frames = d->d_n_frames; p.frame_cap = d->frame_cap;
    p.max_frames_per_stream = d->cfg.max_frames_per_call;
    p.trace = d->d_trace; p.trace_cap = d->cfg.trace_capacity; p.trace_n = d->d_trace_n;
    return launch_rx(d, p, (int)n_launch, st ? st : d->rx_stream);
}

// K8 on the queued frames, results back to the host, frames delivered per stream in sequence order
int rx_finish(lora_b200_decoder *d, uint32_t stream_base, uint32_t n_launch, size_t *consumed, lora_b200_frame_cb cb, void *user) {
    cudaStream_t st = d->rx_stream;
    const int k8_grid = (int)std::min<uint32_t>(d->frame_cap, (uint32_t)d->n_sms * 4u);
    k8_frames_kernel<<<k8_grid, 128, 0, st>>>(d->d_frames, d->d_n_frames, d->frame_cap, d->d_frames_out);
    if (int rc = launched(d)) return rc;
    uint32_t n_frames = 0;
    CU(cudaMemcpyAsync(&n_frames, d->d_n_frames, sizeof n_frames, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(d->h_consumed.data() + stream_base, d->d_consumed + stream_base,
                       sizeof(unsigned long long) * n_launch, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (n_frames > d->frame_cap) n_frames = d->frame_cap;
    if (n_frames) {
        CU(d->h_frames.reserve(d->frame_cap));      // pinned: the D2H runs at link speed
        CU(cudaMemcpyAsync(d->h_frames, d->d_frames_out, sizeof(RxFrameOut) * n_frames, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    }
    for (uint32_t s = 0; s < n_launch; s++) {
        consumed[s] = (size_t)d->h_consumed[stream_base + s];
        d->stdout_last[stream_base + s].clear();
    }
    // queue order is arrival order across streams; deliver per stream in sequence order
    std::vector<uint32_t> order(n_frames);
    for (uint32_t i = 0; i < n_frames; i++) order[i] = i;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
        const RxFrameOut &x = d->h_frames[a], &y = d->h_frames[b];
        return x.stream != y.stream ? x.stream < y.stream : x.seq < y.seq;
    });
    d->h_sorted.resize(n_frames);
    d->rs_info.clear();                           // (lora_b200_rx_info_last describes lora_b200_receive calls only)
    d->rs_chan.clear();
    d->rs_recovered.clear();
    d->rs_toa.clear();
    for (uint32_t k = 0; k < n_frames; k++) {
        const RxFrameOut &f = d->h_frames[order[k]];
        d->h_sorted[k] = f;
        std::string &so = d->stdout_last[f.stream];
        if (f.n_hdr_print) append_hex(so, f.hdr_print, f.n_hdr_print, false, false);    // :832
        append_hex(so, f.bytes + 18, f.len - 18, true, true);                           // :872
        if (cb) cb(user, f.stream, f.bytes, f.len);
    }
    return LORA_B200_OK;
}

int run_rx(lora_b200_decoder *d, const float2 *d_iq, size_t stride_items, size_t n_items, uint32_t stream_base,
           uint32_t n_launch, size_t *consumed, lora_b200_frame_cb cb, void *user) {
    int rc = rx_begin(d);
    if (!rc) rc = rx_launch(d, d_iq, stride_items, n_items, stream_base, n_launch);
    if (!rc) rc = rx_finish(d, stream_base, n_launch, consumed, cb, user);
    return rc;
}

// A3 on a batch of windows: one warp per window, the stream kernel's rw_ifreq on global memory
__global__ void k3_ifreq_kernel(const float2 *__restrict__ iq, size_t n_windows, uint32_t window, float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
    for (size_t w = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < n_windows; w += warps)
        rw_ifreq<false>(iq + w * window, out + w * window, (int)window, lane);
}

// SDR-native ingest: interleaved int16 I/Q -> gr_complex scaled by `scale` (what a host-side sc16 -> fc32 converter does)
__global__ void sc16_to_cf32_kernel(const short2 *__restrict__ in, float2 *__restrict__ out, size_t n, float scale) {
    const size_t stride = (size_t)gridDim.x * blockDim.x * 4;
    for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
        if (i + 4 <= n && (((uintptr_t)(in + i)) & 15u) == 0 && (((uintptr_t)(out + i)) & 15u) == 0) {
            const int4 v = __ldcs(reinterpret_cast<const int4 *>(in + i));
            const short2 s0 = *reinterpret_cast<const short2 *>(&v.x), s1 = *reinterpret_cast<const short2 *>(&v.y);
            const short2 s2 = *reinterpret_cast<const short2 *>(&v.z), s3 = *reinterpret_cast<const short2 *>(&v.w);
            float4 *o = reinterpret_cast<float4 *>(out + i);
            o[0] = make_float4(s0.x * scale, s0.y * scale, s1.x * scale, s1.y * scale);
            o[1] = make_float4(s2.x * scale, s2.y * scale, s3.x * scale, s3.y * scale);
        } else {
            for (size_t k = i; k < n && k < i + 4; k++) out[k] = make_float2(in[k].x * scale, in[k].y * scale);
        }
    }
}

// ... and interleaved int8 I/Q (GNU Radio's interleaved_char_to_complex; 2 bytes per sample over PCIe)
__global__ void sc8_to_cf32_kernel(const char2 *__restrict__ in, float2 *__restrict__ out, size_t n, float scale) {
    const size_t stride = (size_t)gridDim.x * blockDim.x * 8;
    for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
        if (i + 8 <= n && (((uintptr_t)(in + i)) & 15u) == 0 && (((uintptr_t)(out + i)) & 15u) == 0) {
            const int4 v = __ldcs(reinterpret_cast<const int4 *>(in + i));
            const int w[4] = {v.x, v.y, v.z, v.w};
            float4 *o = reinterpret_cast<float4 *>(out + i);
#pragma unroll
            for (int k = 0; k < 4; k++)
                o[k] = make_float4((float)(signed char)(w[k] & 0xff) * scale, (float)(signed char)((w[k] >> 8) & 0xff) * scale,
                                   (float)(signed char)((w[k] >> 16) & 0xff) * scale, (float)(signed char)((w[k] >> 24) & 0xff) * scale);
        } else {
            for (size_t k = i; k < n && k < i + 8; k++) out[k] = make_float2((float)in[k].x * scale, (float)in[k].y * scale);
        }
    }
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

const char *lora_b200_last_error(void) { return g_err.c_str(); }
int lora_b200_abi_version(void) { return LORA_B200_ABI_VERSION; }

// decoder_impl's members as the constructor leaves them (:55-66), for every stream
static cudaError_t init_states(lora_b200_decoder *d) {
    const uint32_t ns = d->cfg.n_streams;
    std::vector<RxStreamState> init(ns);
    for (auto &s : init) rx_state_init(&s, d->phdr1_init);
    return cudaMemcpy(d->d_states, init.data(), sizeof(RxStreamState) * ns, cudaMemcpyHostToDevice);
}

lora_b200_decoder *lora_b200_create(const lora_b200_config *cfg) {
    if (!cfg) { fail(LORA_B200_EINVAL, "null config"); return nullptr; }
    if (cfg->sf < 6 || cfg->sf > 13) {            // decoder_impl.cc:57-61 (the reference prints this and exit(1)s)
        fail(LORA_B200_EINVAL, "[LoRa Decoder] ERROR : Spreading factor should be between 6 and 12 (inclusive)!\n"
                               "                       Other values are currently not supported.");
        return nullptr;
    }
    if (cfg->n_streams == 0) { fail(LORA_B200_EINVAL, "n_streams must be >= 1"); return nullptr; }
    if (cfg->cr > 4) {     // the reference would abort in deinterleave ("More than 8 bits per word", decoder_impl.cc:541-545)
        fail(LORA_B200_EINVAL, "coding rate must be 0..4 (4/4 .. 4/8), got %u", cfg->cr);
        return nullptr;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        fail(LORA_B200_ECUDA, "no CUDA device: liblora_b200 has no CPU fallback");
        return nullptr;
    }
    auto d = std::make_unique<lora_b200_decoder>();     // every return before the last frees it and what it owns
    d->cfg = *cfg;
    if (d->cfg.max_items_per_call == 0) d->cfg.max_items_per_call = 1u << 20;
    if (d->cfg.max_frames_per_call == 0) d->cfg.max_frames_per_call = 8;
    auto bail = [](const char *what, cudaError_t e) {
        fail(LORA_B200_ECUDA, "%s: %s", what, cudaGetErrorString(e));
        return (lora_b200_decoder *)nullptr;
    };
    cudaError_t e;
    d->device = cfg->device;
    if (d->device < 0 && (e = cudaGetDevice(&d->device)) != cudaSuccess) return bail("cudaGetDevice", e);
    if ((e = cudaSetDevice(d->device)) != cudaSuccess) return bail("cudaSetDevice", e);
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, d->device)) != cudaSuccess) return bail("cudaGetDeviceProperties", e);
    d->n_sms = prop.multiProcessorCount;

    // A1: derived parameters, decoder_impl.cc:69-91 (same types, same order)
    static_cast<A1Params &>(*d) = a1_params(*cfg);                      // :74-85
    const uint8_t cr3 = cfg->cr & 7u;                                    // 3-bit field
    d->bits_per_second = (double)cfg->sf * (double)(4.0 / (4.0 + cr3)) / (1u << cfg->sf) * cfg->bandwidth;   // :79
    d->bits_per_symbol = (double)(d->bits_per_second / d->symbols_per_second);   // :82
    d->n_bins_hdr = 1u << (cfg->sf - 2);                                 // :86
    d->decim = d->sps / d->n_bins;                                       // :87
    if (d->sps < 2 * d->n_bins / 2 || d->decim == 0) {
        fail(LORA_B200_EINVAL, "samp_rate %.1f too low for bandwidth %u", cfg->samp_rate, cfg->bandwidth);
        return nullptr;
    }
    d->k1_osr = d->sps % d->n_bins == 0 && with_osr((int)d->decim, [] { return false; }, [](auto) { return true; }) && cfg->sf >= 7 &&
                        cfg->sf <= 12
                    ? (int)d->decim
                    : 0;
    if (cfg->demod == LORA_B200_DEMOD_FFT && d->k1_osr != 8) {
        fail(LORA_B200_EUNSUPPORTED, "FFT demodulator needs samp_rate/bandwidth == 8 and SF7..SF12");
        return nullptr;
    }

    d->toff = build_tables(*d, cfg->bandwidth, d->h_tables);
    table_stats(d.get());
    if ((e = d->d_tables.reserve(d->toff.total)) != cudaSuccess) return bail("cudaMalloc tables", e);
    if ((e = cudaMemcpy(d->d_tables, d->h_tables.data(), d->toff.total, cudaMemcpyHostToDevice)) != cudaSuccess) return bail("upload tables", e);

    const uint32_t ns = d->cfg.n_streams;
    if ((e = d->rx_stream.ensure()) != cudaSuccess) return bail("cudaStreamCreate", e);
    if ((e = d->d_states.reserve(ns)) != cudaSuccess) return bail("cudaMalloc states", e);
    d->phdr1_init = (uint8_t)((cr3 << 5) | ((cfg->crc ? 1u : 0u) << 4));       // :72-73
    if ((e = init_states(d.get())) != cudaSuccess) return bail("init states", e);
    const size_t scr_per = 2 * (size_t)d->sps + d->n_bins;
    if ((e = d->d_scratch.reserve(scr_per * ns)) != cudaSuccess) return bail("cudaMalloc scratch", e);
    if ((e = d->d_consumed.reserve(ns)) != cudaSuccess) return bail("cudaMalloc consumed", e);
    if ((e = cudaMemset(d->d_consumed, 0, sizeof(unsigned long long) * ns)) != cudaSuccess) return bail("memset", e);
    d->frame_cap = ns * d->cfg.max_frames_per_call;
    if ((e = d->d_frames.reserve(d->frame_cap)) != cudaSuccess) return bail("cudaMalloc frames", e);
    if ((e = d->d_frames_out.reserve(d->frame_cap)) != cudaSuccess) return bail("cudaMalloc frames_out", e);
    if ((e = d->d_n_frames.reserve(1)) != cudaSuccess) return bail("cudaMalloc n_frames", e);
    if (d->cfg.trace_capacity) {
        if ((e = d->d_trace.reserve((size_t)d->cfg.trace_capacity * ns)) != cudaSuccess) return bail("cudaMalloc trace", e);
        if ((e = d->d_trace_n.reserve(ns)) != cudaSuccess) return bail("cudaMalloc trace_n", e);
        if ((e = cudaMemset(d->d_trace_n, 0, sizeof(uint32_t) * ns)) != cudaSuccess) return bail("memset trace_n", e);
    }
    d->h_consumed.assign(ns, 0);
    d->stdout_last.assign(ns, std::string());
    d->k2_grid = d->n_sms * 4;
    return d.release();
}

void lora_b200_destroy(lora_b200_decoder *d) {
    if (!d) return;
    cudaSetDevice(d->device);
    cudaDeviceSynchronize();
    delete d;
}

uint32_t lora_b200_samples_per_symbol(const lora_b200_decoder *d) { return d ? d->sps : 0; }
uint32_t lora_b200_bins(const lora_b200_decoder *d) { return d ? d->n_bins : 0; }
uint32_t lora_b200_decimation(const lora_b200_decoder *d) { return d ? d->decim : 0; }
uint64_t lora_b200_launch_count(const lora_b200_decoder *d) { return d ? d->launches : 0; }

int lora_b200_banner(const lora_b200_decoder *d, char *buf, size_t cap) {    // decoder_impl.cc:93-103
    if (!d || !buf) return fail(LORA_B200_EINVAL, "null argument");
    int n = snprintf(buf, cap, "Bits (nominal) per symbol: \t%g\nBins per symbol: \t%u\nSamples per symbol: \t%u\nDecimation: \t\t%u\n",
                     d->bits_per_symbol, d->n_bins, d->sps, d->decim);
    if (d->cfg.disable_drift_correction && n >= 0 && (size_t)n < cap)
        n += snprintf(buf + n, cap - n, "Warning: clock drift correction disabled\n");
    if (d->cfg.implicit && n >= 0 && (size_t)n < cap)
        n += snprintf(buf + n, cap - n, "CR: \t\t%d\nCRC: \t\t%d\n", (int)(d->cfg.cr & 7), (int)(d->cfg.crc ? 1 : 0));
    return n;
}

int lora_b200_set_sf(lora_b200_decoder *d, uint8_t) {                         // :905-909
    return fail(LORA_B200_EUNSUPPORTED, "[LoRa Decoder] WARNING : Setting the spreading factor during execution is currently not supported.\n"
                                        "Nothing set, kept SF of %u.", d ? d->cfg.sf : 0);
}
int lora_b200_set_samp_rate(lora_b200_decoder *d, float) {                    // :911-915
    return fail(LORA_B200_EUNSUPPORTED, "[LoRa Decoder] WARNING : Setting the sample rate during execution is currently not supported.\n"
                                        "Nothing set, kept SR of %u.", d ? d->samples_per_second : 0);
}

size_t lora_b200_tables_build_host(const lora_b200_config *cfg, void *dst, size_t cap) {
    if (!cfg || cfg->sf < 6 || cfg->sf > 13) { fail(LORA_B200_EINVAL, "bad config"); return 0; }
    const A1Params p = a1_params(*cfg);
    if (p.sps < p.n_bins) { fail(LORA_B200_EINVAL, "samp_rate too low"); return 0; }
    std::vector<uint8_t> h;
    const Tables t = build_tables(p, cfg->bandwidth, h);
    if (dst) {
        if (cap < t.total) { fail(LORA_B200_EINVAL, "buffer too small"); return 0; }
        memcpy(dst, h.data(), t.total);
    }
    return t.total;
}

size_t lora_b200_tables_bytes(const lora_b200_decoder *d) { return d ? d->toff.total : 0; }
void *lora_b200_tables_device_ptr(lora_b200_decoder *d) { return d ? d->d_tables.get() : nullptr; }
int lora_b200_tables_export(const lora_b200_decoder *d, void *dst, size_t cap) {
    if (!d || !dst || cap < d->toff.total) return fail(LORA_B200_EINVAL, "tables_export: buffer too small");
    CU(cudaSetDevice(d->device));
    CU(cudaMemcpy(dst, d->d_tables, d->toff.total, cudaMemcpyDeviceToHost));
    return LORA_B200_OK;
}
int lora_b200_tables_import(lora_b200_decoder *d, const void *src, size_t bytes) {
    if (!d || !src || bytes != d->toff.total) return fail(LORA_B200_EINVAL, "tables_import: size mismatch");
    CU(cudaSetDevice(d->device));
    memcpy(d->h_tables.data(), src, bytes);
    table_stats(d);
    CU(cudaMemcpy(d->d_tables, src, bytes, cudaMemcpyHostToDevice));
    return LORA_B200_OK;
}

int lora_b200_tables_commit(lora_b200_decoder *d) {
    if (!d) return fail(LORA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(d->device));
    CU(cudaMemcpy(d->h_tables.data(), d->d_tables, d->toff.total, cudaMemcpyDeviceToHost));
    table_stats(d);
    return LORA_B200_OK;
}

int lora_b200_demod_fft_dev(lora_b200_decoder *d, const void *iq, size_t n_symbols, uint32_t *bins, float *mags, void *stream) {
    if (!d || (!iq && n_symbols) || (!bins && n_symbols)) return fail(LORA_B200_EINVAL, "null argument");
    if (((uintptr_t)iq & 15u) != 0) return fail(LORA_B200_EINVAL, "iq must be 16-byte aligned");
    CU(cudaSetDevice(d->device));
    return dispatch_k1(d, d->k1s[0], (const float2 *)iq, n_symbols, bins, mags, (cudaStream_t)stream);
}

int lora_b200_demod_llr_dev(lora_b200_decoder *d, const void *iq, size_t n_symbols, int reduced, float *llrs, uint32_t *bins, void *stream) {
    if (!d || (n_symbols && (!iq || !llrs))) return fail(LORA_B200_EINVAL, "null argument");
    if (int rc = need_k1(d, "the LLR demodulator")) return rc;
    if (((uintptr_t)iq & 15u) != 0) return fail(LORA_B200_EINVAL, "iq must be 16-byte aligned");
    if (reduced != 0 && reduced != 1) return fail(LORA_B200_EINVAL, "reduced must be 0 or 1, got %d", reduced);
    CU(cudaSetDevice(d->device));
    return dispatch_llr(d, (const float2 *)iq, n_symbols, reduced != 0, llrs, bins, (cudaStream_t)stream);
}

// K1 from host memory: double-buffered 64 MiB chunks, H2D + kernel + D2H overlapped on two streams (each slot owns its
// own keys / exchange scratch).  elem = 8: gr_complex; elem = 4: int16 I/Q, converted on the device right after the copy.
static int demod_fft_host_any(lora_b200_decoder *d, const void *iq, size_t elem, float scale, size_t n_symbols, uint32_t *bins, float *mags) {
    if (!d || (!iq && n_symbols) || (!bins && n_symbols)) return fail(LORA_B200_EINVAL, "null argument");
    if (int rc = need_k1(d, "FFT demodulator")) return rc;
    CU(cudaSetDevice(d->device));
    const size_t sym_bytes = sizeof(float2) * (size_t)d->sps, sym_in = elem * (size_t)d->sps;
    const bool sc16 = elem == 4;
    // the double-buffered pipeline: allocated by the first call that needs each part, costs nothing once it exists
    const size_t chunk_symbols = std::max<size_t>(1, ((size_t)64 << 20) / sym_bytes), chunk_items = chunk_symbols * d->sps;
    cudaPointerAttributes attr;
    bool pinned = cudaPointerGetAttributes(&attr, iq) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    for (int i = 0; i < 2; i++) {
        CU(d->copy_streams[i].ensure());
        CU(d->d_chunk[i].reserve(chunk_items));
        CU(d->d_chunk_bins[i].reserve(chunk_symbols));
        CU(d->d_chunk_mags[i].reserve(chunk_symbols));
        if (sc16) CU(d->d_chunk16[i].reserve(chunk_items));
        if (!pinned) CU(d->h_chunk[i].reserve(chunk_items));
    }
    const uint8_t *src = (const uint8_t *)iq;
    size_t done = 0;
    int k = 0;
    while (done < n_symbols) {
        const size_t n = std::min(chunk_symbols, n_symbols - done);
        const int b = k & 1;
        cudaStream_t st = d->copy_streams[b];
        CU(cudaStreamSynchronize(st));                // buffer b is free again (its D2H finished)
        const void *h = src + done * sym_in;
        if (!pinned) { memcpy(d->h_chunk[b], h, n * sym_in); h = d->h_chunk[b]; }
        if (sc16) {
            CU(cudaMemcpyAsync(d->d_chunk16[b], h, n * sym_in, cudaMemcpyHostToDevice, st));
            const size_t ns = n * (size_t)d->sps;
            const int grid = (int)std::min<size_t>((ns / 4 + 255) / 256, (size_t)d->n_sms * 8);
            sc16_to_cf32_kernel<<<grid, 256, 0, st>>>(d->d_chunk16[b], d->d_chunk[b], ns, scale);
            if (int rc = launched(d)) return rc;
        } else {
            CU(cudaMemcpyAsync(d->d_chunk[b], h, n * sym_bytes, cudaMemcpyHostToDevice, st));
        }
        int rc = dispatch_k1(d, d->k1s[1 + b], d->d_chunk[b], n, d->d_chunk_bins[b], d->d_chunk_mags[b], st);
        if (rc) return rc;
        CU(cudaMemcpyAsync(bins + done, d->d_chunk_bins[b], n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        if (mags) CU(cudaMemcpyAsync(mags + done, d->d_chunk_mags[b], n * sizeof(float), cudaMemcpyDeviceToHost, st));
        done += n;
        k++;
    }
    CU(cudaStreamSynchronize(d->copy_streams[0]));
    CU(cudaStreamSynchronize(d->copy_streams[1]));
    return LORA_B200_OK;
}

int lora_b200_demod_fft_host(lora_b200_decoder *d, const void *iq, size_t n_symbols, uint32_t *bins, float *mags) {
    return demod_fft_host_any(d, iq, sizeof(float2), 1.0f, n_symbols, bins, mags);
}

int lora_b200_demod_fft_host_sc16(lora_b200_decoder *d, const void *iq_sc16, float scale, size_t n_symbols, uint32_t *bins, float *mags) {
    return demod_fft_host_any(d, iq_sc16, sizeof(short2), scale, n_symbols, bins, mags);
}

int lora_b200_demod_gradient_dev(lora_b200_decoder *d, const void *iq, size_t n_symbols, uint32_t *bins, void *stream) {
    if (!d || (!iq && n_symbols) || (!bins && n_symbols)) return fail(LORA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(d->device));
    CU(d->d_k2_scratch.reserve((size_t)d->k2_grid * (d->sps + d->n_bins)));
    if (n_symbols == 0) return LORA_B200_OK;
    const int grid = (int)std::min<size_t>(n_symbols, (size_t)d->k2_grid);
    k2_gradient_kernel<<<grid, RX_THREADS, 0, (cudaStream_t)stream>>>((const float2 *)iq, n_symbols, d->sps, d->n_bins, d->decim,
                                                                     d->d_k2_scratch, bins);
    return launched(d);
}

int lora_b200_ifreq_dev(lora_b200_decoder *d, const void *iq, size_t n_windows, uint32_t window, float *out, void *stream) {
    if (!d || (!iq && n_windows) || (!out && n_windows)) return fail(LORA_B200_EINVAL, "null argument");
    if (window == 0 || window % 128u) return fail(LORA_B200_EINVAL, "window must be a positive multiple of 128");
    CU(cudaSetDevice(d->device));
    if (n_windows == 0) return LORA_B200_OK;
    const int grid = (int)std::min<size_t>((n_windows + 7) / 8, (size_t)d->n_sms * 8);
    k3_ifreq_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const float2 *)iq, n_windows, window, out);
    return launched(d);
}

int lora_b200_decode_codewords_dev(lora_b200_decoder *d, const uint8_t *codewords, const uint32_t *lengths, size_t stride,
                                   const uint8_t *cr, const uint8_t *is_header, size_t n_vec, uint8_t *out,
                                   size_t out_stride, uint32_t *out_len, void *stream) {
    if (!d || !codewords || !lengths || !cr || !is_header || !out || !out_len) return fail(LORA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(d->device));
    if (n_vec == 0) return LORA_B200_OK;
    const int grid = (int)std::min<size_t>(n_vec, (size_t)d->n_sms * 8);
    k8_decode_vectors_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(codewords, lengths, stride, cr, is_header, n_vec, out, out_stride, out_len);
    return launched(d);
}

int lora_b200_deinterleave_dev(lora_b200_decoder *d, const uint32_t *words, uint32_t n_words, uint32_t ppm, size_t n_blocks,
                               uint8_t *codewords, void *stream) {
    if (!d || !words || !codewords) return fail(LORA_B200_EINVAL, "null argument");
    if (n_words == 0 || n_words > 8 || ppm == 0 || ppm > 16) return fail(LORA_B200_EINVAL, "n_words must be 1..8, ppm 1..16");
    CU(cudaSetDevice(d->device));
    if (n_blocks == 0) return LORA_B200_OK;
    k8_deinterleave_kernel<<<(unsigned)((n_blocks + 127) / 128), 128, 0, (cudaStream_t)stream>>>(words, n_words, ppm, n_blocks, codewords);
    return launched(d);
}

// device staging for the host-pointer entry points (grows on demand); the pinned host mirror is only needed by the
// single-stream work() call, whose caller's buffer is pageable GNU Radio memory
static int ensure_stage(lora_b200_decoder *d, size_t items, bool want_host, bool want_sc16) {
    if (items > d->d_stage.capacity()) { d->h_stage.reset(); d->d_stage16.reset(); }    // all three grow together
    CU(d->d_stage.reserve(items));
    if (want_host) CU(d->h_stage.reserve(d->d_stage.capacity()));
    if (want_sc16) CU(d->d_stage16.reserve(d->d_stage.capacity()));
    return LORA_B200_OK;
}

int lora_b200_work(lora_b200_decoder *d, uint32_t stream, const void *iq_host, size_t n_items, size_t *consumed,
                   lora_b200_frame_cb cb, void *user) {
    if (!d || !consumed || (!iq_host && n_items)) return fail(LORA_B200_EINVAL, "null argument");
    if (stream >= d->cfg.n_streams) return fail(LORA_B200_EINVAL, "stream %u out of range", stream);
    CU(cudaSetDevice(d->device));
    if (n_items > d->cfg.max_items_per_call) n_items = d->cfg.max_items_per_call;     // never read past what was staged
    *consumed = 0;
    if (n_items < 2 * (size_t)d->sps) return LORA_B200_OK;                             // output_multiple, :91
    int rc = ensure_stage(d, n_items, true, false);
    if (rc) return rc;
    memcpy(d->h_stage, iq_host, sizeof(float2) * n_items);
    CU(cudaMemcpyAsync(d->d_stage, d->h_stage, sizeof(float2) * n_items, cudaMemcpyHostToDevice, d->rx_stream));
    return run_rx(d, d->d_stage, n_items, n_items, stream, 1, consumed, cb, user);
}

// all streams at once.  Host input is staged in groups of streams: the copy of group g + 1 (copy stream) runs under the
// state machine of group g (rx stream), so the call costs max(PCIe, kernel) instead of their sum.  elem = 8: gr_complex,
// elem = 4: interleaved int16 I/Q converted on the device (x * scale) before the state machine reads it.
static int work_batch_any(lora_b200_decoder *d, const void *iq, size_t elem, float scale, size_t n_items, size_t stride_items,
                          int host_ptr, size_t *consumed, lora_b200_frame_cb cb, void *user) {
    if (!d || !consumed || (!iq && n_items)) return fail(LORA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(d->device));
    const uint32_t ns = d->cfg.n_streams;
    for (uint32_t s = 0; s < ns; s++) consumed[s] = 0;
    if (n_items < 2 * (size_t)d->sps) return LORA_B200_OK;
    const bool sc16 = elem != sizeof(float2);             // an integer format (int16 or int8 I/Q) staged raw, converted on the device
    if (!host_ptr && !sc16) return run_rx(d, (const float2 *)iq, stride_items, n_items, 0, ns, consumed, cb, user);
    if (n_items > d->cfg.max_items_per_call) n_items = d->cfg.max_items_per_call;
    int rc = ensure_stage(d, n_items * ns, false, sc16);
    if (rc) return rc;
    CU(d->copy_streams[0].ensure());
    // groups: one launch each; a group should fill the machine about once (rx_warp_kernel: RW_WARPS streams per CTA, one CTA per
    // SM; rx_stream_kernel: one stream per CTA, two CTAs per SM), small batches stay whole.  Consecutive groups run on two
    // alternating compute streams so that the tail of one launch overlaps the head of the next.
    const uint32_t per_wave = (uint32_t)d->n_sms * (rx_warp_path(d) ? (uint32_t)RW_WARPS : 2u);
    // (a group of per_wave + 1 streams would take two waves: round the number of groups UP, so that the last group -- the
    // only one whose state machine is not hidden under a copy -- is a single wave)
    const uint32_t n_groups = std::max<uint32_t>(1u, std::min<uint32_t>(MAX_STAGE_GROUPS, (ns + per_wave - 1) / per_wave));
    const uint32_t gs = (ns + n_groups - 1) / n_groups;
    CU(d->rx_stream2.ensure());
    CU(d->rx2_done.ensure());
    CU(d->rx_begin_ev.ensure());
    for (uint32_t g = 0; g < n_groups; g++) CU(d->stage_events[g].ensure());
    cudaStream_t cs = d->copy_streams[0];
    if ((rc = rx_begin(d))) return rc;
    CU(cudaEventRecord(d->rx_begin_ev, d->rx_stream));            // the frame counter is reset before any group runs
    CU(cudaStreamWaitEvent(d->rx_stream2, d->rx_begin_ev, 0));
    for (uint32_t g = 0; g * gs < ns; g++) {
        const uint32_t s0 = g * gs, cnt = std::min<uint32_t>(gs, ns - s0);
        cudaStream_t xs = (g & 1) ? d->rx_stream2 : d->rx_stream;
        const uint8_t *src = (const uint8_t *)iq + (size_t)s0 * stride_items * elem;
        void *dst = sc16 ? (void *)((uint8_t *)d->d_stage16.get() + (size_t)s0 * n_items * elem) : (void *)(d->d_stage + (size_t)s0 * n_items);
        if (stride_items == n_items)                                  // dense rows: one linear copy (the 2-D form is for strided captures)
            CU(cudaMemcpyAsync(dst, src, elem * n_items * cnt, host_ptr ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, cs));
        else
            CU(cudaMemcpy2DAsync(dst, elem * n_items, src, elem * stride_items, elem * n_items, cnt,
                                 host_ptr ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, cs));
        CU(cudaEventRecord(d->stage_events[g], cs));
        CU(cudaStreamWaitEvent(xs, d->stage_events[g], 0));
        if (sc16) {
            const size_t n = (size_t)cnt * n_items;
            const int grid = (int)std::min<size_t>((n / 4 + 255) / 256, (size_t)d->n_sms * 8);
            if (elem == 4) sc16_to_cf32_kernel<<<grid, 256, 0, xs>>>(d->d_stage16 + (size_t)s0 * n_items, d->d_stage + (size_t)s0 * n_items, n, scale);
            else sc8_to_cf32_kernel<<<grid, 256, 0, xs>>>((const char2 *)d->d_stage16.get() + (size_t)s0 * n_items, d->d_stage + (size_t)s0 * n_items, n, scale);
            if (int rc = launched(d)) return rc;
        }
        if ((rc = rx_launch(d, d->d_stage + (size_t)s0 * n_items, n_items, n_items, s0, cnt, xs))) return rc;
    }
    CU(cudaEventRecord(d->rx2_done, d->rx_stream2));
    CU(cudaStreamWaitEvent(d->rx_stream, d->rx2_done, 0));
    return rx_finish(d, 0, ns, consumed, cb, user);
}

int lora_b200_work_batch(lora_b200_decoder *d, const void *iq, size_t n_items, size_t stride_items, int host_ptr,
                         size_t *consumed, lora_b200_frame_cb cb, void *user) {
    return work_batch_any(d, iq, sizeof(float2), 1.0f, n_items, stride_items, host_ptr, consumed, cb, user);
}

int lora_b200_work_batch_sc16(lora_b200_decoder *d, const void *iq_sc16, float scale, size_t n_items, size_t stride_items,
                              int host_ptr, size_t *consumed, lora_b200_frame_cb cb, void *user) {
    return work_batch_any(d, iq_sc16, sizeof(short2), scale, n_items, stride_items, host_ptr, consumed, cb, user);
}

int lora_b200_reset(lora_b200_decoder *d) {
    if (!d) return fail(LORA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(d->device));
    CU(cudaStreamSynchronize(d->rx_stream));
    if (d->rx_stream2) CU(cudaStreamSynchronize(d->rx_stream2));
    CU(init_states(d));
    CU(cudaMemset(d->d_consumed, 0, sizeof(unsigned long long) * d->cfg.n_streams));
    if (d->d_trace_n) CU(cudaMemset(d->d_trace_n, 0, sizeof(uint32_t) * d->cfg.n_streams));
    d->h_sorted.clear();
    d->rs_recovered.clear();
    d->rs_toa.clear();
    for (auto &so : d->stdout_last) so.clear();
    return LORA_B200_OK;
}

int lora_b200_tx_symbols_dev(lora_b200_decoder *d, const void *up_table, const uint32_t *values, const float *cfo_hz, float noise_sigma,
                             uint64_t seed, size_t n_symbols, void *out, void *stream) {
    if (!d || (!values && n_symbols) || (!out && n_symbols)) return fail(LORA_B200_EINVAL, "null argument");
    if (d->sps & 1u) return fail(LORA_B200_EUNSUPPORTED, "odd samples per symbol");
    CU(cudaSetDevice(d->device));
    if (n_symbols == 0) return LORA_B200_OK;
    const float2 *up = up_table ? (const float2 *)up_table : tab<float2>(d, d->toff.up);
    const size_t threads = n_symbols * (d->sps / 2);
    const int grid = (int)std::min<size_t>((threads + 255) / 256, (size_t)d->n_sms * 16);
    tx_symbols_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(up, d->sps, d->decim, values, cfo_hz, 1.0 / (double)d->cfg.samp_rate, noise_sigma,
                                                              (unsigned long long)seed, n_symbols, (float2 *)out);
    return launched(d);
}

int lora_b200_tx_expand_dev(lora_b200_decoder *d, const void *base, uint32_t k, size_t n_items, float noise_sigma, uint64_t seed,
                            size_t n_streams, void *out, void *stream) {
    if (!d || !base || !out || k == 0) return fail(LORA_B200_EINVAL, "null argument");
    if (n_items & 1u) return fail(LORA_B200_EINVAL, "n_items must be even");
    CU(cudaSetDevice(d->device));
    if (n_streams == 0 || n_items == 0) return LORA_B200_OK;
    const size_t threads = n_streams * (n_items / 2);
    const int grid = (int)std::min<size_t>((threads + 255) / 256, (size_t)d->n_sms * 16);
    tx_expand_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const float2 *)base, k, n_items, noise_sigma, (unsigned long long)seed, n_streams,
                                                             (float2 *)out);
    return launched(d);
}

// the encoder's view of a configuration; false for one it does not support (SF7..12, CR 4/5..4/8)
static bool tx_code(const lora_b200_config &cfg, TxCode *c) {
    if (cfg.sf < 7 || cfg.sf > 12 || cfg.cr < 1 || cfg.cr > 4) return false;
    *c = TxCode{cfg.sf, cfg.cr, cfg.implicit ? 0u : 1u, cfg.crc ? 1u : 0u, cfg.reduced_rate ? 1u : 0u};
    return true;
}

// upload the per-frame table of a tx call into d->d_tx on `st`, after the previous call that read it has finished (before
// the first call, tx_done has never been recorded and the wait returns at once)
static int tx_upload(lora_b200_decoder *d, const void *src, size_t bytes, cudaStream_t st) {
    CU(d->tx_done.ensure());
    CU(cudaEventSynchronize(d->tx_done));
    CU(d->d_tx.reserve(bytes));
    CU(cudaMemcpyAsync(d->d_tx, src, bytes, cudaMemcpyHostToDevice, st));
    return LORA_B200_OK;
}

static int tx_launched(lora_b200_decoder *d, cudaStream_t st) {
    if (int rc = launched(d)) return rc;
    CU(cudaEventRecord(d->tx_done, st));
    return LORA_B200_OK;
}

uint32_t lora_b200_tx_frame_symbols(const lora_b200_config *cfg, uint32_t payload_len) {
    TxCode c;
    if (!cfg || !tx_code(*cfg, &c) || !tx_length_ok(c, payload_len)) return 0;
    return tx_data_symbols(c, payload_len);
}

int lora_b200_tx_encode_dev(lora_b200_decoder *d, const uint8_t *payloads, const uint32_t *offsets, const uint32_t *lengths,
                            size_t n_frames, uint32_t *shifts, uint32_t max_symbols, void *stream) {
    if (!d || (n_frames && (!offsets || !lengths || !shifts))) return fail(LORA_B200_EINVAL, "null argument");
    TxCode c;
    if (!tx_code(d->cfg, &c)) return fail(LORA_B200_EUNSUPPORTED, "frame encoder needs SF7..SF12 and CR 1..4");
    std::vector<uint2> tab(n_frames);
    for (size_t f = 0; f < n_frames; f++) {
        const uint32_t len = lengths[f];
        if (!tx_length_ok(c, len))
            return fail(LORA_B200_EINVAL, "frame %zu: payload length %u out of range (at most %u%s)", f, len, 255u + 2u * c.crc,
                        c.explicit_hdr && c.crc ? ", at least 2 with CRC" : "");
        if (len && !payloads) return fail(LORA_B200_EINVAL, "null payloads");
        if (tx_data_symbols(c, len) > max_symbols)
            return fail(LORA_B200_EINVAL, "frame %zu needs %u symbols, max_symbols is %u", f, tx_data_symbols(c, len), max_symbols);
        tab[f] = make_uint2(offsets[f], len);
    }
    CU(cudaSetDevice(d->device));
    if (n_frames == 0) return LORA_B200_OK;
    const cudaStream_t st = (cudaStream_t)stream;
    if (int rc = tx_upload(d, tab.data(), sizeof(uint2) * n_frames, st)) return rc;
    const size_t threads = n_frames * max_symbols;
    const int grid = (int)std::min<size_t>((threads + 255) / 256, (size_t)d->n_sms * 16);
    tx_encode_kernel<<<grid, 256, 0, st>>>(c, payloads, (const uint2 *)d->d_tx.get(), n_frames, max_symbols, shifts);
    return tx_launched(d, st);
}

static_assert(sizeof(lora_b200_tx_frame) == 24 && offsetof(lora_b200_tx_frame, stream) == 8 &&
              offsetof(lora_b200_tx_frame, n_symbols) == 12 && offsetof(lora_b200_tx_frame, cfo_hz) == 16 &&
              offsetof(lora_b200_tx_frame, sync_word) == 20, "lora_b200_tx_frame layout");

int lora_b200_tx_frames_dev(lora_b200_decoder *d, const void *up_table, const lora_b200_tx_frame *frames, size_t n_frames,
                            const uint32_t *shifts, uint32_t max_symbols, float noise_sigma, uint64_t seed, size_t n_streams,
                            size_t n_items, void *out, void *stream) {
    return lora_b200_tx_frames_sfo_dev(d, up_table, frames, n_frames, nullptr, shifts, max_symbols, noise_sigma, seed, n_streams,
                                       n_items, out, stream);
}

int lora_b200_tx_frames_sfo_dev(lora_b200_decoder *d, const void *up_table, const lora_b200_tx_frame *frames, size_t n_frames,
                                const float *sfo_ppm, const uint32_t *shifts, uint32_t max_symbols, float noise_sigma, uint64_t seed,
                                size_t n_streams, size_t n_items, void *out, void *stream) {
    if (!d || (n_frames && (!frames || !shifts)) || (n_streams && n_items && !out)) return fail(LORA_B200_EINVAL, "null argument");
    if (n_items & 1u) return fail(LORA_B200_EINVAL, "n_items must be even");
    if (((uintptr_t)out & 15u) != 0) return fail(LORA_B200_EINVAL, "out must be 16-byte aligned");
    if (d->sps & 1u) return fail(LORA_B200_EUNSUPPORTED, "odd samples per symbol");
    if (n_frames >= 0xFFFFFFFFu || n_streams >= 0xFFFFFFFFu) return fail(LORA_B200_EINVAL, "too many frames or streams");
    // sort by (row, start), check placement, then one upload: row_ptr[n_streams + 1] | pad | TxFrameDesc[n_frames]
    std::vector<uint32_t> order(n_frames);
    std::vector<double> rate(n_frames, 1.0);
    std::vector<unsigned long long> n_rx(n_frames);
    for (size_t f = 0; f < n_frames; f++) {
        const lora_b200_tx_frame &fr = frames[f];
        if (fr.stream >= n_streams) return fail(LORA_B200_EINVAL, "frame %zu: stream %u >= n_streams %zu", f, fr.stream, n_streams);
        if (fr.n_symbols > max_symbols) return fail(LORA_B200_EINVAL, "frame %zu: n_symbols %u > max_symbols %u", f, fr.n_symbols, max_symbols);
        if (sfo_ppm && (!std::isfinite(sfo_ppm[f]) || std::fabs(sfo_ppm[f]) > 500.0f))
            return fail(LORA_B200_EINVAL, "frame %zu: sfo_ppm %g is not finite within +-500", f, (double)sfo_ppm[f]);
        if (sfo_ppm) rate[f] = 1.0 + 1e-6 * (double)sfo_ppm[f];
        const unsigned long long len = n_rx[f] = tx_drifted_samples(tx_frame_samples(fr.n_symbols, d->sps), rate[f]);
        if (len > 0xFFFFFFFFull || fr.start > n_items || len > n_items - fr.start)
            return fail(LORA_B200_EINVAL, "frame %zu: samples [%llu, %llu) run past n_items %zu", f, (unsigned long long)fr.start,
                        (unsigned long long)fr.start + len, n_items);
        order[f] = (uint32_t)f;
    }
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
        return frames[a].stream != frames[b].stream ? frames[a].stream < frames[b].stream : frames[a].start < frames[b].start;
    });
    const size_t desc_off = ((n_streams + 1) * sizeof(uint32_t) + 15) & ~(size_t)15;
    std::vector<uint8_t> blob(desc_off + sizeof(TxFrameDesc) * n_frames, 0);
    uint32_t *row_ptr = reinterpret_cast<uint32_t *>(blob.data());
    TxFrameDesc *desc = reinterpret_cast<TxFrameDesc *>(blob.data() + desc_off);
    for (size_t k = 0; k < n_frames; k++) {
        const lora_b200_tx_frame &fr = frames[order[k]];
        if (k && frames[order[k - 1]].stream == fr.stream) {
            const lora_b200_tx_frame &pr = frames[order[k - 1]];
            if (pr.start + n_rx[order[k - 1]] > fr.start)
                return fail(LORA_B200_EINVAL, "frames %u and %u overlap in stream %u", order[k - 1], order[k], fr.stream);
        }
        const uint32_t sync = ((((fr.sync_word >> 4) & 15u) * 8u) % d->n_bins) | ((((fr.sync_word & 15u) * 8u) % d->n_bins) << 16);
        desc[k] = TxFrameDesc{fr.start, fr.n_symbols, fr.cfo_hz, order[k], sync, rate[order[k]], n_rx[order[k]]};
        row_ptr[fr.stream + 1]++;
    }
    for (size_t s = 0; s < n_streams; s++) row_ptr[s + 1] += row_ptr[s];
    CU(cudaSetDevice(d->device));
    if (n_streams == 0 || n_items == 0) return LORA_B200_OK;
    const cudaStream_t st = (cudaStream_t)stream;
    if (int rc = tx_upload(d, blob.data(), blob.size(), st)) return rc;
    const float2 *up = up_table ? (const float2 *)up_table : tab<float2>(d, d->toff.up);
    const size_t threads = n_streams * (n_items / 2);
    const int grid = (int)std::min<size_t>((threads + 255) / 256, (size_t)d->n_sms * 16);
    tx_frames_kernel<<<grid, 256, 0, st>>>(up, d->sps, d->decim, d->n_bins, (const uint32_t *)d->d_tx.get(),
                                           (const TxFrameDesc *)(d->d_tx + desc_off), shifts, max_symbols,
                                           1.0 / (double)d->cfg.samp_rate, noise_sigma, (unsigned long long)seed, n_items, n_streams,
                                           (float2 *)out);
    return tx_launched(d, st);
}

}  // extern "C"

// ---- lora_b200_receive: the dechirp-synchronised receiver (rx_sync.cuh), every launch on rx_stream ----------------------
// one receiver per stream (m = 1: rs_sync_kernel), or per group of m antenna rows (rs_sync_antennas_kernel)
template <int SF, int D, bool DRIFT>
static int rs_launch_sync(lora_b200_decoder *d, const float2 *x, size_t stride, size_t n_items, const RsParams &rp, uint32_t cap,
                          uint32_t m, const float2 *shift) {
    const size_t smem = sizeof(float2) * K1Cfg<SF, D>::SMEM_ELEMS;
    const uint32_t ng = d->cfg.n_streams / m;
    if (m == 1) {
        CU(opt_in_smem((const void *)rs_sync_kernel<SF, D, DRIFT>, d->device, smem));
        rs_sync_kernel<SF, D, DRIFT><<<d->cfg.n_streams * cap, RX_THREADS, smem, d->rx_stream>>>(
            x, stride, n_items, tab<float2>(d, d->toff.down), tab<float2>(d, d->toff.up), tab<float2>(d, d->toff.tw), shift, rp,
            d->d_rs_cands, d->d_rs_ncand, cap, d->d_rs_frames, d->d_rs_nframes, d->cfg.n_streams * cap, d->d_rs_hold);
        return launched(d);
    }
    CU(opt_in_smem((const void *)rs_sync_antennas_kernel<SF, D, DRIFT>, d->device, smem));
    rs_sync_antennas_kernel<SF, D, DRIFT><<<ng * cap, RX_THREADS, smem, d->rx_stream>>>(
        x, stride, n_items, m, tab<float2>(d, d->toff.down), tab<float2>(d, d->toff.up), tab<float2>(d, d->toff.tw), shift, rp,
        d->d_rs_cands, d->d_rs_ncand, cap, d->d_rs_frames, d->d_rs_nframes, ng * cap, d->d_rs_hold, d->d_rs_chan);
    return launched(d);
}

// without a clock offset the synchroniser runs its DRIFT = false instantiation, which does no drift arithmetic; D = sps / N
// (8, 2, 16 or 32) selects the K1 phase functions of its argmax windows; shift: the hypotheses' tables (NULL when rp.hyp = 0)
static int rs_sync(lora_b200_decoder *d, const float2 *x, size_t stride, size_t n_items, const RsParams &rp, uint32_t cap, uint32_t m,
                   const float2 *shift) {
    return with_sf_osr(d->cfg.sf, d->k1_osr, unsupported_sf(d), [&](auto SF, auto D) {
        return with_bool(rs_drift(rp), [&](auto DRIFT) { return rs_launch_sync<SF, D, DRIFT>(d, x, stride, n_items, rp, cap, m, shift); });
    });
}

// the combined screen of ng receivers with m antennas: k1_antennas_kernel over the n_win windows of each row (rows `stride`
// apart), receiver g's results at bins / mags[g * out_stride ..]; chirp: the dechirp table (NULL: the decoder's down-chirp)
template <int SF, int D>
static int rs_screen_launch(lora_b200_decoder *d, const float2 *x, size_t n_win, size_t stride, uint32_t m, uint32_t ng, size_t out_stride,
                            uint32_t *bins, float *mags, cudaStream_t st, const float2 *chirp) {
    using C = K1Cfg<SF, D>;
    const size_t smem = sizeof(float2) * C::SMEM_ELEMS;
    CU(opt_in_smem((const void *)k1_antennas_kernel<SF, D>, d->device, smem));
    const size_t n_work = (n_win + C::G - 1) / C::G * ng;
    const int grid = (int)std::min<size_t>(n_work, (size_t)d->n_sms * 2);
    k1_antennas_kernel<SF, D><<<grid, K1_THREADS, smem, st>>>(K1Args{x, chirp ? chirp : tab<float2>(d, d->toff.down), tab<float2>(d, d->toff.tw), n_win},
                                                             stride, m, ng, out_stride, bins, mags);
    return launched(d);
}
static int rs_screen(lora_b200_decoder *d, const float2 *x, size_t n_win, size_t stride, uint32_t m, uint32_t ng, size_t out_stride,
                     uint32_t *bins, float *mags, cudaStream_t st, const float2 *chirp = nullptr) {
    return with_sf_osr(d->cfg.sf, d->k1_osr, unsupported_sf(d), [&](auto SF, auto D) {
        return rs_screen_launch<SF, D>(d, x, n_win, stride, m, ng, out_stride, bins, mags, st, chirp);
    });
}

// the data windows of frames [slots], as rs_assemble_kernel (m = 1) or combined over m antennas
static int rs_assemble(lora_b200_decoder *d, const float2 *x, size_t stride, size_t n_items, uint32_t m, const RsFrame *frames,
                       const float2 *chan, uint32_t n_frames, const uint32_t *idx, uint32_t first, const uint32_t *offs, uint32_t off_base,
                       const uint32_t *cnts) {
    const int grid = std::min<int>((int)n_frames, d->n_sms * 8);
    if (m == 1)
        rs_assemble_kernel<<<grid, 256, 0, d->rx_stream>>>(x, stride, (long long)n_items, frames, n_frames, idx, first, offs, off_base,
                                                           cnts, d->sps, d->d_rs_win);
    else
        rs_assemble_antennas_kernel<<<grid, 256, 0, d->rx_stream>>>(x, stride, (long long)n_items, m, frames, chan, n_frames, idx, first,
                                                                    offs, off_base, cnts, d->sps, d->d_rs_win);
    return launched(d);
}

// the fine time of arrival of n frames (frames[pub[k]], pub NULL: frames[k]) into toa[k] and nu[k] (may be NULL); DRIFT as
// the synchroniser's (rs_drift)
template <int SF, int D, bool DRIFT>
static int rs_toa_launch(lora_b200_decoder *d, const float2 *x, size_t stride, size_t n_items, uint32_t m, const RsParams &rp,
                         const RsFrame *frames, const uint32_t *pub, uint32_t n, double *toa, float2 *nu) {
    rs_toa_kernel<SF, D, DRIFT><<<n, RX_THREADS, 0, d->rx_stream>>>(x, stride, n_items, m, tab<float2>(d, d->toff.down), tab<float2>(d, d->toff.up),
                                                                    tab<float2>(d, d->toff.tw), rp, frames, pub, toa, nu);
    return launched(d);
}
static int rs_toa(lora_b200_decoder *d, const float2 *x, size_t stride, size_t n_items, uint32_t m, const RsParams &rp, const RsFrame *frames,
                  const uint32_t *pub, uint32_t n, double *toa, float2 *nu) {
    return with_sf_osr(d->cfg.sf, d->k1_osr, unsupported_sf(d), [&](auto SF, auto D) {
        return with_bool(rs_drift(rp), [&](auto DRIFT) { return rs_toa_launch<SF, D, DRIFT>(d, x, stride, n_items, m, rp, frames, pub, n, toa, nu); });
    });
}

// lora_b200_receive (m = 1) and lora_b200_receive_antennas: the receiver of group g reads rows g m .. g m + m - 1
static int rs_receive(lora_b200_decoder *d, const void *iq, size_t n_items, size_t stride_items, int host_ptr, uint32_t m,
                      const lora_b200_rx_params *prm, size_t *consumed) {
    if (!d || !consumed || (!iq && n_items)) return fail(LORA_B200_EINVAL, "null argument");
    if (stride_items < n_items) return fail(LORA_B200_EINVAL, "stride_items %zu < n_items %zu", stride_items, n_items);
    if (int rc = need_k1(d, "the dechirp receiver")) return rc;
    lora_b200_rx_params P;
    memset(&P, 0, sizeof P);
    if (prm) P = *prm;
    const uint32_t crc2 = d->cfg.crc ? 2u : 0u;
    if (d->cfg.implicit && (P.implicit_len == 0 || P.implicit_len > 255u + crc2))
        return fail(LORA_B200_EINVAL, "an implicit-header decoder needs implicit_len in 1..%u, got %u", 255u + crc2, P.implicit_len);
    if (!std::isfinite(P.sfo_ppm) || std::fabs(P.sfo_ppm) > 500.0f)
        return fail(LORA_B200_EINVAL, "sfo_ppm must be finite and within +-500, got %g", (double)P.sfo_ppm);
    if (P.carrier_hz != 0.0 && !(std::isfinite(P.carrier_hz) && P.carrier_hz > d->samples_per_second))
        return fail(LORA_B200_EINVAL, "carrier_hz must be 0 or above the sample rate %g, got %g", d->samples_per_second, P.carrier_hz);
    if (P.soft > 1u) return fail(LORA_B200_EINVAL, "soft must be 0 or 1, got %u", (unsigned)P.soft);
    if (P.crc_list > RS_CRC_MAX_LIST || (P.crc_list && !P.soft))
        return fail(LORA_B200_EINVAL, "crc_list must be 0..%u and needs soft = 1, got %u", RS_CRC_MAX_LIST, (unsigned)P.crc_list);
    if (P.wide_cfo > 1u) return fail(LORA_B200_EINVAL, "wide_cfo must be 0 or 1, got %u", (unsigned)P.wide_cfo);
    if (P.fine_toa > 1u) return fail(LORA_B200_EINVAL, "fine_toa must be 0 or 1, got %u", (unsigned)P.fine_toa);
    const float band_max = (float)((d->samples_per_second - (double)d->cfg.bandwidth) / 2.0);    // (fs - BW) / 2
    if (P.wide_cfo && !(std::isfinite(P.max_cfo_hz) && P.max_cfo_hz > 0.f && P.max_cfo_hz <= band_max))
        return fail(LORA_B200_EINVAL, "wide_cfo needs max_cfo_hz in (0, %g], got %g", (double)band_max, (double)P.max_cfo_hz);
    CU(cudaSetDevice(d->device));
    // rows: ns; receivers (groups of m antenna rows): ng.  m = 1 is lora_b200_receive, launch for launch.
    const uint32_t rows = d->cfg.n_streams, ns = rows / m, sps = d->sps, N = d->n_bins, cap = d->cfg.max_frames_per_call;
    const bool soft = P.soft != 0;
    const uint8_t sw = P.sync_word ? P.sync_word : 0x12;
    const float fs = (float)d->samples_per_second, bin_hz = fs / (float)sps;
    const float max_cfo = P.wide_cfo ? P.max_cfo_hz
                          : P.max_cfo_hz > 0.f && P.max_cfo_hz < d->cfg.bandwidth / 4.0f ? P.max_cfo_hz : d->cfg.bandwidth / 4.0f;
    const float ppm_per_bin = P.carrier_hz > 0.0 ? (float)(1e6 * (double)bin_hz / P.carrier_hz) : 0.0f;
    RsParams rp{sps, N, d->decim, P.sfo_ppm, P.min_preamble ? P.min_preamble : 5u, {((sw >> 4) & 15u) * 8u % N, (sw & 15u) * 8u % N},
                max_cfo / bin_hz, ppm_per_bin, 0};
    rp.hyp = rs_hypotheses(rp.max_cfo_bins, N);
    // end of the window of data symbol n - 1 of a frame (its first n data symbols inside the row)
    auto data_end = [&](const RsFrame &r, long long n) { return rs_sym(r.start, rs_data_j(n - 1), sps, r.sfo_ppm) + (long long)sps; };
    d->rs_info.clear();
    d->h_sorted.clear();
    d->rs_hdr_drops = 0;
    d->rs_chan.clear();
    d->rs_chan_m = m;
    d->rs_recovered.clear();
    d->rs_toa.clear();
    const size_t guard = (size_t)(rp.min_preamble + 4u) * sps, none = ~(size_t)0;
    std::vector<size_t> end_pub(ns, 0), hold(ns, none);
    auto finish = [&]() {
        for (uint32_t s = 0; s < ns; s++) {
            size_t c = n_items > guard ? n_items - guard : 0;
            if (hold[s] < c) c = hold[s];
            consumed[s] = std::max(c, end_pub[s]);
        }
        return LORA_B200_OK;
    };
    if (n_items < (size_t)sps + sps / 2) return finish();
    cudaStream_t st = d->rx_stream;
    // the screen runs K1 straight over the rows when a row is a whole number of windows, else over a padded copy
    const float2 *x = (const float2 *)iq;
    size_t stride = stride_items;
    if (host_ptr || stride % sps || ((uintptr_t)iq & 15u)) {
        stride = (n_items + sps - 1) / sps * sps;
        CU(d->d_rs_stage.reserve(stride * rows));
        CU(cudaMemcpy2DAsync(d->d_rs_stage, sizeof(float2) * stride, iq, sizeof(float2) * stride_items, sizeof(float2) * n_items, rows,
                             host_ptr ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, st));
        x = d->d_rs_stage;
    }
    // wide_cfo: the shifted tables of hypotheses -hyp..hyp, at shift[((c + hyp) * 2 + up) * sps]
    const float2 *shift = nullptr;
    if (rp.hyp > 0) {
        if (rp.hyp > d->rs_shift_hyp) {
            const size_t n_tab = (size_t)(2 * rp.hyp + 1) * 2 * sps;
            d->h_rs_shift.resize(n_tab);
            rs_shift_tables((const float2 *)(d->h_tables.data() + d->toff.down), (const float2 *)(d->h_tables.data() + d->toff.up), sps,
                            d->decim, rp.hyp, d->h_rs_shift.data());
            CU(d->d_rs_shift.reserve(n_tab));
            CU(cudaMemcpyAsync(d->d_rs_shift, d->h_rs_shift.data(), sizeof(float2) * n_tab, cudaMemcpyHostToDevice, st));
            d->rs_shift_hyp = rp.hyp;
        }
        shift = d->d_rs_shift + (size_t)(d->rs_shift_hyp - rp.hyp) * 2 * sps;
    }
    // the screen of hypothesis h - hyp (h = 0 .. 2 hyp) at bins / mags[ph][h * hs ..]; hypothesis 0 dechirps with the
    // decoder's own table
    const size_t hs = (size_t)ns * (stride / sps) + 1, n_hyp = 2 * (size_t)rp.hyp + 1;
    auto screen_chirp = [&](size_t h) { return (int)h == rp.hyp ? nullptr : shift + h * 2 * sps; };
    for (int ph = 0; ph < 2; ph++) {
        CU(d->d_rs_bins[ph].reserve(n_hyp * hs));
        CU(d->d_rs_mags[ph].reserve(n_hyp * hs));
    }
    if (m == 1) {
        const size_t span = (ns - 1) * stride + n_items, nw[2] = {span / sps, (span - sps / 2) / sps};
        for (size_t h = 0; h < n_hyp; h++)
            for (int ph = 0; ph < 2; ph++)
                if (int rc = dispatch_k1(d, d->k1s[0], x + ph * (sps / 2), nw[ph], d->d_rs_bins[ph] + h * hs, d->d_rs_mags[ph] + h * hs, st,
                                         screen_chirp(h)))
                    return rc;
    } else {
        // the combined screen: receiver g's window j of phase ph at bins[ph][g * stride / sps + j], as rs_detect_kernel reads
        // the screen of one row (only the windows it reads are computed)
        const size_t nw[2] = {n_items / sps, n_items >= sps + sps / 2 ? (n_items - sps / 2) / sps : 0};
        for (size_t h = 0; h < n_hyp; h++)
            for (int ph = 0; ph < 2; ph++) {
                if (nw[ph] == 0) continue;
                if (int rc = rs_screen(d, x + ph * (sps / 2), nw[ph], stride, m, ns, stride / sps, d->d_rs_bins[ph] + h * hs,
                                       d->d_rs_mags[ph] + h * hs, st, screen_chirp(h)))
                    return rc;
            }
        CU(d->d_rs_chan.reserve((size_t)ns * cap * 2 * RS_MAX_ANTENNAS));
    }
    // detect, synchronise
    const uint32_t fcap = ns * cap;
    CU(d->d_rs_cands.reserve(fcap));
    CU(d->d_rs_ncand.reserve(ns));
    CU(d->d_rs_dropped.reserve(ns));
    CU(d->d_rs_hold.reserve(ns));
    CU(d->d_rs_frames.reserve(fcap));
    CU(d->d_rs_nframes.reserve(1));
    CU(cudaMemsetAsync(d->d_rs_hold, 0xFF, sizeof(unsigned long long) * ns, st));
    CU(cudaMemsetAsync(d->d_rs_nframes, 0, sizeof(uint32_t), st));
    // the screens bound of the detector: 2 (the one hypothesis c = 0), else that of the decoder's rate (rs_max_screens)
    auto detect = [&](auto S_MAX) {
        rs_detect_kernel<S_MAX><<<(ns + 127) / 128, 128, 0, st>>>(d->d_rs_bins[0], d->d_rs_mags[0], d->d_rs_bins[1], d->d_rs_mags[1], hs,
                                                                  stride, n_items, ns, rp, d->d_rs_cands, cap, d->d_rs_ncand, d->d_rs_dropped);
        return launched(d);
    };
    const int rc_detect = rp.hyp == 0          ? detect(std::integral_constant<int, 2>{})
                          : rp.hyp <= RS_MAX_HYP ? detect(std::integral_constant<int, RS_MAX_SCREENS>{})
                          : rp.hyp <= rs_max_hyp(16) ? detect(std::integral_constant<int, rs_max_screens(16)>{})
                                                     : detect(std::integral_constant<int, rs_max_screens(32)>{});
    if (rc_detect) return rc_detect;
    if (int rc = rs_sync(d, x, stride, n_items, rp, cap, m, shift)) return rc;
    uint32_t n_sync = 0;
    std::vector<long long> dropped(ns);
    std::vector<unsigned long long> shold(ns);
    CU(cudaMemcpyAsync(&n_sync, d->d_rs_nframes, sizeof n_sync, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(dropped.data(), d->d_rs_dropped, sizeof(long long) * ns, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(shold.data(), d->d_rs_hold, sizeof(unsigned long long) * ns, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (uint32_t s = 0; s < ns; s++) {
        if (dropped[s] >= 0) hold[s] = std::min(hold[s], (size_t)dropped[s]);
        if (shold[s] != ~0ull) hold[s] = std::min(hold[s], (size_t)(shold[s] > sps ? shold[s] - sps : 0));
    }
    n_sync = std::min(n_sync, fcap);
    if (n_sync == 0) return finish();
    // header round: 8 windows per frame, assembled and demodulated in batches of at most 256 MiB of windows
    const size_t win_cap = std::max<size_t>(1024, ((size_t)256 << 20) / (sizeof(float2) * sps));
    CU(d->d_rs_win.reserve(win_cap * sps));
    CU(d->d_rs_hbins.reserve((size_t)n_sync * 8));
    // soft decisions: LLRs of ppm values per window (sf - 2 in the header round), corrected into the bins afterwards
    // (with list decoding they go to a buffer of their own, which the payload round does not reuse)
    const uint32_t hppm = d->cfg.sf - 2u, pppm = d->cfg.reduced_rate ? hppm : d->cfg.sf;
    DeviceBuffer<float> &hllr = P.crc_list ? d->d_rs_hllr : d->d_rs_llr;
    if (soft) CU(hllr.reserve((size_t)n_sync * 8 * hppm));
    for (uint32_t f0 = 0; f0 < n_sync; f0 += (uint32_t)(win_cap / 8)) {
        const uint32_t nb = (uint32_t)std::min<size_t>(win_cap / 8, n_sync - f0);
        if (int rc = rs_assemble(d, x, stride, n_items, m, d->d_rs_frames + f0, m > 1 ? d->d_rs_chan + (size_t)f0 * 2 * RS_MAX_ANTENNAS : nullptr,
                                 nb, nullptr, 0, nullptr, 0, nullptr))
            return rc;
        if (soft) {
            if (int rc = dispatch_llr(d, d->d_rs_win, (size_t)nb * 8, true, hllr + (size_t)f0 * 8 * hppm, nullptr, st)) return rc;
        } else if (int rc = dispatch_k1(d, d->k1s[0], d->d_rs_win, (size_t)nb * 8, d->d_rs_hbins + (size_t)f0 * 8, nullptr, st)) {
            return rc;
        }
    }
    RxParams rxp;
    memset(&rxp, 0, sizeof rxp);
    rxp.sps = sps; rxp.n_bins = N; rxp.n_bins_hdr = d->n_bins_hdr; rxp.decim = d->decim; rxp.sf = d->cfg.sf;
    rxp.implicit = d->cfg.implicit; rxp.reduced_rate = d->cfg.reduced_rate;
    if (soft) {
        rs_soft_header_kernel<<<(n_sync + 127) / 128, 128, 0, st>>>(n_sync, rxp, d->phdr1_init, hllr, d->d_rs_hbins);
        if (int rc = launched(d)) return rc;
    }
    rs_header_kernel<<<(n_sync + 127) / 128, 128, 0, st>>>(d->d_rs_frames, d->d_rs_nframes, fcap, rxp, d->phdr1_init, d->d_rs_hbins,
                                                           P.implicit_len);
    if (int rc = launched(d)) return rc;
    std::vector<RsFrame> fr(n_sync);
    CU(cudaMemcpyAsync(fr.data(), d->d_rs_frames, sizeof(RsFrame) * n_sync, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    // one frame per preamble: candidates of one stream whose starts lie within a symbol of the previous synchronised one are
    // the same preamble (found in both screen phases); the group keeps its best member -- a decodable header first, then
    // the higher SNR -- and only that member is held back, dropped or published
    std::vector<uint32_t> order(n_sync), reps, pub;
    for (uint32_t f = 0; f < n_sync; f++) order[f] = f;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
        return fr[a].stream != fr[b].stream ? fr[a].stream < fr[b].stream : fr[a].start < fr[b].start;
    });
    for (uint32_t k = 0; k < n_sync; k++) {
        const uint32_t f = order[k], prev = k ? order[k - 1] : f;
        if (k && fr[prev].stream == fr[f].stream && fr[f].start - fr[prev].start < (long long)sps) {
            const RsFrame &a = fr[reps.back()], &b = fr[f];
            if ((b.n_payload >= 0) > (a.n_payload >= 0) || ((b.n_payload >= 0) == (a.n_payload >= 0) && b.snr_db > a.snr_db)) reps.back() = f;
            continue;
        }
        reps.push_back(f);
    }
    // which frames are whole inside this call
    for (uint32_t f : reps) {
        const RsFrame &r = fr[f];
        if (data_end(r, 8) > (long long)n_items || (r.n_payload >= 0 && data_end(r, 8ll + r.n_payload) > (long long)n_items)) {
            hold[r.stream] = std::min(hold[r.stream], (size_t)std::max<long long>(0, r.start - (long long)sps));
            continue;
        }
        if (r.n_payload < 0) { d->rs_hdr_drops++; continue; }
        pub.push_back(f);
    }
    const uint32_t np = (uint32_t)pub.size();
    if (np == 0) return finish();
    // payload round: table pub | seq | offs | cnts, windows in batches
    std::vector<uint32_t> tabh(4 * (size_t)np);
    uint32_t total = 0, seq = 0;
    for (uint32_t k = 0; k < np; k++) {
        const RsFrame &r = fr[pub[k]];
        seq = (k && fr[pub[k - 1]].stream == r.stream) ? seq + 1 : 0;
        tabh[k] = pub[k]; tabh[np + k] = seq; tabh[2 * np + k] = total; tabh[3 * np + k] = (uint32_t)r.n_payload;
        total += (uint32_t)r.n_payload;
    }
    CU(d->d_rs_tab.reserve(tabh.size()));
    CU(cudaMemcpyAsync(d->d_rs_tab, tabh.data(), sizeof(uint32_t) * tabh.size(), cudaMemcpyHostToDevice, st));
    CU(d->d_rs_pbins.reserve(std::max<uint32_t>(total, 1u)));
    // a batch holds whole frames: the window buffer grows to the longest frame if that is more than a batch
    size_t pwin_cap = win_cap;
    for (uint32_t k = 0; k < np; k++) pwin_cap = std::max<size_t>(pwin_cap, tabh[3 * np + k]);
    CU(d->d_rs_win.reserve(pwin_cap * sps));
    if (soft) CU(d->d_rs_llr.reserve((size_t)std::max<uint32_t>(total, 1u) * pppm));
    const uint32_t *t_pub = d->d_rs_tab, *t_seq = t_pub + np, *t_off = t_pub + 2 * np, *t_cnt = t_pub + 3 * np;
    for (uint32_t g0 = 0; g0 < np;) {
        uint32_t g1 = g0, w = 0;
        while (g1 < np && w + tabh[3 * np + g1] <= pwin_cap) w += tabh[3 * np + g1++];
        if (w) {
            if (int rc = rs_assemble(d, x, stride, n_items, m, d->d_rs_frames, d->d_rs_chan, g1 - g0, t_pub + g0, 8, t_off + g0,
                                     tabh[2 * np + g0], t_cnt + g0))
                return rc;
            const size_t o = tabh[2 * np + g0];
            if (soft) {
                if (int rc = dispatch_llr(d, d->d_rs_win, w, d->cfg.reduced_rate != 0, d->d_rs_llr + o * pppm, nullptr, st)) return rc;
            } else if (int rc = dispatch_k1(d, d->k1s[0], d->d_rs_win, w, d->d_rs_pbins + o, nullptr, st)) {
                return rc;
            }
        }
        g0 = g1;
    }
    if (soft) {
        rs_soft_payload_kernel<<<(np + 127) / 128, 128, 0, st>>>(d->d_rs_frames, t_pub, np, rxp, d->phdr1_init, d->d_rs_hbins, t_off,
                                                                  P.implicit_len, d->d_rs_llr, d->d_rs_pbins);
        if (int rc = launched(d)) return rc;
    }
    if (P.crc_list) {
        CU(d->d_rs_recovered.reserve(np));
        rs_crc_list_kernel<<<(np + RS_CRC_WARPS - 1) / RS_CRC_WARPS, 32 * RS_CRC_WARPS, 0, st>>>(
            d->d_rs_frames, t_pub, np, rxp, d->phdr1_init, P.crc_list, d->d_rs_hbins, t_off, P.implicit_len, d->d_rs_hllr, d->d_rs_llr,
            d->d_rs_pbins, d->d_rs_recovered);
        if (int rc = launched(d)) return rc;
    }
    CU(d->d_rs_recs.reserve(np));
    CU(d->d_rs_out.reserve(np));
    rs_frame_kernel<<<(np + 127) / 128, 128, 0, st>>>(d->d_rs_frames, t_pub, t_seq, np, rxp, d->phdr1_init, d->d_rs_hbins, d->d_rs_pbins,
                                                      t_off, P.implicit_len, d->d_rs_recs);
    if (int rc = launched(d)) return rc;
    CU(cudaMemcpyAsync(d->d_rs_nframes, &np, sizeof np, cudaMemcpyHostToDevice, st));
    // K8 writes a record's first len bytes only: zero the rest, so that a published record never carries stale device
    // memory (after soft decisions, LLRs of an earlier call or decoder)
    CU(cudaMemsetAsync(d->d_rs_out, 0, sizeof(RxFrameOut) * np, st));
    k8_frames_kernel<<<(int)std::min<uint32_t>(np, (uint32_t)d->n_sms * 4u), 128, 0, st>>>(d->d_rs_recs, d->d_rs_nframes, np, d->d_rs_out);
    if (int rc = launched(d)) return rc;
    if (P.fine_toa) {
        CU(d->d_rs_toa.reserve(np));
        if (int rc = rs_toa(d, x, stride, n_items, m, rp, d->d_rs_frames, t_pub, np, d->d_rs_toa, nullptr)) return rc;
        d->rs_toa.resize(np);
        CU(cudaMemcpyAsync(d->rs_toa.data(), d->d_rs_toa, sizeof(double) * np, cudaMemcpyDeviceToHost, st));
    }
    d->h_sorted.resize(np);
    CU(cudaMemcpyAsync(d->h_sorted.data(), d->d_rs_out, sizeof(RxFrameOut) * np, cudaMemcpyDeviceToHost, st));
    std::vector<float2> chan;
    if (m > 1) {
        chan.resize((size_t)n_sync * 2 * RS_MAX_ANTENNAS);
        CU(cudaMemcpyAsync(chan.data(), d->d_rs_chan, sizeof(float2) * chan.size(), cudaMemcpyDeviceToHost, st));
    }
    if (P.crc_list) {
        d->rs_recovered.resize(np);
        CU(cudaMemcpyAsync(d->rs_recovered.data(), d->d_rs_recovered, np, cudaMemcpyDeviceToHost, st));
    }
    CU(cudaStreamSynchronize(st));
    d->rs_info.resize(np);
    for (uint32_t k = 0; k < np; k++) {
        const RsFrame &r = fr[pub[k]];
        const long long d0 = rs_sym(r.start, rs_data_j(0), sps, r.sfo_ppm);
        d->rs_info[k] = lora_b200_rx_info{(uint64_t)r.start, (uint64_t)d0, r.stream, r.cfo_bins * bin_hz, r.snr_db, r.sfo_ppm};
        end_pub[r.stream] = std::max(end_pub[r.stream], (size_t)data_end(r, 8ll + r.n_payload));
        if (m > 1) d->rs_chan.insert(d->rs_chan.end(), chan.begin() + (size_t)pub[k] * 2 * RS_MAX_ANTENNAS,
                                     chan.begin() + (size_t)pub[k] * 2 * RS_MAX_ANTENNAS + m);
    }
    return finish();
}

extern "C" {

int lora_b200_receive(lora_b200_decoder *d, const void *iq, size_t n_items, size_t stride_items, int host_ptr,
                      const lora_b200_rx_params *prm, size_t *consumed) {
    return rs_receive(d, iq, n_items, stride_items, host_ptr, 1, prm, consumed);
}

int lora_b200_receive_antennas(lora_b200_decoder *d, const void *iq, size_t n_items, size_t stride_items, int host_ptr,
                               uint32_t n_antennas, const lora_b200_rx_params *p, size_t *consumed) {
    if (!d) return fail(LORA_B200_EINVAL, "null argument");
    if (n_antennas < 1 || n_antennas > (uint32_t)RS_MAX_ANTENNAS || d->cfg.n_streams % n_antennas)
        return fail(LORA_B200_EINVAL, "n_antennas must be 1..%d and divide n_streams %u, got %u", RS_MAX_ANTENNAS, d->cfg.n_streams,
                    n_antennas);
    return rs_receive(d, iq, n_items, stride_items, host_ptr, n_antennas, p, consumed);
}

size_t lora_b200_rx_channels_last(lora_b200_decoder *d, const float **h, uint32_t *n_antennas) {
    if (!d || !h) { fail(LORA_B200_EINVAL, "null argument"); return 0; }
    *h = reinterpret_cast<const float *>(d->rs_chan.data());
    if (n_antennas) *n_antennas = d->rs_chan_m;
    return d->rs_chan_m > 1 ? d->rs_chan.size() / d->rs_chan_m : 0;
}

int lora_b200_demod_fft_antennas_dev(lora_b200_decoder *d, const void *iq, uint32_t n_groups, uint32_t n_antennas, size_t n_symbols,
                                     size_t row_stride_items, uint32_t *bins, float *mags, void *cuda_stream) {
    if (!d || (n_symbols && n_groups && (!iq || !bins || !mags))) return fail(LORA_B200_EINVAL, "null argument");
    if (int rc = need_k1(d, "the combined screen")) return rc;
    if (n_antennas < 1 || n_antennas > (uint32_t)RS_MAX_ANTENNAS) return fail(LORA_B200_EINVAL, "n_antennas must be 1..%d, got %u", RS_MAX_ANTENNAS, n_antennas);
    if (row_stride_items < n_symbols * d->sps || row_stride_items % 2 || ((uintptr_t)iq & 15u))
        return fail(LORA_B200_EINVAL, "rows must hold n_symbols windows, start 16-byte aligned and lie an even number of samples apart");
    CU(cudaSetDevice(d->device));
    if (n_symbols == 0 || n_groups == 0) return LORA_B200_OK;
    return rs_screen(d, (const float2 *)iq, n_symbols, row_stride_items, n_antennas, n_groups, n_symbols, bins, mags, (cudaStream_t)cuda_stream);
}

static_assert(sizeof(lora_b200_rx_info) == 32 && sizeof(lora_b200_rx_params) == 32 && offsetof(lora_b200_rx_params, soft) == 1 &&
              offsetof(lora_b200_rx_params, crc_list) == 2 && offsetof(lora_b200_rx_params, wide_cfo) == 3 &&
              offsetof(lora_b200_rx_params, implicit_len) == 4 &&
              offsetof(lora_b200_rx_params, sfo_ppm) == 16 && offsetof(lora_b200_rx_params, fine_toa) == 20 &&
              offsetof(lora_b200_rx_params, reserved1) == 21 && offsetof(lora_b200_rx_params, carrier_hz) == 24 && offsetof(lora_b200_rx_info, sfo_ppm) == 28, "lora_b200_rx_* layout");

}  // extern "C"

template <int SF, int D>
static int rs_window_launch(lora_b200_decoder *d, const float2 *x, size_t stride, size_t n_items, uint32_t m, const RsWindowQuery *q,
                            size_t n, float2 *out, float *energy, unsigned long long *key) {
    const size_t smem = sizeof(float2) * K1Cfg<SF, D>::SMEM_ELEMS;   // (the synchronise kernels' dynamic shared memory)
    CU(opt_in_smem((const void *)rs_window_kernel<SF, D>, d->device, smem));
    rs_window_kernel<SF, D><<<(unsigned)n, RX_THREADS, smem, d->rx_stream>>>(x, stride, (long long)n_items, m, tab<float2>(d, d->toff.down),
                                                                             tab<float2>(d, d->toff.up), tab<float2>(d, d->toff.tw), d->sps,
                                                                             q, out, energy, key);
    return launched(d);
}

template <int SF, int D, bool DRIFT>
static int rs_channels_launch(lora_b200_decoder *d, const float2 *x, size_t stride, size_t n_items, uint32_t m, const RsParams &rp,
                              const RsFrame *frames, size_t n, float2 *chan, float *snr_db) {
    rs_channels_kernel<SF, D, DRIFT><<<(unsigned)n, RX_THREADS, 0, d->rx_stream>>>(x, stride, n_items, m, tab<float2>(d, d->toff.down),
                                                                                  tab<float2>(d, d->toff.up), tab<float2>(d, d->toff.tw),
                                                                                  rp, frames, chan, snr_db);
    return launched(d);
}

extern "C" {

int lora_b200_rs_window_dev(lora_b200_decoder *d, const void *iq, size_t n_items, uint32_t m, size_t stride_items, size_t n,
                            const int64_t *pos, const float *cfo_bins, const int32_t *up, const int32_t *bin, void *out, float *energy,
                            uint32_t *argmax_bin, float *argmax_mag) {
    if (!d || (n && (!iq || !pos || !cfo_bins || !up || !bin || !out)))
        return fail(LORA_B200_EINVAL, "null argument");
    if (int rc = need_k1(d, "the dechirp receiver")) return rc;
    if (m < 1 || m > (uint32_t)RS_MAX_ANTENNAS) return fail(LORA_B200_EINVAL, "m must be 1..%d, got %u", RS_MAX_ANTENNAS, m);
    if (m > 1 && stride_items < n_items) return fail(LORA_B200_EINVAL, "stride_items %zu < n_items %zu", stride_items, n_items);
    if (n > 0x7FFFFFFFu) return fail(LORA_B200_EINVAL, "too many windows: %zu", n);
    const long long sps = d->sps, N = d->n_bins;
    // the widest offset the synchroniser evaluates windows at: (fs - BW) / 2 = (D - 1) N / 2 bins (wide_cfo), at least N
    const long long cfo_lim = std::max<long long>(N, ((long long)d->decim - 1) * N / 2);
    std::vector<RsWindowQuery> q(n);
    for (size_t i = 0; i < n; i++) {
        if (pos[i] < 0 || pos[i] + sps > (long long)n_items)
            return fail(LORA_B200_EINVAL, "window %zu: [%lld, %lld) is not inside the row of %zu samples", i, (long long)pos[i],
                        (long long)pos[i] + sps, n_items);
        if (up[i] != 0 && up[i] != 1) return fail(LORA_B200_EINVAL, "window %zu: up must be 0 or 1, got %d", i, up[i]);
        if (bin[i] < -N / 2 || bin[i] >= N / 2) return fail(LORA_B200_EINVAL, "window %zu: bin %d outside -N/2..N/2-1", i, bin[i]);
        if (!std::isfinite(cfo_bins[i]) || std::fabs(cfo_bins[i]) > (float)cfo_lim)
            return fail(LORA_B200_EINVAL, "window %zu: cfo_bins %g is not finite within +-%lld", i, (double)cfo_bins[i], cfo_lim);
        q[i] = RsWindowQuery{(long long)pos[i], cfo_bins[i], up[i], bin[i], 0};
    }
    CU(cudaSetDevice(d->device));
    if (n == 0) return LORA_B200_OK;
    DeviceBuffer<RsWindowQuery> dq;
    DeviceBuffer<unsigned long long> dk;
    CU(dq.reserve(n));
    CU(dk.reserve(n));
    CU(cudaMemcpyAsync(dq, q.data(), sizeof(RsWindowQuery) * n, cudaMemcpyHostToDevice, d->rx_stream));
    int rc = with_sf_osr(d->cfg.sf, d->k1_osr, unsupported_sf(d), [&](auto SF, auto D) {
        return rs_window_launch<SF, D>(d, (const float2 *)iq, stride_items, n_items, m, dq, n, (float2 *)out, energy, dk);
    });
    std::vector<unsigned long long> keys(n);
    if (rc == LORA_B200_OK) CU(cudaMemcpyAsync(keys.data(), dk, sizeof(unsigned long long) * n, cudaMemcpyDeviceToHost, d->rx_stream));
    CU(cudaStreamSynchronize(d->rx_stream));     // (before dq and dk are freed)
    if (rc != LORA_B200_OK) return rc;
    std::vector<uint32_t> kb(n);
    std::vector<float> km(n);
    for (size_t i = 0; i < n; i++) k1_store(kb.data(), km.data(), i, keys[i]);
    if (argmax_bin) CU(cudaMemcpy(argmax_bin, kb.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice));
    if (argmax_mag) CU(cudaMemcpy(argmax_mag, km.data(), sizeof(float) * n, cudaMemcpyHostToDevice));
    return LORA_B200_OK;
}

int lora_b200_rs_frame_dev(lora_b200_decoder *d, const void *iq, size_t n_items, uint32_t m, size_t stride_items, size_t n,
                           const uint32_t *group, const int64_t *start, const float *cfo_bins, const float *sfo_ppm, uint32_t first,
                           uint32_t cnt, void *chan, float *snr_db, void *windows) {
    if (!d || (n && (!iq || !group || !start || !cfo_bins || !sfo_ppm || (cnt && !windows) || (m > 1 && (!chan || !snr_db)))))
        return fail(LORA_B200_EINVAL, "null argument");
    if (int rc = need_k1(d, "the dechirp receiver")) return rc;
    if (m < 1 || m > (uint32_t)RS_MAX_ANTENNAS) return fail(LORA_B200_EINVAL, "m must be 1..%d, got %u", RS_MAX_ANTENNAS, m);
    if (stride_items < n_items) return fail(LORA_B200_EINVAL, "stride_items %zu < n_items %zu", stride_items, n_items);
    if (n > 0x7FFFFFFFu || (size_t)cnt * n > 0xFFFFFFFFu) return fail(LORA_B200_EINVAL, "too many frames or windows: %zu x %u", n, cnt);
    const uint32_t sps = d->sps;
    std::vector<RsFrame> fr(n);
    bool drift = false;
    for (size_t i = 0; i < n; i++) {
        if (!std::isfinite(cfo_bins[i]) || std::fabs(cfo_bins[i]) > (float)d->n_bins || !std::isfinite(sfo_ppm[i]) || std::fabs(sfo_ppm[i]) > 1e4f)
            return fail(LORA_B200_EINVAL, "frame %zu: cfo_bins %g or sfo_ppm %g out of range", i, (double)cfo_bins[i], (double)sfo_ppm[i]);
        if (cnt && rs_sym(start[i], rs_data_j((long long)first), sps, sfo_ppm[i]) < 0)
            return fail(LORA_B200_EINVAL, "frame %zu: data window %u starts before the row", i, first);
        fr[i] = RsFrame{(long long)start[i], group[i], cfo_bins[i], 0.f, RS_OK, 0, sfo_ppm[i]};
        drift = drift || sfo_ppm[i] != 0.f;
    }
    CU(cudaSetDevice(d->device));
    if (n == 0) return LORA_B200_OK;
    std::vector<uint32_t> tabh(2 * n);                // offs | cnts of the assemble kernels
    for (size_t i = 0; i < n; i++) { tabh[i] = (uint32_t)(i * cnt); tabh[n + i] = cnt; }
    DeviceBuffer<RsFrame> df;
    DeviceBuffer<uint32_t> dt;
    CU(df.reserve(n));
    CU(dt.reserve(2 * n));
    CU(cudaMemcpyAsync(df, fr.data(), sizeof(RsFrame) * n, cudaMemcpyHostToDevice, d->rx_stream));
    CU(cudaMemcpyAsync(dt, tabh.data(), sizeof(uint32_t) * 2 * n, cudaMemcpyHostToDevice, d->rx_stream));
    const float2 *x = (const float2 *)iq;
    int rc = LORA_B200_OK;
    if (m > 1) {
        RsParams rp{sps, d->n_bins, d->decim, 0.f, 5u, {0u, 0u}, (float)d->n_bins / 4.0f, 0.f};   // (rs_channels reads sps, decim)
        rc = with_sf_osr(d->cfg.sf, d->k1_osr, unsupported_sf(d), [&](auto SF, auto D) {
            return with_bool(drift, [&](auto DRIFT) {
                return rs_channels_launch<SF, D, DRIFT>(d, x, stride_items, n_items, m, rp, df, n, (float2 *)chan, snr_db);
            });
        });
    }
    if (rc == LORA_B200_OK && cnt) {
        const int grid = std::min<int>((int)n, d->n_sms * 8);
        if (m == 1)
            rs_assemble_kernel<<<grid, 256, 0, d->rx_stream>>>(x, stride_items, (long long)n_items, df, (uint32_t)n, nullptr, first, dt, 0,
                                                               dt + n, sps, (float2 *)windows);
        else
            rs_assemble_antennas_kernel<<<grid, 256, 0, d->rx_stream>>>(x, stride_items, (long long)n_items, m, df, (const float2 *)chan,
                                                                        (uint32_t)n, nullptr, first, dt, 0, dt + n, sps, (float2 *)windows);
        rc = launched(d);
    }
    CU(cudaStreamSynchronize(d->rx_stream));     // (before df and dt are freed)
    return rc;
}

size_t lora_b200_rx_toa_last(lora_b200_decoder *d, const double **toa) {
    if (!d || !toa) { fail(LORA_B200_EINVAL, "null argument"); return 0; }
    *toa = d->rs_toa.data();
    return d->rs_toa.size();
}

int lora_b200_rs_toa_dev(lora_b200_decoder *d, const void *iq, size_t n_items, uint32_t m, size_t stride_items, size_t n,
                         const uint32_t *group, const int64_t *start, const float *cfo_bins, const float *sfo_ppm, float *nu_a,
                         float *nu_b, double *toa) {
    if (!d || (n && (!iq || !group || !start || !cfo_bins || !sfo_ppm || !nu_a || !nu_b || !toa))) return fail(LORA_B200_EINVAL, "null argument");
    if (int rc = need_k1(d, "the dechirp receiver")) return rc;
    if (m < 1 || m > (uint32_t)RS_MAX_ANTENNAS) return fail(LORA_B200_EINVAL, "m must be 1..%d, got %u", RS_MAX_ANTENNAS, m);
    if (stride_items < n_items) return fail(LORA_B200_EINVAL, "stride_items %zu < n_items %zu", stride_items, n_items);
    if (n > 0x7FFFFFFFu) return fail(LORA_B200_EINVAL, "too many frames: %zu", n);
    const long long cfo_lim = std::max<long long>(d->n_bins, ((long long)d->decim - 1) * d->n_bins / 2);   // (as rs_window_dev)
    std::vector<RsFrame> fr(n);
    bool drift = false;
    for (size_t i = 0; i < n; i++) {
        if (!std::isfinite(cfo_bins[i]) || std::fabs(cfo_bins[i]) > (float)cfo_lim || !std::isfinite(sfo_ppm[i]) || std::fabs(sfo_ppm[i]) > 1e4f)
            return fail(LORA_B200_EINVAL, "frame %zu: cfo_bins %g or sfo_ppm %g out of range", i, (double)cfo_bins[i], (double)sfo_ppm[i]);
        fr[i] = RsFrame{(long long)start[i], group[i], cfo_bins[i], 0.f, RS_OK, 0, sfo_ppm[i]};
        drift = drift || sfo_ppm[i] != 0.f;
    }
    CU(cudaSetDevice(d->device));
    if (n == 0) return LORA_B200_OK;
    DeviceBuffer<RsFrame> df;
    DeviceBuffer<double> dt;
    DeviceBuffer<float2> dn;
    CU(df.reserve(n));
    CU(dt.reserve(n));
    CU(dn.reserve(n));
    CU(cudaMemcpyAsync(df, fr.data(), sizeof(RsFrame) * n, cudaMemcpyHostToDevice, d->rx_stream));
    // rs_toa reads sps, decim; DRIFT from any frame's clock offset (a frame with 0 gives the DRIFT = false result either way)
    RsParams rp{d->sps, d->n_bins, d->decim, drift ? 1.f : 0.f, 5u, {0u, 0u}, (float)d->n_bins / 4.0f, 0.f, 0};
    int rc = rs_toa(d, (const float2 *)iq, stride_items, n_items, m, rp, df, nullptr, (uint32_t)n, dt, dn);
    std::vector<float2> nu(n);
    if (rc == LORA_B200_OK) {
        CU(cudaMemcpyAsync(toa, dt, sizeof(double) * n, cudaMemcpyDeviceToHost, d->rx_stream));
        CU(cudaMemcpyAsync(nu.data(), dn, sizeof(float2) * n, cudaMemcpyDeviceToHost, d->rx_stream));
    }
    CU(cudaStreamSynchronize(d->rx_stream));     // (before df, dt and dn are freed)
    for (size_t i = 0; rc == LORA_B200_OK && i < n; i++) { nu_a[i] = nu[i].x; nu_b[i] = nu[i].y; }
    return rc;
}

size_t lora_b200_rx_info_last(lora_b200_decoder *d, const lora_b200_rx_info **info, uint32_t *hdr_drops) {
    if (!d || !info) { fail(LORA_B200_EINVAL, "null argument"); return 0; }
    *info = d->rs_info.data();
    if (hdr_drops) *hdr_drops = d->rs_hdr_drops;
    return d->rs_info.size();
}

int lora_b200_work_batch_sc8(lora_b200_decoder *d, const void *iq_sc8, float scale, size_t n_items, size_t stride_items,
                             int host_ptr, size_t *consumed, lora_b200_frame_cb cb, void *user) {
    return work_batch_any(d, iq_sc8, sizeof(char2), scale, n_items, stride_items, host_ptr, consumed, cb, user);
}

int lora_b200_stream_state(lora_b200_decoder *d, uint32_t stream) {
    if (!d || stream >= d->cfg.n_streams) return fail(LORA_B200_EINVAL, "bad stream");
    CU(cudaSetDevice(d->device));
    int32_t st = 0;
    CU(cudaMemcpy(&st, &d->d_states[stream].state, sizeof st, cudaMemcpyDeviceToHost));
    return st;
}

static_assert(sizeof(lora_b200_frame) == sizeof(RxFrameOut) && LORA_B200_MAX_FRAME_BYTES == LB_MAX_FRAME + 2, "public frame record == K8 output record");

size_t lora_b200_frames_last(lora_b200_decoder *d, const lora_b200_frame **frames) {
    if (!d || !frames) { fail(LORA_B200_EINVAL, "null argument"); return 0; }
    *frames = reinterpret_cast<const lora_b200_frame *>(d->h_sorted.data());
    return d->h_sorted.size();
}

size_t lora_b200_frames_crc_last(lora_b200_decoder *d, const uint8_t **status) {
    if (!d || !status) { fail(LORA_B200_EINVAL, "null argument"); return 0; }
    const size_t n = d->h_sorted.size();
    d->crc_status.resize(n);
    for (size_t k = 0; k < n; k++) {
        const RxFrameOut &f = d->h_sorted[k];
        uint8_t s = (uint8_t)lb_crc_record_status(f.bytes, std::min<uint32_t>(f.len, (uint32_t)sizeof f.bytes));
        if (s == LORA_CRC_OK && k < d->rs_recovered.size() && d->rs_recovered[k]) s = LORA_CRC_RECOVERED;
        d->crc_status[k] = s;
    }
    *status = d->crc_status.data();
    return n;
}

int lora_b200_set_cfo_estimate(lora_b200_decoder *d, int enable) {
    if (!d) return fail(LORA_B200_EINVAL, "null argument");
    d->cfo_estimate = enable != 0;
    return LORA_B200_OK;
}

int lora_b200_last_cfo(lora_b200_decoder *d, uint32_t stream, float *cfo_hz, uint32_t *count) {
    if (!d || stream >= d->cfg.n_streams || !cfo_hz) return fail(LORA_B200_EINVAL, "bad argument");
    CU(cudaSetDevice(d->device));
    struct { float cfo; uint32_t n; } v;
    CU(cudaMemcpy(&v, &d->d_states[stream].cfo_est, sizeof v, cudaMemcpyDeviceToHost));
    *cfo_hz = v.cfo;
    if (count) *count = v.n;
    return LORA_B200_OK;
}

int lora_b200_stdout_last(lora_b200_decoder *d, uint32_t stream, char *buf, size_t cap) {
    if (!d || !buf || stream >= d->cfg.n_streams) return fail(LORA_B200_EINVAL, "bad argument");
    return snprintf(buf, cap, "%s", d->stdout_last[stream].c_str());
}

int lora_b200_trace_read(lora_b200_decoder *d, uint32_t stream, lora_b200_step *steps, size_t cap, size_t *n) {
    if (!d || !steps || !n || stream >= d->cfg.n_streams) return fail(LORA_B200_EINVAL, "bad argument");
    if (!d->d_trace) return fail(LORA_B200_EINVAL, "trace_capacity was 0 at creation");
    CU(cudaSetDevice(d->device));
    uint32_t cnt = 0;
    CU(cudaMemcpy(&cnt, d->d_trace_n + stream, sizeof cnt, cudaMemcpyDeviceToHost));
    size_t m = std::min<size_t>(std::min<size_t>(cnt, d->cfg.trace_capacity), cap);
    if (m) CU(cudaMemcpy(steps, d->d_trace + (size_t)stream * d->cfg.trace_capacity, sizeof(lora_b200_step) * m, cudaMemcpyDeviceToHost));
    *n = cnt;
    return cnt > d->cfg.trace_capacity ? LORA_B200_EOVERFLOW : LORA_B200_OK;
}

}  // extern "C"
