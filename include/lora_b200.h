/*
 * lora_b200.h -- C ABI of liblora_b200.so, the H100 (sm_90a) replacement for the hot path of
 * rpp0/gr-lora: gr::lora::decoder_impl::work() and the DSP helpers it calls
 * (lib/decoder_impl.cc:141-903 of the reference).
 *
 * Drop-in boundary (SURVEY.md 8b): the GNU Radio scheduler, PMT message ports and the
 * hier-block wiring stay on the host.  A thin gr::lora::decoder_impl shim (see
 * INTEGRATION.md) forwards its constructor arguments to lora_b200_create() and its
 * work() buffer to lora_b200_work(); everything numerical happens behind this header.
 * Plain C types only: no torch, no C++ in the signatures.
 *
 * All functions return 0 on success or a negative LORA_B200_E* code; the message of the
 * last failure on the calling thread is available from lora_b200_last_error().
 * There is NO CPU fallback: without a CUDA device lora_b200_create() fails.
 */
#ifndef LORA_B200_H
#define LORA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LORA_B200_ABI_VERSION 1

enum {
    LORA_B200_OK = 0,
    LORA_B200_EINVAL = -1,     /* bad argument (the reference exit(1)s for sf outside [6,13], decoder_impl.cc:57-61) */
    LORA_B200_ECUDA = -2,      /* CUDA runtime failure / no device */
    LORA_B200_ENOMEM = -3,
    LORA_B200_EUNSUPPORTED = -4,
    LORA_B200_EOVERFLOW = -5   /* per-call frame or trace capacity exhausted */
};

/* demodulator selection for demodulate() (decoder_impl.cc:499-500) */
enum {
    LORA_B200_DEMOD_GRADIENT = 0,  /* max_frequency_gradient_idx: what the reference runs today (:499)      */
    LORA_B200_DEMOD_FFT = 1        /* dechirp + FFT + argmax (get_shift_fft :430-464), mapped (bin-1) mod N */
};

/* decoder states, lib/decoder_impl.h:40-48 */
enum { LORA_B200_DETECT = 0, LORA_B200_SYNC, LORA_B200_FIND_SFD, LORA_B200_PAUSE,
       LORA_B200_DECODE_HEADER, LORA_B200_DECODE_PAYLOAD, LORA_B200_STOP };

/* Replaces the argument list of lora::decoder::make (include/lora/decoder.h:705,
 * lib/decoder_impl.cc:41-44,49): the first eight fields are exactly those arguments. */
typedef struct lora_b200_config {
    float    samp_rate;
    uint32_t bandwidth;
    uint8_t  sf;
    uint8_t  implicit;
    uint8_t  cr;
    uint8_t  crc;
    uint8_t  reduced_rate;
    uint8_t  disable_drift_correction;
    uint8_t  demod;              /* LORA_B200_DEMOD_*                                         */
    uint8_t  reserved0;
    uint32_t n_streams;          /* independent (channel, SF) streams sharing this config; >=1 */
    int32_t  device;             /* CUDA device ordinal; -1 = current device                   */
    uint32_t max_items_per_call; /* capacity of the per-stream staging buffer (0 = 1<<20)      */
    uint32_t max_frames_per_call;/* per stream (0 = 8)                                         */
    uint32_t trace_capacity;     /* per-stream lora_b200_step records kept per call (0 = none) */
} lora_b200_config;

typedef struct lora_b200_decoder lora_b200_decoder;

/* one state-machine step, for parity tests against the oracle's work() trace */
typedef struct lora_b200_step {
    int32_t state;       /* state at entry of the step                        */
    int32_t consumed;    /* what the reference would pass to consume_each      */
    int32_t bin;         /* raw demodulated bin, -1 when the step has none     */
    int32_t fine_sync;   /* d_fine_sync after the step                         */
    float   metric;      /* autocorr (DETECT), max corr (SYNC), pearson (FIND_SFD) */
} lora_b200_step;

/* Frame callback: replaces message_port_pub("frames", blob) (decoder_impl.cc:607-608).
 * `frame` = 15-byte loratap header | 3-byte loraphy header | payload (decoder_impl.cc:588-601);
 * valid only during the callback. */
typedef void (*lora_b200_frame_cb)(void *user, uint32_t stream, const uint8_t *frame, size_t len);

/* ---- lifecycle: decoder::make / ~decoder_impl (decoder_impl.cc:41-139) ---- */
lora_b200_decoder *lora_b200_create(const lora_b200_config *cfg);
void lora_b200_destroy(lora_b200_decoder *d);
/* Every stream back to the state of a freshly made block (DETECT, empty power queue, no partial frame, counters 0): what
 * stopping and restarting the flowgraph does to decoder_impl's members (:55-66).  Device buffers and tables are kept. */
int lora_b200_reset(lora_b200_decoder *d);
const char *lora_b200_last_error(void);
int lora_b200_abi_version(void);

/* derived parameters (decoder_impl.cc:69-91) and the constructor's stdout banner (:93-103) */
uint32_t lora_b200_samples_per_symbol(const lora_b200_decoder *d);
uint32_t lora_b200_bins(const lora_b200_decoder *d);
uint32_t lora_b200_decimation(const lora_b200_decoder *d);
int lora_b200_banner(const lora_b200_decoder *d, char *buf, size_t cap);
/* set_sf / set_samp_rate are unsupported at run time in the reference too (:905-915): they
 * return LORA_B200_EUNSUPPORTED and leave the decoder untouched. */
int lora_b200_set_sf(lora_b200_decoder *d, uint8_t sf);
int lora_b200_set_samp_rate(lora_b200_decoder *d, float samp_rate);

/* ---- chirp / twiddle tables (build_ideal_chirps, decoder_impl.cc:141-175) ----
 * One contiguous device blob: downchirp cf32[sps] | upchirp cf32[sps] | down_ifreq f32[sps] |
 * up_ifreq f32[sps] | up_ifreq_v f32[3*sps] | FFT twiddles cf32[sps].  Rank 0 builds it, the
 * other ranks receive it by ONE ncclBroadcast at init (SURVEY.md 8e) and call _commit. */
size_t lora_b200_tables_bytes(const lora_b200_decoder *d);
/* host-only: build the blob for `cfg` into dst (no device needed); returns its size in bytes
 * (dst == NULL: size query), 0 on error.  Layout: the six arrays above, back to back,
 * total rounded up to 256 bytes. */
size_t lora_b200_tables_build_host(const lora_b200_config *cfg, void *dst, size_t cap);
void *lora_b200_tables_device_ptr(lora_b200_decoder *d);
int lora_b200_tables_export(const lora_b200_decoder *d, void *host_dst, size_t cap);
int lora_b200_tables_import(lora_b200_decoder *d, const void *host_src, size_t bytes);
/* after writing the device blob in place (e.g. ncclBroadcast into lora_b200_tables_device_ptr):
 * refresh the host copy and the constants derived from it */
int lora_b200_tables_commit(lora_b200_decoder *d);

/* ---- K1: dechirp + FFT + argmax on aligned symbol windows (get_shift_fft, :430-464) ----
 * iq: n_symbols * sps interleaved cf32.  bins[i] in [0, N), mags[i] = |tmp[bin]| (may be NULL).
 * _dev: all pointers are device pointers, the launch is asynchronous on `cuda_stream`
 * (a cudaStream_t passed as void*, NULL = default stream).
 * _host: host pointers; copies (pinned, chunked, overlapped with compute) are inside.
 * samp_rate / bandwidth 8 (the tuned kernels of each SF) or 2 (one kernel generic in the oversampling factor), SF7..SF12;
 * otherwise LORA_B200_EUNSUPPORTED. */
int lora_b200_demod_fft_dev(lora_b200_decoder *d, const void *iq, size_t n_symbols,
                            uint32_t *bins, float *mags, void *cuda_stream);
int lora_b200_demod_fft_host(lora_b200_decoder *d, const void *iq, size_t n_symbols,
                             uint32_t *bins, float *mags);
/* Soft output of the same windows, for soft-decision decoding here (lora_b200_rx_params.soft) or in the caller's own FEC:
 * llrs[i * ppm + j] = max |tmp[k]| over the kept bins k whose demodulated word has bit j = 0, minus the same over bit j = 1
 * (> 0: bit 0), j < ppm.  The demodulated word of bin k is the receiver's: gray((k - 1) mod N), with (k - 1) mod N first
 * folded to N / 4 bins as reduced-rate symbols are (reduced = 1, ppm = SF - 2; reduced = 0: ppm = SF).  bins (may be NULL)
 * = lora_b200_demod_fft_dev's argmax of the same computation.  iq 16-byte aligned; device pointers, async on cuda_stream.
 * LORA_B200_EUNSUPPORTED unless samp_rate / bandwidth is 8, 2, 16 or 32 and SF7..SF12 (4 is refused). */
int lora_b200_demod_llr_dev(lora_b200_decoder *d, const void *iq, size_t n_symbols, int reduced, float *llrs, uint32_t *bins,
                            void *cuda_stream);
/* The window sums the dechirp receiver's synchroniser (lora_b200_receive, lora_b200_receive_antennas) measures, on their own,
 * to check them against a reference.  One receiver of m (1..4) antennas, row a = iq + a * stride_items (n_items samples
 * each; stride_items is ignored for m = 1).  For window i and antenna a, out[i * m + a] = sum_n x_a[pos[i] + n] c[n]
 * exp(-2 pi j (cfo_bins[i] (pos[i] + n) + bin[i] n) / sps), n < sps, c the down-chirp table (up[i] = 0) or the up-chirp
 * table (up[i] = 1); energy[i * m + a] = sum |x_a|^2 over the window; argmax_bin[i] / argmax_mag[i] = the first argmax of
 * the combined spectrum P[k] = sum_a |tmp_a[k]|^2 of the raw windows at pos[i] dechirped with c (as
 * lora_b200_demod_fft_antennas_dev, at any position) and sqrt(P[bin]).  m = 1 runs the one-row synchroniser's arithmetic,
 * m >= 2 the antenna synchroniser's.  Every window inside the row, bin in -N/2..N/2-1, |cfo_bins| <= max(N, (D - 1) N / 2) (D = fs / bw:
 * the widest offset of wide_cfo, 3.5 N at fs / bw = 8).  iq, out
 * (float2[n][m]), energy (float[n][m]), argmax_bin and argmax_mag are device pointers (energy, argmax_bin and argmax_mag
 * may be NULL), pos, cfo_bins, up and bin host arrays; returns when the results are written.  Test entry point. */
int lora_b200_rs_window_dev(lora_b200_decoder *d, const void *iq, size_t n_items, uint32_t m, size_t stride_items, size_t n,
                            const int64_t *pos, const float *cfo_bins, const int32_t *up, const int32_t *bin, void *out, float *energy,
                            uint32_t *argmax_bin, float *argmax_mag);
/* The channel estimates, weights and data windows the dechirp receiver forms for given frames, on their own: frame i (start[i],
 * its CFO cfo_bins[i] in bins, its clock offset sfo_ppm[i]) lies on receiver group[i], rows group[i] * m + a =
 * iq + (group[i] * m + a) * stride_items, n_items samples each.  m >= 2: chan[i][0..4) = h, chan[i][4..8) = w (float2, 0 above
 * m) and snr_db[i], as lora_b200_receive_antennas computes them after synchronising (rx_channels_last is h).  windows[(i cnt + k)
 * sps ..] = data window first + k of frame i as the receiver demodulates it: sum_a w_a x_a (m = 1: x_0) from rs_sym(start[i],
 * 12.25 + first + k) on, de-rotated by cfo_bins[i], 0 past n_items.  Data window `first` must start inside the row.  iq, chan
 * (float2[n][8], m >= 2), snr_db (float[n], m >= 2) and windows (float2[n cnt sps]) are device pointers, group, start,
 * cfo_bins and sfo_ppm host arrays; returns when the results are written.  Test entry point. */
int lora_b200_rs_frame_dev(lora_b200_decoder *d, const void *iq, size_t n_items, uint32_t m, size_t stride_items, size_t n,
                           const uint32_t *group, const int64_t *start, const float *cfo_bins, const float *sfo_ppm, uint32_t first,
                           uint32_t cnt, void *chan, float *snr_db, void *windows);
/* The fine time of arrival of given frames on its own (the procedure of lora_b200_rx_params.fine_toa): frame i (start[i], CFO
 * cfo_bins[i] in bins, clock offset sfo_ppm[i]) on receiver group[i], rows iq + (group[i] * m + a) * stride_items of n_items
 * samples, m = 1..4.  nu_a[i] / nu_b[i] = the peaks of the summed preamble / SFD window powers in bins from the CFO, toa[i]
 * the time of arrival (lora_b200_rx_toa_last).  iq is a device pointer, the rest host arrays; returns when the results are
 * written.  Test entry point. */
int lora_b200_rs_toa_dev(lora_b200_decoder *d, const void *iq, size_t n_items, uint32_t m, size_t stride_items, size_t n,
                         const uint32_t *group, const int64_t *start, const float *cfo_bins, const float *sfo_ppm, float *nu_a,
                         float *nu_b, double *toa);
/* The combined screen of the dechirp receiver with several antennas (lora_b200_receive_antennas) on its own, so that it can be
 * held to a reference: n_groups groups of n_antennas (1..4) rows, row r = iq + r * row_stride_items, each holding n_symbols
 * aligned windows of sps samples.  For window i of group g, with tmp_a the kept bins of lora_b200_demod_fft_dev's spectrum of
 * antenna a's window, P[k] = sum_a |tmp_a[k]|^2: bins[g * n_symbols + i] = the first argmax of P, mags[..] = sqrt(P[bin]).
 * iq 16-byte aligned, row_stride_items even and >= n_symbols * sps; device pointers, async on cuda_stream. */
int lora_b200_demod_fft_antennas_dev(lora_b200_decoder *d, const void *iq, uint32_t n_groups, uint32_t n_antennas, size_t n_symbols,
                                     size_t row_stride_items, uint32_t *bins, float *mags, void *cuda_stream);
/* SDR-native ingest: iq_sc16 = interleaved little-endian int16 I/Q (what a USRP / file source delivers before the
 * host-side conversion to gr_complex); the device converts x * scale right after the copy, so PCIe moves 4 instead of
 * 8 bytes per sample.  Results equal lora_b200_demod_fft_host on the host-converted buffer bit for bit. */
int lora_b200_demod_fft_host_sc16(lora_b200_decoder *d, const void *iq_sc16, float scale, size_t n_symbols,
                                  uint32_t *bins, float *mags);
/* K2: max_frequency_gradient_idx on aligned windows (:466-491), same layout */
int lora_b200_demod_gradient_dev(lora_b200_decoder *d, const void *iq, size_t n_symbols,
                                 uint32_t *bins, void *cuda_stream);
/* A3: instantaneous_frequency (:224-244) of n_windows windows of `window` gr_complex each (window a multiple of 128),
 * out[n_windows][window] floats; the last value of a window repeats the one before it (:243).  The arg() per sample is
 * the stream kernels' own (1.8 ulp; the values agree with libm-based ones to 1e-6 rad); device pointers, async on cuda_stream. */
int lora_b200_ifreq_dev(lora_b200_decoder *d, const void *iq, size_t n_windows, uint32_t window, float *out, void *cuda_stream);

/* ---- synthetic transmitter / channel on the device (SURVEY 8(f) N3; the reference is a receiver only) ----
 * tx_symbols: n_symbols aligned data symbols, out[s][n] = up[(n + decim * values[s]) mod sps] * e^{j 2 pi cfo_hz[s] n / fs}
 *   + noise_sigma * (N(0,1) + j N(0,1)).  up_table = device cf32[sps] or NULL for the decoder's own ideal up-chirp
 *   (lib/decoder_impl.cc:149-160: (1 + 1j) e^{j phase}, i.e. amplitude sqrt 2); cfo_hz = device float[n_symbols] or NULL; noise_sigma = 0: no noise.  The noise is a
 *   counter-based generator (Philox4x32-10) keyed by `seed`: the same call gives the same samples on any launch geometry.
 * tx_expand: n_streams concurrent channels from k base captures, out[s] = base[s mod k] + the stream's own noise
 *   (base device cf32[k][n_items], n_items even).  Device pointers, async on cuda_stream. */
int lora_b200_tx_symbols_dev(lora_b200_decoder *d, const void *up_table, const uint32_t *values, const float *cfo_hz,
                             float noise_sigma, uint64_t seed, size_t n_symbols, void *out, void *cuda_stream);
int lora_b200_tx_expand_dev(lora_b200_decoder *d, const void *base, uint32_t k, size_t n_items, float noise_sigma, uint64_t seed,
                            size_t n_streams, void *out, void *cuda_stream);

/* ---- frame encoder and frame modulator on the device (the inverse of B1-B5 + chirp synthesis + sync word + SFD) ----
 * The specification is the host encoder gr_lora_b200/tx.py: encode_frame, modulate_frame and channel.
 *
 * tx_frame_symbols (host only, no device needed): data symbols (the 8-symbol header block + the payload blocks) of one frame
 *   carrying payload_len bytes under cfg's sf / cr / implicit / crc / reduced_rate; the whole frame is
 *   (8 + 2 + 2) * sps + sps / 4 + that * sps samples.  0 for an unsupported configuration or length.
 * tx_encode: payload bytes -> chirp shifts.  Frame f = payloads[offsets[f] .. + lengths[f]) (payloads, shifts: device;
 *   offsets, lengths: host arrays, validated and uploaded inside the call); shifts[f * max_symbols + i] for
 *   i < tx_frame_symbols(lengths[f]) equals tx.encode_frame(payload, sf, cr, explicit=not implicit, has_crc=crc,
 *   reduced_rate).shifts, the rest of each row is not written.  A payload is the bytes the receiver prints after the header:
 *   with CRC on, the caller supplies the two CRC bytes at its end (no payload CRC is computed).  Supported for SF7..SF12 and
 *   CR 1..4 at the decoder's own settings, else LORA_B200_EUNSUPPORTED.  LORA_B200_EINVAL, before any launch, for a length
 *   above 255 + 2 * crc, below 2 with CRC on and an explicit header, or needing more than max_symbols symbols.
 *   One thread per (frame, data symbol).  Async on cuda_stream.
 * tx_frames: whole streams of frames.  out = device cf32 [n_streams][n_items] (n_items even, 16-byte aligned), every sample
 *   written once: frame samples at [start, start + frame length) of row `stream` -- 8 preamble up-chirps, 2 sync symbols,
 *   2.25 down-chirps (conj(up)), then data symbol k = up[(n + decim * shifts[f * max_symbols + k]) mod sps] -- rotated by
 *   e^{j 2 pi cfo_hz n / fs} (n = sample index in the row, phase reduced in double as tx_symbols does), 0 outside every
 *   frame, then noise_sigma * (N(0,1) + j N(0,1)) added exactly as tx_expand adds it: tx_frames(sigma, seed) equals
 *   tx_expand(base = tx_frames(0), k = n_streams, sigma, seed) bit for bit.  up_table as for tx_symbols (NULL: the decoder's
 *   own ideal up-chirp).  frames (host) may come in any order; LORA_B200_EINVAL, before any launch, for frames that overlap
 *   in one row, a frame that runs past n_items, stream >= n_streams or n_symbols > max_symbols.  The per-frame tables of
 *   tx_encode / tx_frames are uploaded on cuda_stream into one buffer per decoder: a call first waits (on the host) for the
 *   previous such call's kernel to finish. */
typedef struct lora_b200_tx_frame {
    uint64_t start;      /* first preamble sample, index into its row (may be odd)                                   */
    uint32_t stream;     /* row of out                                                                               */
    uint32_t n_symbols;  /* data symbols, read from shifts[f * max_symbols ..], f = index of this descriptor          */
    float    cfo_hz;     /* rotation e^{j 2 pi cfo_hz n / fs}, n = sample index in the row (as tx.channel)            */
    uint8_t  sync_word;  /* two symbols of ((sw >> 4) & 15) * 8 and (sw & 15) * 8 bins (tx.modulate_frame)            */
    uint8_t  pad[3];
} lora_b200_tx_frame;
uint32_t lora_b200_tx_frame_symbols(const lora_b200_config *cfg, uint32_t payload_len);
int lora_b200_tx_encode_dev(lora_b200_decoder *d, const uint8_t *payloads, const uint32_t *offsets, const uint32_t *lengths,
                            size_t n_frames, uint32_t *shifts, uint32_t max_symbols, void *cuda_stream);
int lora_b200_tx_frames_dev(lora_b200_decoder *d, const void *up_table, const lora_b200_tx_frame *frames, size_t n_frames,
                            const uint32_t *shifts, uint32_t max_symbols, float noise_sigma, uint64_t seed, size_t n_streams,
                            size_t n_items, void *out, void *cuda_stream);
/* tx_frames_sfo: tx_frames with frames from transmitters whose clock is off.  sfo_ppm = host float[n_frames], parallel to
 *   frames, or NULL (= tx_frames).  Frame f's clock is off by delta = sfo_ppm[f] * 1e-6 (> 0: fast), so row sample n holds
 *   transmitter time u = (n - start) (1 + delta) samples; the frame covers the row samples with 0 <= u < frame length, and
 *   those are what the overlap and n_items checks see.  A frame with delta != 0 is evaluated at the fractional u from the
 *   phase law of tx.base_upchirp, e^{j 2 pi m (m - sps) / (2 decim sps)} at chirp position m (cyclic shifts at fractional
 *   positions, the conjugate for the SFD), in double and reduced to revolutions, times up_table[0]; tx.modulate_frame(...,
 *   sfo_ppm) is its specification.  The CFO rotation and the noise are tx_frames'; a frame with delta = 0 is tx_frames' own.
 *   LORA_B200_EINVAL, before any launch, for an sfo_ppm that is not finite or beyond +-500. */
int lora_b200_tx_frames_sfo_dev(lora_b200_decoder *d, const void *up_table, const lora_b200_tx_frame *frames, size_t n_frames,
                                const float *sfo_ppm, const uint32_t *shifts, uint32_t max_symbols, float noise_sigma, uint64_t seed,
                                size_t n_streams, size_t n_items, void *out, void *cuda_stream);

/* ---- K8: integer decode of whole code-word vectors (decode(), :567-586, B2-B4) ----
 * For each of n_vec vectors: codewords[i*stride .. +lengths[i]) -> deshuffle, dewhiten,
 * Hamming decode.  out[i*out_stride ..]; out_len[i] = bytes produced.  cr[i] = d_phdr.cr,
 * is_header[i] as in decode(is_header).  Device pointers, async on cuda_stream. */
int lora_b200_decode_codewords_dev(lora_b200_decoder *d, const uint8_t *codewords, const uint32_t *lengths,
                                   size_t stride, const uint8_t *cr, const uint8_t *is_header, size_t n_vec,
                                   uint8_t *out, size_t out_stride, uint32_t *out_len, void *cuda_stream);
/* B1 + Gray: words (u32, one per symbol) of one interleaver block -> ppm code words; batch of blocks */
int lora_b200_deinterleave_dev(lora_b200_decoder *d, const uint32_t *words, uint32_t n_words, uint32_t ppm,
                               size_t n_blocks, uint8_t *codewords, void *cuda_stream);

/* ---- the drop-in: decoder_impl::work (decoder_impl.cc:740-903) ----
 * Feeds `n_items` cf32 items of stream `stream` (HOST pointer, as GNU Radio hands them to
 * work(); not retained after return).  Runs the whole state machine on the GPU for as many
 * steps as fit (each step needs 2*sps items of look-ahead, the block's output_multiple :91),
 * sets *consumed to the number of items the caller must drop (the sum of the reference's
 * consume_each() calls) and invokes cb once per completed frame, in order.
 * The caller re-presents the unconsumed tail at the start of the next call. */
int lora_b200_work(lora_b200_decoder *d, uint32_t stream, const void *iq_host, size_t n_items,
                   size_t *consumed, lora_b200_frame_cb cb, void *user);
/* Same for all streams at once: iq is [n_streams][n_items] (row stride `stride_items`).
 * host_ptr != 0: iq is host memory (copied inside); 0: iq is device memory. */
int lora_b200_work_batch(lora_b200_decoder *d, const void *iq, size_t n_items, size_t stride_items,
                         int host_ptr, size_t *consumed /* [n_streams] */, lora_b200_frame_cb cb, void *user);
/* the same with int16 I/Q input (see lora_b200_demod_fft_host_sc16); frames, consume amounts and stdout equal those of
 * lora_b200_work_batch on the host-converted buffer. */
int lora_b200_work_batch_sc16(lora_b200_decoder *d, const void *iq_sc16, float scale, size_t n_items, size_t stride_items,
                              int host_ptr, size_t *consumed /* [n_streams] */, lora_b200_frame_cb cb, void *user);
/* ... and with int8 I/Q (interleaved signed bytes, GNU Radio's interleaved_char_to_complex followed by a multiply):
 * a quarter of the gr_complex bytes over PCIe, the only lever left once the copy is the bound. */
int lora_b200_work_batch_sc8(lora_b200_decoder *d, const void *iq_sc8, float scale, size_t n_items, size_t stride_items,
                             int host_ptr, size_t *consumed /* [n_streams] */, lora_b200_frame_cb cb, void *user);
/* Bulk access to what the last work / work_batch call published, for hosts that drain thousands of streams per call and do
 * not want one callback per frame (cb may be NULL then): records in delivery order (by stream, then by sequence), valid
 * until the next work call on this decoder.  `bytes` = loratap | loraphy | payload, `len` of them valid
 * (decoder_impl.cc:588-601); hdr_print = the header bytes the reference prints first (:832). */
#define LORA_B200_MAX_FRAME_BYTES 564
typedef struct lora_b200_frame {
    uint32_t stream, seq, len;
    uint8_t  n_hdr_print;
    uint8_t  hdr_print[4];
    uint8_t  pad[3];
    uint8_t  bytes[LORA_B200_MAX_FRAME_BYTES];
} lora_b200_frame;
size_t lora_b200_frames_last(lora_b200_decoder *d, const lora_b200_frame **frames);
/* The payload CRC status of every frame of lora_b200_frames_last, parallel to it (valid after work, work_batch*, receive and
 * receive_antennas, until the next call): LORA_B200_CRC_NONE when the frame's header (or the implicit configuration) carries
 * no CRC or its payload is shorter than 2 bytes, _OK, _BAD, or _RECOVERED: OK only after CRC-aided list decoding
 * (lora_b200_rx_params.crc_list).  Semtech's CRC: CRC-16, polynomial 0x1021, initial value 0, over payload[0 .. L-2), XORed
 * with payload[L-1] | payload[L-2] << 8; the radio sends it low byte first, unwhitened, and the decode chain dewhitens it
 * like every payload nibble, so the published CRC bytes are crc ^ W(L), a fixed XOR (DESIGN.md section 5).  Computed on the
 * host from the published records: no launch, no copy, nothing published changes; frames that fail are still published. */
#define LORA_B200_CRC_NONE 0
#define LORA_B200_CRC_OK 1
#define LORA_B200_CRC_BAD 2
#define LORA_B200_CRC_RECOVERED 3
size_t lora_b200_frames_crc_last(lora_b200_decoder *d, const uint8_t **status);
/* ---- dechirp-synchronised receiver: frames below the noise floor (an opt-in path beside the reference state machine) ----
 * iq = [n_streams][n_items] cf32 (row stride stride_items; host_ptr != 0: host memory, copied inside; 0: device memory).
 * Every stream is screened by K1 (dechirp + FFT + argmax) on windows at hops of sps/2; runs of >= min_preamble windows whose
 * bins agree within one bin are preamble candidates, each synchronised by one CTA: integer CFO and timing from the preamble and
 * SFD bins, fractional CFO from the preamble peak's phase advance, timing to the sample, then the two sync-word symbols are
 * checked.  Data windows are de-rotated by the frame's CFO and demodulated by the K1 batch kernels; the FFT demodulator's
 * (bin - 1) mod N mapping and the stream path's integer chain follow.  Explicit headers whose 5-bit checksum fails are dropped
 * (and counted); frames whose payload CRC fails are published too (lora_b200_frames_crc_last reports it).  Implicit headers carry implicit_len payload bytes (0 with an implicit-header
 * decoder: LORA_B200_EINVAL).  Needs the FFT kernels (samp_rate / bandwidth == 8, 2, 16 or 32, SF7..SF12), else LORA_B200_EUNSUPPORTED;
 * at 2 (e.g. 500 kHz channels at 1 MS/s, or a channelizer's output at 2 samples per chip) timing is refined to +-1 sample.
 * Clock offset: a transmitter whose clock is off by delta = ppm * 1e-6 (delta > 0: fast against the receiver) sends TX symbol
 * position j (0..7 preamble, 8, 9 sync word, 10..12.25 SFD, 12.25 + k data symbol k) at receiver sample
 * start + llround(j * sps / (1 + delta)); every window of a frame is placed by this rule.  A frame's delta is
 * p->sfo_ppm * 1e-6 + cfo_hz / p->carrier_hz: one crystal sets a radio's carrier and its sample clock, so with carrier_hz
 * (the RF frequency of the channel, 0 = none) each frame's clock offset follows from its own measured CFO.  Both 0: timing
 * fixed per frame, which holds while ppm x frame length stays below about a quarter chip.  sfo_ppm must be finite within
 * +-500 and carrier_hz 0 or finite and above the sample rate, else LORA_B200_EINVAL.
 * Carrier offsets beyond BW / 4 (p->wide_cfo = 1): the screen searches coarse offsets c * BW / 2, c = -C..C with
 * C = max(0, ceil((max_cfo_hz - BW / 4) / (BW / 2))), each with its own shifted dechirp tables (one more screen per c, about
 * 2 C + 1 times the screen's cost), and the synchroniser scores the three candidates of the N / 2 ambiguity; max_cfo_hz is
 * taken as given and must be finite in (0, (fs - BW) / 2], the widest offset at which a frame still lies inside the sampled
 * band (3.5 BW at fs / bw = 8, BW / 2 at 2).  wide_cfo other than 0 and 1, or an out-of-range max_cfo_hz with wide_cfo = 1:
 * LORA_B200_EINVAL before any launch.  wide_cfo = 0 is the receiver without the search, max_cfo_hz clamped to BW / 4; with
 * max_cfo_hz <= BW / 4 both give the same frames.
 * Limits: |CFO| <= max_cfo_hz <= BW / 4 ((fs - BW) / 2 with wide_cfo), no blind drift estimation (the clock offset is given or follows the CFO), data
 * windows placed to the nearest sample, one frame at a time per stream, the decoder's SF only, several antennas per receiver
 * through lora_b200_receive_antennas (below).  The stream state machine's
 * per-stream state is not touched.
 * Streaming: a frame is published only when its last sample lies inside the call; consumed[s] is where the caller must
 * re-present stream s from: the earliest preamble whose frame was incomplete, else n_items minus a guard of
 * (min_preamble + 4) symbols, never before the end of a published frame.  consumed[s] == 0 with more samples pending means
 * stream s holds a frame longer than this call's n_items: present a longer chunk (there is no per-call size limit; buffers
 * grow as needed).  At most max_frames_per_call frames per stream;
 * further preambles are held back the same way.  Frames come back through lora_b200_frames_last (delivery order: by stream,
 * then by start), their synchronisation through lora_b200_rx_info_last.
 * Soft decisions (p->soft = 1; other values than 0 and 1: LORA_B200_EINVAL): the data windows go through the LLR
 * demodulator (lora_b200_demod_llr_dev) instead of K1, each code word is decoded to the nibble whose encoder code word best
 * matches its bits' LLRs, and the bins of the re-encoded code words replace the argmax bins before the integer chain.
 * CRC-aided list decoding (p->crc_list = K, 1..12, needs soft = 1; other values: LORA_B200_EINVAL before any launch): a frame
 * whose payload CRC fails gets its K least reliable payload / CRC code words (smallest metric gap to the runner-up nibble)
 * tried at their runner-ups, and the cheapest combination (least summed gap) that satisfies the CRC is published, with status
 * LORA_B200_CRC_RECOVERED.  The price: a frame whose errors lie outside the list passes a wrong combination with probability
 * about (2^K - 1) / 2^16, which is why K is capped and the option is off by default.  0 changes nothing.
 * Fine time of arrival (p->fine_toa = 1; other values than 0 and 1: LORA_B200_EINVAL before any launch): each published
 * frame's arrival to a fraction of a sample, from the dechirped preamble and SFD windows (lora_b200_rx_toa_last).  Reported
 * only: nothing published changes, and 0 launches nothing more. */
typedef struct lora_b200_rx_params {
    uint8_t  sync_word;          /* 0 = 0x12                                                    */
    uint8_t  soft;               /* 1: soft-decision decoding (per-bit LLRs, ML code words)      */
    uint8_t  crc_list;           /* CRC-aided list decoding of K code words (0 = off), see above */
    uint8_t  wide_cfo;           /* 1: search carrier offsets up to max_cfo_hz beyond BW / 4      */
    uint32_t implicit_len;       /* payload bytes of implicit-header frames (incl. CRC bytes)  */
    uint32_t min_preamble;       /* windows of one phase (0 = 5)                                */
    float    max_cfo_hz;         /* 0 = BW / 4; larger values are clamped to BW / 4 (wide_cfo = 0);
                                    with wide_cfo = 1 taken as given, (0, (fs - BW) / 2]          */
    float    sfo_ppm;            /* clock offset of every frame in ppm (> 0: transmitter fast)  */
    uint8_t  fine_toa;           /* 1: each published frame's time of arrival to a fraction of a
                                    sample, lora_b200_rx_toa_last (0 = off)                      */
    uint8_t  reserved1[3];
    double   carrier_hz;         /* RF carrier of the channel: each frame's clock offset also
                                    follows its CFO, cfo_hz / carrier_hz (0 = not given)        */
} lora_b200_rx_params;
typedef struct lora_b200_rx_info {
    uint64_t start;              /* first preamble sample in the row of this call               */
    uint64_t data_start;         /* first sample of the first data symbol                       */
    uint32_t stream;
    float    cfo_hz;
    float    snr_db;             /* estimated SNR in the LoRa bandwidth                         */
    float    sfo_ppm;            /* clock offset its windows were placed with (0: none asked)   */
} lora_b200_rx_info;
int lora_b200_receive(lora_b200_decoder *d, const void *iq, size_t n_items, size_t stride_items, int host_ptr,
                      const lora_b200_rx_params *p, size_t *consumed /* [n_streams] */);
/* per published frame of the last lora_b200_receive call, parallel to lora_b200_frames_last; *hdr_drops (may be NULL) =
 * synchronised explicit-header frames dropped for a failed header checksum */
size_t lora_b200_rx_info_last(lora_b200_decoder *d, const lora_b200_rx_info **info, uint32_t *hdr_drops);
/* Per published frame of the last lora_b200_receive / lora_b200_receive_antennas call with p->fine_toa = 1, parallel to
 * lora_b200_frames_last: *toa[k] = the row position, in the call's row coordinates like rx_info.start, at which the frame's
 * first preamble sample (transmitter time 0) arrived, to a fraction of a sample: start + eps, eps from the peaks of the
 * dechirped preamble windows 1..6 and SFD windows 10, 11 (DESIGN.md section 5).  NaN for a frame without a preamble or
 * SFD window inside the row.  Returns 0 (no values) after a call without fine_toa and after the work entry points, which
 * replace lora_b200_frames_last's records. */
size_t lora_b200_rx_toa_last(lora_b200_decoder *d, const double **toa);
/* The dechirp receiver on several phase-coherent antennas per receiver (one LO and one sample clock, e.g. both RX channels of
 * a B210): rows g * n_antennas .. g * n_antennas + n_antennas - 1 of iq ([n_streams][n_items], as lora_b200_receive) are
 * the antennas of receiver g.  Timing and CFO are common to a receiver's antennas: the screen takes the argmax of the
 * combined spectrum sum_a |tmp_a[k]|^2, the synchroniser sums its statistics over the antennas, and each frame's data
 * windows are y = sum_a w_a x_a with maximum-ratio weights w_a = conj(h_a) / noise_a (scaled to sum |w_a|^2 = 1) from the
 * per-antenna channel h_a and noise power measured on the preamble; y then goes through the demodulators, soft decisions and
 * decoding of lora_b200_receive unchanged.  Receiver g gets one consumed[g] (consumed has n_streams / n_antennas entries),
 * frames and rx_info with stream == g, and snr_db = the combined (post-MRC) SNR, the sum of the antennas' SNRs.
 * n_antennas must be 1..4 and divide n_streams, else LORA_B200_EINVAL; everything else as lora_b200_receive.
 * n_antennas == 1 is lora_b200_receive. */
int lora_b200_receive_antennas(lora_b200_decoder *d, const void *iq, size_t n_items, size_t stride_items, int host_ptr,
                               uint32_t n_antennas, const lora_b200_rx_params *p, size_t *consumed /* [n_streams / n_antennas] */);
/* per published frame of the last receive_antennas call, parallel to lora_b200_frames_last: n_antennas complex channel
 * estimates (float2: re, im), in row order -- the mean preamble peak of each antenna over (1 + j) sps, the amplitude per
 * sample with a phase reference common to the frame's antennas.  *n_antennas (may be NULL) = that call's n_antennas.
 * Returns the number of frames; 0 after lora_b200_receive, after n_antennas == 1 (no weights to form) and after work calls. */
size_t lora_b200_rx_channels_last(lora_b200_decoder *d, const float **h, uint32_t *n_antennas);
/* current state of a stream (LORA_B200_DETECT ...) */
int lora_b200_stream_state(lora_b200_decoder *d, uint32_t stream);
/* N4 (SURVEY.md 8f): the CFO estimate the reference computes in experimental_determine_cfo (lib/decoder_impl.cc:730-738:
 * instantaneous frequency of samples x downchirp at index 256 of the synchronised preamble symbol, in Hz) and would
 * publish as ("cfo" . x) on its "control" port for the channelizer (:774-776, commented out there; consumer
 * lib/controller_impl.cc:52-57 -> channelizer_impl::apply_cfo).  Off by default: nothing observable changes.  With it
 * enabled every SYNC step stores the estimate; _last_cfo returns the latest one and how many there have been, for the
 * host to forward to lora_b200_channelizer_apply_cfo. */
int lora_b200_set_cfo_estimate(lora_b200_decoder *d, int enable);
int lora_b200_last_cfo(lora_b200_decoder *d, uint32_t stream, float *cfo_hz, uint32_t *count);
/* the reference's std::cout hex lines for the frames delivered by the last work call of this
 * stream (" 04 90 40" + " de ad ... (ascii)\n", decoder_impl.cc:832,872).  A frame's header bytes are delivered together
 * with its payload line, by the call in which the frame completes; the reference prints them as soon as the header block
 * is decoded, so input that ends inside a frame leaves it one unterminated header print ahead. */
int lora_b200_stdout_last(lora_b200_decoder *d, uint32_t stream, char *buf, size_t cap);
/* per-step trace of the last work call (needs trace_capacity > 0): *n = the number of steps the stream made in that call,
 * steps[0 .. min(*n, trace_capacity, cap)) = the FIRST of them (later steps are not recorded).  LORA_B200_EOVERFLOW when
 * *n > trace_capacity (steps[] and *n are valid), LORA_B200_EINVAL without a trace. */
int lora_b200_trace_read(lora_b200_decoder *d, uint32_t stream, lora_b200_step *steps, size_t cap, size_t *n);

/* ---- N1 (SURVEY.md 8f): the channelizer in front of the decoder -------------------------------------
 * Replaces lora::channelizer::make(samp_rate, center_freq, channel_list, bandwidth, decimation)
 * (include/lora/channelizer.h:49, lib/channelizer_impl.cc:40-60): GNU Radio's
 * freq_xlating_fir_filter_ccf with firdes::low_pass(1, fs, bw/2 + 15000, 10000, Hamming) taps.  The
 * reference wires only channel_list[0]; here every listed channel is produced by one FIR-bank launch:
 * out[ch][n] for n < n_in / decimation (device pointers, async on cuda_stream).  Filter history and
 * rotator phase carry over between calls like a GNU Radio block's. */
typedef struct lora_b200_channelizer lora_b200_channelizer;
lora_b200_channelizer *lora_b200_channelizer_create(float samp_rate, float center_freq, const float *channel_list,
                                                    uint32_t n_channels, uint32_t bandwidth, uint32_t decimation,
                                                    int32_t device);
void lora_b200_channelizer_destroy(lora_b200_channelizer *c);
const char *lora_b200_channelizer_last_error(void);
uint32_t lora_b200_channelizer_ntaps(const lora_b200_channelizer *c);
int lora_b200_channelizer_taps(const lora_b200_channelizer *c, float *out, size_t cap);
/* channelizer_impl::apply_cfo (lib/channelizer_impl.cc:68-71), driven by the "cfo" control message
 * (lib/controller_impl.cc:52-57) */
int lora_b200_channelizer_apply_cfo(lora_b200_channelizer *c, uint32_t channel, float cfo);
/* conj != 0: every output sample is conjugated on its way out -- the blocks.conjugate_cc that lora_receiver(conj=True)
 * wires between the channelizer and the decoder (python/lora_receiver.py:50,70-75), without a host round trip */
int lora_b200_channelizer_set_conjugate(lora_b200_channelizer *c, int conj);
int lora_b200_channelizer_work_dev(lora_b200_channelizer *c, const void *in_dev, size_t n_in, void *out_dev,
                                   size_t out_stride, size_t *n_out, void *cuda_stream);
/* host entry: uploads `in_host`, filters into an internal device buffer; _output() returns the DEVICE
 * pointer of one channel's n_out items (valid until the next call) so the decoder can consume it
 * without a host round trip (lora_b200_work_batch(..., host_ptr = 0)). */
int lora_b200_channelizer_work_host(lora_b200_channelizer *c, const void *in_host, size_t n_in, size_t *n_out);
const void *lora_b200_channelizer_output(const lora_b200_channelizer *c, uint32_t channel, size_t *stride_items);
/* host copy of one channel's output of the last _work_host call (what a GNU Radio block's work() hands downstream) */
int lora_b200_channelizer_read_output(const lora_b200_channelizer *c, uint32_t channel, void *host_dst, size_t n_items);
uint64_t lora_b200_channelizer_launch_count(const lora_b200_channelizer *c);

/* how many kernels this library has launched since creation (bench.py's gpu_launches) */
uint64_t lora_b200_launch_count(const lora_b200_decoder *d);

#ifdef __cplusplus
}
#endif
#endif /* LORA_B200_H */
