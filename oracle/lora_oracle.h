/*
 * lora_oracle.h -- CPU ORACLE for the gr-lora decoder hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * This is a dependency-free C restatement of the algorithm in the reference's
 * lib/decoder_impl.cc (rpp0/gr-lora @ 90343d45).  It exists so that the CUDA path can be
 * checked against the reference's arithmetic.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load it; the product
 * (gr_lora_b200/, include/) never links, imports or calls anything in oracle/.
 *
 * Pinning status (SURVEY.md 8c).  The reference ships no IQ fixtures and its cmake build needs GNU Radio, VOLK,
 * liquid-dsp and Boost, none of which is installed.  This restatement is pinned by
 *   - THE REFERENCE'S OWN CODE: oracle/_ref/liblora_ref.so is lib/decoder_impl.cc + lib/debugger.cc compiled
 *     unmodified from /root/reference against stand-in headers for those libraries (oracle/ref_wrap.cc,
 *     oracle/ref_standins/README.md).  tests/test_ref_pins_oracle.py requires restatement == reference, bit for bit,
 *     for parameters, banner, chirp tables, instantaneous frequency, gradient demodulator, fine sync, the three
 *     detectors, energy, deinterleave / deshuffle / dewhiten / Hamming / nibble order, and per work() call the state,
 *     consume amount, bin, fine-sync correction, frames and stdout on the 13 golden cases, the SF x CR x payload
 *     matrix of the reference's `short` suite, clock drift, frame offsets, CFO and noise; get_shift_fft bins equal
 *     and magnitudes within fp32 FFT rounding.  tests/golden/golden.json is generated only if both agree,
 *   - the README console golden (README.md:62-71): banner numbers and the frame bytes
 *     " 04 90 40 de ad be ef 70 0d", through TX -> oracle and TX -> compiled reference,
 *   - the in-tree Hamming(8,4) code book (include/lora/utilities.h:257-264) and the
 *     single-error behaviour of hamming_decode_soft_byte (utilities.h:288-339),
 *   - the whitening tables' sha256 (lib/tables.h:30-44).
 * Still unpinned, because it lives in the absent third-party libraries and not in the reference's source: the
 * Hamming(8,4) decision for code words with >= 2 bit errors (liquid-dsp's table), the rounding of liquid's FFT (any
 * correct unnormalised forward DFT is equivalent within fp32 rounding) and the summation order of VOLK's SIMD
 * kernels (stand-in: generic protokernel order, which is also this file's order).
 *
 * Deliberate deviations where the reference has undefined behaviour (SURVEY.md 5):
 *   D1 fine_sync reads d_upchirp_ifreq_v past its end when bin==N-1 (decoder_impl.cc:310):
 *      out-of-range entries read as the last valid entry.
 *   D2 dewhiten reads past the 516/518-entry tables for maximal payloads (:643): reads 0.
 *   D3 fec_decode reads 2n encoded bytes but only len exist (:658-661): missing bytes read 0.
 *   D4 d_snr uninitialised when the power ring holds <2 entries (:377-383,597): starts at 1.0f.
 *   D5 print/publish may read d_decoded past its size (:872,601): missing bytes read 0.
 *   D6 (uint8_t) cast of a negative double (:597): value is truncated to int then to 8 bits.
 */
#ifndef LORA_ORACLE_H
#define LORA_ORACLE_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { float re, im; } lo_cf;

/* decoder states, lib/decoder_impl.h:40-48 */
enum { LO_DETECT = 0, LO_SYNC, LO_FIND_SFD, LO_PAUSE, LO_DECODE_HEADER, LO_DECODE_PAYLOAD, LO_STOP };

/* demodulator used by demodulate() (decoder_impl.cc:499-500) */
enum { LO_DEMOD_GRADIENT = 0,   /* live reference path: max_frequency_gradient_idx            */
       LO_DEMOD_FFT = 1 };      /* north-star path: (get_shift_fft(x) - 1) mod N  (SURVEY A7)  */

typedef struct lo_decoder lo_decoder;

/* trace of one work() call (state BEFORE the call, what it did) */
typedef struct {
    int32_t state;       /* state at entry                                   */
    int32_t consumed;    /* items passed to consume_each                      */
    int32_t bin;         /* raw demod bin (before /4 and Gray), -1 if none    */
    int32_t fine_sync;   /* d_fine_sync at exit                               */
    float   metric;      /* autocorr (DETECT), max correlation (SYNC), pearson c (FIND_SFD), else 0 */
} lo_step;

/* lifecycle: mirrors decoder::make (include/lora/decoder.h:705, lib/decoder_impl.cc:41-122).
 * Returns NULL for sf outside [6,13] (reference exits, :57-61). */
lo_decoder *lo_create(float samp_rate, uint32_t bandwidth, uint8_t sf, int implicit, uint8_t cr,
                      int crc, int reduced_rate, int disable_drift_correction);
void lo_destroy(lo_decoder *d);
void lo_set_demod(lo_decoder *d, int method);

/* derived parameters (A1, decoder_impl.cc:69-91) */
uint32_t lo_sps(const lo_decoder *d);
uint32_t lo_bins(const lo_decoder *d);
uint32_t lo_decim(const lo_decoder *d);
double   lo_bits_per_symbol(const lo_decoder *d);

/* tables (A2, :141-175); pointers stay valid for the decoder's lifetime */
const lo_cf *lo_downchirp(const lo_decoder *d);
const lo_cf *lo_upchirp(const lo_decoder *d);
const float *lo_downchirp_ifreq(const lo_decoder *d);
const float *lo_upchirp_ifreq(const lo_decoder *d);
const float *lo_upchirp_ifreq_v(const lo_decoder *d);   /* 3*sps entries */

/* float-stage entry points (each restates one reference function) */
void     lo_instantaneous_frequency(const lo_cf *in, float *out, uint32_t window);   /* A3 :224-244 */
uint32_t lo_get_shift_fft(lo_decoder *d, const lo_cf *samples, float *mag_out);       /* A4 :430-464 */
uint32_t lo_max_frequency_gradient_idx(lo_decoder *d, const lo_cf *samples);         /* A5 :466-491 */
int32_t  lo_fine_sync(lo_decoder *d, const lo_cf *samples, int32_t bin_idx, int32_t search_space); /* A6 :300-338, returns d_fine_sync */
float    lo_detect_preamble_autocorr(lo_decoder *d, const lo_cf *samples);           /* A8 :340-366 (has side effects) */
float    lo_detect_upchirp(lo_decoder *d, const lo_cf *samples, int32_t *index);     /* A9 :392-413 */
float    lo_detect_downchirp(lo_decoder *d, const lo_cf *samples);                   /* A10 :385-390 */
float    lo_determine_energy(lo_decoder *d, const lo_cf *samples);                   /* A11 :368-375 */

/* batch helper for benchmarks/parity: n aligned symbols of sps samples each */
void lo_demod_fft_batch(lo_decoder *d, const lo_cf *iq, size_t n_symbols, uint32_t *bins, float *mags);
void lo_demod_grad_batch(lo_decoder *d, const lo_cf *iq, size_t n_symbols, uint32_t *bins);

/* the state machine (A12 :740-903).  `in` must hold at least 2*sps items (the block's
 * output_multiple, :91).  Returns the number of items consumed by this call. */
int lo_work(lo_decoder *d, const lo_cf *in, lo_step *trace);
/* fake scheduler: feeds work() until fewer than 2*sps items remain; returns total consumed.
 * If steps!=NULL records up to max_steps traces; *n_steps gets the number of calls made. */
size_t lo_run(lo_decoder *d, const lo_cf *in, size_t n_items, lo_step *steps, size_t max_steps, size_t *n_steps);
int lo_state(const lo_decoder *d);

/* frames published on port "frames" (msg_lora_frame, :588-609): loratap(15) | phy(3) | payload */
size_t lo_frame_count(const lo_decoder *d);
size_t lo_frame_len(const lo_decoder *d, size_t idx);
const uint8_t *lo_frame_data(const lo_decoder *d, size_t idx);
void lo_frames_clear(lo_decoder *d);
/* everything the reference writes to std::cout (banner :93-103, hex lines :832,872) */
const char *lo_stdout(const lo_decoder *d);

/* integer-stage pure functions (B1-B4) for unit tests and the K8 parity tests */
uint32_t lo_rotl(uint32_t bits, uint32_t count, uint32_t size);                      /* utilities.h:96-103 */
uint32_t lo_gray(uint32_t bin);                                                      /* :512 */
uint32_t lo_reduce_bin(uint32_t bin, uint32_t n_bins_hdr);                           /* :508 */
void lo_deinterleave_words(const uint32_t *words, uint32_t n_words, uint32_t ppm, uint8_t *out /* ppm */); /* B1 :535-565 */
uint8_t lo_deshuffle_byte(uint8_t v);                                                /* B2 :611-624 */
uint8_t lo_hamming84_encode(uint8_t nibble);                                         /* utilities.h:257-264 */
uint8_t lo_hamming84_decode(uint8_t codeword);                                       /* liquid fec_hamming84 stand-in */
uint8_t lo_hamming_decode_soft_byte(uint8_t v);                                      /* utilities.h:288-339 */
/* full B2-B4 chain on a codeword vector: returns number of bytes written (decode(), :567-586).
 * `cr` is d_phdr.cr at the time of the call. */
size_t lo_decode_codewords(const uint8_t *demodulated, size_t n, int is_header, uint8_t cr,
                           uint8_t *out, size_t out_cap, size_t *consumed);
/* B5: payload symbol count from the decoded header (:838-847) */
int32_t lo_payload_symbols(uint32_t payload_len, uint8_t cr, uint8_t sf, int reduced_rate);

#ifdef __cplusplus
}
#endif
#endif
