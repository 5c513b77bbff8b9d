// tx_channel.cuh -- synthetic transmitter and channel on the device (SURVEY 8(f) N3).
//
// The reference is a receiver only (its README points at a hardware transmitter), so this has no reference counterpart; it
// is what tests and the benchmark need to put known LoRa traffic into HBM without a pass over PCIe:
//   * tx_symbols_kernel   aligned data symbols: out[s][n] = up[(n + decim * value[s]) mod sps] * e^{j 2 pi cfo[s] n / fs}
//                         + sigma (N(0,1) + j N(0,1)) -- the cyclic-shift modulator of gr_lora_b200/tx.py::modulate_shifts
//                         (bit-identical to it when given the same chirp table and no noise / CFO);
//   * tx_expand_kernel    a batch of concurrent channels from K base captures: out[s] = base[s mod K] + the stream's own
//                         noise (64 channels that replay one capture would correlate perfectly);
//   * tx_frames_kernel    whole streams of placed frames (preamble, sync word, SFD, the data symbols tx_encode_kernel of
//                         tx_encode.cuh produced), per-frame CFO, the noise of tx_expand_kernel: every stream its own payloads.
// Noise: Philox4x32-10 keyed by the seed, counter = (sample pair, row), Box-Muller on the four 32-bit outputs -- a
// counter-based generator, so the result does not depend on the launch geometry.  Both kernels are HBM-write bound.
#pragma once
#include "lora_common.cuh"

namespace lb {
#ifdef __CUDACC__
LB_HD uint32_t philox_mulhi(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (uint32_t)(((unsigned long long)a * b) >> 32);
#endif
}
LB_HD void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
    const uint32_t hi0 = philox_mulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = philox_mulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
}
// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3"): c <- ten rounds under key (k0, k1)
LB_HD void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; r++) {
        philox_round(c, k0, k1);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
}
// four normal deviates for (row, pair index i) under `seed`
LB_D float4 philox_normal4(unsigned long long seed, unsigned long long row, unsigned long long i) {
    uint32_t c[4] = {(uint32_t)i, (uint32_t)(i >> 32), (uint32_t)row, (uint32_t)(row >> 32)};
    philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
    const float s = 2.3283064365386963e-10f;                    // 2^-32
    const float u0 = ((float)c[0] + 0.5f) * s, u1 = (float)c[1] * s, u2 = ((float)c[2] + 0.5f) * s, u3 = (float)c[3] * s;
    const float r0 = sqrtf(-2.0f * __logf(fminf(u0, 0.99999994f))), r1 = sqrtf(-2.0f * __logf(fminf(u2, 0.99999994f)));
    float s0, c0, s1, c1;
    sincospif(2.0f * u1, &s0, &c0);
    sincospif(2.0f * u3, &s1, &c1);
    return make_float4(r0 * c0, r0 * s0, r1 * c1, r1 * s1);
}

// one thread = two consecutive samples of one symbol
__global__ void tx_symbols_kernel(const float2 *__restrict__ up, uint32_t sps, uint32_t decim, const uint32_t *__restrict__ values,
                                  const float *__restrict__ cfo_hz, double inv_fs, float sigma, unsigned long long seed,
                                  size_t n_symbols, float2 *__restrict__ out) {
    const size_t pairs = (size_t)sps / 2, total = n_symbols * pairs;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
        const size_t s = g / pairs;
        const uint32_t n = (uint32_t)(g - s * pairs) * 2u;
        const uint32_t sh = values[s] * decim;
        float2 a = up[(n + sh) % sps], b = up[(n + 1u + sh) % sps];
        if (cfo_hz) {
            const double rev = (double)cfo_hz[s] * inv_fs;        // revolutions per sample
            double t0 = rev * (double)n, t1 = rev * (double)(n + 1u);
            t0 -= floor(t0); t1 -= floor(t1);
            float s0, c0, s1, c1;
            sincospif(2.0f * (float)t0, &s0, &c0);
            sincospif(2.0f * (float)t1, &s1, &c1);
            a = make_float2(a.x * c0 - a.y * s0, a.x * s0 + a.y * c0);
            b = make_float2(b.x * c1 - b.y * s1, b.x * s1 + b.y * c1);
        }
        if (sigma != 0.0f) {
            const float4 z = philox_normal4(seed, s, n / 2u);
            a.x = fmaf(sigma, z.x, a.x); a.y = fmaf(sigma, z.y, a.y);
            b.x = fmaf(sigma, z.z, b.x); b.y = fmaf(sigma, z.w, b.y);
        }
        __stcs(reinterpret_cast<float4 *>(out + s * sps + n), make_float4(a.x, a.y, b.x, b.y));
    }
}

// out[s][i] = base[s % k][i] + noise(seed, s, i); n_items even
__global__ void tx_expand_kernel(const float2 *__restrict__ base, uint32_t k, size_t n_items, float sigma, unsigned long long seed,
                                 size_t n_streams, float2 *__restrict__ out) {
    const size_t pairs = n_items / 2, total = n_streams * pairs;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
        const size_t s = g / pairs, i = (g - s * pairs) * 2;
        const float4 v = __ldg(reinterpret_cast<const float4 *>(base + (s % k) * n_items + i));
        float4 o = v;
        if (sigma != 0.0f) {
            const float4 z = philox_normal4(seed, s, i / 2);
            o = make_float4(fmaf(sigma, z.x, v.x), fmaf(sigma, z.y, v.y), fmaf(sigma, z.z, v.z), fmaf(sigma, z.w, v.w));
        }
        __stcs(reinterpret_cast<float4 *>(out + s * n_items + i), o);
    }
}

// one placed frame of tx_frames_kernel; a row's frames are sorted by start and do not overlap
struct TxFrameDesc {
    unsigned long long start;   // first preamble sample in the row
    uint32_t n_symbols;         // data symbols, shifts[shift_row * max_symbols ..]
    float cfo_hz;
    uint32_t shift_row;
    uint32_t sync;              // bins of the two sync symbols, low and high half
    double rate;                // 1 + delta: transmitter samples per row sample (1: no clock offset)
    unsigned long long n_rx;    // row samples the frame covers: those with (n - start) * rate < tx_frame_samples
};

// samples of a frame: 8 preamble up-chirps, 2 sync symbols, 2.25 down-chirps (conj(up)), then the data symbols
LB_HD unsigned long long tx_frame_samples(uint32_t n_symbols, uint32_t sps) { return (12ull + n_symbols) * sps + sps / 4u; }

// row samples i >= 0 of a frame of len transmitter samples with i * rate < len, rate = 1 + delta (rx_sync.cuh's convention)
inline unsigned long long tx_drifted_samples(unsigned long long len, double rate) {
    unsigned long long n = (unsigned long long)ceil((double)len / rate);
    while (n && (double)(n - 1) * rate >= (double)len) n--;
    while ((double)n * rate < (double)len) n++;
    return n;
}

// sample o (< tx_frame_samples) of frame fr, before the CFO rotation
LB_D float2 tx_frame_sample(const float2 *__restrict__ up, uint32_t sps, uint32_t decim, const TxFrameDesc &fr,
                            const uint32_t *__restrict__ shifts, uint32_t max_symbols, uint32_t n_bins, uint32_t o) {
    const uint32_t q = o / sps, r = o - q * sps;
    if (q < 8u) return __ldg(up + r);
    if (q < 10u) return __ldg(up + (r + ((q == 8u ? fr.sync : fr.sync >> 16) & 0xFFFFu) * decim) % sps);
    const uint32_t sfd_end = 12u * sps + sps / 4u;
    if (o < sfd_end) {                 // conj(up), with +0 for a zero imaginary part, as tx.channel's complex scaling leaves it
        const float2 u = __ldg(up + r);
        return make_float2(u.x, __fsub_rn(0.0f, u.y));
    }
    const uint32_t d = o - sfd_end, k = d / sps, rr = d - k * sps;
    const uint32_t sh = __ldg(shifts + (size_t)fr.shift_row * max_symbols + k) % n_bins;
    return __ldg(up + (rr + sh * decim) % sps);
}

// the same at fractional transmitter time u (a frame with a clock offset), from the phase law of tx.base_upchirp:
// up(m) = e^{j 2 pi m (m - sps) / (2 decim sps)} for 0 <= m < sps, in double and reduced to revolutions, times up[0] (the
// table's value at phase 0, so that its amplitude and rotation carry over); a cyclic shift by sh bins reads up at
// (m + sh decim) mod sps, the SFD is the conjugate
LB_D float2 tx_frame_sample_at(const float2 *__restrict__ up, uint32_t sps, uint32_t decim, const TxFrameDesc &fr,
                               const uint32_t *__restrict__ shifts, uint32_t max_symbols, uint32_t n_bins, double u) {
    const double S = (double)sps;
    double q = floor(u / S), m = u - q * S;
    bool conj = false;
    if (q >= 8.0 && q < 10.0) {
        m += (double)(((q == 8.0 ? fr.sync : fr.sync >> 16) & 0xFFFFu) * decim);
    } else if (q >= 10.0) {
        const double d = u - 12.25 * S;
        if (d < 0.0) {
            conj = true;
        } else {
            const double k = floor(d / S);
            const uint32_t sh = __ldg(shifts + (size_t)fr.shift_row * max_symbols + (uint32_t)k) % n_bins;
            m = d - k * S + (double)(sh * decim);
        }
    }
    if (m >= S) m -= S;
    double rev = m * (m - S) / (2.0 * (double)decim * S);
    rev -= floor(rev);
    float sn, cs;
    sincospif(2.0f * (float)rev, &sn, &cs);
    const float2 v = cmul(__ldg(up), make_float2(cs, sn));
    return conj ? make_float2(v.x, -v.y) : v;
}

// whole streams of frames: out[s][n] = frame sample (0 outside every frame) * e^{j 2 pi cfo n / fs} + noise(seed, s, n), the
// noise exactly tx_expand_kernel's, so that with sigma > 0 the output equals tx_expand over the sigma = 0 output.  One thread
// = one sample pair; the covering frame comes from a binary search of the row's sorted list (row_ptr: CSR over rows).
__global__ void tx_frames_kernel(const float2 *__restrict__ up, uint32_t sps, uint32_t decim, uint32_t n_bins,
                                 const uint32_t *__restrict__ row_ptr, const TxFrameDesc *__restrict__ frames,
                                 const uint32_t *__restrict__ shifts, uint32_t max_symbols, double inv_fs, float sigma,
                                 unsigned long long seed, size_t n_items, size_t n_streams, float2 *__restrict__ out) {
    const size_t pairs = n_items / 2, total = n_streams * pairs;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
        const size_t s = g / pairs, i = (g - s * pairs) * 2;
        // last frame of the row that starts at or before sample i + 1
        uint32_t lo = __ldg(row_ptr + s), hi = __ldg(row_ptr + s + 1);
        const uint32_t first = lo;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (frames[mid].start <= i + 1) lo = mid + 1; else hi = mid;
        }
        float2 v[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
        for (int e = 0; e < 2 && lo > first; e++) {
            const size_t n = i + e;
            // sample i may still belong to the frame before one that starts at i + 1
            const uint32_t k = (e == 0 && frames[lo - 1].start > n) ? lo - 2 : lo - 1;
            if (k < first || k == 0xFFFFFFFFu) continue;
            const TxFrameDesc fr = frames[k];
            if (n < fr.start || n - fr.start >= fr.n_rx) continue;
            float2 a = fr.rate == 1.0 ? tx_frame_sample(up, sps, decim, fr, shifts, max_symbols, n_bins, (uint32_t)(n - fr.start))
                                      : tx_frame_sample_at(up, sps, decim, fr, shifts, max_symbols, n_bins, (double)(n - fr.start) * fr.rate);
            if (fr.cfo_hz != 0.0f) {                                 // as tx_symbols_kernel: phase reduced in double
                double t = (double)fr.cfo_hz * inv_fs * (double)n;
                t -= floor(t);
                float sn, cs;
                sincospif(2.0f * (float)t, &sn, &cs);
                a = make_float2(a.x * cs - a.y * sn, a.x * sn + a.y * cs);
            }
            v[e] = a;
        }
        float4 o = make_float4(v[0].x, v[0].y, v[1].x, v[1].y);
        if (sigma != 0.0f) {
            const float4 z = philox_normal4(seed, s, i / 2);
            o = make_float4(fmaf(sigma, z.x, o.x), fmaf(sigma, z.y, o.y), fmaf(sigma, z.z, o.z), fmaf(sigma, z.w, o.w));
        }
        __stcs(reinterpret_cast<float4 *>(out + s * n_items + i), o);
    }
}
#endif
}  // namespace lb
