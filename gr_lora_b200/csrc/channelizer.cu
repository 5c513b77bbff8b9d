// channelizer.cu -- SURVEY.md 8f row N1: the block in front of the decoder.
//
// The reference's channelizer (lib/channelizer_impl.cc:40-60) is a hier block around GNU Radio's
// freq_xlating_fir_filter_ccf(decimation, firdes::low_pass(1, fs, bw/2 + 15000, 10000, WIN_HAMMING),
// channel_list[0] - center_freq, fs); it wires only channel_list[0].  gr-filter is not part of the
// reference tree, so the arithmetic below restates GNU Radio's published algorithm
//   taps   firdes::low_pass: windowed sinc, ntaps = odd(int(53 fs / (22 tw))), unity DC gain
//   filter y[n] = rot^n * sum_k (taps[k] e^{j w k}) x[n D - k],  rot = e^{-j w D},  w = 2 pi f_off / fs
// and parity is "unpinned" (SURVEY.md 8c): it is checked against a float64 restatement in the tests.
// Here every channel of channel_list is produced (one FIR bank launch, the wideband input is staged in
// shared memory once per tile and reused by all channels), output stays in HBM for the decoder.
#include "../../include/lora_b200.h"
#include "cuda_owned.h"
#include "device_once.h"
#include <cuda_runtime.h>
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

extern "C" const char *lora_b200_last_error(void);
namespace lbc {
extern thread_local std::string g_err_chan;
thread_local std::string g_err_chan;
}

struct lora_b200_channelizer {
    float samp_rate, center_freq;
    uint32_t bandwidth, decimation, n_channels, ntaps;
    int device;
    std::vector<float> channel_list, taps;
    std::vector<double> cfo, w, phase;            // per channel: applied CFO, rad/sample, rotator phase at the next output
    // device memory, owned by the members and freed by the destructor (cuda_owned.h)
    lb::DeviceBuffer<float2> d_ctaps;             // [n_channels][ntaps]
    lb::DeviceBuffer<float2> d_hist;              // last ntaps-1 input samples
    lb::DeviceBuffer<double> d_phase, d_dphase;
    lb::DeviceBuffer<float2> d_in, d_out;         // internal staging for the host entry point; d_out is [n_channels][out_cap()]
    uint64_t launches = 0;
    bool conj_out = false;                        // conjugate every output sample (the hier block's optional conjugate_cc)
    std::string err;
    size_t out_cap() const { return d_out.capacity() / n_channels; }     // items per channel
};

namespace {

constexpr int CH_TN = 128;      // outputs per block
constexpr int CH_CT = 4;        // channels per block (register accumulators)

__global__ void __launch_bounds__(CH_TN)
chan_fir_kernel(const float2 *__restrict__ hist, const float2 *__restrict__ x, size_t n_in, uint32_t D, uint32_t ntaps,
                const float2 *__restrict__ ctaps, const double *__restrict__ phase0, const double *__restrict__ dphase,
                float2 *__restrict__ out, size_t out_stride, size_t n_out, uint32_t n_channels, float conj_sign) {
    extern __shared__ float2 ch_smem[];
    const uint32_t seg = (CH_TN - 1) * D + ntaps;            // input samples this tile needs
    float2 *xs = ch_smem;                                     // [seg]
    float2 *ts = ch_smem + seg;                               // [CH_CT][ntaps]
    const size_t n0 = (size_t)blockIdx.x * CH_TN;
    const uint32_t c0 = blockIdx.y * CH_CT;
    // xs[i] = x_ext[n0*D - (ntaps-1) + i], x_ext = history followed by this call's input
    const long long first = (long long)n0 * D - (long long)(ntaps - 1);
    for (uint32_t i = threadIdx.x; i < seg; i += CH_TN) {
        const long long idx = first + i;
        float2 v = make_float2(0.f, 0.f);
        if (idx < 0) v = hist[idx + (long long)(ntaps - 1)];
        else if ((size_t)idx < n_in) v = x[idx];
        xs[i] = v;
    }
    for (uint32_t i = threadIdx.x; i < CH_CT * ntaps; i += CH_TN) {
        const uint32_t c = c0 + i / ntaps;
        ts[i] = c < n_channels ? ctaps[(size_t)c * ntaps + i % ntaps] : make_float2(0.f, 0.f);
    }
    __syncthreads();
    const size_t n = n0 + threadIdx.x;
    float2 acc[CH_CT];
#pragma unroll
    for (int c = 0; c < CH_CT; c++) acc[c] = make_float2(0.f, 0.f);
    const float2 *xp = xs + (size_t)threadIdx.x * D + (ntaps - 1);       // x[nD - k] = xp[-k]
    for (uint32_t k = 0; k < ntaps; k++) {
        const float2 xv = xp[-(int)k];
#pragma unroll
        for (int c = 0; c < CH_CT; c++) {
            const float2 t = ts[c * ntaps + k];
            acc[c].x = fmaf(t.x, xv.x, fmaf(-t.y, xv.y, acc[c].x));
            acc[c].y = fmaf(t.x, xv.y, fmaf(t.y, xv.x, acc[c].y));
        }
    }
    if (n < n_out) {
#pragma unroll
        for (int c = 0; c < CH_CT; c++) {
            const uint32_t ch = c0 + c;
            if (ch < n_channels) {
                double s, co;
                sincos(phase0[ch] + dphase[ch] * (double)n, &s, &co);   // rotator e^{-j w D n}, phase kept in double
                const float cr = (float)co, sr = (float)s;
                // conj_sign = -1: the blocks.conjugate_cc the reference wires between channelizer and decoder (python/lora_receiver.py:70-75)
                out[(size_t)ch * out_stride + n] = make_float2(acc[c].x * cr - acc[c].y * sr, conj_sign * (acc[c].x * sr + acc[c].y * cr));
            }
        }
    }
}

int cfail(lora_b200_channelizer *c, int code, const char *msg) {
    if (c) c->err = msg;
    lbc::g_err_chan = msg;
    return code;
}

// firdes::low_pass(gain=1, fs, cutoff, transition_width, WIN_HAMMING) as published by GNU Radio
std::vector<float> firdes_low_pass(double fs, double cutoff, double tw) {
    int ntaps = (int)(53.0 * fs / (22.0 * tw));               // max_attenuation(Hamming) = 53 dB
    if ((ntaps & 1) == 0) ntaps++;
    std::vector<float> taps(ntaps), w(ntaps);
    const int M = (ntaps - 1) / 2;
    for (int n = 0; n < ntaps; n++) w[n] = (float)(0.54 - 0.46 * cos((2.0 * M_PI * n) / (ntaps - 1)));
    const double fwT0 = 2.0 * M_PI * cutoff / fs;
    for (int n = -M; n <= M; n++) {
        if (n == 0) taps[n + M] = (float)(fwT0 / M_PI * w[n + M]);
        else taps[n + M] = (float)(sin(n * fwT0) / (n * M_PI) * w[n + M]);
    }
    double fmax = taps[M];
    for (int n = 1; n <= M; n++) fmax += 2.0 * taps[n + M];
    const double gain = 1.0 / fmax;
    for (int i = 0; i < ntaps; i++) taps[i] = (float)(taps[i] * gain);
    return taps;
}

int upload_channel(lora_b200_channelizer *c, uint32_t ch) {
    // freq_xlating_fir_filter::build_composite_fir: ctaps[i] = taps[i] e^{j i w}; rotator increment e^{-j w D}
    const double f_off = (double)c->channel_list[ch] - (double)c->center_freq + c->cfo[ch];
    const double w = 2.0 * M_PI * f_off / (double)c->samp_rate;
    c->w[ch] = w;
    std::vector<float2> ct(c->ntaps);
    for (uint32_t i = 0; i < c->ntaps; i++) ct[i] = make_float2((float)(c->taps[i] * cos(w * i)), (float)(c->taps[i] * sin(w * i)));
    if (cudaMemcpy(c->d_ctaps + (size_t)ch * c->ntaps, ct.data(), sizeof(float2) * c->ntaps, cudaMemcpyHostToDevice) != cudaSuccess)
        return cfail(c, LORA_B200_ECUDA, "channelizer: upload of composite taps failed");
    return LORA_B200_OK;
}

}  // namespace

extern "C" {

const char *lora_b200_channelizer_last_error(void) { return lbc::g_err_chan.c_str(); }

lora_b200_channelizer *lora_b200_channelizer_create(float samp_rate, float center_freq, const float *channel_list,
                                                    uint32_t n_channels, uint32_t bandwidth, uint32_t decimation, int32_t device) {
    if (!channel_list || n_channels == 0 || decimation == 0 || samp_rate <= 0) { cfail(nullptr, LORA_B200_EINVAL, "channelizer: bad argument"); return nullptr; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cfail(nullptr, LORA_B200_ECUDA, "no CUDA device: liblora_b200 has no CPU fallback"); return nullptr; }
    lora_b200_channelizer *c = new lora_b200_channelizer();
    c->samp_rate = samp_rate; c->center_freq = center_freq; c->bandwidth = bandwidth; c->decimation = decimation;
    c->n_channels = n_channels;
    c->channel_list.assign(channel_list, channel_list + n_channels);
    if (device < 0) cudaGetDevice(&device);
    c->device = device;
    cudaSetDevice(device);
    c->taps = firdes_low_pass(samp_rate, (double)(bandwidth / 2) + 15000.0, 10000.0);      // lib/channelizer_impl.cc:46
    c->ntaps = (uint32_t)c->taps.size();
    c->cfo.assign(n_channels, 0.0); c->w.assign(n_channels, 0.0); c->phase.assign(n_channels, 0.0);
    bool ok = c->d_ctaps.reserve((size_t)n_channels * c->ntaps) == cudaSuccess &&
              c->d_hist.reserve(c->ntaps) == cudaSuccess &&
              c->d_phase.reserve(n_channels) == cudaSuccess &&
              c->d_dphase.reserve(n_channels) == cudaSuccess &&
              cudaMemset(c->d_hist, 0, sizeof(float2) * c->ntaps) == cudaSuccess;
    for (uint32_t ch = 0; ok && ch < n_channels; ch++) ok = upload_channel(c, ch) == LORA_B200_OK;
    if (!ok) { cfail(nullptr, LORA_B200_ECUDA, "channelizer: device allocation failed"); delete c; return nullptr; }
    return c;
}

void lora_b200_channelizer_destroy(lora_b200_channelizer *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    delete c;
}

uint32_t lora_b200_channelizer_ntaps(const lora_b200_channelizer *c) { return c ? c->ntaps : 0; }
int lora_b200_channelizer_taps(const lora_b200_channelizer *c, float *out, size_t cap) {
    if (!c || !out || cap < c->ntaps) return cfail(nullptr, LORA_B200_EINVAL, "channelizer_taps: buffer too small");
    for (uint32_t i = 0; i < c->ntaps; i++) out[i] = c->taps[i];
    return (int)c->ntaps;
}

int lora_b200_channelizer_set_conjugate(lora_b200_channelizer *c, int on) {
    if (!c) return cfail(c, LORA_B200_EINVAL, "channelizer_set_conjugate: null argument");
    c->conj_out = on != 0;
    return LORA_B200_OK;
}

int lora_b200_channelizer_apply_cfo(lora_b200_channelizer *c, uint32_t channel, float cfo) {   // channelizer_impl::apply_cfo :68-71
    if (!c || channel >= c->n_channels) return cfail(c, LORA_B200_EINVAL, "channelizer_apply_cfo: bad channel");
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    c->cfo[channel] += cfo;
    return upload_channel(c, channel);
}

int lora_b200_channelizer_work_dev(lora_b200_channelizer *c, const void *in_dev, size_t n_in, void *out_dev,
                                   size_t out_stride, size_t *n_out, void *cuda_stream) {
    if (!c || (!in_dev && n_in) || !out_dev || !n_out) return cfail(c, LORA_B200_EINVAL, "channelizer_work: null argument");
    if (n_in % c->decimation) return cfail(c, LORA_B200_EINVAL, "channelizer_work: n_in must be a multiple of the decimation");
    const size_t no = n_in / c->decimation;
    *n_out = no;
    if (no == 0) return LORA_B200_OK;
    if (out_stride < no) return cfail(c, LORA_B200_EINVAL, "channelizer_work: out_stride < n_out");
    cudaSetDevice(c->device);
    cudaStream_t st = (cudaStream_t)cuda_stream;
    std::vector<double> dph(c->n_channels);
    for (uint32_t ch = 0; ch < c->n_channels; ch++) dph[ch] = -c->w[ch] * (double)c->decimation;
    if (cudaMemcpyAsync(c->d_phase, c->phase.data(), sizeof(double) * c->n_channels, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(c->d_dphase, dph.data(), sizeof(double) * c->n_channels, cudaMemcpyHostToDevice, st) != cudaSuccess)
        return cfail(c, LORA_B200_ECUDA, "channelizer_work: phase upload failed");
    cudaStreamSynchronize(st);                       // dph is a stack vector
    const uint32_t seg = (CH_TN - 1) * c->decimation + c->ntaps;
    const size_t smem = sizeof(float2) * ((size_t)seg + (size_t)CH_CT * c->ntaps);
    if (smem > 48 * 1024 && lb::opt_in_smem((const void *)chan_fir_kernel, c->device, 200 * 1024) != cudaSuccess)
        return cfail(c, LORA_B200_ECUDA, "channelizer_work: shared memory attribute");
    if (smem > 200 * 1024) return cfail(c, LORA_B200_EUNSUPPORTED, "channelizer_work: filter too long for one tile");
    dim3 grid((unsigned)((no + CH_TN - 1) / CH_TN), (c->n_channels + CH_CT - 1) / CH_CT);
    chan_fir_kernel<<<grid, CH_TN, smem, st>>>(c->d_hist, (const float2 *)in_dev, n_in, c->decimation, c->ntaps, c->d_ctaps,
                                              c->d_phase, c->d_dphase, (float2 *)out_dev, out_stride, no, c->n_channels, c->conj_out ? -1.0f : 1.0f);
    c->launches++;
    if (cudaGetLastError() != cudaSuccess) return cfail(c, LORA_B200_ECUDA, "channelizer_work: launch failed");
    // history for the next call: the last ntaps-1 samples of (history ++ input)
    const size_t h = c->ntaps - 1;
    if (n_in >= h) {
        if (cudaMemcpyAsync(c->d_hist, (const float2 *)in_dev + (n_in - h), sizeof(float2) * h, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
            return cfail(c, LORA_B200_ECUDA, "channelizer_work: history copy failed");
    } else {
        std::vector<float2> tmp(h), in(n_in), nh(h);
        if (cudaStreamSynchronize(st) != cudaSuccess ||
            cudaMemcpy(tmp.data(), c->d_hist, sizeof(float2) * h, cudaMemcpyDeviceToHost) != cudaSuccess ||
            cudaMemcpy(in.data(), in_dev, sizeof(float2) * n_in, cudaMemcpyDeviceToHost) != cudaSuccess)
            return cfail(c, LORA_B200_ECUDA, "channelizer_work: history copy failed");
        for (size_t i = 0; i < h; i++) nh[i] = (i + n_in < h) ? tmp[i + n_in] : in[i + n_in - h];
        if (cudaMemcpy(c->d_hist, nh.data(), sizeof(float2) * h, cudaMemcpyHostToDevice) != cudaSuccess)
            return cfail(c, LORA_B200_ECUDA, "channelizer_work: history copy failed");
    }
    for (uint32_t ch = 0; ch < c->n_channels; ch++) c->phase[ch] = fmod(c->phase[ch] + dph[ch] * (double)no, 2.0 * M_PI);
    return LORA_B200_OK;
}

int lora_b200_channelizer_work_host(lora_b200_channelizer *c, const void *in_host, size_t n_in, size_t *n_out) {
    if (!c || (!in_host && n_in) || !n_out) return cfail(c, LORA_B200_EINVAL, "channelizer_work_host: null argument");
    cudaSetDevice(c->device);
    const size_t no = n_in / c->decimation;
    if (c->d_in.reserve(n_in) != cudaSuccess) return cfail(c, LORA_B200_ENOMEM, "channelizer: input staging");
    if (c->d_out.reserve(no * c->n_channels) != cudaSuccess) return cfail(c, LORA_B200_ENOMEM, "channelizer: output buffer");
    if (n_in && cudaMemcpy(c->d_in, in_host, sizeof(float2) * n_in, cudaMemcpyHostToDevice) != cudaSuccess)
        return cfail(c, LORA_B200_ECUDA, "channelizer: H2D failed");
    int rc = lora_b200_channelizer_work_dev(c, c->d_in, n_in, c->d_out, c->out_cap(), n_out, nullptr);
    if (rc) return rc;
    if (cudaDeviceSynchronize() != cudaSuccess) return cfail(c, LORA_B200_ECUDA, "channelizer: kernel failed");
    return LORA_B200_OK;
}

const void *lora_b200_channelizer_output(const lora_b200_channelizer *c, uint32_t channel, size_t *stride_items) {
    if (!c || channel >= c->n_channels || !c->d_out) return nullptr;
    if (stride_items) *stride_items = c->out_cap();
    return c->d_out + (size_t)channel * c->out_cap();
}

int lora_b200_channelizer_read_output(const lora_b200_channelizer *c, uint32_t channel, void *host_dst, size_t n_items) {
    if (!c || channel >= c->n_channels || !c->d_out || (!host_dst && n_items)) return cfail(nullptr, LORA_B200_EINVAL, "channelizer_read_output: bad argument");
    if (n_items > c->out_cap()) return cfail(nullptr, LORA_B200_EINVAL, "channelizer_read_output: more items than the last call produced");
    cudaSetDevice(c->device);
    if (n_items && cudaMemcpy(host_dst, c->d_out + (size_t)channel * c->out_cap(), sizeof(float2) * n_items, cudaMemcpyDeviceToHost) != cudaSuccess)
        return cfail(nullptr, LORA_B200_ECUDA, "channelizer_read_output: D2H failed");
    return LORA_B200_OK;
}

uint64_t lora_b200_channelizer_launch_count(const lora_b200_channelizer *c) { return c ? c->launches : 0; }

}  // extern "C"
