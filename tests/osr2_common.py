"""Shared helpers of the fs/bw = 2 tests (no torch): the decoder's tables at 250 kS/s, K1 test batches, the float64 max-log
LLR definition, the host emulation's oversampling-aware entry points and frames modulated at fs = 2 bw."""
from __future__ import annotations

import ctypes as C

import numpy as np

import gr_lora_b200 as G
from gr_lora_b200 import build, tx
from k1_reference import CHUNK_BYTES, K1Reference

OSR = 2
BW = 125e3
FS = OSR * BW
CAP = 16
CARRIER = 868.1e6

# symbols per CTA batch of k1_fft_kernel<SF, 2> (K1Cfg<SF, 2>::G = 8192 / (2 NP), NP = N up to SF11, N / 2 at SF12)
BATCH = {7: 32, 8: 16, 9: 8, 10: 4, 11: 2, 12: 2}

_TABLES: dict[int, tuple] = {}


def tables(sf):
    """(down, up, tw) of the decoder at fs = 250 kS/s, BW = 125 kHz."""
    if sf not in _TABLES:
        t = G.split_tables(G.tables_build_host(samp_rate=FS, sf=sf), OSR << sf)
        _TABLES[sf] = tuple(np.ascontiguousarray(t[k]) for k in ("downchirp", "upchirp", "twiddles"))
    return _TABLES[sf]


class K1ReferenceOsr(K1Reference):
    """tests/k1_reference.py's float64 get_shift_fft (and its tau criterion, through check_k1) for symbols of sps = osr N
    samples dechirped with `chirp`, the decoder's down-chirp at that rate: tmp[0:N/2] = F[0:N/2], tmp[N/2:N] =
    F[sps-N/2:sps], tmp[N/2] += F[N/2] -- at osr = 2, F[3N/2] + F[N/2]."""

    def __init__(self, x, sf, chirp, osr=OSR):
        n_bins, sps = 1 << sf, osr << sf
        x = np.asarray(x).reshape(-1, sps)
        c = np.asarray(chirp).astype(np.complex128)
        n = x.shape[0]
        self.sf, self.sps, self.n_bins = sf, sps, n_bins
        self.m64 = np.empty((n, n_bins), np.float64)
        self.ynorm = np.empty(n, np.float64)
        step = max(1, CHUNK_BYTES // (16 * sps))
        h = n_bins // 2
        for s in range(0, n, step):
            e = min(n, s + step)
            y = x[s:e].astype(np.complex128) * c
            self.ynorm[s:e] = np.sqrt(np.sum(y.real ** 2 + y.imag ** 2, axis=1))
            f = np.fft.fft(y, axis=1)
            tmp = np.concatenate([f[:, :h], f[:, sps - h:]], axis=1)
            tmp[:, h] += f[:, h]
            self.m64[s:e] = np.abs(tmp)


def k1_batch(sf, rng, n_clean=None):
    """Clean symbols (every bin up to SF10, a spread of bins with the edges and N/2 +- 1 above), symbols at -3 dB per-sample
    SNR, a half-bin frequency offset and pure noise, at fs/bw = 2."""
    n, sps = 1 << sf, OSR << sf
    if n_clean is None:
        vals = np.arange(n) if sf <= 10 else np.unique(np.r_[0, 1, n // 2 - 1, n // 2, n // 2 + 1, n - 1, rng.integers(0, n, 26)])
    else:
        vals = rng.integers(0, n, n_clean)
    clean = tx.modulate_shifts(vals, sf, BW, FS).reshape(-1, sps)
    v2 = rng.integers(0, n, 6)
    noisy = tx.modulate_shifts(v2[:3], sf, BW, FS).reshape(-1, sps) + tx.awgn(3 * sps, -3.0, rng).reshape(-1, sps)
    half = tx.modulate_shifts(v2[3:5], sf, BW, FS).reshape(-1, sps) * np.exp(1j * np.pi * np.arange(sps) / sps)
    noise = (rng.standard_normal(2 * sps) + 1j * rng.standard_normal(2 * sps)).reshape(-1, sps)
    return np.ascontiguousarray(np.concatenate([clean, noisy, half, noise]), np.complex64)


def words_of_bins(sf, reduced):
    """w(k) for every kept bin k: gray((k - 1) mod N), folded to N/4 bins first for reduced-rate symbols."""
    n = 1 << sf
    v = (np.arange(n) - 1) % n
    if reduced:
        v = ((v + 2) >> 2) % (n // 4)
    return v ^ (v >> 1)


def llr64(m64, sf, reduced):
    """The max-log LLR definition in float64 over the float64 |tmp| of every kept bin."""
    ppm = sf - 2 if reduced else sf
    w = words_of_bins(sf, reduced)
    out = np.empty((m64.shape[0], ppm))
    for j in range(ppm):
        b = (w >> j) & 1
        out[:, j] = m64[:, b == 0].max(axis=1) - m64[:, b == 1].max(axis=1)
    return out


def check_llrs(llr, bins, ref, sf, reduced, what):
    """Every LLR within 2 tau of the float64 one; its sign that of the reported bin's bits when no second bin lies in the (A)
    band of tests/k1_reference.py."""
    want = llr64(ref.m64, sf, reduced)
    mx = ref.m64.max(axis=1)
    tau = ref.tau(mx)[:, None]
    err = np.abs(llr.astype(np.float64) - want)
    assert np.all(err <= 2 * tau), f"{what}: worst |LLR - LLR64| / tau = {np.max(err / tau):.3g}"
    band = np.sum(ref.m64 >= (mx - 2 * ref.tau(mx))[:, None], axis=1)
    w = words_of_bins(sf, reduced)[np.asarray(bins, np.int64)]
    for i in np.flatnonzero(band == 1):
        bits = (w[i] >> np.arange(llr.shape[1])) & 1
        assert np.array_equal(llr[i] < 0, bits == 1), (what, i, llr[i], bits)


_EMUL = None


def emul():
    """build/host_emul.so with the argument types of its oversampling-aware entry points."""
    global _EMUL
    if _EMUL is None:
        L = C.CDLL(str(build.build_host_emul()))
        L.lb_k1_emulate_osr.restype = C.c_int
        L.lb_k1_emulate_osr.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.lb_k1_llr_emulate_osr.restype = C.c_int
        L.lb_k1_llr_emulate_osr.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                            C.c_void_p]
        f = L.lb_emul_rx_receive_osr
        f.restype = C.c_uint32
        f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_int,
                      C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
        _EMUL = L
    return _EMUL


def k1_emulate(x, sf, osr=OSR, chirp=None, tw=None):
    x = np.ascontiguousarray(x, np.complex64)
    if chirp is None:
        chirp, _, tw = tables(sf)
    n = x.size // (osr << sf)
    bins = np.zeros(n, np.uint32)
    mags = np.zeros(n, np.float32)
    assert emul().lb_k1_emulate_osr(sf, osr, x.ctypes.data, n, chirp.ctypes.data, tw.ctypes.data, bins.ctypes.data, mags.ctypes.data) == 0
    return bins, mags


def llr_emulate(x, sf, reduced, osr=OSR):
    x = np.ascontiguousarray(x, np.complex64)
    down, _, tw = tables(sf)
    n = x.size // (osr << sf)
    llr = np.zeros((n, sf - 2 if reduced else sf), np.float32)
    bins = np.zeros(n, np.uint32)
    assert emul().lb_k1_llr_emulate_osr(sf, osr, x.ctypes.data, n, down.ctypes.data, tw.ctypes.data, int(reduced), llr.ctypes.data,
                                        bins.ctypes.data) == 0
    return llr, bins


def receive_emul(x, sf, cr=4, rr=False, soft=False, sfo_ppm=0.0, carrier_hz=0.0, implicit=False, crc=True, implicit_len=0,
                 sync_word=0x12, min_preamble=0):
    """lb_emul_rx_receive_osr at fs/bw = 2 on one row: a dict per synchronised frame."""
    x = np.ascontiguousarray(x, np.complex64)
    down, up, tw = tables(sf)
    start = np.zeros(CAP, np.int64)
    cfo = np.zeros(CAP, np.float32)
    snr = np.zeros(CAP, np.float32)
    status = np.zeros(CAP, np.int32)
    sfo = np.zeros(CAP, np.float32)
    pay = np.zeros((CAP, 256), np.uint8)
    ln = np.zeros(CAP, np.uint32)
    n = emul().lb_emul_rx_receive_osr(x.ctypes.data, x.size, down.ctypes.data, up.ctypes.data, tw.ctypes.data, sf, OSR, cr,
                                      int(implicit), int(crc), int(rr), sync_word, implicit_len, min_preamble, float(sfo_ppm),
                                      float(carrier_hz), int(soft), start.ctypes.data, cfo.ctypes.data, snr.ctypes.data,
                                      status.ctypes.data, sfo.ctypes.data, pay.ctypes.data, ln.ctypes.data, CAP)
    return [dict(start=int(start[k]), cfo=float(cfo[k]), snr=float(snr[k]), status=int(status[k]), sfo=float(sfo[k]),
                 payload=bytes(pay[k, : ln[k]])) for k in range(n)]


def frame_row(sf, payload, cfo_hz, offset, *, snr_db=None, seed=0, cr=4, rr=None, sfo_ppm=0.0, tail=3):
    """One frame modulated at fs = 2 bw at sample `lead + offset` of a row (CFO in Hz, the transmitter's clock off by sfo_ppm),
    SNR in the 125 kHz band (None: no noise).  Returns (row, lead, frame length)."""
    rr = sf > 10 if rr is None else rr
    sps = OSR << sf
    f = tx.modulate_frame(tx.encode_frame(payload, sf, cr, reduced_rate=rr), sf, fs=FS, sfo_ppm=sfo_ppm)
    lead = 2 * sps + offset
    x = np.zeros(lead + f.size + tail * sps, np.complex128)
    x[lead: lead + f.size] = f
    x *= np.exp(2j * np.pi * cfo_hz * np.arange(x.size) / FS)
    if snr_db is not None:
        x += tx.awgn(x.size, snr_db - 10 * np.log10(OSR), np.random.default_rng(seed))
    return x.astype(np.complex64), lead, f.size
