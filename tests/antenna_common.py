"""Shared helpers of the several-antenna receiver tests: the host emulation's antenna entry points, captures of one frame on
M antennas with per-antenna complex gains and independent noise (host: tx.modulate_frame; device: tx_frames, a torch
multiply and tx_expand), and the float64 combined spectrum the screen is held to."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

import gr_lora_b200 as G
from gr_lora_b200 import build, tx
from k1_reference import CHUNK_BYTES, U_FP32

BW = 125e3
CAP = 16
CARRIER = 868.1e6
# per-antenna SNR (125 kHz) at which one antenna decodes every frame (fs/bw = 8 and 2, DESIGN section 5)
SENSITIVITY = {7: -2.0, 8: -5.0, 9: -7.5, 10: -10.0, 11: -12.5, 12: -15.0}

_TABLES: dict[tuple, tuple] = {}


def tables(sf, osr):
    """(down, up, tw) of the decoder at fs = osr * 125 kHz."""
    if (sf, osr) not in _TABLES:
        t = G.split_tables(G.tables_build_host(samp_rate=osr * BW, sf=sf), osr << sf)
        _TABLES[sf, osr] = tuple(np.ascontiguousarray(t[k]) for k in ("downchirp", "upchirp", "twiddles"))
    return _TABLES[sf, osr]


_EMUL = None

_RX_ARGS = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_double,
            C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]


def emul():
    global _EMUL
    if _EMUL is None:
        L = C.CDLL(str(build.build_host_emul()))
        L.lb_k1_antennas_emulate_osr.restype = C.c_int
        L.lb_k1_antennas_emulate_osr.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_uint32, C.c_size_t, C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.c_void_p]
        L.lb_emul_rx_receive_osr.restype = C.c_uint32
        L.lb_emul_rx_receive_osr.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, *_RX_ARGS, C.c_uint32]
        L.lb_emul_rx_receive_antennas.restype = C.c_uint32
        L.lb_emul_rx_receive_antennas.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, *_RX_ARGS,
                                                  C.c_void_p, C.c_uint32]
        _EMUL = L
    return _EMUL


def k1_antennas_emulate(X, sf, osr):
    """The combined screen of one group: X [M, n_windows * sps] -> (bins, mags) per window position."""
    X = np.ascontiguousarray(X, np.complex64)
    down, _, tw = tables(sf, osr)
    m, n = X.shape[0], X.shape[1] // (osr << sf)
    bins = np.zeros(n, np.uint32)
    mags = np.zeros(n, np.float32)
    assert emul().lb_k1_antennas_emulate_osr(sf, osr, X.ctypes.data, X.shape[1], m, n, down.ctypes.data, tw.ctypes.data,
                                             bins.ctypes.data, mags.ctypes.data) == 0
    return bins, mags


def receive_emul(X, sf, osr, *, antennas=None, cr=4, rr=None, soft=False, sfo_ppm=0.0, carrier_hz=0.0, implicit=False, crc=True,
                 implicit_len=0, sync_word=0x12, min_preamble=0):
    """One receiver on the host: lb_emul_rx_receive_antennas over the rows of X [M, n] (antennas=True), or
    lb_emul_rx_receive_osr over the row X [n] (antennas=None with a 1-D X).  A dict per synchronised frame, with h (M complex
    channel estimates) from the antenna entry point."""
    X = np.ascontiguousarray(X, np.complex64)
    rr = sf > 10 if rr is None else rr
    down, up, tw = tables(sf, osr)
    start = np.zeros(CAP, np.int64)
    cfo = np.zeros(CAP, np.float32)
    snr = np.zeros(CAP, np.float32)
    status = np.zeros(CAP, np.int32)
    sfo = np.zeros(CAP, np.float32)
    pay = np.zeros((CAP, 256), np.uint8)
    ln = np.zeros(CAP, np.uint32)
    common = (sf, osr, cr, int(implicit), int(crc), int(rr), sync_word, implicit_len, min_preamble, float(sfo_ppm), float(carrier_hz),
              int(soft), start.ctypes.data, cfo.ctypes.data, snr.ctypes.data, status.ctypes.data, sfo.ctypes.data, pay.ctypes.data,
              ln.ctypes.data)
    h = None
    if X.ndim == 1:
        n = emul().lb_emul_rx_receive_osr(X.ctypes.data, X.size, down.ctypes.data, up.ctypes.data, tw.ctypes.data, *common, CAP)
    else:
        m = X.shape[0]
        h = np.zeros((CAP, m), np.complex64)
        n = emul().lb_emul_rx_receive_antennas(X.ctypes.data, X.shape[1], m, down.ctypes.data, up.ctypes.data, tw.ctypes.data, *common,
                                               h.ctypes.data, CAP)
    return [dict(start=int(start[k]), cfo=float(cfo[k]), snr=float(snr[k]), status=int(status[k]), sfo=float(sfo[k]),
                 payload=bytes(pay[k, : ln[k]]), h=None if h is None else h[k].copy()) for k in range(n)]


def frame_rows(sf, osr, payload, cfo_hz, offset, gains, *, snr_db=None, seed=0, cr=4, rr=None, sfo_ppm=0.0, tail=3, noise_only=()):
    """One frame at sample `lead + offset` on len(gains) antennas: row a = gains[a] * frame (CFO in Hz, the transmitter's
    clock off by sfo_ppm) + its own noise at snr_db in 125 kHz for a unit gain (None: no noise; a sequence: one level per
    antenna, None for a noiseless row).  Rows in noise_only carry noise at that level whatever snr_db is.  Returns (X [M, n]
    complex64, lead, frame length)."""
    rr = sf > 10 if rr is None else rr
    fs, sps = osr * BW, osr << sf
    f = tx.modulate_frame(tx.encode_frame(payload, sf, cr, reduced_rate=rr), sf, fs=fs, sfo_ppm=sfo_ppm)
    lead = 2 * sps + offset
    s = np.zeros(lead + f.size + tail * sps, np.complex128)
    s[lead: lead + f.size] = f
    s *= np.exp(2j * np.pi * cfo_hz * np.arange(s.size) / fs)
    rng = np.random.default_rng(seed)
    X = np.empty((len(gains), s.size), np.complex128)
    for a, g in enumerate(gains):
        X[a] = 0.0 if a in noise_only else g * s
        level = snr_db[a] if np.ndim(snr_db) else snr_db
        level = level if level is not None else (10.0 if a in noise_only else None)
        if level is not None:
            X[a] += tx.awgn(s.size, level - 10 * np.log10(osr), rng)
    return X.astype(np.complex64), lead, f.size


def k1_batch(sf, osr, rng, n_clean=None):
    """Clean symbols (every bin up to SF10, a spread of bins with the edges and N/2 +- 1 above), symbols at -3 dB per-sample
    SNR, a half-bin frequency offset and pure noise, at fs = osr * 125 kHz; [n, sps]."""
    n, sps, fs = 1 << sf, osr << sf, osr * BW
    if n_clean is None:
        vals = np.arange(n) if sf <= 10 else np.unique(np.r_[0, 1, n // 2 - 1, n // 2, n // 2 + 1, n - 1, rng.integers(0, n, 10)])
    else:
        vals = rng.integers(0, n, n_clean)
    vals = rng.permutation(vals)
    clean = tx.modulate_shifts(vals, sf, BW, fs).reshape(-1, sps)
    v2 = rng.integers(0, n, 6)
    noisy = tx.modulate_shifts(v2[:3], sf, BW, fs).reshape(-1, sps) + tx.awgn(3 * sps, -3.0, rng).reshape(-1, sps)
    half = tx.modulate_shifts(v2[3:5], sf, BW, fs).reshape(-1, sps) * np.exp(1j * np.pi * np.arange(sps) / sps)
    noise = (rng.standard_normal(2 * sps) + 1j * rng.standard_normal(2 * sps)).reshape(-1, sps)
    return np.concatenate([clean, noisy, half, noise])


class CombinedReference:
    """The float64 combined spectrum P[k] = sum_a m64_a[k]^2 of M antennas' windows X [M, n, sps] (m64_a: tests/
    k1_reference.py's |tmp| of antenna a, at fs/bw = osr; dechirped with the down-chirp, or with `chirp`), with the rounding
    band summed over the antennas:
        tau_a[k] = u log2(sps) (m64_a[k] + ||y_a||),   tau_P[k] = sum_a (2 m64_a[k] + tau_a[k]) tau_a[k]."""

    def __init__(self, X, sf, osr, antennas=None, chirp=None):
        X = np.asarray(X)
        m, n, sps = X.shape
        n_bins, h = 1 << sf, (1 << sf) // 2
        c = (tables(sf, osr)[0] if chirp is None else np.asarray(chirp)).astype(np.complex128)
        self.P = np.zeros((n, n_bins))
        self.tauP = np.zeros((n, n_bins))
        step = max(1, CHUNK_BYTES // (16 * sps))
        for a in (range(m) if antennas is None else antennas):
            for s in range(0, n, step):
                e = min(n, s + step)
                y = X[a, s:e].astype(np.complex128) * c
                ynorm = np.sqrt(np.sum(np.abs(y) ** 2, axis=1))[:, None]
                f = np.fft.fft(y, axis=1)
                tmp = np.concatenate([f[:, :h], f[:, sps - h:]], axis=1)
                tmp[:, h] += f[:, h]
                m64 = np.abs(tmp)
                tau = U_FP32 * math.log2(sps) * (m64 + ynorm)
                self.P[s:e] += m64 ** 2
                self.tauP[s:e] += (2 * m64 + tau) * tau

    def check(self, bins, mags, what="combined screen"):
        """(A) P[b] + tau_P[b] >= max_k (P[k] - tau_P[k]); (M) |mag - sqrt P[b]| <= tau_P[b] / sqrt P[b] + 4 u sqrt P[b]
        (the fp32 sum over antennas and the square root).  Returns the number of windows whose band held more than one bin."""
        bins = np.asarray(bins).astype(np.int64)
        mags = np.asarray(mags, np.float64)
        rows = np.arange(bins.size)
        assert bins.size == self.P.shape[0], what
        pb, tb = self.P[rows, bins], self.tauP[rows, bins]
        lo = (self.P - self.tauP).max(axis=1)
        bad = pb + tb < lo
        sq = np.sqrt(pb)
        with np.errstate(divide="ignore", invalid="ignore"):
            lim = np.where(sq > 0, tb / sq, 0.0) + 4 * U_FP32 * sq
        bad |= np.abs(mags - sq) > lim
        if bad.any():
            i = np.flatnonzero(bad)[:6]
            raise AssertionError(f"{what}: {int(bad.sum())} of {bins.size} windows outside the band: windows {i.tolist()}, bins "
                                 f"{bins[i].tolist()}, argmax {self.P[i].argmax(axis=1).tolist()}")
        return int(np.sum((self.P + self.tauP >= lo[:, None]).sum(axis=1) > 1))


def rayleigh(rng, shape):
    """Independent complex-Gaussian gains of mean power 1."""
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)) / np.sqrt(2.0)


def sigma_for(snr_125k_db, fs):
    """The noise_sigma of tx_frames / tx_expand for an SNR in 125 kHz (unit-amplitude frames)."""
    return float(np.sqrt(10 ** (-(snr_125k_db - 10 * np.log10(fs / BW)) / 10) / 2))


def synth_antennas(torch, sf, osr, pays, n_items, snr_db, gains, seed, *, rr=False, cr=4, sfo_ppm=0.0, cfo=None):
    """Device capture of len(pays) receivers x M antennas: each receiver's frames (tx_frames, no noise) times gains[g, a]
    (one complex gain per frame and antenna: one frame per receiver) into rows g * M + a, then independent noise on every
    row (tx_expand with k = n_rows).  Returns ([n_rows, n_items] complex64 tensor, placed)."""
    fs = osr * BW
    rng = np.random.default_rng(seed)
    gen = G.decoder(fs, BW, sf, False, cr, True, rr, quiet=True)
    up = torch.from_numpy(tx.base_upchirp(sf, BW, fs).astype(np.complex64)).cuda()
    if cfo is None:
        cfo = [[float(rng.uniform(-0.9, 0.9) * BW / 4) for _ in p] for p in pays]
    clean, placed = gen.synth_streams(pays, n_items, lead_symbols=float(rng.uniform(1.0, 3.0)), gap_symbols=float(rng.uniform(3.0, 5.0)),
                                      cfo_hz=cfo, noise_sigma=0.0, seed=seed, up_table_dev=up, sfo_ppm=sfo_ppm)
    g = torch.from_numpy(np.asarray(gains, np.complex64)).cuda()               # [n_receivers, M]
    m = g.shape[1]
    base = (clean[:, None, :] * g[:, :, None]).reshape(-1, n_items).contiguous()
    if snr_db is None:
        out = base
    else:
        out = torch.empty_like(base)
        gen.tx_expand(base, base.shape[0], n_items, base.shape[0], out, sigma_for(snr_db, fs), seed + 1,
                      torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    gen.close()
    return out, placed
