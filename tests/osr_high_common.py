"""Shared helpers of the fs/bw = 16 and 32 tests (no torch): the K1 configuration at those rates, the host emulation of the
kernels and of the receiver at any oversampling, and the shared-memory replay of k1_fft_kernel<SF, D>."""
from __future__ import annotations

import ctypes as C

import numpy as np

from antenna_common import BW, CAP, _RX_ARGS, tables
from osr2_common import emul

RATES = (16, 32)
SENSITIVITY = {7: -2.0, 8: -5.0, 9: -7.5, 10: -10.0, 11: -12.5, 12: -15.0}


def sub_bins(sf, osr):
    """NP: bins per sub-problem, min(N, 2048, 8192 / D)."""
    return min(1 << sf, 2048, 8192 // osr)


def split(sf, osr):
    """S: sub-problems per symbol."""
    return (1 << sf) // sub_bins(sf, osr)


def batch(sf, osr):
    """G: symbols per CTA batch, 8192 / (D NP)."""
    return 8192 // (osr * sub_bins(sf, osr))


def k1_emulate(x, sf, osr, chirp=None):
    """lb_k1_emulate_osr: k1_fft_kernel<SF, D> on the host, dechirping with the down-chirp (or `chirp`)."""
    x = np.ascontiguousarray(x, np.complex64)
    down, _, tw = tables(sf, osr)
    chirp = down if chirp is None else np.ascontiguousarray(chirp, np.complex64)
    n = x.size // (osr << sf)
    bins = np.zeros(n, np.uint32)
    mags = np.zeros(n, np.float32)
    assert emul().lb_k1_emulate_osr(sf, osr, x.ctypes.data, n, chirp.ctypes.data, tw.ctypes.data, bins.ctypes.data, mags.ctypes.data) == 0
    return bins, mags


def llr_emulate(x, sf, osr, reduced):
    """lb_k1_llr_emulate_osr: k1_llr_kernel<SF, D> on the host -> (llrs [n, ppm], bins)."""
    x = np.ascontiguousarray(x, np.complex64)
    down, _, tw = tables(sf, osr)
    n = x.size // (osr << sf)
    llr = np.zeros((n, sf - 2 if reduced else sf), np.float32)
    bins = np.zeros(n, np.uint32)
    assert emul().lb_k1_llr_emulate_osr(sf, osr, x.ctypes.data, n, down.ctypes.data, tw.ctypes.data, int(reduced), llr.ctypes.data,
                                        bins.ctypes.data) == 0
    return llr, bins


def _lib():
    L = emul()
    if not hasattr(L, "_osr_high"):
        f = L.lb_emul_rx_receive_toa
        f.restype = C.c_uint32
        f.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, *_RX_ARGS[:12], C.c_float, *_RX_ARGS[12:],
                      C.c_void_p, C.c_uint32]
        L.lb_k1_smem_replay.restype = C.c_long
        L.lb_k1_smem_replay.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_long]
        L._osr_high = True
    return L


def receive(X, sf, osr, *, max_cfo_bins=0.0, cr=4, rr=None, soft=False, sfo_ppm=0.0, carrier_hz=0.0, sync_word=0x12):
    """lb_emul_rx_receive_toa over one receiver (X [n] or [M, n]): max_cfo_bins > 0 searches |CFO| up to it (wide_cfo), else
    |CFO| <= N/4.  A dict per synchronised frame: start, cfo (bins), snr, status, sfo, payload, toa."""
    X = np.ascontiguousarray(X, np.complex64)
    rows = X if X.ndim == 2 else X[None]
    rr = sf > 10 if rr is None else rr
    down, up, tw = tables(sf, osr)
    start = np.zeros(CAP, np.int64)
    cfo = np.zeros(CAP, np.float32)
    snr = np.zeros(CAP, np.float32)
    status = np.zeros(CAP, np.int32)
    sfo = np.zeros(CAP, np.float32)
    pay = np.zeros((CAP, 256), np.uint8)
    ln = np.zeros(CAP, np.uint32)
    toa = np.zeros(CAP, np.float64)
    n = _lib().lb_emul_rx_receive_toa(rows.ctypes.data, rows.shape[1], rows.shape[0], down.ctypes.data, up.ctypes.data, tw.ctypes.data,
                                      sf, osr, cr, 0, 1, int(rr), sync_word, 0, 0, float(sfo_ppm), float(carrier_hz), int(soft),
                                      float(max_cfo_bins), start.ctypes.data, cfo.ctypes.data, snr.ctypes.data, status.ctypes.data,
                                      sfo.ctypes.data, pay.ctypes.data, ln.ctypes.data, toa.ctypes.data, CAP)
    return [dict(start=int(start[k]), cfo=float(cfo[k]), snr=float(snr[k]), status=int(status[k]), sfo=float(sfo[k]),
                 payload=bytes(pay[k, : ln[k]]), toa=float(toa[k])) for k in range(n)]


PHASES = ("pass0", "pass1", "pass2", "combine")


def smem_replay(sf, osr):
    """lb_k1_smem_replay: for each phase of k1_fft_kernel<SF, D>, the float2 index every thread touches at every shared-memory
    instruction of one batch -> {phase: [n_instructions, 256] int64, -1 where the thread is idle}."""
    L = _lib()
    n = L.lb_k1_smem_replay(sf, osr, None, None, 0)
    assert n > 0, (sf, osr)
    idx = np.zeros(n, np.int32)
    ph = np.zeros(n // 256, np.int32)
    assert L.lb_k1_smem_replay(sf, osr, idx.ctypes.data, ph.ctypes.data, n) == n
    idx = idx.reshape(-1, 256)
    return {name: idx[ph == k].astype(np.int64) for k, name in enumerate(PHASES) if np.any(ph == k)}


def bank_multiplicity(acc):
    """Worst bank multiplicity of [n_instructions, 256] float2 indices: per instruction and half-warp (16 lanes, 128 B: a
    float2 spans the bank pair 2 (i mod 16), 2 (i mod 16) + 1), the largest number of distinct indices with one i mod 16."""
    worst = 1
    for row in acc:
        for h in range(0, 256, 16):
            i = np.unique(row[h: h + 16])
            i = i[i >= 0]
            if i.size:
                worst = max(worst, int(np.bincount(i % 16).max()))
    return worst
