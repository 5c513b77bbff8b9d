"""Shared helpers of the coarse-offset search tests (rx_params.wide_cfo): the host emulation's lb_emul_rx_receive_wide and the
shifted dechirp tables of one hypothesis, restated in numpy."""
from __future__ import annotations

import ctypes as C

import numpy as np

from antenna_common import CAP, _RX_ARGS, emul, tables

BW = 125e3


def _lib():
    L = emul()
    if not hasattr(L, "_wide"):
        f = L.lb_emul_rx_receive_wide
        f.restype = C.c_uint32
        f.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, *_RX_ARGS[:12], C.c_float, *_RX_ARGS[12:],
                      C.c_uint32]
        L._wide = True
    return L


def receive_wide(X, sf, osr, max_cfo_bins, *, cr=4, rr=None, soft=False, sfo_ppm=0.0, carrier_hz=0.0, sync_word=0x12, min_preamble=0):
    """lb_emul_rx_receive_wide over one receiver: X [n] (one antenna) or X [M, n].  A dict per synchronised frame, as
    antenna_common.receive_emul."""
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
    n = _lib().lb_emul_rx_receive_wide(rows.ctypes.data, rows.shape[1], rows.shape[0], down.ctypes.data, up.ctypes.data, tw.ctypes.data,
                                       sf, osr, cr, 0, 1, int(rr), sync_word, 0, min_preamble, float(sfo_ppm), float(carrier_hz), int(soft),
                                       float(max_cfo_bins), start.ctypes.data, cfo.ctypes.data, snr.ctypes.data, status.ctypes.data,
                                       sfo.ctypes.data, pay.ctypes.data, ln.ctypes.data, CAP)
    return [dict(start=int(start[k]), cfo=float(cfo[k]), snr=float(snr[k]), status=int(status[k]), sfo=float(sfo[k]),
                 payload=bytes(pay[k, : ln[k]])) for k in range(n)]


def dedup(frames, sps):
    """lora_b200_receive's rule for one stream's synchronised frames, restated (as test_gpu_rx_sync_parity.dedup): in order of
    start, a frame less than one symbol after the previous one belongs to its group, and a group keeps its best member -- a
    decodable header first, then the higher SNR.  Incomplete frames (status 2) are left out."""
    reps, prev = [], None
    for f in sorted((f for f in frames if f["status"] != 2), key=lambda f: f["start"]):
        if prev is not None and f["start"] - prev["start"] < sps:
            a = reps[-1]
            if (f["status"] == 0) > (a["status"] == 0) or ((f["status"] == 0) == (a["status"] == 0) and f["snr"] > a["snr"]):
                reps[-1] = f
        else:
            reps.append(f)
        prev = f
    return reps


def band_limit_bins(sf, osr):
    """(fs - BW) / 2 in bins: the widest max_cfo_bins wide_cfo takes."""
    return (osr - 1) * (1 << sf) / 2


def shifted_chirp(sf, osr, c, up=False):
    """down_c[n] = down[n] e^{-j pi c n / D} (up_c likewise): the table hypothesis c dechirps with, in float64."""
    down, upc, _ = tables(sf, osr)
    n = np.arange(osr << sf)
    t = (upc if up else down).astype(np.complex128)
    return (t * np.exp(-1j * np.pi * ((c * n) % (2 * osr)) / osr)).astype(np.complex64)
