"""Shared helpers of the payload CRC / list decoding tests: the host emulation's entry points (lb_emul_rx_receive_crc,
lb_emul_rx_crc_list) and frames that carry a valid CRC (tx.crc_bytes)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from antenna_common import CAP, emul, tables
from gr_lora_b200 import tx

NONE, OK, BAD, RECOVERED = 0, 1, 2, 3


def crc_emul():
    L = emul()
    if not hasattr(L, "_crc_ready"):
        f = L.lb_emul_rx_receive_crc
        f.restype = C.c_uint32
        f.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                      C.c_int, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_double, C.c_int, C.c_uint32, C.c_void_p,
                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
        g = L.lb_emul_rx_crc_list
        g.restype = C.c_int
        g.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p,
                      C.c_void_p, C.c_void_p]
        L._crc_ready = True
    return L


def receive_crc(X, sf, osr, *, crc_list=0, soft=True, cr=4, rr=None):
    """One receiver on the host (rows of X [M, n], or one row X [n]) with list decoding: a dict per synchronised frame with its
    status (0 published), payload and CRC status."""
    X = np.ascontiguousarray(X, np.complex64)
    if X.ndim == 1:
        X = X[None, :]
    rr = sf > 10 if rr is None else rr
    down, up, tw = tables(sf, osr)
    start = np.zeros(CAP, np.int64)
    cfo, snr, sfo = np.zeros(CAP, np.float32), np.zeros(CAP, np.float32), np.zeros(CAP, np.float32)
    status = np.zeros(CAP, np.int32)
    pay = np.zeros((CAP, 256), np.uint8)
    ln = np.zeros(CAP, np.uint32)
    crc = np.zeros(CAP, np.uint8)
    n = crc_emul().lb_emul_rx_receive_crc(X.ctypes.data, X.shape[1], X.shape[0], down.ctypes.data, up.ctypes.data, tw.ctypes.data, sf,
                                          osr, cr, 0, 1, int(rr), 0x12, 0, 0, 0.0, 0.0, int(soft), crc_list, start.ctypes.data,
                                          cfo.ctypes.data, snr.ctypes.data, status.ctypes.data, sfo.ctypes.data, pay.ctypes.data,
                                          ln.ctypes.data, crc.ctypes.data, CAP)
    return [dict(start=int(start[k]), cfo=float(cfo[k]), snr=float(snr[k]), status=int(status[k]), payload=bytes(pay[k, : ln[k]]),
                 crc=int(crc[k])) for k in range(n)]


def with_crc(payload: bytes, cr: int) -> bytes:
    """The bytes to hand tx.encode_frame for the frame a radio sends with this payload."""
    return payload + tx.crc_bytes(payload, cr)
