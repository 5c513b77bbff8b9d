"""The fine time of arrival of the dechirp receiver (lora_b200_rx_params.fine_toa, rs_toa in csrc/rx_sync.cuh) restated in
float64 from its definition (DESIGN.md section 5), and the host emulation's entry points for it.

A frame with integer start t, CFO F bins and clock offset delta = sfo_ppm 1e-6 is evaluated on the preamble windows j = 1..6
and the SFD windows j = 10, 11, each at pos_j = t + llround(j sps / (1 + delta)) (t + j sps without a clock offset), whose own
rounding r_j = pos_j - t - j sps / (1 + delta) it cancels:
    P_up(nu) = sum_j sum_a |sum_n x_a[pos_j + n] down[n] e^{-2 pi i (F + nu + r_j / D) (pos_j + n) / sps}|^2   (j = 1..6)
    P_dn(nu) = the same over j = 10, 11 with the up-chirp table and F + nu - r_j / D
nu_A = argmax P_up, nu_B = argmax P_dn over |nu| <= W = (D / 2 + 1) / D + 1/4, and toa = t + D (nu_B - nu_A) / 2 + delta sps / 2.
The argmax is taken here by a dense grid and a bounded scalar search, not by the receiver's grid and parabolas."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
from scipy.optimize import minimize_scalar

from antenna_common import CAP, _RX_ARGS, emul, tables
from gr_lora_b200 import tx

BW = 125e3
# |nu_emul - nu_ref| in bins within which the host emulation and the device must hold the definition: the receiver's grid
# and two parabolic refinements against the dense search, plus float32 window sums and frequencies (tests/test_rx_toa_host.py
# and tests/test_gpu_rx_toa.py measure it)
NU_BOUND = 2e-3


SENSITIVITY = {7: -2.0, 8: -5.0, 9: -7.5, 10: -10.0, 11: -12.5, 12: -15.0}
PAY = b"fine toa"


def frame_rows(sf, osr, delay, cfo_bins, gains=(1.0,), *, ppm=0.0, snr_db=None, seed=0, lead_syms=2, payload=PAY):
    """One frame whose first preamble sample arrives at row position truth = lead + delay (delay fractional,
    tx.modulate_frame(delay=)), CFO in bins, the transmitter's clock off by ppm, on len(gains) antennas with their own noise
    at snr_db in 125 kHz for a unit gain.  Returns (X [M, n] complex64, truth)."""
    sps = osr << sf
    f = tx.modulate_frame(tx.encode_frame(payload, sf, 4, reduced_rate=sf > 10), sf, fs=osr * BW, sfo_ppm=ppm, delay=delay)
    lead = lead_syms * sps
    s = np.zeros(lead + f.size + 3 * sps, np.complex128)
    s[lead: lead + f.size] = f
    s *= np.exp(2j * np.pi * cfo_bins * np.arange(s.size) / sps)
    rng = np.random.default_rng(seed)
    X = np.array([g * s for g in gains])
    if snr_db is not None:
        for a in range(len(gains)):
            X[a] += tx.awgn(s.size, snr_db - 10 * np.log10(osr), rng)
    return X.astype(np.complex64), lead + delay


def rms(e):
    return float(np.sqrt(np.mean(np.square(e))))


def toa_bound(osr):
    """|toa - toa_ref| in samples that NU_BOUND on both peaks allows."""
    return osr * NU_BOUND


def half_width(osr):
    return (osr / 2 + 1) / osr + 0.25


def window_pos(start, j, sps, ppm):
    """rs_pos: the row position of TX symbol j and its rounding r_j."""
    if ppm == 0:
        return start + j * sps, 0.0
    rate = 1.0 + 1e-6 * float(np.float32(ppm))
    u = j * sps / rate
    p = start + int(math.floor(abs(u) + 0.5)) * (1 if u >= 0 else -1)     # llround
    return p, (p - start) - u


def reference(X, sf, osr, start, cfo_bins, sfo_ppm=0.0, *, sign=1, rounding=True, sfd=True, antennas=None):
    """(nu_A, nu_B, toa) of one frame on the rows X [M, n] (or one row [n]).  The keywords restate known mistakes, for
    showing that the tests catch them: sign=-1 flips the result, rounding=False drops the r_j correction, sfd=False times
    from the preamble alone (toa = t - D nu_A + delta sps / 2), antennas= a subset of the rows."""
    X = np.atleast_2d(np.asarray(X))
    n_bins, sps = 1 << sf, osr << sf
    down, up, _ = tables(sf, osr)
    rows = range(X.shape[0]) if antennas is None else antennas
    n = np.arange(sps)
    W = half_width(osr)
    delta = 1e-6 * float(np.float32(sfo_ppm))

    def windows(js, table, sgn):
        ys = []
        for j in js:
            p, r = window_pos(start, j, sps, sfo_ppm)
            if p < 0 or p + sps > X.shape[1]:
                continue
            f = float(np.float32(cfo_bins)) + (sgn * r / osr if rounding else 0.0)
            rot = np.exp(-2j * np.pi * f * (p + n) / sps) * table.astype(np.complex128)
            ys += [X[a, p: p + sps].astype(np.complex128) * rot for a in rows]
        return np.array(ys)

    def power(ys, nu):
        return float(np.sum(np.abs(ys @ np.exp(-2j * np.pi * nu * n / sps)) ** 2))

    def peak(ys):
        grid = np.linspace(-W, W, 129)
        e = np.exp(-2j * np.pi * np.outer(n, grid) / sps)
        P = np.sum(np.abs(ys @ e) ** 2, axis=0)
        k = int(np.argmax(P))
        h = grid[1] - grid[0]
        res = minimize_scalar(lambda v: -power(ys, v), bounds=(grid[k] - h, grid[k] + h), method="bounded",
                              options=dict(xatol=1e-7))
        return float(res.x)

    A = windows(range(1, 7), down, +1)
    B = windows((10, 11), up, -1)
    if len(A) == 0 or len(B) == 0:
        return math.nan, math.nan, math.nan
    nu_a, nu_b = peak(A), peak(B)
    eps = osr * (nu_b - nu_a) / 2 if sfd else -osr * nu_a
    return nu_a, nu_b, start + sign * (eps + delta * sps / 2)


def emul_toa(X, sf, osr, starts, cfos, sfos):
    """lb_emul_rs_toa on given frames of the rows X [M, n]: (nu_a, nu_b, toa) arrays."""
    L = emul()
    if not hasattr(L, "_toa"):
        L.lb_emul_rs_toa.restype = C.c_int
        L.lb_emul_rs_toa.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                     C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        f = L.lb_emul_rx_receive_toa
        f.restype = C.c_uint32
        f.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, *_RX_ARGS[:12], C.c_float, *_RX_ARGS[12:],
                      C.c_void_p, C.c_uint32]
        L._toa = True
    X = np.ascontiguousarray(np.atleast_2d(X), np.complex64)
    down, up, tw = tables(sf, osr)
    s = np.ascontiguousarray(starts, np.int64)
    c = np.ascontiguousarray(cfos, np.float32)
    q = np.ascontiguousarray(sfos, np.float32)
    nu_a, nu_b, toa = np.zeros(s.size, np.float32), np.zeros(s.size, np.float32), np.zeros(s.size, np.float64)
    assert L.lb_emul_rs_toa(X.ctypes.data, X.shape[1], X.shape[0], down.ctypes.data, up.ctypes.data, tw.ctypes.data, sf, osr, s.size,
                            s.ctypes.data, c.ctypes.data, q.ctypes.data, nu_a.ctypes.data, nu_b.ctypes.data, toa.ctypes.data) == 0
    return nu_a, nu_b, toa


def receive_toa(X, sf, osr, *, cr=4, rr=None, soft=False, sfo_ppm=0.0, carrier_hz=0.0, max_cfo_bins=0.0, sync_word=0x12):
    """lb_emul_rx_receive_toa over one receiver X [n] or [M, n]: a dict per synchronised frame, as
    antenna_common.receive_emul, with its toa."""
    emul_toa(np.zeros((1, 1), np.complex64), sf, osr, [], [], [])      # (binds the entry points)
    L = emul()
    X = np.ascontiguousarray(np.atleast_2d(X), np.complex64)
    rr = sf > 10 if rr is None else rr
    down, up, tw = tables(sf, osr)
    start, cfo, snr = np.zeros(CAP, np.int64), np.zeros(CAP, np.float32), np.zeros(CAP, np.float32)
    status, sfo, toa = np.zeros(CAP, np.int32), np.zeros(CAP, np.float32), np.zeros(CAP, np.float64)
    pay, ln = np.zeros((CAP, 256), np.uint8), np.zeros(CAP, np.uint32)
    n = L.lb_emul_rx_receive_toa(X.ctypes.data, X.shape[1], X.shape[0], down.ctypes.data, up.ctypes.data, tw.ctypes.data, sf, osr, cr, 0, 1,
                                 int(rr), sync_word, 0, 0, float(sfo_ppm), float(carrier_hz), int(soft), float(max_cfo_bins),
                                 start.ctypes.data, cfo.ctypes.data, snr.ctypes.data, status.ctypes.data, sfo.ctypes.data,
                                 pay.ctypes.data, ln.ctypes.data, toa.ctypes.data, CAP)
    return [dict(start=int(start[k]), cfo=float(cfo[k]), snr=float(snr[k]), status=int(status[k]), sfo=float(sfo[k]),
                 payload=bytes(pay[k, : ln[k]]), toa=float(toa[k])) for k in range(n)]
