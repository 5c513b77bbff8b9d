"""CPU: frames from a transmitter whose clock is off, through the host specification of the modulator (tx.modulate_frame(...,
sfo_ppm)) and the host emulation of the dechirp-synchronised receiver (lb_emul_rx_receive_sfo), which runs the same
__host__ __device__ placement and synchronisation as lora_b200_receive."""
import ctypes as C

import numpy as np
import pytest

import gr_lora_b200 as G
from gr_lora_b200 import build, tx

CAP = 16
CARRIER = 868.1e6
BW, FS = 125e3, 1e6


@pytest.fixture(scope="module")
def emul():
    L = C.CDLL(str(build.build_host_emul()))
    f = L.lb_emul_rx_receive_sfo
    f.restype = C.c_uint32
    f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int,
                  C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    return f


_TABLES = {}


def tables(sf):
    if sf not in _TABLES:
        t = G.split_tables(G.tables_build_host(sf=sf), 8 << sf)
        _TABLES[sf] = tuple(np.ascontiguousarray(t[k]) for k in ("downchirp", "upchirp", "twiddles"))
    return _TABLES[sf]


def receive(emul, x, sf, sfo_ppm=0.0, carrier_hz=0.0, cr=4, rr=False):
    x = np.ascontiguousarray(x, np.complex64)
    down, up, tw = tables(sf)
    start = np.zeros(CAP, np.int64)
    cfo = np.zeros(CAP, np.float32)
    snr = np.zeros(CAP, np.float32)
    status = np.zeros(CAP, np.int32)
    sfo = np.zeros(CAP, np.float32)
    pay = np.zeros((CAP, 256), np.uint8)
    ln = np.zeros(CAP, np.uint32)
    n = emul(x.ctypes.data, x.size, down.ctypes.data, up.ctypes.data, tw.ctypes.data, sf, cr, 0, 1, int(rr), 0x12, 0, 0,
             float(sfo_ppm), float(carrier_hz), start.ctypes.data, cfo.ctypes.data, snr.ctypes.data, status.ctypes.data,
             sfo.ctypes.data, pay.ctypes.data, ln.ctypes.data, CAP)
    return [dict(start=int(start[k]), cfo=float(cfo[k]), status=int(status[k]), sfo=float(sfo[k]), payload=bytes(pay[k, : ln[k]]))
            for k in range(n)]


def drift_chips(sf, n_samples, ppm):
    """Timing error at the end of a frame of n_samples, in chips (decim samples)."""
    return abs(ppm) * 1e-6 * n_samples / 8


def test_zero_offset_is_the_undrifted_frame():
    for sf in (7, 10, 12):
        e = tx.encode_frame(bytes(range(20)), sf, 4, reduced_rate=sf > 10)
        a, b = tx.modulate_frame(e, sf), tx.modulate_frame(e, sf, sfo_ppm=0.0)
        assert a.dtype == b.dtype and np.array_equal(a, b)


@pytest.mark.parametrize("sf,ppm", [(7, 200.0), (7, -200.0), (9, 200.0), (9, -200.0)])
def test_drifted_frame_matches_the_resampled_capture(sf, ppm):
    """The drifted frame equals tests/conftest.py::make_capture's resampling of the undrifted frame (linear interpolation at
    n (1 + delta)) within that interpolation's error at 8x oversampling; samples interpolated across a symbol boundary, where
    the chirp's phase jumps, are left out.  The opposite sign would be off by whole samples and fail: this pins the sign."""
    sps = 8 << sf
    e = tx.encode_frame(bytes(range(12)), sf, 4)
    x = tx.modulate_frame(e, sf)
    got = tx.modulate_frame(e, sf, sfo_ppm=ppm)
    assert got.size == tx.drifted_length(x.size, ppm)
    t = np.arange(int(x.size / (1 + ppm * 1e-6))) * (1 + ppm * 1e-6)
    i0 = np.floor(t).astype(np.int64)
    fr = t - i0
    i1 = np.minimum(i0 + 1, x.size - 1)
    want = x[i0] * (1 - fr) + x[i1] * fr
    n = min(want.size, got.size) - 1
    data0 = 12 * sps + sps // 4
    edge = (i1[:n] % sps == 0) | ((i1[:n] >= data0) & ((i1[:n] - data0) % sps == 0))
    err = np.abs(got[:n] - want[:n])[~edge]
    assert err.max() < 0.025, err.max()
    flipped = tx.modulate_frame(e, sf, sfo_ppm=-ppm)
    m = min(n, flipped.size)
    assert np.abs(flipped[:m] - want[:m])[~edge[:m]].max() > 0.5


def drifted_row(sf, payload, ppm, cfo_hz, offset, rr):
    sps = 8 << sf
    f = tx.modulate_frame(tx.encode_frame(payload, sf, 4, reduced_rate=rr), sf, sfo_ppm=ppm)
    lead = 2 * sps + offset
    x = np.zeros(lead + f.size + 3 * sps, np.complex128)
    x[lead: lead + f.size] = f
    x *= np.exp(2j * np.pi * cfo_hz * np.arange(x.size) / FS)
    return x.astype(np.complex64), lead, f.size


# (sf, ppm, coupled): coupled = a crystal offset on carrier and clock (cfo = ppm * 868.1 Hz, carrier_hz given), else a clock
# offset alone given through sfo_ppm
CASES = ([(sf, p, True) for sf in (7, 8, 9, 10) for p in (20.0, -20.0)] + [(sf, p, False) for sf in (7, 8, 9, 10) for p in (200.0, -200.0)]
         + [(11, 20.0, True), (12, -20.0, True), (11, -20.0, False)])


@pytest.mark.parametrize("sf,ppm,coupled", CASES)
def test_drifted_frames_are_synchronised_and_decoded(emul, sf, ppm, coupled):
    """Clean 64-byte frames from a drifting transmitter: start within one sample, CFO within 1/8 bin, the reported clock offset
    within the CFO tolerance mapped through the carrier, and the payload.  The same frame received with neither parameter
    loses its payload wherever the drift at its end exceeds one chip."""
    rr = sf > 10
    N, sps = 1 << sf, 8 << sf
    bin_hz = BW / N
    rng = np.random.default_rng(sf * 1000 + int(ppm) + 7 * coupled)
    payload = bytes(rng.integers(0, 256, 64, dtype=np.uint8))
    cfo_hz = ppm * CARRIER * 1e-6 if coupled else float(rng.uniform(-0.5, 0.5) * BW / 4)
    x, start, flen = drifted_row(sf, payload, ppm, cfo_hz, int(rng.integers(0, sps)), rr)
    kw = dict(carrier_hz=CARRIER) if coupled else dict(sfo_ppm=ppm)
    got = receive(emul, x, sf, rr=rr, **kw)
    assert len(got) == 1, got
    g = got[0]
    assert abs(g["cfo"] - cfo_hz / bin_hz) <= 1 / 8, (g, cfo_hz / bin_hz)
    assert abs(g["start"] - start) <= 1, (g, start)
    tol = bin_hz / 8 / CARRIER * 1e6 if coupled else 1e-4
    assert abs(g["sfo"] - ppm) <= tol, (g["sfo"], ppm, tol)
    assert g["status"] == 0 and g["payload"] == payload, g
    if drift_chips(sf, flen, ppm) > 1.0:
        plain = receive(emul, x, sf, rr=rr)
        assert not any(p["status"] == 0 and p["payload"] == payload for p in plain), plain


def test_zero_offset_entry_point_matches(emul):
    """lb_emul_rx_receive_sfo with both parameters 0 reports what lb_emul_rx_receive does, and a clock offset of 0."""
    L = C.CDLL(str(build.build_host_emul()))
    f = L.lb_emul_rx_receive
    f.restype = C.c_uint32
    sf, sps = 8, 8 << 8
    x, _, _ = drifted_row(sf, b"0123456789", 0.0, 1234.0, 77, False)
    got = receive(emul, x, sf)
    down, up, tw = tables(sf)
    start, cfo, snr = np.zeros(CAP, np.int64), np.zeros(CAP, np.float32), np.zeros(CAP, np.float32)
    status, pay, ln = np.zeros(CAP, np.int32), np.zeros((CAP, 256), np.uint8), np.zeros(CAP, np.uint32)
    n = f(C.c_void_p(x.ctypes.data), C.c_size_t(x.size), C.c_void_p(down.ctypes.data), C.c_void_p(up.ctypes.data),
          C.c_void_p(tw.ctypes.data), C.c_uint32(sf), C.c_uint32(4), C.c_int(0), C.c_int(1), C.c_int(0), C.c_uint32(0x12),
          C.c_uint32(0), C.c_uint32(0), C.c_void_p(start.ctypes.data), C.c_void_p(cfo.ctypes.data), C.c_void_p(snr.ctypes.data),
          C.c_void_p(status.ctypes.data), C.c_void_p(pay.ctypes.data), C.c_void_p(ln.ctypes.data), C.c_uint32(CAP))
    assert n == len(got) == 1
    assert (got[0]["start"], got[0]["cfo"], got[0]["status"], got[0]["sfo"]) == (int(start[0]), float(cfo[0]), int(status[0]), 0.0)
    assert got[0]["payload"] == bytes(pay[0, : ln[0]]) == b"0123456789"
