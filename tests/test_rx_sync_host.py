"""CPU: the dechirp-synchronised receive path (csrc/rx_sync.cuh) through its host emulation -- the screen (K1's CPU
emulation), preamble detection, synchronisation and the integer chain, the same __host__ __device__ functions the kernels of
lora_b200_receive run."""
import ctypes as C

import numpy as np
import pytest

import gr_lora_b200 as G
from gr_lora_b200 import build, tx

CAP = 16


@pytest.fixture(scope="module")
def emul():
    L = C.CDLL(str(build.build_host_emul()))
    f = L.lb_emul_rx_receive
    f.restype = C.c_uint32
    f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int,
                  C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_uint32]
    return f


_TABLES = {}


def tables(sf):
    if sf not in _TABLES:
        t = G.split_tables(G.tables_build_host(sf=sf), 8 << sf)
        _TABLES[sf] = tuple(np.ascontiguousarray(t[k]) for k in ("downchirp", "upchirp", "twiddles"))
    return _TABLES[sf]


def receive(emul, x, sf, cr=4, implicit=False, crc=True, rr=False, sync_word=0x12, implicit_len=0, min_preamble=0):
    x = np.ascontiguousarray(x, np.complex64)
    down, up, tw = tables(sf)
    start = np.zeros(CAP, np.int64)
    cfo = np.zeros(CAP, np.float32)
    snr = np.zeros(CAP, np.float32)
    status = np.zeros(CAP, np.int32)
    pay = np.zeros((CAP, 256), np.uint8)
    ln = np.zeros(CAP, np.uint32)
    n = emul(x.ctypes.data, x.size, down.ctypes.data, up.ctypes.data, tw.ctypes.data, sf, cr, int(implicit), int(crc), int(rr),
             sync_word, implicit_len, min_preamble, start.ctypes.data, cfo.ctypes.data, snr.ctypes.data, status.ctypes.data,
             pay.ctypes.data, ln.ctypes.data, CAP)
    return [dict(start=int(start[k]), cfo=float(cfo[k]), snr=float(snr[k]), status=int(status[k]),
                 payload=bytes(pay[k, : ln[k]])) for k in range(n)]


def one_frame(sf, payload, cfo_bins, offset, snr_db=None, seed=0, cr=4, rr=None, sync_word=0x12):
    """One frame at sample `lead + offset` of a row, CFO in bins; SNR in the 125 kHz band (None: no noise)."""
    rr = sf > 10 if rr is None else rr
    sps = 8 << sf
    e = tx.encode_frame(payload, sf, cr, reduced_rate=rr)
    f = tx.modulate_frame(e, sf, sync_word=sync_word)
    lead = 2 * sps + offset
    x = np.zeros(lead + f.size + 3 * sps, np.complex128)
    x[lead: lead + f.size] = f
    x *= np.exp(2j * np.pi * cfo_bins * np.arange(x.size) / sps)
    if snr_db is not None:
        x += tx.awgn(x.size, snr_db - 10 * np.log10(8), np.random.default_rng(seed))
    return x.astype(np.complex64), lead


@pytest.mark.parametrize("sf", range(7, 13))
def test_estimator_recovers_cfo_and_timing(emul, sf):
    """Clean frames: integer + fractional CFO within 1/8 bin and the start within one sample, for CFOs of 0, +-0.37, +-5.5 and
    +-0.9 N/4 bins and start offsets across the whole symbol."""
    N, sps = 1 << sf, 8 << sf
    rng = np.random.default_rng(sf)
    cfos = [0.0, 0.37, -0.37, 5.5, -5.5, 0.9 * N / 4, -0.9 * N / 4]
    offsets = [0, 1, 3, 7, sps // 2 + 5, sps - 1] + rng.integers(0, sps, 2).tolist()
    if sf >= 11:                                     # (the CPU emulation of K1 at SF11/12 is slow)
        offsets = offsets[::3]
    pay = b"\x01\x02\x03\x04"
    for k, cfo in enumerate(cfos):
        off = offsets[k % len(offsets)] if sf >= 11 else None
        for o in ([off] if off is not None else offsets):
            x, start = one_frame(sf, pay + b"\x00\x00", cfo, o)
            got = receive(emul, x, sf, rr=sf > 10)
            assert len(got) == 1, (cfo, o, got)
            g = got[0]
            assert abs(g["cfo"] - cfo) <= 1 / 8, (cfo, o, g)
            assert abs(g["start"] - start) <= 1, (cfo, o, g, start)
            assert g["status"] == 0 and g["payload"] == pay + b"\x00\x00", (cfo, o, g)


@pytest.mark.parametrize("sf", [7, 8])
def test_pipeline_decodes_below_the_noise_floor(emul, sf):
    """A few frames at 0 dB SNR in 125 kHz, random CFO within +-BW/4 and random start: decoded to the transmitted bytes."""
    N, sps = 1 << sf, 8 << sf
    rng = np.random.default_rng(100 + sf)
    ok = 0
    for k in range(4):
        pay = bytes(rng.integers(0, 256, 8, dtype=np.uint8))
        cfo = float(rng.uniform(-0.9, 0.9) * N / 4)
        x, start = one_frame(sf, pay, cfo, int(rng.integers(0, sps)), snr_db=0.0, seed=k)
        got = [g for g in receive(emul, x, sf) if g["status"] == 0]
        ok += len(got) == 1 and got[0]["payload"] == pay
    assert ok == 4


def test_pure_noise_yields_no_frame(emul):
    for sf in (7, 8):
        rng = np.random.default_rng(sf)
        x = (rng.standard_normal(300 * (8 << sf)) + 1j * rng.standard_normal(300 * (8 << sf))).astype(np.complex64)
        assert [g for g in receive(emul, x, sf) if g["status"] == 0] == []


def test_other_sync_word_is_rejected(emul):
    x, _ = one_frame(7, b"abcdef", 3.2, 17, sync_word=0x34)
    assert receive(emul, x, 7, sync_word=0x12) == []
    assert [g["payload"] for g in receive(emul, x, 7, sync_word=0x34)] == [b"abcdef"]


def test_implicit_header_uses_the_given_length(emul):
    sf, sps = 8, 8 << 8
    pay = b"implicit!"
    e = tx.encode_frame(pay, sf, 3, explicit=False, has_crc=False)
    f = tx.modulate_frame(e, sf)
    x = np.zeros(3 * sps + f.size + 4 * sps, np.complex64)
    x[3 * sps: 3 * sps + f.size] = f
    got = receive(emul, x, sf, cr=3, implicit=True, crc=False, implicit_len=len(pay))
    assert [g["payload"] for g in got] == [pay]
