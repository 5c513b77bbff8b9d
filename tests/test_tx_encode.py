"""CPU: the device frame encoder (gr_lora_b200/csrc/tx_encode.cuh) run on the host through build/host_emul.so, and the host-only
lora_b200_tx_frame_symbols, against the host encoder gr_lora_b200/tx.py::encode_frame on every SF x CR x header mode x CRC x
reduced-rate combination."""
import ctypes as C

import numpy as np
import pytest

import gr_lora_b200 as G
from gr_lora_b200 import _native as N
from gr_lora_b200 import build as B
from gr_lora_b200 import tx
from gr_lora_b200.decoder import decoder


@pytest.fixture(scope="module")
def emul():
    L = C.CDLL(str(B.build_host_emul()))
    L.lb_emul_tx_encode.restype = C.c_uint32
    L.lb_emul_tx_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_uint32]
    L.lb_emul_header_checksum.restype = C.c_uint32
    L.lb_emul_header_checksum.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
    return L


def max_len(crc):
    return 255 + 2 * int(crc)


def min_len(implicit, crc):
    return 2 if (crc and not implicit) else 0


def sweep_lengths(implicit, crc, rng):
    """Every length up to 20 (from the smallest allowed), then a random sweep to the maximum."""
    lo, hi = min_len(implicit, crc), max_len(crc)
    return list(range(lo, 21)) + sorted(set(rng.integers(21, hi, 6).tolist())) + [hi]


def cases(sf, cr, implicit, crc, rr):
    """(length, payload) pairs: random payloads on the sweep, all-0x00 and all-0xFF at the smallest, a middle and the largest."""
    rng = np.random.default_rng(1000 * sf + 100 * cr + 8 * implicit + 4 * crc + 2 * rr)
    out = [(n, bytes(rng.integers(0, 256, n, dtype=np.uint8))) for n in sweep_lengths(implicit, crc, rng)]
    for n in (min_len(implicit, crc), 37, max_len(crc)):
        out += [(n, bytes(n)), (n, b"\xff" * n)]
    return out


def emul_encode(L, payload, sf, cr, implicit, crc, rr, cap=4096):
    buf = np.frombuffer(payload, np.uint8).copy() if payload else np.zeros(1, np.uint8)
    out = np.full(cap, 0xFFFFFFFF, np.uint32)
    n = L.lb_emul_tx_encode(buf.ctypes.data, len(payload), sf, cr, int(implicit), int(crc), int(rr), out.ctypes.data, cap)
    return out[:n].tolist()


CONFIGS = [(implicit, crc, rr) for implicit in (False, True) for crc in (False, True) for rr in (False, True)]


@pytest.mark.parametrize("cr", [1, 2, 3, 4])
@pytest.mark.parametrize("sf", range(7, 13))
def test_encoder_equals_host_encoder(emul, sf, cr):
    for implicit, crc, rr in CONFIGS:
        for n, p in cases(sf, cr, implicit, crc, rr):
            want = tx.encode_frame(p, sf, cr, explicit=not implicit, has_crc=crc, reduced_rate=rr).shifts
            got = emul_encode(emul, p, sf, cr, implicit, crc, rr)
            assert got == want, (sf, cr, implicit, crc, rr, n, p.hex())


@pytest.mark.parametrize("cr", [1, 2, 3, 4])
@pytest.mark.parametrize("sf", range(7, 13))
def test_frame_symbols_equal_host_encoder(emul, sf, cr):
    out = np.zeros(4096, np.uint32)
    scratch = np.zeros(1, np.uint8)
    for implicit, crc, rr in CONFIGS:
        for n, p in cases(sf, cr, implicit, crc, rr):
            want = len(tx.encode_frame(p, sf, cr, explicit=not implicit, has_crc=crc, reduced_rate=rr).shifts)
            assert G.tx_frame_symbols(n, sf, cr, implicit, crc, rr) == want, (sf, cr, implicit, crc, rr, n)
        # out of range: refused before the payload is read
        for n in list(range(max_len(crc) + 1, max_len(crc) + 4)) + [1000, 2 ** 32 - 1] + list(range(min_len(implicit, crc))):
            assert G.tx_frame_symbols(n, sf, cr, implicit, crc, rr) == 0, (sf, cr, implicit, crc, rr, n)
            assert emul.lb_emul_tx_encode(scratch.ctypes.data, n, sf, cr, int(implicit), int(crc), int(rr), out.ctypes.data, out.size) == 0


def test_unsupported_configurations_have_no_frame_length():
    for sf, cr in ((6, 4), (13, 4), (7, 0), (7, 5), (12, 7)):
        assert G.tx_frame_symbols(10, sf, cr, False, True, False) == 0, (sf, cr)
    assert N.lib().lora_b200_tx_frame_symbols(None, 10) == 0


def test_header_checksum_equals_host(emul):
    for length in range(256):
        for cr in range(8):
            for crc in (0, 1):
                assert emul.lb_emul_header_checksum(length, cr, crc) == tx.header_checksum(length, cr, crc), (length, cr, crc)
    # the README golden 04 90 40: length 4, CR 4/8, CRC on
    assert tx.header_bytes(4, 4, 1).hex() == "049040"


def test_readme_golden_frame(emul):
    """The frame the reference's README decodes (04 90 40 | de ad be ef 70 0d) at SF7 CR4/8 with CRC."""
    p = bytes.fromhex("deadbeef700d")
    got = emul_encode(emul, p, 7, 4, False, True, False)
    assert got == tx.encode_frame(p, 7, 4).shifts and len(got) == G.tx_frame_symbols(6, 7, 4, False, True, False)


def test_tx_frame_layout_matches_header():
    assert C.sizeof(N.TxFrame) == 24
    assert (N.TxFrame.start.offset, N.TxFrame.stream.offset, N.TxFrame.n_symbols.offset, N.TxFrame.cfo_hz.offset,
            N.TxFrame.sync_word.offset, N.TxFrame.pad.offset) == (0, 8, 12, 16, 20, 21)
    dt = decoder.TX_FRAME_DTYPE
    assert dt.itemsize == 24
    assert [dt.fields[k][1] for k in ("start", "stream", "n_symbols", "cfo_hz", "sync_word", "pad")] == [0, 8, 12, 16, 20, 21]
