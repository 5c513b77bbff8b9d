"""CPU: the payload CRC of published frames -- its definition (tx.payload_crc, csrc/lora_crc.h) against an independent
polynomial restatement, the reference's known answer, and every length and coding rate through the oracle's decode chain."""
import ctypes as C

import numpy as np
import pytest

from gr_lora_b200 import build, loraphy, tx, whitening

NONE, OK, BAD = loraphy.CRC_NONE, loraphy.CRC_OK, loraphy.CRC_BAD


@pytest.fixture(scope="module")
def L():
    lib = C.CDLL(str(build.build_host_emul()))
    lib.lb_emul_crc_record_status.restype = C.c_uint32
    lib.lb_emul_crc_record_status.argtypes = [C.c_char_p, C.c_uint32]
    lib.lb_emul_crc16.restype = C.c_uint32
    lib.lb_emul_crc16.argtypes = [C.c_char_p, C.c_uint32]
    return lib


def crc16_polydiv(msg: bytes) -> int:
    """The remainder of M(x) x^16 modulo x^16 + x^12 + x^5 + 1, M's first bit the highest power: a CRC-16 with initial value 0,
    no reflection and no final XOR, as long division on one integer."""
    m = int.from_bytes(msg, "big") << 16 if msg else 0
    poly = 0x11021
    for bit in range(m.bit_length() - 1, 15, -1):
        if m >> bit & 1:
            m ^= poly << (bit - 16)
    return m


def record(body: bytes, length: int, cr: int, has_crc: int) -> bytes:
    """A published blob: loratap (15 zero bytes), the PHY header, the payload bytes as decoded."""
    return bytes(15) + tx.header_bytes(length, cr, has_crc) + body


def test_definition_against_polynomial_division(L):
    rng = np.random.default_rng(1)
    for n in list(range(2, 40)) + [178, 255]:
        for _ in range(3):
            p = bytes(rng.integers(0, 256, n, dtype=np.uint8))
            want = crc16_polydiv(p[:-2]) ^ p[-1] ^ (p[-2] << 8)
            assert tx.payload_crc(p) == want, p.hex()
            assert L.lb_emul_crc16(p[:-2], n - 2) ^ p[-1] ^ (p[-2] << 8) == want


def test_known_answer_of_the_reference_readme(L):
    pay = bytes.fromhex("deadbeef")
    assert tx.payload_crc(pay) == 0xEC80
    assert tx.crc_whitening(4, 4) == 0xE1F0                  # nibbles 8..11 of PRNG_PAYLOAD_CR78: 00 ff d2 2d -> 0, 15, 1, 14
    assert tx.crc_bytes(pay, 4) == bytes.fromhex("700d")
    blob = record(pay + bytes.fromhex("700d"), 4, 4, 1)
    assert loraphy.crc_status(blob) == OK and L.lb_emul_crc_record_status(blob, len(blob)) == OK


def test_golden_frames_statuses(L):
    """The reference's golden frames: every 'de ad be ef 70 0d' frame checks at every coding rate; the others carry arbitrary
    trailing bytes (BAD) or no CRC (NONE)."""
    import json
    from pathlib import Path
    g = json.loads((Path(__file__).parent / "golden" / "golden.json").read_text())["frames"]
    seen_ok = 0
    for name, case in g.items():
        for h in case["frames"]:
            blob = bytes.fromhex(h)
            f = loraphy.parse_frame(blob)
            st = loraphy.crc_status(blob)
            assert L.lb_emul_crc_record_status(blob, len(blob)) == st, name
            if not f.has_mac_crc:
                assert st == NONE, name
            elif f.payload == bytes.fromhex("deadbeef700d"):
                assert st == OK, name
                seen_ok += 1
    assert seen_ok >= 10


def test_table_entry_359_is_not_a_code_word():
    """The CRC's last nibble at L = 178 sits on entry 359 of the CR 4/7-4/8 table, 0xC7: one bit from 0x87, whose data is 3."""
    assert whitening.PRNG_PAYLOAD_CR78[359] == 0xC7
    assert 0xC7 not in tx.HAMMING84 and tx.HAMMING84.index(0x87) == 3
    assert (tx.crc_whitening(178, 4) >> 12) == 3


@pytest.mark.parametrize("cr", [1, 2, 3, 4])
def test_round_trip_every_length_through_the_oracle_chain(L, oracle, cr):
    """payload || crc_bytes through tx.encode_frame and the oracle's integer chain (deinterleaved code words -> bytes): the
    published frame checks at every length 2..255 (L = 178 reaches table entry 359 at CR 3/4)."""
    rng = np.random.default_rng(cr)
    for n in range(2, 256):
        pay = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        e = tx.encode_frame(pay + tx.crc_bytes(pay, cr), 7, cr)
        out, _ = oracle.decode_codewords(e.codewords[5:], False, cr)
        body = out[: n + 2]
        assert body[:n] == pay, n
        blob = record(body, n, cr, 1)
        assert loraphy.crc_status(blob) == OK, (n, cr)
        assert L.lb_emul_crc_record_status(blob, len(blob)) == OK, (n, cr)


@pytest.mark.parametrize("n", [2, 3, 4, 17, 178, 255])
@pytest.mark.parametrize("cr", [1, 4])
def test_every_single_bit_error_is_bad(L, n, cr):
    rng = np.random.default_rng(n * 10 + cr)
    pay = bytes(rng.integers(0, 256, n, dtype=np.uint8))
    body = bytearray(pay + tx.crc_bytes(pay, cr))
    assert loraphy.crc_status(record(bytes(body), n, cr, 1)) == OK
    for bit in range(8 * len(body)):
        b = bytearray(body)
        b[bit >> 3] ^= 1 << (bit & 7)
        blob = record(bytes(b), n, cr, 1)
        assert loraphy.crc_status(blob) == BAD, bit
        assert L.lb_emul_crc_record_status(blob, len(blob)) == BAD, bit


def test_no_crc_or_short_payload_is_none(L):
    for body, has_crc in ((b"\x01\x02", 1), (b"\x01\x02\x03", 1), (bytes.fromhex("deadbeef700d"), 0), (b"", 1)):
        blob = record(body, max(len(body) - 2 * has_crc, 0), 4, has_crc)
        assert loraphy.crc_status(blob) == NONE, body
        assert L.lb_emul_crc_record_status(blob, len(blob)) == NONE, body
