"""CPU: CRC-aided list decoding of the dechirp receiver through the host emulation (lb_emul_rx_crc_list, the procedure of
rs_crc_list_kernel as plain loops) on LLRs built from known code words, and the emulated receiver with crc_list."""
import ctypes as C

import numpy as np
import pytest

from crc_common import BAD, NONE, OK, RECOVERED, crc_emul, receive_crc, with_crc
from antenna_common import receive_emul
from gr_lora_b200 import tx, whitening

SF, CR = 8, 4                                         # explicit header, CRC, CR 4/8: one payload nibble in the header block
HPPM, PPM, SPB = SF - 2, SF, CR + 4


def soft_decode_fns():
    L = crc_emul()
    L.lb_emul_soft_header.restype = C.c_uint32
    L.lb_emul_soft_header.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.lb_emul_soft_block.restype = None
    L.lb_emul_soft_block.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.lb_emul_rx_decode.restype = C.c_int32
    L.lb_emul_rx_decode.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                    C.c_void_p]
    return L


def slot_cw(q, s):
    """Code word of nibble s at slot q: header nibbles 0..4, then payload nibble p = q - 5 (whitened with CR 4/8's table)."""
    if q < 5:
        return tx.shuffle_byte(tx.HAMMING84[s] ^ whitening.PRNG_HEADER[q])
    nbits = 8 if q < HPPM else SPB
    return tx.shuffle_byte(tx.HAMMING84[s] ^ whitening.PRNG_PAYLOAD_CR78[q - 5]) & ((1 << nbits) - 1)


def slot_geom(q):
    """(block, x, n_words, ppm) of slot q; block -1 is the header block."""
    if q < HPPM:
        return -1, q, 8, HPPM
    b, x = divmod(q - HPPM, PPM)
    return b, x, SPB, PPM


def sgn(cw, n):
    return np.array([-1.0 if (cw >> i) & 1 else 1.0 for i in range(n)])


class Frame:
    """A frame's LLRs set slot by slot: every slot clean (+-1 from its true code word) unless made weak."""

    def __init__(self, payload):
        self.body = with_crc(payload, CR)
        e = tx.encode_frame(self.body, SF, CR)
        self.n_payload = len(e.shifts) - 8
        self.nb = self.n_payload // SPB
        hdr = tx.header_bytes(len(payload), CR, 1)
        nib = [hdr[0] >> 4, hdr[0] & 15, hdr[1] >> 4, hdr[1] & 15, hdr[2] >> 4]
        for b in self.body:
            nib += [b & 15, b >> 4]
        self.n_slots = HPPM + self.nb * PPM
        self.true = nib + [0] * (self.n_slots - len(nib))
        self.hllr = np.zeros((8, HPPM), np.float32)
        self.pllr = np.zeros((self.nb * SPB, PPM), np.float32)
        for q in range(self.n_slots):
            self.set(q, sgn(slot_cw(q, self.true[q]), slot_geom(q)[2]))

    def set(self, q, v):
        b, x, n, ppm = slot_geom(q)
        a, r0 = (self.hllr, 0) if b < 0 else (self.pllr, b * SPB)
        for i in range(n):
            a[r0 + i, (x - i) % ppm] = v[i]

    def metrics(self, q):
        b, x, n, ppm = slot_geom(q)
        a, r0 = (self.hllr, 0) if b < 0 else (self.pllr, b * SPB)
        l = np.array([a[r0 + i, (x - i) % ppm] for i in range(n)], np.float64)
        return [float(np.dot(sgn(slot_cw(q, s), n), l)) for s in range(16)]

    def weak(self, q, top, second, scale):
        """Slot q's LLRs a mix of two code words: `top` wins, `second` is the runner-up.  Returns the gap, or None when another
        nibble would come between them."""
        n = slot_geom(q)[2]
        self.set(q, scale * (0.625 * sgn(slot_cw(q, top), n) + 0.375 * sgn(slot_cw(q, second), n)))
        m = self.metrics(q)
        order = sorted(range(16), key=lambda s: (-m[s], s))
        return m[top] - m[second] if order[:2] == [top, second] else None

    def soft_bins(self, L):
        hb = np.zeros(8, np.uint32)
        L.lb_emul_soft_header(SF, CR, 0, 1, 0, np.ascontiguousarray(self.hllr).ctypes.data, hb.ctypes.data, None)
        pb = np.zeros(self.n_payload, np.uint32)
        for b in range(self.nb):
            blk = np.ascontiguousarray(self.pllr[b * SPB:(b + 1) * SPB])
            out = np.zeros(SPB, np.uint32)
            L.lb_emul_soft_block(SF, CR, 0, 1, 0, b, blk.ctypes.data, out.ctypes.data, None)
            pb[b * SPB:(b + 1) * SPB] = out
        return hb, pb

    def list_decode(self, L, K):
        hb, pb = self.soft_bins(L)
        hb2, pb2 = hb.copy(), pb.copy()
        h = np.ascontiguousarray(self.hllr)
        p = np.ascontiguousarray(self.pllr)
        rec = L.lb_emul_rx_crc_list(SF, CR, 0, 1, 0, 0, K, self.n_payload, h.ctypes.data, p.ctypes.data, hb2.ctypes.data, pb2.ctypes.data)
        return rec, (hb, pb), (hb2, pb2)

    def decode(self, L, bins):
        b = np.ascontiguousarray(np.concatenate(bins), np.uint32)
        out = np.zeros(256, np.uint8)
        k = L.lb_emul_rx_decode(SF, CR, 0, 1, 0, 0, b.ctypes.data, None, b.size, out.ctypes.data)
        return bytes(out[:k])


def crc_ok(body):
    return tx.crc_bytes(body[:-2], CR) == body[-2:]


def message_slots(f):
    """The list candidates: the slots of payload[0 .. L-2), the CRC's message (slot 5 sits in the header block)."""
    return np.arange(5, 5 + 2 * (len(f.body) - 4))


def delta(n, p, v):
    """The syndrome change of XORing nibble p of an n-byte payload with v: the CRC of that nibble alone in the message."""
    m = bytearray(n)
    m[p >> 1] = v << (4 * (p & 1))
    return tx.payload_crc(bytes(m))


def wrong_with_runner_up(f, q, rng, scale):
    """Make slot q decode to a wrong nibble whose runner-up is the true one; returns the gap."""
    for s in rng.permutation(16):
        if s != f.true[q]:
            g = f.weak(q, int(s), f.true[q], scale)
            if g is not None:
                return g
    raise AssertionError(q)


def correct_with_runner_up(f, q, u, scale):
    return f.weak(q, f.true[q], u, scale)


@pytest.mark.parametrize("n_wrong,K", [(1, 1), (2, 4), (3, 8), (5, 12)])
def test_weak_wrong_code_words_in_the_list_are_recovered(n_wrong, K):
    L = soft_decode_fns()
    rng = np.random.default_rng(n_wrong * 100 + K)
    for trial in range(6):
        f = Frame(bytes(rng.integers(0, 256, int(rng.integers(8, 40)), dtype=np.uint8)))
        cands = message_slots(f)
        for q in rng.choice(cands, n_wrong, replace=False):
            wrong_with_runner_up(f, int(q), rng, 0.125)
        rec, soft, listed = f.list_decode(L, K)
        assert f.decode(L, soft) != f.body and not crc_ok(f.decode(L, soft)), trial
        assert rec == 1 and f.decode(L, listed) == f.body, trial


def test_error_outside_the_list_stays_bad_and_unchanged():
    L = soft_decode_fns()
    rng = np.random.default_rng(7)
    K = 4
    for trial in range(6):
        f = Frame(bytes(rng.integers(0, 256, 24, dtype=np.uint8)))
        qs = rng.choice(message_slots(f), K + 1, replace=False)
        wrong_with_runner_up(f, int(qs[0]), rng, 0.5)       # the error: a larger gap than ...
        for q in qs[1:]:                                       # ... the K weakest, which are right
            u = next(s for s in rng.permutation(16) if correct_with_runner_up(f, int(q), int(s), 0.125) is not None)
        rec, soft, listed = f.list_decode(L, K)
        assert rec == 0 and all(np.array_equal(a, b) for a, b in zip(soft, listed)), trial
        assert not crc_ok(f.decode(L, soft))


def test_list_ties_go_to_the_lowest_nibble_index():
    """Three weak slots of equal gap, the wrong one last: K = 2 lists the first two (BAD), K = 3 all three (RECOVERED)."""
    L = soft_decode_fns()
    rng = np.random.default_rng(11)
    f = Frame(bytes(rng.integers(0, 256, 20, dtype=np.uint8)))
    gaps = []
    for q in (9, 14):
        gaps.append(next(g for s in range(16) if s != f.true[q] and (g := correct_with_runner_up(f, q, s, 0.125)) is not None))
    for s in range(16):
        if s != f.true[21] and (g := f.weak(21, s, f.true[21], 0.125)) == gaps[0]:
            break
    assert gaps[0] == gaps[1] == g
    assert f.list_decode(L, 2)[0] == 0
    rec, _, listed = f.list_decode(L, 3)
    assert rec == 1 and f.decode(L, listed) == f.body


@pytest.mark.parametrize("scale_a,want_sent", [(0.125, True), (0.5, False), (0.25, False)])
def test_least_cost_subset_wins_and_ties_go_to_the_lowest_subset(scale_a, want_sent):
    """Two subsets that both satisfy the CRC: {A} (A received wrong, the true nibble its runner-up) and {B, C} (both received
    right, runner-ups whose syndrome changes sum to A's).  B and C have gap 0.25 each; A's gap 0.25 makes {A} the cheaper
    (the sent payload), 1.0 makes {B, C} the cheaper (a wrong payload that checks), and 0.5 ties: {B, C}, listed first, is
    the lower subset mask and wins."""
    L = soft_decode_fns()
    rng = np.random.default_rng(5)
    f = Frame(bytes(rng.integers(0, 256, 60, dtype=np.uint8)))
    n = len(f.body) - 2
    slots = [int(q) for q in message_slots(f)]
    table = {delta(n, q - 5, v): (q, v) for q in slots for v in range(1, 15)}
    found = None
    for qa in rng.permutation(slots)[:20]:
        for va in range(1, 15):
            for qb in slots:
                for vb in range(1, 15):
                    hit = table.get(delta(n, qa - 5, va) ^ delta(n, qb - 5, vb))
                    if qb != qa and hit and hit[0] not in (qa, qb):
                        found = (int(qa), va, qb, vb, *hit)
                        break
                if found:
                    break
            if found:
                break
        if found:
            break
    qa, va, qb, vb, qc, vc = found
    assert f.weak(qa, f.true[qa] ^ va, f.true[qa], scale_a) == 2 * scale_a
    assert f.weak(qb, f.true[qb], f.true[qb] ^ vb, 0.125) == 0.25 and f.weak(qc, f.true[qc], f.true[qc] ^ vc, 0.125) == 0.25
    rec, _, listed = f.list_decode(L, 3)
    got = f.decode(L, listed)
    assert rec == 1 and crc_ok(got)
    assert (got == f.body) == want_sent


# ---- the emulated receiver ------------------------------------------------------------------------------------------------
def capture(sf, osr, pays, snr_db, seed, cr=4):
    rng = np.random.default_rng(seed)
    sps, fs = osr << sf, osr * 125e3
    rows = []
    for p in pays:
        f = tx.modulate_frame(tx.encode_frame(p, sf, cr, reduced_rate=sf > 10), sf, fs=fs)
        lead = 2 * sps + int(rng.integers(0, sps))
        x = np.zeros(lead + f.size + 3 * sps, np.complex128)
        x[lead: lead + f.size] = f
        x *= np.exp(2j * np.pi * rng.uniform(-0.9, 0.9) * 125e3 / 4 * np.arange(x.size) / fs)
        x += tx.awgn(x.size, snr_db - 10 * np.log10(osr), rng)
        rows.append(x.astype(np.complex64))
    return rows


@pytest.mark.parametrize("osr", [8, 2])
def test_crc_list_off_is_the_soft_receiver(osr):
    rng = np.random.default_rng(osr)
    pays = [with_crc(bytes(rng.integers(0, 256, 12, dtype=np.uint8)), 1) for _ in range(3)]
    for x in capture(7, osr, pays, -3.0, 10 + osr, cr=1):
        a = receive_crc(x, 7, osr, crc_list=0, cr=1)
        b = receive_emul(x, 7, osr, soft=True, cr=1)
        assert [(e["start"], e["cfo"], e["snr"], e["status"], e["payload"]) for e in a] == \
               [(e["start"], e["cfo"], e["snr"], e["status"], e["payload"]) for e in b]
        assert all(e["crc"] in (OK, BAD) if e["status"] == 0 else e["crc"] == NONE for e in a)


@pytest.mark.parametrize("cr", [1, 4])
def test_emulated_receiver_at_low_snr_publishes_only_sent_payloads_as_ok(cr):
    """SF7 frames with valid CRCs at -5.5 dB: with crc_list = 8 every frame reported OK or RECOVERED carries a payload that
    was sent, OK frames are those of crc_list = 0, and the CRC-correct frames are at least those of soft decisions alone."""
    rng = np.random.default_rng(30 + cr)
    pays = [with_crc(bytes(rng.integers(0, 256, 16, dtype=np.uint8)), cr) for _ in range(16)]
    n = {0: 0, 8: 0}
    recovered = 0
    for x, p in zip(capture(7, 8, pays, -5.5, 40 + cr, cr=cr), pays):
        for K in (0, 8):
            good = [e for e in receive_crc(x, 7, 8, crc_list=K, cr=cr) if e["status"] == 0 and e["crc"] in (OK, RECOVERED)]
            assert all(e["payload"] == p for e in good), K
            n[K] += bool(good)
            recovered += K == 8 and any(e["crc"] == RECOVERED for e in good)
    print(f"SF7 CR 4/{4 + cr} at -5.5 dB, 16 frames: CRC-correct soft {n[0]}, soft + list(8) {n[8]} ({recovered} recovered)")
    assert n[8] >= n[0]
