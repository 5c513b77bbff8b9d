"""CPU: soft-decision decoding of the dechirp-synchronised receiver through the host emulation -- the LLR demodulator
(csrc/k1_llr.cuh) against a float64 spectrum, the soft block decoder (csrc/rx_sync.cuh) against a brute-force
maximum-likelihood decoder built from the host encoder (gr_lora_b200/tx.py, whitening.py), and the whole receive path with
soft decisions."""
import ctypes as C
import itertools

import numpy as np
import pytest

import gr_lora_b200 as G
from gr_lora_b200 import build, tx, whitening
from k1_reference import K1Reference

CAP = 16


@pytest.fixture(scope="module")
def L():
    lib = C.CDLL(str(build.build_host_emul()))
    lib.lb_k1_llr_emulate.restype = C.c_int
    lib.lb_k1_llr_emulate.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.lb_emul_soft_header.restype = C.c_uint32
    lib.lb_emul_soft_header.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.lb_emul_soft_block.restype = None
    lib.lb_emul_soft_block.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    f = lib.lb_emul_rx_receive_soft
    f.restype = C.c_uint32
    f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int,
                  C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    return lib


_TABLES = {}


def tables(sf):
    if sf not in _TABLES:
        t = G.split_tables(G.tables_build_host(sf=sf), 8 << sf)
        _TABLES[sf] = tuple(np.ascontiguousarray(t[k]) for k in ("downchirp", "upchirp", "twiddles"))
    return _TABLES[sf]


# ---- the definition in numpy ------------------------------------------------------------------------------------------------
def words_of_bins(sf, reduced):
    """w(k) for every kept bin k: gray((k - 1) mod N), folded to N/4 bins first for reduced-rate symbols."""
    n = 1 << sf
    v = (np.arange(n) - 1) % n
    if reduced:
        v = ((v + 2) >> 2) % (n // 4)
    return v ^ (v >> 1)


def llr64(m64, sf, reduced):
    ppm = sf - 2 if reduced else sf
    w = words_of_bins(sf, reduced)
    out = np.empty((m64.shape[0], ppm))
    for j in range(ppm):
        b = (w >> j) & 1
        out[:, j] = m64[:, b == 0].max(axis=1) - m64[:, b == 1].max(axis=1)
    return out


def symbols(sf, rng, n_clean=3):
    """Clean symbols, symbols at -3 dB (per-sample SNR), a half-bin offset and pure noise."""
    n, sps = 1 << sf, 8 << sf
    vals = rng.integers(0, n, n_clean + 2)
    clean = tx.modulate_shifts(vals[:n_clean], sf).reshape(n_clean, sps)
    noisy = tx.modulate_shifts(vals[n_clean:n_clean + 1], sf).reshape(1, sps)
    noisy = noisy + tx.awgn(sps, -3.0, rng).reshape(1, sps)
    half = tx.modulate_shifts(vals[-1:], sf).reshape(1, sps) * np.exp(1j * np.pi * np.arange(sps) / sps)
    noise = (rng.standard_normal(sps) + 1j * rng.standard_normal(sps)).reshape(1, sps)
    return np.ascontiguousarray(np.concatenate([clean, noisy, half, noise]), np.complex64)


def check_llrs(llr, bins, x, sf, reduced, what):
    """Every LLR within 2 tau of the float64 max-log LLR; its sign that of the reported bin's bits when no second bin lies in
    the (A) band."""
    ref = K1Reference(x, sf)
    want = llr64(ref.m64, sf, reduced)
    mx = ref.m64.max(axis=1)
    tau = ref.tau(mx)[:, None]
    err = np.abs(llr.astype(np.float64) - want)
    assert np.all(err <= 2 * tau), f"{what}: worst |LLR - LLR64| / tau = {np.max(err / tau):.3g}"
    band = np.sum(ref.m64 >= (mx - 2 * ref.tau(mx))[:, None], axis=1)
    w = words_of_bins(sf, reduced)[bins]
    for i in np.flatnonzero(band == 1):
        bits = (w[i] >> np.arange(llr.shape[1])) & 1
        assert np.array_equal(llr[i] < 0, bits == 1), (what, i, llr[i], bits)


@pytest.mark.parametrize("sf", range(7, 13))
@pytest.mark.parametrize("reduced", [0, 1])
def test_llr_emulation_against_float64(L, sf, reduced):
    down, _, tw = tables(sf)
    x = symbols(sf, np.random.default_rng(10 * sf + reduced), n_clean=3 if sf < 11 else 1)
    ppm = sf - 2 if reduced else sf
    llr = np.zeros((x.shape[0], ppm), np.float32)
    bins = np.zeros(x.shape[0], np.uint32)
    assert L.lb_k1_llr_emulate(sf, x.ctypes.data, x.shape[0], down.ctypes.data, tw.ctypes.data, reduced, llr.ctypes.data,
                               bins.ctypes.data) == 0
    check_llrs(llr, bins, x, sf, reduced, f"SF{sf} reduced={reduced}")
    kb = np.zeros(x.shape[0], np.uint32)
    km = np.zeros(x.shape[0], np.float32)
    L.lb_k1_emulate.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.lb_k1_emulate(sf, x.ctypes.data, x.shape[0], down.ctypes.data, tw.ctypes.data, kb.ctypes.data, km.ctypes.data)
    assert np.array_equal(bins, kb)                  # the same phase functions and argmax key as K1


# ---- brute-force maximum-likelihood block decoder ---------------------------------------------------------------------------
def header_cw(s, x, explicit, cr):
    if explicit and x < 5:
        return tx.shuffle_byte(tx.HAMMING84[s] ^ whitening.PRNG_HEADER[x])
    return payload_cw(s, x - (5 if explicit else 0), cr, 8)


def payload_cw(s, p, cr, nbits):
    prng = whitening.payload_sequence(cr)
    return tx.shuffle_byte(tx.HAMMING84[s] ^ (prng[p] if p < len(prng) else 0)) & ((1 << nbits) - 1)


def ml_nibble(llr, n_words, ppm, x, cand):
    metric = [sum((-1 if (cand(s) >> i) & 1 else 1) * llr[i, (x - i) % ppm] for i in range(n_words)) for s in range(16)]
    return int(np.argmax(metric))                    # the first maximum: the lowest nibble on ties


def shifts_of(cws, n_words, ppm, sf, reduced):
    n = 1 << sf
    out = []
    for w in tx.interleave_block(cws, n_words, ppm):
        g = tx.gray_decode(w)
        if reduced:
            g = (4 * g) % n
        out.append((g + 1) % n)
    return out


def brute_header(llr, sf, cr, explicit):
    ppm = sf - 2
    nib = []
    for x in range(ppm if not explicit else 5):
        nib.append(ml_nibble(llr, 8, ppm, x, lambda s: header_cw(s, x, explicit, cr)))
    if explicit:
        cr = min(nib[2] >> 1, 4)
        for x in range(5, ppm):
            nib.append(ml_nibble(llr, 8, ppm, x, lambda s: header_cw(s, x, explicit, cr)))
    return nib, shifts_of([header_cw(s, x, explicit, cr) for x, s in enumerate(nib)], 8, ppm, sf, True), cr


def brute_block(llr, sf, cr, explicit, rr, b):
    ppm, spb = (sf - 2 if rr else sf), cr + 4
    p0 = sf - 2 - (5 if explicit else 0) + b * ppm
    nib = [ml_nibble(llr, spb, ppm, x, lambda s: payload_cw(s, p0 + x, cr, spb)) for x in range(ppm)]
    return nib, shifts_of([payload_cw(s, p0 + x, cr, spb) for x, s in enumerate(nib)], spb, ppm, sf, rr)


def soft_header(L, llr, sf, cr, explicit, crc, rr):
    llr = np.ascontiguousarray(llr, np.float32)
    bins, nib = np.zeros(8, np.uint32), np.zeros(sf - 2, np.uint32)
    fcr = L.lb_emul_soft_header(sf, cr, int(not explicit), int(crc), int(rr), llr.ctypes.data, bins.ctypes.data, nib.ctypes.data)
    return nib.tolist(), bins.tolist(), int(fcr)


def soft_block(L, llr, sf, cr, explicit, crc, rr, b):
    llr = np.ascontiguousarray(llr, np.float32)
    ppm = sf - 2 if rr else sf
    bins, nib = np.zeros(cr + 4, np.uint32), np.zeros(ppm, np.uint32)
    L.lb_emul_soft_block(sf, cr, int(not explicit), int(crc), int(rr), b, llr.ctypes.data, bins.ctypes.data, nib.ctypes.data)
    return nib.tolist(), bins.tolist()


MATRIX = list(itertools.product(range(7, 13), range(1, 5), [True, False], [True, False], [False, True]))


@pytest.mark.parametrize("sf,cr,explicit,crc,rr", MATRIX)
def test_soft_block_decoder_against_brute_force(L, sf, cr, explicit, crc, rr):
    """Random LLRs on a grid of 1/64 (every sum exact in float32 and float64), and integer LLRs in -2..2, whose many exact
    ties must go to the lowest nibble."""
    rng = np.random.default_rng(hash((sf, cr, explicit, crc, rr)) & 0xFFFFFFFF)
    ppm = sf - 2 if rr else sf
    for trial in range(4):
        draw = (lambda n: rng.integers(-128, 129, n) / 64.0) if trial % 2 == 0 else (lambda n: rng.integers(-2, 3, n).astype(float))
        lh = draw(8 * (sf - 2)).reshape(8, sf - 2)
        nib, bins, fcr = soft_header(L, lh, sf, cr, explicit, crc, rr)
        bn, bb, bcr = brute_header(lh, sf, cr, explicit)
        assert (nib, bins, fcr) == (bn, bb, bcr), ("header", trial)
        for b in (0, 3):
            lp = draw((cr + 4) * ppm).reshape(cr + 4, ppm)
            assert soft_block(L, lp, sf, cr, explicit, crc, rr, b) == brute_block(lp, sf, cr, explicit, rr, b), ("block", b, trial)


def rx_words(shifts, sf, reduced):
    n = 1 << sf
    return [int(words_of_bins(sf, reduced)[s % n]) for s in shifts]


def clean_llrs(words, ppm):
    return np.array([[-1.0 if (w >> j) & 1 else 1.0 for j in range(ppm)] for w in words], np.float32)


@pytest.mark.parametrize("sf,cr,explicit,crc,rr", MATRIX)
def test_clean_llrs_give_the_transmitted_shifts(L, sf, cr, explicit, crc, rr):
    rng = np.random.default_rng(sf * 100 + cr)
    pay = bytes(rng.integers(0, 256, int(rng.integers(2, 24)), dtype=np.uint8))
    e = tx.encode_frame(pay, sf, cr, explicit=explicit, has_crc=crc, reduced_rate=rr)
    ppm, spb = (sf - 2 if rr else sf), cr + 4
    _, hb, fcr = soft_header(L, clean_llrs(rx_words(e.shifts[:8], sf, True), sf - 2), sf, cr, explicit, crc, rr)
    assert hb == list(e.shifts[:8]) and fcr == cr
    rest = e.shifts[8:]
    for b in range(len(rest) // spb):
        blk = rest[b * spb:(b + 1) * spb]
        _, bins = soft_block(L, clean_llrs(rx_words(blk, sf, rr), ppm), sf, cr, explicit, crc, rr, b)
        assert bins == list(blk), b


def hard_nibbles(words, n_words, ppm, p0, cr):
    """The hard decoder on one payload block's words: deinterleave, deshuffle, dewhiten, then Hamming(8,4) nearest code
    word (CR 4/7, 4/8) or the data bits (CR 4/5, 4/6) -- int_chain.cuh's decode_byte."""
    prng = whitening.payload_sequence(cr)
    out = []
    for x in range(ppm):
        cw = sum((((words[i] >> ((x - i) % ppm)) & 1) << i) for i in range(n_words))
        v = sum((((cw >> src) & 1) << j) for j, src in enumerate(tx.SHUFFLE_PATTERN)) ^ (prng[p0 + x] if p0 + x < len(prng) else 0)
        if cr >= 3:
            out.append(min(range(16), key=lambda s: (bin(v ^ tx.HAMMING84[s]).count("1"), s)))
        else:
            out.append(((v >> 1) & 1) | (((v >> 2) & 1) << 1) | (((v >> 3) & 1) << 2) | (((v >> 5) & 1) << 3))
    return out


def weak_errors(words, ppm, which, rng, n_bins_mask):
    """LLRs of ±1 from the true words, except symbols `which`, whose words are replaced by wrong ones at weight 0.1."""
    bad = list(words)
    for i in which:
        bad[i] = words[i] ^ (int(rng.integers(1, 1 << ppm)) & n_bins_mask)
    llr = clean_llrs(bad, ppm)
    for i in which:
        llr[i] *= 0.1
    return bad, llr


def test_two_weak_wrong_symbols_in_a_cr48_block_are_corrected(L):
    sf, cr = 7, 4
    rng = np.random.default_rng(3)
    fixed = 0
    for trial in range(20):
        pay = bytes(rng.integers(0, 256, 16, dtype=np.uint8))
        e = tx.encode_frame(pay, sf, cr)
        blk = e.shifts[8:16]
        words = rx_words(blk, sf, False)
        i, j = rng.choice(8, 2, replace=False)
        bad, llr = weak_errors(words, sf, (i, j), rng, (1 << sf) - 1)
        nib, bins = soft_block(L, llr, sf, cr, True, True, False, 0)
        assert bins == list(blk), trial
        p0 = sf - 2 - 5
        true = hard_nibbles(words, 8, sf, p0, cr)
        fixed += hard_nibbles(bad, 8, sf, p0, cr) != true
    assert fixed >= 10                               # hard decoding of the same bins fails in most draws


def test_weak_wrong_symbol_on_a_parity_bit_in_a_cr45_block_is_corrected(L):
    sf, cr = 8, 1
    rng = np.random.default_rng(4)
    for trial in range(12):
        pay = bytes(rng.integers(0, 256, 16, dtype=np.uint8))
        e = tx.encode_frame(pay, sf, cr)
        blk = e.shifts[8:13]
        words = rx_words(blk, sf, False)
        i = int(rng.choice([0, 1, 2]))                # d0, d1, d2: the data bits the one parity bit covers
        bad, llr = weak_errors(words, sf, (i,), rng, (1 << sf) - 1)
        nib, bins = soft_block(L, llr, sf, cr, True, True, False, 0)
        assert bins == list(blk), trial
        p0 = sf - 2 - 5
        assert hard_nibbles(bad, 5, sf, p0, cr) != hard_nibbles(words, 5, sf, p0, cr)


# ---- the whole receive path ---------------------------------------------------------------------------------------------
def receive(L, x, sf, soft, cr=4, rr=False):
    x = np.ascontiguousarray(x, np.complex64)
    down, up, tw = tables(sf)
    start = np.zeros(CAP, np.int64)
    cfo, snr = np.zeros(CAP, np.float32), np.zeros(CAP, np.float32)
    status, ln = np.zeros(CAP, np.int32), np.zeros(CAP, np.uint32)
    pay = np.zeros((CAP, 256), np.uint8)
    n = L.lb_emul_rx_receive_soft(x.ctypes.data, x.size, down.ctypes.data, up.ctypes.data, tw.ctypes.data, sf, cr, 0, 1, int(rr),
                                  0x12, 0, 0, 0.0, 0.0, int(soft), start.ctypes.data, cfo.ctypes.data, snr.ctypes.data,
                                  status.ctypes.data, None, pay.ctypes.data, ln.ctypes.data, CAP)
    return [(int(start[k]), int(status[k]), bytes(pay[k, : ln[k]])) for k in range(n)]


@pytest.mark.parametrize("sf,cr", [(7, 4), (7, 1), (8, 2)])
def test_emulated_soft_receive_equals_hard_at_high_snr(L, sf, cr):
    sps = 8 << sf
    rng = np.random.default_rng(sf + cr)
    for k in range(2):
        pay = bytes(rng.integers(0, 256, 10, dtype=np.uint8))
        f = tx.modulate_frame(tx.encode_frame(pay, sf, cr), sf)
        lead = 2 * sps + int(rng.integers(0, sps))
        x = np.zeros(lead + f.size + 3 * sps, np.complex128)
        x[lead: lead + f.size] = f
        x *= np.exp(2j * np.pi * 2.3 * np.arange(x.size) / sps)
        x += tx.awgn(x.size, 10.0 - 10 * np.log10(8), rng)
        hard, soft = receive(L, x, sf, False, cr), receive(L, x, sf, True, cr)
        assert soft == hard and [g[2] for g in hard if g[1] == 0] == [pay]


def decode(L, sf, cr, implicit, crc, rr, n, bins=None, llr=None, implicit_len=0):
    f = L.lb_emul_rx_decode
    f.restype = C.c_int32
    f.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    out = np.zeros(256, np.uint8)
    bp = None if bins is None else np.ascontiguousarray(bins, np.uint32)
    lp = None if llr is None else np.ascontiguousarray(llr, np.float32)
    k = f(sf, cr, int(implicit), int(crc), int(rr), implicit_len, None if bp is None else bp.ctypes.data,
          None if lp is None else lp.ctypes.data, n, out.ctypes.data)
    return bytes(out[:k]) if k >= 0 else k


@pytest.mark.parametrize("sf,cr,implicit,rr", [(7, 4, False, False), (8, 1, False, False), (11, 3, False, True), (9, 2, True, False)])
def test_frame_decode_entry_from_bins_and_llrs(L, sf, cr, implicit, rr):
    """lb_emul_rx_decode: a frame's transmitted shifts, as bins or as clean LLRs, give back its payload."""
    pay = bytes(range(40, 52))
    e = tx.encode_frame(pay, sf, cr, explicit=not implicit, has_crc=True, reduced_rate=rr)
    n = len(e.shifts)
    ppm = sf - 2 if rr else sf
    llr = np.concatenate([clean_llrs(rx_words(e.shifts[:8], sf, True), sf - 2).ravel(),
                          clean_llrs(rx_words(e.shifts[8:], sf, rr), ppm).ravel()])
    il = len(pay) if implicit else 0
    assert decode(L, sf, cr, implicit, True, rr, n, bins=e.shifts, implicit_len=il) == pay
    assert decode(L, sf, cr, implicit, True, rr, n, llr=llr, implicit_len=il) == pay
