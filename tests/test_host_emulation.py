"""CPU: the kernels' __host__ __device__ phase functions (K1 passes, integer chain) executed on
the host through build/host_emul.so and compared with the oracle.  This is the same source the
GPU compiles (gr_lora_b200/csrc/k1_fft.cuh, int_chain.cuh); only the thread loop is emulated."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest

from conftest import FRAME_CASES, case_decoder_args, make_case_iq, twiddle_table
from gr_lora_b200 import build as B, tx, whitening

GOLD = json.loads((Path(__file__).parent / "golden" / "golden.json").read_text())


@pytest.fixture(scope="module")
def emul():
    L = C.CDLL(str(B.build_host_emul()))
    L.lb_k1_emulate.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.lb_k1_emulate_warp_sf7.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.lb_k1_emulate_group.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.lb_k1_emulate_rows.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.lb_emul_decode.restype = C.c_uint32
    L.lb_emul_decode.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_uint32, C.c_void_p, C.c_uint32]
    L.lb_emul_deinterleave.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    for n in ("lb_emul_reduce_bin",):
        getattr(L, n).restype = C.c_uint32
        getattr(L, n).argtypes = [C.c_uint32, C.c_uint32]
    L.lb_emul_gray.restype = C.c_uint32
    L.lb_emul_gray.argtypes = [C.c_uint32]
    for n in ("lb_emul_hamming84_decode", "lb_emul_hamming84_encode", "lb_emul_deshuffle"):
        getattr(L, n).restype = C.c_uint8
        getattr(L, n).argtypes = [C.c_uint8]
    L.lb_emul_payload_symbols.restype = C.c_int32
    L.lb_emul_payload_symbols.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_int]
    L.lb_emul_atan2f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    L.lb_emul_philox4x32_10.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.lb_emul_rx_replay.restype = C.c_uint32
    L.lb_emul_rx_replay.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int, C.c_uint32, C.c_int, C.c_int,
                                    C.c_void_p, C.c_void_p, C.c_uint32]
    L.lb_emul_rx_frame_rec_size.restype = C.c_uint32
    return L


@pytest.mark.parametrize("sf", range(7, 13))
def test_k1_emulation_matches_oracle(emul, oracle, sf):
    from golden.make_golden import k1_case
    g = GOLD["k1"][str(sf)]
    vals, x = k1_case(sf, g["n"], g["snr_db"], g["seed"])
    d = oracle.Decoder(sf=sf)
    chirp, tw = d.downchirp, twiddle_table(d.sps)
    n = len(vals)
    bins, mags = np.zeros(n, np.uint32), np.zeros(n, np.float32)
    assert emul.lb_k1_emulate(sf, x.ctypes.data, n, chirp.ctypes.data, tw.ctypes.data, bins.ctypes.data, mags.ctypes.data) == 0
    ob, om = d.demod_fft_batch(x)
    assert np.array_equal(bins, ob)
    assert [int(b) for b in bins] == g["fft_bins"]
    np.testing.assert_allclose(mags, om, rtol=1e-5)


@pytest.mark.parametrize("which", ["warp7", "group8", "group9", "group10"])
def test_k1_fast_kernels_emulation_matches_oracle(emul, oracle, which):
    """k1_warp.cuh (SF7, warp per symbol), k1_group.cuh (SF8-9, group per symbol) and k1_sf10.cuh: lane/thread
    functions run on the host; bins must equal the oracle on the fixture, the edge bins and on noise."""
    from golden.make_golden import k1_case
    sf = int(which[-2:]) if which[-2:].isdigit() else int(which[-1])
    g = GOLD["k1"][str(sf)]
    vals, x = k1_case(sf, g["n"], g["snr_db"], g["seed"])
    rng = np.random.default_rng(77)
    d = oracle.Decoder(sf=sf)
    nn = 9 if sf < 10 else 3
    noise = (rng.standard_normal(nn * d.sps) + 1j * rng.standard_normal(nn * d.sps)).astype(np.complex64)
    chirp, tw = d.downchirp, twiddle_table(d.sps)
    for sig in (x, noise):
        n = sig.size // d.sps
        bins, mags = np.zeros(n, np.uint32), np.zeros(n, np.float32)
        if which == "warp7":
            emul.lb_k1_emulate_warp_sf7(sig.ctypes.data, n, chirp.ctypes.data, tw.ctypes.data, bins.ctypes.data, mags.ctypes.data)
        else:
            assert emul.lb_k1_emulate_group(sf, sig.ctypes.data, n, chirp.ctypes.data, tw.ctypes.data, bins.ctypes.data, mags.ctypes.data) == 0
        ob, om = d.demod_fft_batch(sig)
        assert np.array_equal(bins, ob)
        np.testing.assert_allclose(mags, om, rtol=1e-5)
    assert [int(b) for b in ob] != []


def test_k1_emulation_ragged_batch_and_noise_only(emul, oracle):
    """n_symbols not a multiple of the CTA batch (G=8 at SF7); pure noise: bins within +-0 of the oracle
    except where the two fp32 evaluation orders break a near-tie differently."""
    sf = 7
    d = oracle.Decoder(sf=sf)
    rng = np.random.default_rng(5)
    n = 13
    x = (rng.standard_normal(n * d.sps) + 1j * rng.standard_normal(n * d.sps)).astype(np.complex64)
    bins, mags = np.zeros(n, np.uint32), np.zeros(n, np.float32)
    chirp, tw = d.downchirp, twiddle_table(d.sps)      # keep the arrays alive across the call
    emul.lb_k1_emulate(sf, x.ctypes.data, n, chirp.ctypes.data, tw.ctypes.data, bins.ctypes.data, mags.ctypes.data)
    ob, om = d.demod_fft_batch(x)
    np.testing.assert_allclose(mags, om, rtol=1e-4)
    assert np.mean(bins == ob) >= 0.9


def test_integer_chain_matches_oracle(emul, oracle):
    L = oracle.lib()
    for v in range(256):
        assert emul.lb_emul_hamming84_decode(v) == L.lo_hamming84_decode(v)
        assert emul.lb_emul_deshuffle(v) == L.lo_deshuffle_byte(v)
    for v in range(16):
        assert emul.lb_emul_hamming84_encode(v) == L.lo_hamming84_encode(v)
    for b in range(0, 8192):
        assert emul.lb_emul_gray(b) == L.lo_gray(b)
        for nh in (32, 1024):
            assert emul.lb_emul_reduce_bin(b, nh) == L.lo_reduce_bin(b, nh)
    for ln in range(0, 300, 7):
        for cr in range(1, 5):
            for sf in (7, 10, 12):
                for rr in (0, 1):
                    assert emul.lb_emul_payload_symbols(ln, cr, sf, rr) == L.lo_payload_symbols(ln, cr, sf, rr)


def test_deinterleave_and_decode_match_oracle(emul, oracle):
    rng = np.random.default_rng(9)
    for _ in range(200):
        ppm = int(rng.integers(5, 13))
        nw = int(rng.integers(5, 9))
        words = rng.integers(0, 1 << ppm, nw).astype(np.uint32)
        out = np.zeros(16, np.uint8)
        emul.lb_emul_deinterleave(words.ctypes.data, nw, ppm, out.ctypes.data)
        assert np.array_equal(out[:ppm], oracle.deinterleave(words, ppm))
    for _ in range(300):
        n = int(rng.integers(5, 600))
        cr = int(rng.integers(1, 5))
        hdr = bool(rng.integers(0, 2))
        cw = rng.integers(0, 256, n).astype(np.uint8)
        out = np.zeros(1024, np.uint8)
        k = emul.lb_emul_decode(cw.ctypes.data, n, int(hdr), cr, out.ctypes.data, out.size)
        ref, _ = oracle.decode_codewords(cw, hdr, cr)
        assert bytes(out[:k]) == ref


def test_tx_inverts_the_integer_chain(emul):
    """encode_frame -> (deinterleave, decode) returns the payload: the TX really is the inverse."""
    for sf, cr in ((7, 4), (8, 1), (9, 2), (10, 3), (12, 4)):
        payload = bytes(range(17))
        fs = tx.encode_frame(payload, sf, cr, explicit=True, has_crc=False)
        words = np.array(fs.words, np.uint32)
        cws = []
        out = np.zeros(16, np.uint8)
        emul.lb_emul_deinterleave(words[:8].ctypes.data, 8, sf - 2, out.ctypes.data)
        cws += list(out[:sf - 2])
        for b in range((len(words) - 8) // (4 + cr)):
            w = np.ascontiguousarray(words[8 + b * (4 + cr): 8 + (b + 1) * (4 + cr)])
            emul.lb_emul_deinterleave(w.ctypes.data, 4 + cr, sf, out.ctypes.data)
            cws += list(out[:sf])
        cws = np.array(cws, np.uint8)
        dec = np.zeros(1024, np.uint8)
        k = emul.lb_emul_decode(cws.ctypes.data, cws.size, 1, 4, dec.ctypes.data, dec.size)
        assert bytes(dec[:3]) == tx.header_bytes(len(payload), cr, 0)
        rest = np.ascontiguousarray(cws[5:])
        k = emul.lb_emul_decode(rest.ctypes.data, rest.size, 0, cr, dec.ctypes.data, dec.size)
        if cr >= 3 or True:
            got = bytes(dec[:len(payload)])
            if cr == 3:      # 7-bit code words: bit 7 is lost on air; single-error decode restores it
                assert got == payload
            else:
                assert got == payload


# lb::RxFrameRec (rx_stream.cuh)
FRAME_REC = np.dtype([("stream", "<u4"), ("seq", "<u4"), ("n_cw", "<u4"), ("cr", "<u4"), ("payload_length", "<u4"), ("snr", "<f4"),
                      ("phdr", "u1", 3), ("n_hdr_print", "u1"), ("hdr_print", "u1", 4), ("cw", "u1", 1024)])


def _hex(v):
    return "".join(f" {int(b):02x}" for b in v)


@pytest.mark.parametrize("case", FRAME_CASES, ids=[c[0] for c in FRAME_CASES])
def test_rx_bookkeeping_replays_the_oracle(emul, oracle, case):
    """The stream kernels' bookkeeping after each step (rx_stream.cuh: DETECT and FIND_SFD verdicts, reduced-rate fold,
    Gray, deinterleave, header parse with the erase of 5, payload countdown, frame record) replayed on the host over the
    oracle's steps (state, metric, bin): every next state is the oracle's, and the frames' header and payload bytes
    (decoded by decode_byte, as K8 does) and printed lines are the oracle's.  The SNR byte is not compared: the steps
    carry no energies."""
    x, _, _ = make_case_iq(case)
    _replay_matches_oracle(emul, oracle, x, case_decoder_args(case))


def test_rx_bookkeeping_clamps_the_header_cr(emul, oracle):
    """A header whose CR field reads 7 (the reference never checks the header checksum): the bookkeeping clamps it to 4
    (:834-835) as the oracle does, and the CR 4/8 payload after it decodes."""
    payload = bytes.fromhex("0badc0ffee0102")
    fs = tx.encode_frame(payload, 8, 4, has_crc=True, header=tx.header_bytes(len(payload) - 2, 7, 1))
    x = tx.channel([tx.modulate_frame(fs, 8)] * 2, sf=8, snr_db=40.0, seed=23)
    frames = _replay_matches_oracle(emul, oracle, x, dict(sf=8, implicit=False, cr=4, crc=True, reduced_rate=False))
    assert [f[16] >> 5 for f in frames] == [4, 4] and [f[18:] for f in frames] == [payload] * 2


def _replay_matches_oracle(emul, oracle, x, args):
    sf, implicit, cr, crc, rr = args["sf"], args["implicit"], args["cr"], args["crc"], args["reduced_rate"]
    d = oracle.Decoder(**args)
    _, steps = d.run(x)
    want = d.frames()
    states = np.ascontiguousarray(steps["state"])
    metrics = np.ascontiguousarray(steps["metric"])
    bins = np.ascontiguousarray(steps["bin"])
    nxt = np.empty(states.size, np.int32)
    recs = np.zeros(4, FRAME_REC)
    assert emul.lb_emul_rx_frame_rec_size() == FRAME_REC.itemsize
    k = emul.lb_emul_rx_replay(states.ctypes.data, metrics.ctypes.data, bins.ctypes.data, states.size, sf, int(implicit), cr,
                               int(crc), int(rr), nxt.ctypes.data, recs.ctypes.data, len(recs))
    after = np.append(states[1:], d.state)
    replayed = nxt >= 0
    assert np.count_nonzero(np.isin(states[replayed], (4, 5))) > 0
    assert np.array_equal(nxt[replayed], after[replayed])
    assert k == len(want) == 2
    text = ""
    for r, f in zip(recs[:k], want):
        cw = np.ascontiguousarray(r["cw"][:r["n_cw"]])
        dec = np.zeros(1024, np.uint8)
        m = emul.lb_emul_decode(cw.ctypes.data, int(r["n_cw"]), 0, int(r["cr"]), dec.ctypes.data, dec.size)
        plen = int(r["payload_length"])
        payload = bytes(dec[:min(m, plen)]) + bytes(max(0, plen - m))      # missing bytes read 0 (oracle D5)
        assert bytes(r["phdr"]) + payload == f[15:]
        text += _hex(r["hdr_print"][:r["n_hdr_print"]]) + _hex(payload)
        text += " (" + "".join(chr(b) for b in payload if 32 <= b <= 126) + ")\n"
    assert d.stdout.endswith(text)
    return want


@pytest.mark.parametrize("sf", [11, 12])
def test_k1_rows_emulation_matches_oracle(emul, oracle, sf):
    """k1_rows.cuh (SF11: one CTA per symbol; SF12: two CTAs, branches 4c..4c+3 each): the rotating slot pool, the in-place
    swizzled passes, the lane-pair and CTA-pair partial sums and the bin-N/2 double evaluation, thread by thread on the
    host; edge bins and noise down to -14 dB."""
    d = oracle.Decoder(sf=sf)
    nb = 1 << sf
    chirp, tw = d.downchirp, twiddle_table(d.sps)
    rng = np.random.default_rng(sf)
    n = 40                                     # more than two turns of the 28 / 26-slot pool
    vals = rng.integers(0, nb, n)
    vals[:6] = [0, 1, nb // 2 - 1, nb // 2, nb // 2 + 1, nb - 1]
    for snr in (None, -3.0, -14.0):
        x = tx.synth_symbols(vals, sf, snr_db=snr, seed=5)
        bins, mags = np.zeros(n, np.uint32), np.zeros(n, np.float32)
        assert emul.lb_k1_emulate_rows(sf, x.ctypes.data, n, chirp.ctypes.data, tw.ctypes.data, bins.ctypes.data, mags.ctypes.data) == 0
        ob, om = d.demod_fft_batch(x)
        assert np.array_equal(bins, ob)
        np.testing.assert_allclose(mags, om, rtol=2e-6)


def test_atan2_of_the_stream_kernels(emul):
    """lb_atan2f (lora_common.cuh), the arg() of the instantaneous-frequency passes: within 2 ulp of the exact value on
    2e6 points over all octants and 60 decades of magnitude (measured maximum 1.8), and C99's results for zeros, infinities and NaN.  (The GPU executes the same source with the same IEEE operations.)"""
    rng = np.random.default_rng(3)
    n = 2_000_000
    mag = np.float32(10.0) ** rng.uniform(-30, 30, n).astype(np.float32)
    x = (rng.standard_normal(n).astype(np.float32) * mag).astype(np.float32)
    y = (rng.standard_normal(n).astype(np.float32) * mag * np.float32(10.0) ** rng.uniform(-3, 3, n).astype(np.float32)).astype(np.float32)
    y[np.isinf(y)] = 1.0
    out = np.empty(n, np.float32)
    emul.lb_emul_atan2f(y.ctypes.data, x.ctypes.data, out.ctypes.data, n)
    exact = np.arctan2(y.astype(np.float64), x.astype(np.float64))
    ulp = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
    err = np.abs(out.astype(np.float64) - exact) / ulp
    assert err.max() < 2.0, err.max()
    assert np.all(np.abs(out) <= np.float32(np.pi))
    sp_y = np.array([0.0, -0.0, 0.0, -0.0, 1.0, -1.0, 0.0, -0.0, np.inf, -np.inf, np.inf, -np.inf, 1.0, 1.0, np.inf, np.nan, 1.0], np.float32)
    sp_x = np.array([0.0, 0.0, -0.0, -0.0, 0.0, 0.0, -1.0, -1.0, np.inf, np.inf, -np.inf, -np.inf, np.inf, -np.inf, 1.0, 1.0, np.nan], np.float32)
    got = np.empty(sp_y.size, np.float32)
    emul.lb_emul_atan2f(sp_y.ctypes.data, sp_x.ctypes.data, got.ctypes.data, sp_y.size)
    want = np.arctan2(sp_y.astype(np.float64), sp_x.astype(np.float64)).astype(np.float32)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.allclose(got[ok], want[ok], rtol=0, atol=2.4e-7) and np.array_equal(np.signbit(got[ok]), np.signbit(want[ok]))


def _philox4x32_10(ctr, key):
    """Philox4x32-10 written from the paper (Salmon, Moraes, Dror, Shaw, SC'11), independent of the product source."""
    c = [int(v) for v in ctr]
    k = [int(v) for v in key]
    for _ in range(10):
        p0 = 0xD2511F53 * c[0]
        p1 = 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k[0]) & 0xFFFFFFFF, p1 & 0xFFFFFFFF, ((p0 >> 32) ^ c[3] ^ k[1]) & 0xFFFFFFFF, p0 & 0xFFFFFFFF]
        k = [(k[0] + 0x9E3779B9) & 0xFFFFFFFF, (k[1] + 0xBB67AE85) & 0xFFFFFFFF]
    return c


def test_philox_of_the_tx_kernels(emul):
    """The noise generator of csrc/tx_channel.cuh is the standard Philox4x32-10: Random123's known answer for the all-zero
    counter and key, and an independent implementation on random counters / keys."""
    def product(ctr, key):
        c = np.array(ctr, np.uint32)
        k = np.array(key, np.uint32)
        o = np.empty(4, np.uint32)
        emul.lb_emul_philox4x32_10(c.ctypes.data, k.ctypes.data, o.ctypes.data)
        return [int(v) for v in o]

    assert product([0, 0, 0, 0], [0, 0]) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    rng = np.random.default_rng(5)
    for _ in range(200):
        ctr = rng.integers(0, 1 << 32, 4, dtype=np.uint64)
        key = rng.integers(0, 1 << 32, 2, dtype=np.uint64)
        assert product(ctr, key) == _philox4x32_10(ctr, key)
    assert product([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2) == _philox4x32_10([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2)
