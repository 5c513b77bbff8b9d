"""Soft-decision decoding on the device: the LLR demodulator (lora_b200_demod_llr_dev) against a float64 spectrum, and
lora_b200_receive with soft decisions against hard decisions -- identical at high SNR, fewer frame errors near sensitivity."""
import ctypes as C

import numpy as np
import pytest

from conftest import FRAME_CASES, make_case_iq
from k1_reference import K1Reference, symbols_per_pass
from test_rx_soft_host import check_llrs, symbols

pytestmark = pytest.mark.gpu

BW, FS = 125000, 1e6
SENSITIVITY = [(7, -2.0), (8, -5.0), (9, -7.5), (10, -10.0), (11, -12.5), (12, -15.0)]


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


@pytest.fixture(scope="module")
def emul():
    from gr_lora_b200 import build
    L = C.CDLL(str(build.build_host_emul()))
    f = L.lb_emul_rx_decode
    f.restype = C.c_int32
    f.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    return f


def make_dec(sf, cr=4, implicit=False, crc=True, rr=False, **kw):
    import gr_lora_b200 as G
    return G.decoder(FS, BW, sf, implicit, cr, crc, rr, quiet=True, demod="fft", **kw)


def sigma_for(snr_125k_db):
    return float(np.sqrt(10 ** (-(snr_125k_db - 10 * np.log10(FS / BW)) / 10) / 2))


def payloads_of(frames):
    out = {}
    for r in frames:
        out.setdefault(int(r["stream"]), []).append(bytes(r["bytes"][15: int(r["len"])]))
    return out


# ---- the LLR demodulator ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sf", range(7, 13))
@pytest.mark.parametrize("reduced", [0, 1])
def test_demod_llr_dev_against_float64(torch, sf, reduced):
    """Batches of clean, -3 dB, half-bin and noise windows around the kernel's symbols per pass: every LLR within 2 tau of
    the float64 max-log LLR, bins equal to demod_fft_dev's outside near ties, two runs bit-identical."""
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    dec = make_dec(sf)
    ppm = sf - 2 if reduced else sf
    per_pass = 2 * n_sms * max(1, 1024 >> sf)          # CTAs of one wave x symbols per CTA batch
    rng = np.random.default_rng(sf * 2 + reduced)
    base = symbols(sf, rng, n_clean=3)
    for n in sorted({1, per_pass - 1, per_pass, per_pass + 1, symbols_per_pass(sf, n_sms) + 1}):
        x = np.ascontiguousarray(np.resize(base, (n, base.shape[1])), np.complex64)
        xd = torch.from_numpy(x).cuda()
        llr = torch.zeros(n * ppm, dtype=torch.float32, device="cuda")
        bins = torch.zeros(n, dtype=torch.int32, device="cuda")
        dec.demod_llr(xd, n, llr, bins, reduced=bool(reduced))
        kb = torch.zeros(n, dtype=torch.int32, device="cuda")
        dec.demod_fft(xd, n, kb)
        llr2 = torch.zeros_like(llr)
        dec.demod_llr(xd, n, llr2, None, reduced=bool(reduced))
        torch.cuda.synchronize()
        L, B = llr.cpu().numpy().reshape(n, ppm), bins.cpu().numpy().astype(np.int64)
        ref = K1Reference(x, sf)
        check_llrs(L, B, x, sf, reduced, f"SF{sf} reduced={reduced} n={n}")
        mx = ref.m64.max(axis=1)
        band = np.sum(ref.m64 >= (mx - 2 * ref.tau(mx))[:, None], axis=1)
        clear = band == 1
        assert np.array_equal(B[clear], kb.cpu().numpy().astype(np.int64)[clear])
        assert torch.equal(llr, llr2)
    dec.close()


def test_demod_llr_dev_needs_the_fft_kernels(torch):
    import gr_lora_b200 as G
    from gr_lora_b200 import _native as N
    dec = G.decoder(500e3, BW, 7, False, 4, True, False, quiet=True)      # fs / bw = 4
    x = torch.zeros(dec.sps * 2, dtype=torch.complex64, device="cuda")
    llr = torch.zeros(14, dtype=torch.float32, device="cuda")
    with pytest.raises(N.LoraB200Error) as e:
        dec.demod_llr(x, 2, llr)
    assert e.value.code == N.EUNSUPPORTED
    dec.close()


# ---- receive(soft=True) -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", FRAME_CASES, ids=[c[0] for c in FRAME_CASES])
def test_high_snr_soft_equals_hard(torch, case):
    """Every FRAME_CASES capture: soft and hard decisions publish byte-identical frame records (all of each record),
    rx_info, consumed and header drops."""
    name, sf, cr, implicit, crc, rr, payload_hex, snr, seed = case
    x, _, payload = make_case_iq(case)
    x = x[: x.size // 2 * 2]
    sw = 0x78 if sf >= 11 else 0x12
    out = []
    for soft in (False, True, False):                 # (the last decoder may reuse the soft one's device memory)
        d = make_dec(sf, cr, implicit, crc, rr, max_items_per_call=x.size)
        c, frames, info = d.receive(x[None, :], sync_word=sw, implicit_len=len(payload) if implicit else 0, soft=soft)
        out.append((c.tobytes(), frames.tobytes(), info.tobytes(), d.header_drops))
        assert len(frames) == 2
        d.close()
    assert out[0] == out[1] == out[2]


def test_soft_flag_is_checked_and_noise_gives_no_frames(torch):
    from gr_lora_b200 import _native as N
    d = make_dec(7, n_streams=4, max_items_per_call=200 * 1024)
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(4, 200 * 1024, dtype=torch.complex64, device="cuda", generator=g)
    _, frames, _ = d.receive(x, n_items=200 * 1024, soft=True)
    assert len(frames) == 0
    with pytest.raises(N.LoraB200Error) as e:
        d.receive(x, n_items=200 * 1024, soft=2)
    assert e.value.code == N.EINVAL
    d.close()


def test_lora_receiver_soft_needs_the_dechirp_receiver():
    import gr_lora_b200 as G
    with pytest.raises(ValueError):
        G.lora_receiver(FS, 868e6, [868e6], BW, 7, False, 4, True, disable_channelization=True, sync="reference", soft=True)


# ---- genie decoding: known timing, no CFO --------------------------------------------------------------------------------
def genie_frames(torch, emul, sf, cr, rr, snr, n_frames, seed, plen=16):
    """n_frames frames of plen random bytes encoded by tx_encode_dev, their data symbols made by tx_symbols_dev at this SNR;
    decoded on the host from demod_fft_dev bins (hard) and from demod_llr_dev LLRs (soft).  Returns the wrong frames of each."""
    hard = soft = 0
    for c in range(0, n_frames, 256):                # (an SF12 chunk of 256 frames is 2 GB of IQ)
        h, s = genie_chunk(torch, emul, sf, cr, rr, snr, min(256, n_frames - c), seed * 1000 + c, plen)
        hard, soft = hard + h, soft + s
    return hard, soft


def genie_chunk(torch, emul, sf, cr, rr, snr, n_frames, seed, plen):
    import gr_lora_b200 as G
    rng = np.random.default_rng(seed)
    pays = rng.integers(0, 256, (n_frames, plen), dtype=np.uint8)
    d = make_dec(sf, cr, False, True, rr)
    ns = G.tx_frame_symbols(plen, sf, cr, False, True, rr)
    shifts = torch.zeros(n_frames * ns, dtype=torch.int32, device="cuda")
    d.tx_encode(torch.from_numpy(pays.ravel()).cuda(), np.arange(n_frames) * plen, np.full(n_frames, plen), shifts, ns)
    x = torch.zeros(n_frames * ns * d.sps, dtype=torch.complex64, device="cuda")
    d.tx_symbols(shifts, x, n_frames * ns, noise_sigma=sigma_for(snr), seed=seed)
    bins = torch.zeros(n_frames * ns, dtype=torch.int32, device="cuda")
    d.demod_fft(x, n_frames * ns, bins)
    ppm = sf - 2 if rr else sf
    xs = x.view(n_frames, ns, d.sps)
    hx = xs[:, :8].contiguous()
    px = xs[:, 8:].contiguous()
    hl = torch.zeros(n_frames * 8 * (sf - 2), dtype=torch.float32, device="cuda")
    pl = torch.zeros(n_frames * (ns - 8) * ppm, dtype=torch.float32, device="cuda")
    d.demod_llr(hx, n_frames * 8, hl, reduced=True)
    d.demod_llr(px, n_frames * (ns - 8), pl, reduced=rr)
    torch.cuda.synchronize()
    B = bins.cpu().numpy().astype(np.uint32).reshape(n_frames, ns)
    HL = hl.cpu().numpy().reshape(n_frames, -1)
    PL = pl.cpu().numpy().reshape(n_frames, -1)
    d.close()
    out = np.zeros(256, np.uint8)
    hard = soft = 0
    for f in range(n_frames):
        want = bytes(pays[f])
        b = np.ascontiguousarray(B[f])
        k = emul(sf, cr, 0, 1, int(rr), 0, b.ctypes.data, None, ns, out.ctypes.data)
        hard += not (k == plen and bytes(out[:k]) == want)
        llr = np.ascontiguousarray(np.concatenate([HL[f], PL[f]]), np.float32)
        k = emul(sf, cr, 0, 1, int(rr), 0, None, llr.ctypes.data, ns, out.ctypes.data)
        soft += not (k == plen and bytes(out[:k]) == want)
    return hard, soft


@pytest.mark.parametrize("sf,cr,rr,snr0", [(7, 4, False, -2.0), (7, 1, False, -2.0), (10, 4, False, -10.0), (12, 4, True, -15.0)])
def test_genie_soft_beats_hard(torch, emul, sf, cr, rr, snr0):
    """Frames of known timing and no CFO: at an SNR where hard decoding loses 10 % to 50 % of 1024 frames (found by stepping
    down 0.5 dB at a time from snr0, a sensitivity point of the synchronised receiver, on 256 frames), soft decoding loses
    strictly fewer.  (tx_symbols' chirps have amplitude sqrt 2: the SNRs printed are those of a unit-amplitude chirp.)"""
    snr = snr0
    for _ in range(40):
        h, _ = genie_frames(torch, emul, sf, cr, rr, snr, 256, seed=int(-snr * 10) + sf)
        if h >= 0.2 * 256:
            break
        snr -= 0.5
    n = 1024
    hard, soft = genie_frames(torch, emul, sf, cr, rr, snr, n, seed=99 + sf + cr)
    print(f"genie SF{sf} CR 4/{4 + cr}{' reduced' if rr else ''} at {snr:+.1f} dB: hard {hard}/{n} frame errors, soft {soft}/{n}")
    assert 0.10 * n <= hard <= 0.50 * n, (snr, hard)
    assert soft < hard


# ---- end to end ---------------------------------------------------------------------------------------------------------------
def synth(torch, sf, pays, n_items, snr_db, seed, rr=False, cr=4):
    from gr_lora_b200 import tx
    rng = np.random.default_rng(seed)
    gen = make_dec(sf, cr, False, True, rr)
    up = torch.from_numpy(tx.base_upchirp(sf).astype(np.complex64)).cuda()
    cfo = [[float(rng.uniform(-0.9, 0.9) * BW / 4) for _ in p] for p in pays]
    out, placed = gen.synth_streams(pays, n_items, lead_symbols=float(rng.uniform(1.0, 3.0)), gap_symbols=float(rng.uniform(3.0, 5.0)),
                                    cfo_hz=cfo, noise_sigma=sigma_for(snr_db), seed=seed, up_table_dev=up)
    torch.cuda.synchronize()
    gen.close()
    return out, placed


def test_end_to_end_near_sensitivity(torch):
    """At the sensitivity points soft decisions still decode >= 90 % of the frames; 2 dB below them soft decodes at least
    hard - 1 per SF and more than hard over the six SFs, and no frame soft decisions publish carries a payload that was not
    sent.  (Hard decisions may publish one: the payload CRC is not checked.)"""
    import gr_lora_b200 as G
    tot = {False: 0, True: 0}
    for sf, snr0 in SENSITIVITY:
        rr, ns, sps = sf >= 11, 48, 8 << sf
        rng = np.random.default_rng(sf)
        pays = [[bytes(rng.integers(0, 256, 10, dtype=np.uint8))] for _ in range(ns)]
        n_items = (int((12 + G.tx_frame_symbols(10, sf, 4, False, True, rr)) * sps + sps // 4 + 9 * sps) // 2) * 2
        for snr, at_point in ((snr0, True), (snr0 - 2.0, False)):
            out, placed = synth(torch, sf, pays, n_items, snr, seed=2000 + sf + int(-snr * 10), rr=rr)
            sent = {(s, p) for s, _, p in placed}
            ok = {}
            for soft in (False, True):
                rx = make_dec(sf, 4, False, True, rr, n_streams=ns, max_items_per_call=n_items)
                _, frames, _ = rx.receive(out, n_items=n_items, soft=soft)
                got = [(int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in frames]
                if soft:
                    assert all(g in sent for g in got), (sf, snr)
                ok[soft] = len(set(got) & sent)
                rx.close()
            print(f"SF{sf} at {snr:+.1f} dB: hard {ok[False]}/{ns}, soft {ok[True]}/{ns}")
            if at_point:
                assert ok[True] >= 0.9 * ns, (sf, snr, ok)
            else:
                assert ok[True] >= ok[False] - 1, (sf, snr, ok)
                tot[False] += ok[False]
                tot[True] += ok[True]
    print(f"2 dB below the sensitivity points, six SFs: hard {tot[False]}, soft {tot[True]}")
    assert tot[True] > tot[False]


def test_config5_soft_against_hard(torch):
    """test_config5_end_to_end's capture (SF10, implicit header, CR 4/5, no CRC, -10 dB): soft FER <= hard FER."""
    from gr_lora_b200 import tx
    sf, ns = 10, 256
    rng = np.random.default_rng(5)
    pays = [[bytes(rng.integers(0, 256, 16, dtype=np.uint8))] for _ in range(ns)]
    gen = make_dec(sf, 1, True, False)
    up = torch.from_numpy(tx.base_upchirp(sf).astype(np.complex64)).cuda()
    cfo = [[float(rng.uniform(-0.9, 0.9) * BW / 4)] for _ in range(ns)]
    n_items = (12 + 40) * (8 << sf)
    out, placed = gen.synth_streams(pays, n_items, lead_symbols=2.3, cfo_hz=cfo, noise_sigma=sigma_for(-10.0), seed=55, up_table_dev=up)
    torch.cuda.synchronize()
    fer = {}
    for soft in (False, True):
        rx = make_dec(sf, 1, True, False, n_streams=ns, max_items_per_call=n_items)
        _, frames, _ = rx.receive(out, n_items=n_items, implicit_len=16, soft=soft)
        got = payloads_of(frames)
        ok = sum(1 for s, _, p in placed if got.get(s, [b""])[0][3:] == p)
        fer[soft] = 1 - ok / ns
        rx.close()
    print(f"config 5 (SF10, implicit, CR 4/5, no CRC, -10 dB): hard FER {fer[False]:.4f}, soft FER {fer[True]:.4f} over {ns} frames")
    assert fer[True] <= fer[False]
