"""The dechirp-synchronised receiver (lora_b200_receive) through the C ABI: sensitivity below the noise floor, parity with
lora_b200_work_batch at high SNR, many streams, chunked captures under the consumed rule, determinism and false alarms."""
import ctypes as C

import numpy as np
import pytest

from conftest import FRAME_CASES, make_capture, make_case_iq

pytestmark = pytest.mark.gpu

BW, FS = 125000, 1e6


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def make_dec(sf, cr=4, implicit=False, crc=True, rr=False, **kw):
    import gr_lora_b200 as G
    return G.decoder(FS, BW, sf, implicit, cr, crc, rr, quiet=True, demod="fft", **kw)


def sigma_for(snr_125k_db):
    """Noise sigma per real component for a unit-amplitude chirp at this SNR in the 125 kHz band (fs = 8 BW)."""
    return float(np.sqrt(10 ** (-(snr_125k_db - 10 * np.log10(FS / BW)) / 10) / 2))


def payloads_of(frames):
    out = {}
    for r in frames:
        out.setdefault(int(r["stream"]), []).append(bytes(r["bytes"][15: int(r["len"])]))
    return out


def synth(torch, sf, pays, n_items, snr_db, seed, rr=False, cr=4, sync_word=0x12, cfo_frac=0.9, lead=None):
    """Streams of frames with a random CFO within +-cfo_frac BW/4 per frame and random starts; unit-amplitude chirps."""
    from gr_lora_b200 import tx
    rng = np.random.default_rng(seed)
    gen = make_dec(sf, cr, False, True, rr)
    up = torch.from_numpy(tx.base_upchirp(sf).astype(np.complex64)).cuda()
    cfo = [[float(rng.uniform(-cfo_frac, cfo_frac) * BW / 4) for _ in p] for p in pays]
    out, placed = gen.synth_streams(pays, n_items, lead_symbols=float(rng.uniform(1.0, 3.0)) if lead is None else lead,
                                    gap_symbols=float(rng.uniform(3.0, 5.0)), cfo_hz=cfo, sync_word=sync_word,
                                    noise_sigma=sigma_for(snr_db), seed=seed, up_table_dev=up)
    torch.cuda.synchronize()
    gen.close()
    return out, placed


def frame_len(sf, plen, cr=4, rr=False):
    import gr_lora_b200 as G
    return (12 + G.tx_frame_symbols(plen, sf, cr, False, True, rr)) * (8 << sf) + (8 << sf) // 4


SENSITIVITY = [(7, -2.0), (8, -5.0), (9, -7.5), (10, -10.0), (11, -12.5), (12, -15.0)]


@pytest.mark.parametrize("sf,snr", SENSITIVITY)
def test_sensitivity_below_the_noise_floor(torch, sf, snr):
    """CR 4/8, explicit header, random CFO within +-BW/4 and random starts: >= 90 % of the frames decode byte-exact at the
    sensitivity point; the reference state machine (work_batch) decodes none of them."""
    rr = sf >= 11
    ns, per = 48, 1
    rng = np.random.default_rng(sf)
    pays = [[bytes(rng.integers(0, 256, 10, dtype=np.uint8)) for _ in range(per)] for _ in range(ns)]
    sps = 8 << sf
    n_items = (int(frame_len(sf, 10, rr=rr) + 9 * sps) // 2) * 2
    out, placed = synth(torch, sf, pays, n_items, snr, seed=1000 + sf, rr=rr)
    assert len(placed) == ns * per
    rx = make_dec(sf, 4, False, True, rr, n_streams=ns, max_items_per_call=n_items)
    _, frames, info = rx.receive(out, n_items=n_items)
    got = payloads_of(frames)
    ok = sum(1 for s, _, p in placed if any(g[3:] == p for g in got.get(s, [])))
    assert ok >= 0.9 * len(placed), (sf, snr, ok, len(placed))
    assert len(frames) <= len(placed) + 0                   # nothing but the placed frames
    ref = make_dec(sf, 4, False, True, rr, n_streams=ns, max_items_per_call=n_items)
    ref.work_batch(out, n_items=n_items, stride_items=n_items, host=0, callbacks=False)
    old = payloads_of(ref.frames_last())
    assert sum(1 for s, _, p in placed if any(g[3:] == p for g in old.get(s, []))) == 0


@pytest.mark.parametrize("case", FRAME_CASES, ids=[c[0] for c in FRAME_CASES])
def test_high_snr_parity_with_the_state_machine(torch, case):
    """Every FRAME_CASES capture: the same frames, bytes[15:], as work_batch with the FFT demodulator; implicit frames carry
    implicit_len = len(payload) bytes, the first implicit_len of the state machine's."""
    name, sf, cr, implicit, crc, rr, payload_hex, snr, seed = case
    x, _, payload = make_case_iq(case)
    x = x[: x.size // 2 * 2]
    sw = 0x78 if sf >= 11 else 0x12
    old = make_dec(sf, cr, implicit, crc, rr, max_items_per_call=x.size)
    old.work_batch(x[None, :])
    want = [bytes(r["bytes"][15: int(r["len"])]) for r in old.frames_last()]
    new = make_dec(sf, cr, implicit, crc, rr, max_items_per_call=x.size)
    _, frames, info = new.receive(x[None, :], sync_word=sw, implicit_len=len(payload) if implicit else 0)
    got = [bytes(r["bytes"][15: int(r["len"])]) for r in frames]
    assert len(want) == 2 and len(got) == 2, (want, got)
    for g, w in zip(got, want):
        if implicit:
            assert g[3:] == w[3: 3 + len(payload)] == payload
        else:
            assert g == w


# CFOs of a fraction of a bin, which the state machine's FFT demodulator (no CFO correction) decodes on these captures
@pytest.mark.parametrize("sf,cfo", [(7, 300.0), (8, -200.0), (9, 40.0), (10, -50.0), (11, 20.0), (12, 10.0)])
def test_high_snr_parity_with_cfo(torch, sf, cfo):
    """make_capture captures with CFO and no clock drift: the same frames, bytes[15:], as work_batch with the FFT demodulator."""
    payload = bytes.fromhex("deadbeef700d")
    x = make_capture(payload, sf, 4, True, seed=sf, n_frames=2, cfo_hz=cfo)
    x = x[: x.size // 2 * 2]
    rr, sw = sf > 10, 0x78 if sf >= 11 else 0x12
    old = make_dec(sf, 4, False, True, rr, max_items_per_call=x.size)
    old.work_batch(x[None, :])
    want = [bytes(r["bytes"][15: int(r["len"])]) for r in old.frames_last()]
    new = make_dec(sf, 4, False, True, rr, max_items_per_call=x.size)
    _, frames, info = new.receive(x[None, :], sync_word=sw)
    got = [bytes(r["bytes"][15: int(r["len"])]) for r in frames]
    assert len(want) == 2 and got == want and all(g[3:] == payload for g in got), (got, want)
    assert np.all(np.abs(info["cfo_hz"] - cfo) < BW / (1 << sf) / 8)


@pytest.mark.parametrize("sf,cfo", [(7, 2500.0), (8, -7000.0), (9, 11000.0), (10, -1234.5), (12, 20000.0)])
def test_large_cfo_decodes_the_payload(torch, sf, cfo):
    """CFOs of many bins (the state machine's FFT demodulator misreads these captures): both frames carry the transmitted
    payload and the estimated CFO is within 1/8 bin."""
    payload = bytes.fromhex("deadbeef700d")
    x = make_capture(payload, sf, 4, True, seed=sf, n_frames=2, cfo_hz=cfo)
    x = x[: x.size // 2 * 2]
    rr, sw = sf > 10, 0x78 if sf >= 11 else 0x12
    new = make_dec(sf, 4, False, True, rr, max_items_per_call=x.size)
    _, frames, info = new.receive(x[None, :], sync_word=sw)
    got = [bytes(r["bytes"][15: int(r["len"])]) for r in frames]
    assert len(got) == 2 and all(g[3:] == payload for g in got), got
    assert np.all(np.abs(info["cfo_hz"] - cfo) < BW / (1 << sf) / 8)


@pytest.mark.parametrize("sf,plen,channelizer", [(12, 6, False), (12, 6, True), (10, 128, False)])
def test_lora_receiver_dechirp_frames_longer_than_a_call(torch, sf, plen, channelizer):
    """lora_receiver(sync="dechirp") with the default max_items_per_call (1 << 20): frames longer than one call (an SF12 frame
    of 6 bytes, an SF10 frame of 128 bytes) are decoded; run() returns the samples it consumed."""
    import gr_lora_b200 as G
    from gr_lora_b200 import tx
    rng = np.random.default_rng(sf * 1000 + plen)
    pays = [bytes(rng.integers(0, 256, plen, dtype=np.uint8)) for _ in range(2)]
    frames = [tx.modulate_frame(tx.encode_frame(p, sf, 4, reduced_rate=sf > 10), sf) for p in pays]
    assert min(f.size for f in frames) > 1 << 20
    x = tx.channel(frames, sf=sf, snr_db=10.0, seed=sf, cfo_hz=1500.0)
    center = 868.0e6
    rx = G.lora_receiver(FS, center, [center], BW, sf, False, 4, True, sf > 10, disable_channelization=not channelizer,
                         sync="dechirp", quiet=True)
    n = rx.run(x)
    assert [f[18:] for _, f in rx.frames] == pays
    assert 0 < n <= x.size


def test_config5_end_to_end(torch):
    """SF10, implicit header, CR 4/5, no CRC, -10 dB in 125 kHz, no genie: frame and bit error rates."""
    sf, ns = 10, 256
    rng = np.random.default_rng(5)
    pays = [[bytes(rng.integers(0, 256, 16, dtype=np.uint8))] for _ in range(ns)]
    from gr_lora_b200 import tx
    gen = make_dec(sf, 1, True, False)
    up = torch.from_numpy(tx.base_upchirp(sf).astype(np.complex64)).cuda()
    cfo = [[float(rng.uniform(-0.9, 0.9) * BW / 4)] for _ in range(ns)]
    n_items = (12 + 40) * (8 << sf)
    out, placed = gen.synth_streams(pays, n_items, lead_symbols=2.3, cfo_hz=cfo, noise_sigma=sigma_for(-10.0), seed=55, up_table_dev=up)
    torch.cuda.synchronize()
    assert len(placed) == ns
    rx = make_dec(sf, 1, True, False, n_streams=ns, max_items_per_call=n_items)
    _, frames, _ = rx.receive(out, n_items=n_items, implicit_len=16)
    got = payloads_of(frames)
    bit_err, ok = 0, 0
    for s, _, p in placed:
        g = got.get(s, [None])[0]
        if g is None:
            bit_err += 8 * len(p)
            continue
        ok += g[3:] == p
        bit_err += int(np.unpackbits(np.frombuffer(g[3:], np.uint8) ^ np.frombuffer(p, np.uint8)).sum())
    fer, ber = 1 - ok / ns, bit_err / (8 * 16 * ns)
    print(f"config 5 (SF10, implicit, CR 4/5, no CRC, -10 dB, no genie): FER {fer:.4f} BER {ber:.5f} over {ns} frames "
          f"({ns - ok} frames wrong, {bit_err} of {8 * 16 * ns} payload bits)")
    assert fer <= 0.1


def check_exact(placed, frames, n_streams):
    got = payloads_of(frames)
    want = {}
    for s, _, p in placed:
        want.setdefault(s, []).append(p)
    bad = [s for s in range(n_streams) if [g[3:] for g in got.get(s, [])] != want.get(s, [])]
    assert not bad, (len(bad), bad[:4], [(got.get(s), want.get(s)) for s in bad[:2]])


def test_4096_sf7_streams(torch):
    """4096 SF7 streams, every stream its own payloads and CFO, 3 dB above the sensitivity point: every frame once."""
    sf, ns = 7, 4096
    rng = np.random.default_rng(77)
    pays = [[s.to_bytes(2, "little") + bytes([k]) + bytes(rng.integers(0, 256, 7, dtype=np.uint8)) for k in range(3)] for s in range(ns)]
    n_items = 3 * frame_len(sf, 10) + 20 * (8 << sf)
    out, placed = synth(torch, sf, pays, n_items, 1.0, seed=7)
    assert len(placed) == 3 * ns
    rx = make_dec(sf, 4, False, True, n_streams=ns, max_items_per_call=n_items)
    _, frames, _ = rx.receive(out, n_items=n_items)
    check_exact(placed, frames, ns)


def test_mixed_sf_streams(torch):
    """384 streams, 64 per SF7..SF12 (one decoder per SF), each SF 3 dB above its sensitivity point: every frame once."""
    for sf, snr in SENSITIVITY:
        rr, ns = sf >= 11, 64
        rng = np.random.default_rng(sf + 40)
        pays = [[bytes([s, k]) + bytes(rng.integers(0, 256, 6, dtype=np.uint8)) for k in range(2)] for s in range(ns)]
        n_items = (2 * frame_len(sf, 8, rr=rr) + 16 * (8 << sf)) // 2 * 2
        out, placed = synth(torch, sf, pays, n_items, snr + 3.0, seed=sf + 400, rr=rr)
        rx = make_dec(sf, 4, False, True, rr, n_streams=ns, max_items_per_call=n_items)
        _, frames, _ = rx.receive(out, n_items=n_items)
        try:
            check_exact(placed, frames, ns)
        except AssertionError as e:
            raise AssertionError((sf, str(e)[:400])) from None


def test_chunks_and_determinism(torch):
    """One capture fed in random chunk sizes under the consumed rule publishes what the one-shot call does; two runs are
    bit-identical."""
    sf, ns = 8, 16
    rng = np.random.default_rng(3)
    pays = [[bytes([s, k]) + bytes(rng.integers(0, 256, 8, dtype=np.uint8)) for k in range(6)] for s in range(ns)]
    flen = frame_len(sf, 10)
    n_items = 6 * flen + 40 * (8 << sf)
    out, placed = synth(torch, sf, pays, n_items, 0.0, seed=9)
    rx = make_dec(sf, 4, False, True, n_streams=ns, max_items_per_call=n_items)
    _, f1, i1 = rx.receive(out, n_items=n_items)
    f1, i1 = f1.copy(), i1.copy()
    _, f2, i2 = rx.receive(out, n_items=n_items)
    assert f1.tobytes() == f2.tobytes() and i1.tobytes() == i2.tobytes()
    check_exact(placed, f1, ns)
    host = out.cpu().numpy()
    got = {s: [] for s in range(ns)}
    for s in range(ns):                                  # each stream its own chunking
        one = make_dec(sf, 4, False, True, n_streams=1, max_items_per_call=n_items)
        pos = 0
        while pos < n_items:
            n = min(n_items - pos, int(rng.integers(2 * flen, 4 * flen)))
            c, fr, info = one.receive(host[s: s + 1, pos: pos + n])
            got[s] += [bytes(r["bytes"][18: int(r["len"])]) for r in fr]
            if pos + n >= n_items:
                break
            assert c[0] > 0
            pos += int(c[0])
    want = {s: [bytes(r["bytes"][18: int(r["len"])]) for r in f1 if int(r["stream"]) == s] for s in range(ns)}
    assert got == want


def test_false_alarms(torch):
    """384 streams x 2 s of pure noise publish nothing; neither do frames with another sync word."""
    sf, ns, n_items = 7, 384, 2_000_000
    g = torch.Generator(device="cuda").manual_seed(1)
    noise = torch.randn((ns, n_items), dtype=torch.complex64, device="cuda", generator=g)
    rx = make_dec(sf, 4, False, True, n_streams=ns, max_items_per_call=n_items, max_frames_per_call=64)
    _, frames, _ = rx.receive(noise, n_items=n_items)
    assert len(frames) == 0
    del noise
    rng = np.random.default_rng(4)
    pays = [[bytes(rng.integers(0, 256, 8, dtype=np.uint8)) for _ in range(2)] for _ in range(32)]
    for sf in (7, 10):
        out, placed = synth(torch, sf, pays, 2 * frame_len(sf, 8) + 16 * (8 << sf), 10.0, seed=5, sync_word=0x34)
        rx = make_dec(sf, 4, False, True, n_streams=32, max_items_per_call=out.shape[1])
        assert len(rx.receive(out)[1]) == 0
        assert len(rx.receive(out, sync_word=0x34)[1]) == len(placed)


def test_implicit_len_zero_is_refused(torch):
    import gr_lora_b200._native as N
    rx = make_dec(7, 4, True, True)
    x = np.zeros((1, 8192), np.complex64)
    with pytest.raises(N.LoraB200Error) as e:
        rx.receive(x)
    assert e.value.code == N.EINVAL


def test_state_machine_state_untouched(torch):
    x, _, _ = make_case_iq(FRAME_CASES[0])
    x = x[: x.size // 2 * 2]
    rx = make_dec(7, 4, False, True, max_items_per_call=x.size)
    rx.work_batch(x[None, : x.size // 3])
    st = rx.state(0)
    _, frames, _ = rx.receive(x[None, :])
    assert len(frames) == 2 and rx.state(0) == st
