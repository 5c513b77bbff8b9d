"""lora_b200_receive_antennas on the device: M = 1 is lora_b200_receive byte for byte, M = 2 frame by frame against its host
emulation (lb_emul_rx_receive_antennas), the array gain in white noise and the diversity gain under Rayleigh fading, and the
call's edges (drift, chunked feeding, pure noise, the channelizer path, bad antenna counts)."""
import numpy as np
import pytest

from antenna_common import BW, CARRIER, SENSITIVITY, frame_rows, rayleigh, receive_emul, synth_antennas

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def make_dec(sf, osr=8, rr=False, **kw):
    import gr_lora_b200 as G
    return G.decoder(osr * BW, BW, sf, False, 4, True, rr, quiet=True, **kw)


def n_items_for(sf, osr, n_bytes, rr, ppm=0.0):
    import gr_lora_b200 as G
    sps = osr << sf
    return int((12 + G.tx_frame_symbols(n_bytes, sf, 4, False, True, rr)) * sps * (1 + abs(ppm) * 1e-6) + sps // 4 + 9 * sps) // 8 * 8


def decoded(frames, sent):
    got = {(int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in frames}
    return got & sent, got


# ---- the combined screen against float64 ---------------------------------------------------------------------------------------------
# windows per CTA batch of k1_antennas_kernel<SF, D> (K1Cfg<SF, D>::G)
GROUP = {8: {7: 8, 8: 4, 9: 2, 10: 1, 11: 1, 12: 1}, 2: {7: 32, 8: 16, 9: 8, 10: 4, 11: 2, 12: 2}}


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf", range(7, 13))
def test_combined_screen_against_float64(torch, sf, osr):
    """k1_antennas_kernel through lora_b200_demod_fft_antennas_dev: every bin clean (a spread at SF11/12), -3 dB, half-bin and
    noise windows, each antenna its own symbols and gain, M = 2, 3 and 4, two groups, in batches around the kernel's windows per
    grid pass (more work items than CTAs): bins and magnitudes inside the band of the float64 sum_a |tmp_a|^2
    (antenna_common.CombinedReference), two runs bit-identical."""
    from antenna_common import CombinedReference, k1_batch
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    sps, ng = osr << sf, 2
    per_pass = 2 * n_sms * GROUP[osr][sf]
    dec = make_dec(sf, osr)
    rng = np.random.default_rng(300 * sf + osr)
    for m in (2, 3, 4):
        base = [k1_batch(sf, osr, np.random.default_rng(1000 * sf + 10 * osr + a), n_clean=24 if sf >= 11 else None)
                for a in range(ng * m)]
        for n in sorted({min(b.shape[0] for b in base), per_pass // ng + 1}):
            gains = np.exp(2j * np.pi * rng.uniform(size=ng * m)) * 10 ** (rng.uniform(-3, 3, ng * m) / 20)
            X = np.stack([g * np.resize(b, (n, sps)) for g, b in zip(gains, base)]).astype(np.complex64)   # [ng m, n, sps]
            xd = torch.from_numpy(X.reshape(ng * m, n * sps)).cuda()
            out = []
            for _ in range(2):
                bins = torch.zeros(ng * n, dtype=torch.int32, device="cuda")
                mags = torch.zeros(ng * n, dtype=torch.float32, device="cuda")
                dec.demod_fft_antennas(xd, ng, m, n, n * sps, bins, mags)
                torch.cuda.synchronize()
                out.append((bins.cpu().numpy(), mags.cpu().numpy()))
            assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1].view(np.uint32), out[1][1].view(np.uint32))
            for g in range(ng):
                ref = CombinedReference(X[g * m: g * m + m], sf, osr)
                ref.check(out[0][0][g * n: (g + 1) * n], out[0][1][g * n: (g + 1) * n], f"SF{sf} fs/bw={osr} M={m} n={n} group {g}")
            del xd
    dec.close()


# ---- M = 1 is lora_b200_receive ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("soft", [False, True])
def test_one_antenna_is_byte_identical(torch, osr, soft):
    """Several streams, host and device input, with carrier_hz: frames, rx_info, header drops and consumed of
    receive(antennas=1) through lora_b200_receive_antennas equal lora_b200_receive's byte for byte."""
    import ctypes as C
    from gr_lora_b200 import _native as N
    sf, ns = 8, 6
    rng = np.random.default_rng(osr + 10 * soft)
    pays = [[bytes(rng.integers(0, 256, 10, dtype=np.uint8))] for _ in range(ns)]
    n = n_items_for(sf, osr, 10, False)
    x, _ = synth_antennas(torch, sf, osr, pays, n, SENSITIVITY[sf] + 1.0, np.ones((ns, 1)), seed=5 + osr)
    dec = make_dec(sf, osr, n_streams=ns, max_items_per_call=n)
    for src, host in ((x, 0), (x.cpu().numpy(), 1)):
        ref = dec.receive(src, n_items=n, soft=soft, carrier_hz=CARRIER)
        ref_drops = dec.header_drops
        p = N.RxParams(sync_word=0x12, carrier_hz=CARRIER, soft=int(soft))
        cons = np.zeros(ns, np.uint64)
        ptr = src.ctypes.data if host else int(src.data_ptr())
        N.check(dec._L.lora_b200_receive_antennas(dec._h, ptr, n, n, host, 1, C.byref(p), cons.ctypes.data_as(C.POINTER(C.c_size_t))), "x")
        frames = dec.frames_last()
        iptr, drops = C.c_void_p(0), C.c_uint32(0)
        k = int(dec._L.lora_b200_rx_info_last(dec._h, C.byref(iptr), C.byref(drops)))
        info = np.frombuffer(C.string_at(iptr.value, k * dec.RX_INFO_DTYPE.itemsize), dec.RX_INFO_DTYPE) if k else np.zeros(0, dec.RX_INFO_DTYPE)
        assert np.array_equal(cons.astype(np.int64), ref[0])
        assert frames.tobytes() == ref[1].tobytes() and info.tobytes() == ref[2].tobytes() and int(drops.value) == ref_drops
        assert len(frames) > 0
    dec.close()


# ---- M = 2 against the host emulation ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf,m", [(sf, 2) for sf in range(7, 13)] + [(8, 3), (11, 3)] + [(7, 4), (9, 4), (12, 4)])
def test_antennas_match_host_emulation(torch, sf, m, osr):
    """M = 2 (every SF), M = 3 (SF8, 11) and M = 4 (SF7, 9, 12) at +10 dB and at sensitivity - 1.5 dB per antenna, random relative phases and
    gains within +-3 dB: per receiver the device publishes the set of payloads the host emulation publishes (at +10 dB: the
    one sent), and frames both sides place within 2 samples of each other have the same start and payload and CFOs within 1e-3
    bin."""
    rr = sf > 10
    n_rx = 4 if sf <= 10 else 2
    rng = np.random.default_rng(20 * sf + osr + 100 * m)
    sps = osr << sf
    for snr in (10.0, SENSITIVITY[sf] - 1.5):
        rows, truth = [], []
        for g in range(n_rx):
            pay = bytes(rng.integers(0, 256, 8, dtype=np.uint8))
            gains = [1.0] + [10 ** (rng.uniform(-3, 3) / 20) * np.exp(2j * np.pi * rng.uniform()) for _ in range(m - 1)]
            X, _, _ = frame_rows(sf, osr, pay, float(rng.uniform(-0.9, 0.9) * BW / 4), int(rng.integers(0, sps)), gains, snr_db=snr,
                                 seed=int(rng.integers(1 << 30)), rr=rr)
            rows.append(X)
            truth.append(pay)
        n = max(X.shape[1] for X in rows)
        Y = np.zeros((m * n_rx, n), np.complex64)
        for g, X in enumerate(rows):
            Y[m * g: m * g + m, : X.shape[1]] = X
        dec = make_dec(sf, osr, rr, n_streams=m * n_rx, max_items_per_call=n)
        _, frames, info = dec.receive(Y, antennas=m)
        h = dec.rx_channels_last()
        assert h.shape == (len(frames), m)
        dev = {}
        for f, i in zip(frames, info):
            dev.setdefault(int(f["stream"]), []).append((int(i["start"]), float(i["cfo_hz"]) / (BW / (1 << sf)), bytes(f["bytes"][18: int(f["len"])])))
        for g in range(n_rx):
            host = [(e["start"], e["cfo"], e["payload"]) for e in receive_emul(Y[m * g: m * g + m], sf, osr, rr=rr) if e["status"] == 0]
            d = dev.get(g, [])
            # (the emulation publishes every synchronised candidate; the device keeps one frame per preamble, so a preamble
            # both phases of the screen found may appear twice on the host side)
            assert {a[2] for a in d} == {b[2] for b in host}, (snr, g, d, host)
            if snr >= 10.0:
                assert {a[2] for a in d} == {truth[g]}, (g, d, host)
            for a in d:
                for b in host:
                    if abs(a[0] - b[0]) <= 2:
                        assert a[0] == b[0] and a[2] == b[2] and abs(a[1] - b[1]) <= 1e-3, (snr, g, a, b)
        dec.close()


# ---- array gain in white noise, diversity gain under fading ----------------------------------------------------------------------
def antenna_run(torch, sf, snr, gains, seed, soft=False, osr=8, n_bytes=10):
    """One capture of len(gains) receivers x M antennas: frames decoded with the M antennas combined, and by each antenna alone
    through lora_b200_receive (the same rows)."""
    rr = sf >= 11
    ng, m = np.shape(gains)
    rng = np.random.default_rng(seed)
    pays = [[bytes(rng.integers(0, 256, n_bytes, dtype=np.uint8))] for _ in range(ng)]
    n = n_items_for(sf, osr, n_bytes, rr)
    x, placed = synth_antennas(torch, sf, osr, pays, n, snr, gains, seed, rr=rr)
    sent = {(s, p) for s, _, p in placed}
    rx = make_dec(sf, osr, rr, n_streams=ng * m, max_items_per_call=n)
    comb, got = decoded(rx.receive(x, n_items=n, soft=soft, antennas=m)[1], sent)
    rx.close()
    single = []
    one = make_dec(sf, osr, rr, n_streams=ng, max_items_per_call=n)
    for a in range(m):
        xa = x.view(ng, m, n)[:, a, :].contiguous()
        torch.cuda.synchronize()                      # (receive reads device input on its own stream)
        single.append(len(decoded(one.receive(xa, n_items=n, soft=soft)[1], sent)[0]))
    one.close()
    return len(comb), single, len(sent)


def test_two_antennas_gain_in_white_noise(torch):
    """Two antennas with independent noise and random relative phase.  Each at its SF's sensitivity point - 2 dB: at least 47
    of 48 frames decode per SF (hard), and at least what each antenna decodes alone.  One antenna alone still decodes nearly
    every frame there, so the gain itself is checked 4 dB below the sensitivity points as well: per SF at least what each
    antenna decodes alone, and strictly more summed over SFs."""
    for off in (-2.0, -4.0):
        tot_c, tot_s = 0, [0, 0]
        for sf in range(7, 13):
            rng = np.random.default_rng(sf + 40)
            gains = np.stack([np.ones(48), np.exp(2j * np.pi * rng.uniform(size=48))], axis=1)
            c, s, ns = antenna_run(torch, sf, SENSITIVITY[sf] + off, gains, seed=700 + sf + int(10 * off))
            print(f"SF{sf} at {SENSITIVITY[sf] + off:+.1f} dB per antenna: 2 antennas {c}/{ns}, alone {s[0]}, {s[1]}")
            assert ns == 48 and c >= max(s), (sf, off, c, s)
            if off == -2.0:
                assert c >= 47, (sf, c, s)
            tot_c += c
            tot_s = [tot_s[0] + s[0], tot_s[1] + s[1]]
        if off == -4.0:
            assert tot_c > max(tot_s), (tot_c, tot_s)


def test_two_antennas_under_rayleigh_fading(torch):
    """Independent complex-Gaussian gains per frame and antenna (mean power 1), mean SNR at the sensitivity point + 3 dB: two
    antennas lose at most half as many frames as the better single antenna on the same capture."""
    for sf in (7, 9, 12):
        rng = np.random.default_rng(sf + 90)
        gains = rayleigh(rng, (96, 2))
        c, s, ns = antenna_run(torch, sf, SENSITIVITY[sf] + 3.0, gains, seed=900 + sf)
        lost_c, lost_s = ns - c, ns - max(s)
        print(f"SF{sf} Rayleigh at {SENSITIVITY[sf] + 3.0:+.1f} dB mean: 2 antennas lose {lost_c}/{ns}, alone {ns - s[0]}, {ns - s[1]}")
        assert 2 * lost_c <= lost_s, (sf, lost_c, s)


# ---- edges -----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ppm", [20.0, -20.0])
def test_sf12_drifted_frames_decode_with_carrier(torch, ppm):
    """SF12 64-byte frames from transmitters whose crystal is off by +-20 ppm, two antennas, found through carrier_hz."""
    sf, ng = 12, 3
    rng = np.random.default_rng(int(ppm) + 70)
    pays = [[bytes(rng.integers(0, 256, 64, dtype=np.uint8))] for _ in range(ng)]
    n = n_items_for(sf, 8, 64, True, ppm)
    gains = np.stack([np.ones(ng), 0.7 * np.exp(2j * np.pi * rng.uniform(size=ng))], axis=1)
    x, placed = synth_antennas(torch, sf, 8, pays, n, SENSITIVITY[sf] + 3.0, gains, seed=31 + int(ppm), rr=True, sfo_ppm=ppm,
                               cfo=[[ppm * CARRIER * 1e-6] for _ in range(ng)])
    rx = make_dec(sf, 8, True, n_streams=2 * ng, max_items_per_call=n)
    _, frames, info = rx.receive(x, n_items=n, carrier_hz=CARRIER, antennas=2)
    ok, got = decoded(frames, {(s, p) for s, _, p in placed})
    assert got == {(s, p) for s, _, p in placed}
    assert all(abs(float(i["sfo_ppm"]) - ppm) < 0.5 for i in info)
    rx.close()


def test_chunked_feeding_publishes_every_frame(torch):
    """Several frames per receiver fed in chunks under the consumed rule (one consumed per receiver): every frame is published
    once, as in one call over the whole capture."""
    sf, osr, ng, m = 8, 8, 3, 2
    rng = np.random.default_rng(3)
    pays = [[bytes(rng.integers(0, 256, 12, dtype=np.uint8)) for _ in range(6)] for _ in range(ng)]
    n = 6 * n_items_for(sf, osr, 12, False)
    gains = np.stack([np.ones(ng), np.exp(2j * np.pi * rng.uniform(size=ng))], axis=1)
    x, placed = synth_antennas(torch, sf, osr, pays, n, SENSITIVITY[sf] + 2.0, gains, seed=17)
    X = x.cpu().numpy()
    sent = [(s, p) for s, _, p in placed]
    whole = make_dec(sf, osr, n_streams=ng * m, max_items_per_call=n)
    ref = sorted((int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in whole.receive(X, antennas=m)[1])
    whole.close()
    rx = make_dec(sf, osr, n_streams=ng * m, max_items_per_call=n)
    pos, got, chunk = np.zeros(ng, np.int64), [], 9 * (osr << sf) + 123
    while (pos < n).any():
        L = int(min(chunk, n - pos.min()))
        part = np.zeros((ng * m, L), np.complex64)
        for g in range(ng):
            seg = X[g * m: g * m + m, pos[g]: pos[g] + L]
            part[g * m: g * m + m, : seg.shape[1]] = seg
        c, frames, _ = rx.receive(part, antennas=m)
        got += [(int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in frames]
        assert c.shape == (ng,)
        if (pos + L >= n).all():
            break
        pos += np.where(pos + L >= n, 0, c)
        chunk = chunk if c.min() > 0 else 2 * chunk
    rx.close()
    assert sorted(got) == ref == sorted(sent)


def test_pure_noise_publishes_nothing(torch):
    """64 receivers x 2 antennas x 2 s of noise: no frame, hard or soft."""
    x = torch.randn(128, 2_000_000, dtype=torch.complex64, device="cuda")
    for soft in (False, True):
        rx = make_dec(7, 8, n_streams=128, max_items_per_call=x.shape[1])
        c, frames, _ = rx.receive(x, n_items=x.shape[1], soft=soft, antennas=2)
        assert len(frames) == 0 and c.shape == (64,), (soft, len(frames))
        rx.close()


def test_bad_antenna_counts_are_rejected(torch):
    """M not dividing n_streams, M = 0 and M = 5: LORA_B200_EINVAL before any launch."""
    from gr_lora_b200 import _native as N
    rx = make_dec(7, 8, n_streams=6, max_items_per_call=1 << 16)
    x = np.zeros((6, 1 << 16), np.complex64)
    before = rx.launch_count()
    for m in (0, 4, 5):
        with pytest.raises(N.LoraB200Error) as e:
            rx.receive(x, antennas=m)
        assert e.value.code == N.EINVAL
    assert rx.launch_count() == before
    rx.close()


def test_channelizer_path_with_two_antennas(torch):
    """A two-row 1 MS/s capture through lora_receiver(..., decimation=4, sync="dechirp", antennas=2) (one channelizer per
    antenna) publishes what decimation=1 publishes on the same capture."""
    import gr_lora_b200 as G
    center = 868.1e6
    for sf in (7, 9):
        rng = np.random.default_rng(sf + 77)
        pays = [bytes(rng.integers(0, 256, 10, dtype=np.uint8)) for _ in range(5)]
        rows = [1.0, 0.8 * np.exp(1j * 2.1)]                      # the antennas' gains
        n_each = int((12 + G.tx_frame_symbols(10, sf, 4, False, True, False) + 8) * (8 << sf))
        sig = np.zeros(len(pays) * n_each + 8 * (8 << sf), np.complex128)
        for k, p in enumerate(pays):
            X, lead, fl = frame_rows(sf, 8, p, float(rng.uniform(-0.5, 0.5) * BW / 4), int(rng.integers(0, 8 << sf)), [1.0])
            sig[k * n_each: k * n_each + X.shape[1]] += X[0][: min(X.shape[1], sig.size - k * n_each)]
        noise = np.random.default_rng(sf)
        cap = np.stack([g * sig for g in rows])
        from gr_lora_b200 import tx
        snr = SENSITIVITY[sf] + 1.5
        cap = cap + np.stack([tx.awgn(sig.size, snr - 10 * np.log10(8), noise) for _ in rows])
        cap = cap[:, : cap.shape[1] // 8 * 8].astype(np.complex64)
        res = {}
        for decim in (1, 4):
            rx = G.lora_receiver(1e6, center, [center], 125000, sf, False, 4, True, decimation=decim, sync="dechirp", antennas=2, quiet=True)
            rx.run(cap)
            res[decim] = [bytes(f[18:]) for _, f in rx.frames]
        print(f"SF{sf}: decimation 1 {len(res[1])}, decimation 4 {len(res[4])} of {len(pays)}")
        assert res[4] == res[1] == pays, (sf, res)
    with pytest.raises(ValueError):
        G.lora_receiver(1e6, center, [center], 125000, 7, False, 4, True, antennas=2)
