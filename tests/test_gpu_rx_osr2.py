"""fs/bw = 2 on the device: k1_fft_kernel<SF, 2> and k1_llr_kernel<SF, 2> (demod_fft_dev / demod_llr_dev of a decoder at
250 kS/s) against a float64 get_shift_fft, lora_b200_receive frame by frame against its host emulation
(lb_emul_rx_receive_osr), its sensitivity, and the channelizer path lora_receiver(..., decimation=4, sync="dechirp")."""
import numpy as np
import pytest

from k1_reference import check_k1
from osr2_common import BATCH, BW, CARRIER, FS, OSR, K1ReferenceOsr, check_llrs, frame_row, k1_batch, receive_emul

pytestmark = pytest.mark.gpu

SENSITIVITY = [(7, -2.0), (8, -5.0), (9, -7.5), (10, -10.0), (11, -12.5), (12, -15.0)]


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def make_dec(sf, cr=4, implicit=False, crc=True, rr=False, fs=FS, **kw):
    import gr_lora_b200 as G
    return G.decoder(fs, BW, sf, implicit, cr, crc, rr, quiet=True, **kw)


def sigma_for(snr_125k_db, fs=FS):
    return float(np.sqrt(10 ** (-(snr_125k_db - 10 * np.log10(fs / BW)) / 10) / 2))


# ---- K1 and the LLR demodulator -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sf", range(7, 13))
def test_demod_fft_dev_against_float64(torch, sf):
    """Every bin clean (a spread at SF11/12), -3 dB, half-bin and noise windows in batches around the kernel's symbols per
    grid pass: bins and magnitudes inside the float64 rounding band, two runs bit-identical."""
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    dec = make_dec(sf)
    assert dec.sps == OSR << sf and dec.decim == OSR
    from osr2_common import tables
    down = tables(sf)[0]
    base = k1_batch(sf, np.random.default_rng(sf))
    per_pass = 2 * n_sms * BATCH[sf]
    for n in sorted({base.shape[0], per_pass - 1, per_pass, per_pass + 1}):
        x = np.ascontiguousarray(np.resize(base, (n, base.shape[1])), np.complex64)
        xd = torch.from_numpy(x).cuda()
        bins = torch.zeros(n, dtype=torch.int32, device="cuda")
        mags = torch.zeros(n, dtype=torch.float32, device="cuda")
        dec.demod_fft(xd, n, bins, mags)
        bins2 = torch.zeros_like(bins)
        mags2 = torch.zeros_like(mags)
        dec.demod_fft(xd, n, bins2, mags2)
        torch.cuda.synchronize()
        check_k1(bins.cpu().numpy(), mags.cpu().numpy(), None, sf, ref=K1ReferenceOsr(x, sf, down), what=f"SF{sf} n={n}")
        assert torch.equal(bins, bins2) and torch.equal(mags, mags2)
        if sf <= 10 and n >= 1 << sf:                     # an up-chirp shifted by v dechirps to bin v
            assert np.array_equal(bins.cpu().numpy()[: 1 << sf], np.arange(1 << sf))
    dec.close()


@pytest.mark.parametrize("sf", range(7, 13))
@pytest.mark.parametrize("reduced", [0, 1])
def test_demod_llr_dev_against_float64(torch, sf, reduced):
    """LLRs within 2 tau of the float64 max-log LLR; their bins equal demod_fft_dev's bit for bit; two runs bit-identical."""
    from osr2_common import tables
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    dec = make_dec(sf)
    ppm = sf - 2 if reduced else sf
    down = tables(sf)[0]
    base = k1_batch(sf, np.random.default_rng(10 * sf + reduced), n_clean=3)
    per_pass = 2 * n_sms * BATCH[sf]
    for n in sorted({1, base.shape[0], per_pass - 1, per_pass, per_pass + 1}):
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
        check_llrs(L, B, K1ReferenceOsr(x, sf, down), sf, reduced, f"SF{sf} reduced={reduced} n={n}")
        assert torch.equal(bins, kb)
        assert torch.equal(llr, llr2)
    dec.close()


# ---- the receiver against its host emulation ------------------------------------------------------------------------------------
def rows(sf, snr_db, n_rows, seed, rr, sfo_ppm=0.0, coupled=False):
    """n_rows rows of one frame each at fs/bw = 2 (random CFO, start, payload), equal length."""
    rng = np.random.default_rng(seed)
    sps = OSR << sf
    out, truth = [], []
    for k in range(n_rows):
        pay = bytes(rng.integers(0, 256, 12, dtype=np.uint8))
        cfo = sfo_ppm * CARRIER * 1e-6 if coupled else float(rng.uniform(-0.9, 0.9) * BW / 4)
        x, lead, _ = frame_row(sf, pay, cfo, int(rng.integers(0, sps)), snr_db=snr_db, seed=seed * 100 + k, rr=rr,
                               sfo_ppm=sfo_ppm, tail=3 + k % 3)
        out.append(x)
        truth.append((lead, pay))
    m = max(x.size for x in out)
    X = np.zeros((n_rows, m), np.complex64)
    for k, x in enumerate(out):
        X[k, : x.size] = x
        if snr_db is not None and x.size < m:
            X[k, x.size:] = tx_noise(m - x.size, snr_db, seed * 100 + k + 50)
    return X, truth


def tx_noise(n, snr_db, seed):
    from gr_lora_b200 import tx
    return tx.awgn(n, snr_db - 10 * np.log10(OSR), np.random.default_rng(seed)).astype(np.complex64)


@pytest.mark.parametrize("sf", range(7, 13))
@pytest.mark.parametrize("soft", [False, True])
def test_receive_matches_host_emulation(torch, sf, soft):
    """Per row, at +10 dB and 1 dB above the sensitivity points (hard and soft): the device publishes the payloads the host
    emulation publishes (at +10 dB: the one sent), and frames both sides place within 2 samples of each other have the same
    start and payload and CFOs within 1e-3 bin."""
    rr = sf > 10
    snr_sens = dict(SENSITIVITY)[sf]
    n_rows = 8 if sf <= 10 else 3
    for snr in (10.0, snr_sens + 1.0):
        X, truth = rows(sf, snr, n_rows, seed=sf * 10 + int(soft) + int(snr), rr=rr)
        dec = make_dec(sf, rr=rr, n_streams=n_rows, max_items_per_call=X.shape[1])
        _, frames, info = dec.receive(X, soft=soft)
        dev = {}
        for f, i in zip(frames, info):
            dev.setdefault(int(f["stream"]), []).append((int(i["start"]), float(i["cfo_hz"]) / (BW / (1 << sf)),
                                                         bytes(f["bytes"][18: int(f["len"])])))
        for s in range(n_rows):
            host = [(g["start"], g["cfo"], g["payload"]) for g in receive_emul(X[s], sf, rr=rr, soft=soft) if g["status"] == 0]
            d = dev.get(s, [])
            if snr >= 10.0:
                assert {a[2] for a in d} == {b[2] for b in host} == {truth[s][1]}, (s, d, host)
            for a in d:
                for b in host:
                    if abs(a[0] - b[0]) <= 2:
                        assert a[0] == b[0] and a[2] == b[2] and abs(a[1] - b[1]) <= 1e-3, (s, a, b)
            if snr >= 10.0:
                continue
            assert {a[2] for a in d} == {b[2] for b in host}, (sf, soft, s, d, host)
        dec.close()


# ---- sensitivity ---------------------------------------------------------------------------------------------------------------
def synth(torch, sf, pays, n_items, snr_db, seed, rr=False, cr=4, sfo_ppm=0.0, cfo=None):
    from gr_lora_b200 import tx
    rng = np.random.default_rng(seed)
    gen = make_dec(sf, cr, False, True, rr)
    up = torch.from_numpy(tx.base_upchirp(sf, BW, FS).astype(np.complex64)).cuda()
    if cfo is None:
        cfo = [[float(rng.uniform(-0.9, 0.9) * BW / 4) for _ in p] for p in pays]
    out, placed = gen.synth_streams(pays, n_items, lead_symbols=float(rng.uniform(1.0, 3.0)), gap_symbols=float(rng.uniform(3.0, 5.0)),
                                    cfo_hz=cfo, noise_sigma=sigma_for(snr_db) if snr_db is not None else 0.0, seed=seed,
                                    up_table_dev=up, sfo_ppm=sfo_ppm)
    torch.cuda.synchronize()
    gen.close()
    return out, placed


def test_sensitivity_points(torch):
    """48 frames per SF at the fs/bw = 8 sensitivity points (SF7 -2 ... SF12 -15 dB in 125 kHz, SF11/12 reduced rate): all
    decode, hard and soft, and soft decisions publish no payload that was not sent."""
    import gr_lora_b200 as G
    for sf, snr in SENSITIVITY:
        rr, ns, sps = sf >= 11, 48, OSR << sf
        rng = np.random.default_rng(sf)
        pays = [[bytes(rng.integers(0, 256, 10, dtype=np.uint8))] for _ in range(ns)]
        n_items = (int((12 + G.tx_frame_symbols(10, sf, 4, False, True, rr)) * sps + sps // 4 + 9 * sps) // 2) * 2
        out, placed = synth(torch, sf, pays, n_items, snr, seed=3000 + sf, rr=rr)
        sent = {(s, p) for s, _, p in placed}
        assert len(sent) == ns
        for soft in (False, True):
            rx = make_dec(sf, 4, False, True, rr, n_streams=ns, max_items_per_call=n_items)
            _, frames, _ = rx.receive(out, n_items=n_items, soft=soft)
            got = [(int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in frames]
            print(f"fs/bw = 2, SF{sf} at {snr:+.1f} dB: {'soft' if soft else 'hard'} {len(set(got) & sent)}/{ns}")
            if soft:
                assert all(g in sent for g in got), (sf, snr)
            assert len(set(got) & sent) == ns, (sf, snr, soft)
            rx.close()


def test_pure_noise_publishes_nothing(torch):
    """64 streams x 2 s of noise at 250 kS/s: no frame, hard or soft."""
    for sf in (7, 9):
        x = torch.randn(64, int(2 * FS), dtype=torch.complex64, device="cuda")
        for soft in (False, True):
            rx = make_dec(sf, n_streams=64, max_items_per_call=x.shape[1])
            _, frames, _ = rx.receive(x, n_items=x.shape[1], soft=soft)
            assert len(frames) == 0, (sf, soft, len(frames))
            rx.close()


@pytest.mark.parametrize("ppm", [20.0, -20.0])
def test_sf12_drifted_frames_decode_with_carrier(torch, ppm):
    """SF12 64-byte frames from transmitters whose crystal is off by +-20 ppm (carrier and clock), found through carrier_hz."""
    sf, ns = 12, 4
    rng = np.random.default_rng(int(ppm) + 99)
    pays = [[bytes(rng.integers(0, 256, 64, dtype=np.uint8))] for _ in range(ns)]
    import gr_lora_b200 as G
    sps = OSR << sf
    n_items = int((12 + G.tx_frame_symbols(64, sf, 4, False, True, True)) * sps * 1.001 + 9 * sps) // 2 * 2
    out, placed = synth(torch, sf, pays, n_items, 0.0, seed=77 + int(ppm), rr=True, sfo_ppm=ppm,
                        cfo=[[ppm * CARRIER * 1e-6] for _ in range(ns)])
    rx = make_dec(sf, 4, False, True, True, n_streams=ns, max_items_per_call=n_items)
    _, frames, info = rx.receive(out, n_items=n_items, carrier_hz=CARRIER)
    got = {(int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in frames}
    assert got == {(s, p) for s, _, p in placed}
    assert all(abs(float(i["sfo_ppm"]) - ppm) < 0.5 for i in info)
    rx.close()


# ---- the channelizer path --------------------------------------------------------------------------------------------------------
def test_channelizer_decimation_4_matches_decimation_1(torch):
    """A 1 MS/s capture made by the fs/bw = 8 decoder's transmitter, through lora_receiver(..., decimation=4, sync="dechirp"):
    the frames reach the receiver at fs/bw = 2 with fractional-chip offsets and it publishes the payloads decimation=1
    publishes on the same capture, 1.5 dB above the sensitivity points."""
    import gr_lora_b200 as G
    from gr_lora_b200 import tx
    center = 868.1e6
    for sf, snr in SENSITIVITY[:4]:
        snr += 1.5
        fs8 = 1e6
        rng = np.random.default_rng(sf + 500)
        pays = [bytes(rng.integers(0, 256, 10, dtype=np.uint8)) for _ in range(6)]
        gen = make_dec(sf, fs=fs8)
        up = torch.from_numpy(tx.base_upchirp(sf, BW, fs8).astype(np.complex64)).cuda()
        sps8 = 8 << sf
        n_items = int(len(pays) * (12 + G.tx_frame_symbols(10, sf, 4, False, True, False) + 8) * sps8 + 8 * sps8) // 8 * 8
        cfo = [[float(rng.uniform(-0.5, 0.5) * BW / 4) for _ in pays]]
        out, placed = gen.synth_streams([pays], n_items, lead_symbols=2.37, gap_symbols=4.61, cfo_hz=cfo,
                                        noise_sigma=sigma_for(snr, fs8), seed=sf, up_table_dev=up)
        torch.cuda.synchronize()
        gen.close()
        x = out[0].cpu().numpy()
        res = {}
        for decim in (1, 4):
            rx = G.lora_receiver(fs8, center, [center], 125000, sf, False, 4, True, decimation=decim, sync="dechirp", quiet=True)
            rx.run(x)
            res[decim] = [bytes(f[18:]) for _, f in rx.frames]
        sent = [p for _, _, p in placed]
        print(f"SF{sf} at {snr:+.1f} dB: decimation 1 {len(res[1])}, decimation 4 {len(res[4])} of {len(sent)}")
        assert res[4] == res[1] == sent, (sf, res, sent)
