"""fs/bw = 16 and 32 on the device: k1_fft_kernel<SF, D>, k1_llr_kernel<SF, D> and k1_antennas_kernel<SF, D> against a float64
get_shift_fft, the synchroniser's window sums across the sampled band, lora_b200_receive frame by frame against its host
emulation (hard, soft, list decoding, two antennas, wide_cfo, fine_toa), its sensitivity, and the channelizer at
decimation=1."""
import math

import numpy as np
import pytest

from antenna_common import BW, CombinedReference, frame_rows, k1_batch, synth_antennas, tables
from antenna_reference import window_sum
from k1_reference import check_k1
from osr2_common import K1ReferenceOsr, check_llrs
from osr_high_common import RATES, SENSITIVITY, batch, receive

pytestmark = pytest.mark.gpu

CARRIER = 868.1e6


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def make_dec(sf, osr, rr=False, bw=BW, **kw):
    import gr_lora_b200 as G
    return G.decoder(osr * bw, bw, sf, False, 4, True, rr, quiet=True, **kw)


def per_pass(torch, sf, osr):
    """symbols per grid pass of the K1 kernels: 2 CTAs per SM, G symbols each"""
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count * batch(sf, osr)


# ---- K1, the LLR demodulator and the combined screen ------------------------------------------------------------------------
@pytest.mark.parametrize("osr", RATES)
@pytest.mark.parametrize("sf", range(7, 13))
def test_demod_fft_dev_against_float64(torch, sf, osr):
    """Clean, -3 dB, half-bin and noise windows in batches around the symbols per grid pass: bins and magnitudes inside the
    float64 rounding band, two runs bit-identical, an up-chirp shifted by v at bin v."""
    dec = make_dec(sf, osr)
    assert dec.sps == osr << sf and dec.decim == osr
    down = tables(sf, osr)[0]
    base = k1_batch(sf, osr, np.random.default_rng(sf + osr), n_clean=24)
    pp = per_pass(torch, sf, osr)
    for n in sorted({base.shape[0], pp - 1, pp, pp + 1}):
        x = np.ascontiguousarray(np.resize(base, (n, base.shape[1])), np.complex64)
        xd = torch.from_numpy(x).cuda()
        bins = torch.zeros(n, dtype=torch.int32, device="cuda")
        mags = torch.zeros(n, dtype=torch.float32, device="cuda")
        dec.demod_fft(xd, n, bins, mags)
        bins2, mags2 = torch.zeros_like(bins), torch.zeros_like(mags)
        dec.demod_fft(xd, n, bins2, mags2)
        torch.cuda.synchronize()
        check_k1(bins.cpu().numpy(), mags.cpu().numpy(), None, sf, ref=K1ReferenceOsr(x, sf, down, osr=osr), what=f"SF{sf} D={osr} n={n}")
        assert torch.equal(bins, bins2) and torch.equal(mags, mags2)
        del xd
    dec.close()


@pytest.mark.parametrize("osr", RATES)
@pytest.mark.parametrize("sf", range(7, 13))
def test_demod_llr_dev_against_float64(torch, sf, osr):
    """LLRs within 2 tau of the float64 max-log LLR (normal and reduced rate); bins equal demod_fft_dev's; two runs identical."""
    dec = make_dec(sf, osr)
    down = tables(sf, osr)[0]
    pp = per_pass(torch, sf, osr)
    for reduced in (0, 1):
        ppm = sf - 2 if reduced else sf
        base = k1_batch(sf, osr, np.random.default_rng(10 * sf + reduced + osr), n_clean=3)
        for n in sorted({1, base.shape[0], pp + 1}):
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
            check_llrs(llr.cpu().numpy().reshape(n, ppm), bins.cpu().numpy().astype(np.int64), K1ReferenceOsr(x, sf, down, osr=osr), sf,
                       reduced, f"SF{sf} D={osr} reduced={reduced} n={n}")
            assert torch.equal(bins, kb) and torch.equal(llr, llr2)
            del xd
    dec.close()


@pytest.mark.parametrize("osr", RATES)
@pytest.mark.parametrize("sf", range(7, 13))
def test_demod_fft_antennas_dev_against_float64(torch, sf, osr):
    """The combined screen of 3 groups x 2 antennas: each argmax inside the float64 combined band; two runs identical."""
    dec = make_dec(sf, osr)
    sps = osr << sf
    rng = np.random.default_rng(sf * 3 + osr)
    base = k1_batch(sf, osr, rng, n_clean=6)
    ng, m = 3, 2
    n = max(base.shape[0], batch(sf, osr) + 1)
    X = np.stack([np.resize(np.roll(base, k, axis=0), (n, sps)) * (0.5 + rng.uniform()) for k in range(ng * m)])
    X = np.ascontiguousarray(X.reshape(ng * m, n * sps), np.complex64)
    xd = torch.from_numpy(X).cuda()
    out = []
    for _ in range(2):
        bins = torch.zeros(ng * n, dtype=torch.int32, device="cuda")
        mags = torch.zeros(ng * n, dtype=torch.float32, device="cuda")
        dec.demod_fft_antennas(xd, ng, m, n, n * sps, bins, mags)
        out.append((bins, mags))
    torch.cuda.synchronize()
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    b, mg = out[0][0].cpu().numpy().reshape(ng, n), out[0][1].cpu().numpy().reshape(ng, n)
    for g in range(ng):
        CombinedReference(X[g * m: g * m + m].reshape(m, n, sps), sf, osr).check(b[g], mg[g], f"SF{sf} D={osr} group {g}")
    dec.close()


@pytest.mark.parametrize("osr", RATES)
@pytest.mark.parametrize("sf", [7, 9, 12])
def test_window_sums_across_the_band(torch, sf, osr):
    """rs_window_dev on a 2^24-sample row: window sums against float64 at |cfo_bins| up to (D - 1) N / 2, the edge of the
    sampled band, both chirps and the special bins."""
    sps, N = osr << sf, 1 << sf
    rng = np.random.default_rng(40 * osr + sf)
    n = (1 << 24) + 3
    down, up, _ = tables(sf, osr)
    dec = make_dec(sf, osr)
    g = torch.Generator(device="cuda").manual_seed(sf + osr)
    row = torch.randn(1, n, dtype=torch.complex64, device="cuda", generator=g)
    q = 32
    pos = np.concatenate([[0, n - sps], rng.integers(0, n - sps, q - 2)]).astype(np.int64)
    lim = (osr - 1) * N / 2
    cfo = rng.uniform(-lim, lim, q).astype(np.float32)
    cfo[:4] = [lim, -lim, N / 4, 0.5]
    bins = np.resize([0, 1, -1, 8, 16, -N // 2, N // 2 - 1], q).astype(np.int32)
    upf = rng.integers(0, 2, q).astype(np.int32)
    out = torch.zeros(q, dtype=torch.complex64, device="cuda")
    dec.rs_window(row, n, pos, cfo, upf, bins, out)
    idx = torch.from_numpy(pos).cuda()[:, None] + torch.arange(sps, device="cuda")[None, :]
    W = row[0, idx].cpu().numpy()
    got = out.cpu().numpy()
    for i in range(q):
        X, tol = window_sum(W[i], up if upf[i] else down, pos[i], cfo[i], bins[i])
        assert abs(got[i] - X) <= tol, (i, int(pos[i]), float(cfo[i]), int(bins[i]), got[i], X, tol)
    dec.close()


# ---- the receiver against its host emulation ------------------------------------------------------------------------------------
def rows(sf, osr, snr_db, n_rx, m, seed, cfo_lim):
    """n_rx receivers of m rows with one frame each (random CFO within +-cfo_lim bins, start, payload, gains), equal length."""
    rng = np.random.default_rng(seed)
    sps = osr << sf
    out, truth = [], []
    for k in range(n_rx):
        pay = bytes(rng.integers(0, 256, 10, dtype=np.uint8))
        cfo = float(rng.uniform(-cfo_lim, cfo_lim)) * BW / (1 << sf)
        gains = [1.0] if m == 1 else list(np.exp(2j * np.pi * rng.uniform(size=m)) * rng.uniform(0.7, 1.3, m))
        X, lead, _ = frame_rows(sf, osr, pay, cfo, int(rng.integers(0, sps)), gains, snr_db=snr_db, seed=seed * 10 + k, tail=3 + k % 2)
        out.append(X)
        truth.append((lead, pay))
    L = max(x.shape[1] for x in out)
    Y = np.zeros((n_rx * m, L), np.complex64)
    for k, x in enumerate(out):
        Y[k * m: k * m + m, : x.shape[1]] = x
    return Y, truth


VARIANTS = [dict(), dict(soft=True), dict(soft=True, crc_list=4), dict(m=2), dict(wide=True), dict(fine_toa=True),
            dict(m=2, soft=True, wide=True, fine_toa=True)]


@pytest.mark.parametrize("osr", RATES)
@pytest.mark.parametrize("sf", [7, 8])
@pytest.mark.parametrize("variant", range(len(VARIANTS)))
def test_receive_matches_host_emulation(torch, sf, osr, variant):
    """Per receiver, 2 dB above the sensitivity point: the device publishes the payloads the host emulation publishes, and
    frames at the same start have the same payload, CFOs within 1e-3 bin and (fine_toa) toa within 1e-3 sample."""
    v = VARIANTS[variant]
    m, soft, wide, toa = v.get("m", 1), v.get("soft", False), v.get("wide", False), v.get("fine_toa", False)
    N = 1 << sf
    lim = (osr - 1) * N / 2
    n_rx = 6
    Y, truth = rows(sf, osr, SENSITIVITY[sf] + 2.0, n_rx, m, seed=sf * 100 + osr + variant, cfo_lim=(0.9 * lim if wide else 0.9 * N / 4))
    dec = make_dec(sf, osr, n_streams=n_rx * m, max_items_per_call=Y.shape[1])
    kw = dict(soft=soft, antennas=m, crc_list=v.get("crc_list", 0), fine_toa=toa)
    if wide:
        kw.update(wide_cfo=True, max_cfo_hz=lim * BW / N)
    _, frames, info = dec.receive(Y, **kw)
    toas = dec.rx_toa_last() if toa else None
    dev = {}
    for k, (f, i) in enumerate(zip(frames, info)):
        dev.setdefault(int(f["stream"]), []).append((int(i["start"]), float(i["cfo_hz"]) / (BW / N), bytes(f["bytes"][18: int(f["len"])]),
                                                     float(toas[k]) if toa else 0.0))
    for r in range(n_rx):
        X = Y[r * m: r * m + m] if m > 1 else Y[r]
        host = [(g["start"], g["cfo"], g["payload"], g["toa"]) for g in receive(X, sf, osr, soft=soft, max_cfo_bins=lim if wide else 0.0)
                if g["status"] == 0]
        d = dev.get(r, [])
        assert {a[2] for a in d} == {b[2] for b in host}, (r, d, host)
        assert truth[r][1] in {a[2] for a in d}, (r, d)
        for a in d:
            for b in host:
                if a[0] == b[0]:
                    assert a[2] == b[2] and abs(a[1] - b[1]) <= 1e-3, (r, a, b)
                    if toa:
                        assert abs(a[3] - b[3]) <= 1e-3, (r, a, b)
    dec.close()


# ---- sensitivity, noise, drift ---------------------------------------------------------------------------------------------------
def n_items_for(sf, osr, n_bytes, rr, scale=1.0):
    import gr_lora_b200 as G
    sps = osr << sf
    return int((12 + G.tx_frame_symbols(n_bytes, sf, 4, False, True, rr)) * sps * scale + sps // 4 + 9 * sps) // 2 * 2


@pytest.mark.parametrize("osr", RATES)
def test_sensitivity_points(torch, osr):
    """48 frames per SF at the fs/bw = 8 sensitivity points (SF7 -2 ... SF12 -15 dB in 125 kHz, SF11/12 reduced rate), at 2 MS/s
    (D = 16) or 4 MS/s (D = 32): all decode, hard and soft, and nothing is published that was not sent."""
    for sf, snr in SENSITIVITY.items():
        rr, ns = sf >= 11, 48
        rng = np.random.default_rng(sf + osr)
        pays = [[bytes(rng.integers(0, 256, 10, dtype=np.uint8))] for _ in range(ns)]
        n_items = n_items_for(sf, osr, 10, rr)
        out, placed = synth_antennas(torch, sf, osr, pays, n_items, snr, np.ones((ns, 1)), seed=3000 + sf + osr, rr=rr)
        sent = {(s, p) for s, _, p in placed}
        assert len(sent) == ns
        for soft in (False, True):
            rx = make_dec(sf, osr, rr, n_streams=ns, max_items_per_call=n_items)
            _, frames, _ = rx.receive(out, n_items=n_items, soft=soft)
            got = [(int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in frames]
            print(f"fs/bw = {osr}, SF{sf} at {snr:+.1f} dB: {'soft' if soft else 'hard'} {len(set(got) & sent)}/{ns}")
            assert all(g in sent for g in got) and len(set(got) & sent) == ns, (sf, snr, soft)
            rx.close()
        del out


@pytest.mark.parametrize("osr", RATES)
def test_pure_noise_through_the_widest_search(torch, osr):
    """16 streams x 0.5 s of noise through wide_cfo at max_cfo_hz = (fs - BW) / 2: nothing published, hard or soft."""
    for sf in (7, 9):
        fs = osr * BW
        x = torch.randn(16, int(0.5 * fs), dtype=torch.complex64, device="cuda")
        for soft in (False, True):
            rx = make_dec(sf, osr, n_streams=16, max_items_per_call=x.shape[1])
            _, frames, _ = rx.receive(x, n_items=x.shape[1], soft=soft, wide_cfo=True, max_cfo_hz=(fs - BW) / 2)
            assert len(frames) == 0, (sf, soft, len(frames))
            rx.close()


@pytest.mark.parametrize("osr", RATES)
@pytest.mark.parametrize("ppm", [20.0, -20.0])
def test_sf12_drifted_frames_decode_with_carrier(torch, osr, ppm):
    """SF12 64-byte frames from transmitters whose crystal is off by +-20 ppm (carrier and clock), found through carrier_hz."""
    sf, ns = 12, 3
    rng = np.random.default_rng(abs(int(ppm)) * 10 + osr + (ppm < 0))
    pays = [[bytes(rng.integers(0, 256, 64, dtype=np.uint8))] for _ in range(ns)]
    n_items = n_items_for(sf, osr, 64, True, 1.001)
    out, placed = synth_antennas(torch, sf, osr, pays, n_items, 0.0, np.ones((ns, 1)), seed=77 + int(ppm), rr=True, sfo_ppm=ppm,
                                 cfo=[[ppm * CARRIER * 1e-6] for _ in range(ns)])
    rx = make_dec(sf, osr, True, n_streams=ns, max_items_per_call=n_items)
    _, frames, info = rx.receive(out, n_items=n_items, carrier_hz=CARRIER)
    assert {(int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in frames} == {(s, p) for s, _, p in placed}
    assert all(abs(float(i["sfo_ppm"]) - ppm) < 0.5 for i in info)
    rx.close()


def test_narrow_channel_with_crystal_offsets(torch):
    """A 31.25 kHz channel at 1 MS/s (D = 32), SF9, transmitters with +-20 ppm crystals at 868.1 MHz (+-17.4 kHz: more than half
    the bandwidth), received with wide_cfo and carrier_hz."""
    import gr_lora_b200 as G
    from gr_lora_b200 import tx
    sf, osr, bw, ns = 9, 32, 31250.0, 8
    fs = osr * bw
    rng = np.random.default_rng(31)
    ppms = rng.uniform(-20, 20, ns)
    ppms[:2] = [20.0, -20.0]
    pays = [[bytes(rng.integers(0, 256, 12, dtype=np.uint8))] for _ in range(ns)]
    sps = osr << sf
    n_items = int((12 + G.tx_frame_symbols(12, sf, 4, False, True, False)) * sps * 1.0001 + 9 * sps) // 2 * 2
    gen = make_dec(sf, osr, bw=bw)
    up = torch.from_numpy(tx.base_upchirp(sf, bw, fs).astype(np.complex64)).cuda()
    out, placed = gen.synth_streams(pays, n_items, lead_symbols=2.0, gap_symbols=4.0, cfo_hz=[[p * CARRIER * 1e-6] for p in ppms],
                                    noise_sigma=float(np.sqrt(10 ** (-(0.0 - 10 * np.log10(osr)) / 10) / 2)), seed=5, up_table_dev=up,
                                    sfo_ppm=[[float(p)] for p in ppms])
    torch.cuda.synchronize()
    gen.close()
    rx = make_dec(sf, osr, bw=bw, n_streams=ns, max_items_per_call=n_items)
    _, frames, info = rx.receive(out, n_items=n_items, carrier_hz=CARRIER, wide_cfo=True, max_cfo_hz=20e-6 * CARRIER * 1.1)
    got = {(int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in frames}
    assert got == {(s, p) for s, _, p in placed}
    for i in info:
        assert abs(float(i["sfo_ppm"]) - ppms[int(i["stream"])]) < 0.5, (i, ppms)
    rx.close()


# ---- the channelizer at decimation=1 ------------------------------------------------------------------------------------------
def test_channelizer_decimation_1_matches_decimation_2(torch):
    """A 2 MS/s capture through lora_receiver(2e6, c, [c], 125000, decimation=1, sync="dechirp") -- fs/bw = 16 -- publishes the
    payloads decimation=2 (fs/bw = 8) publishes, 1.5 dB above the sensitivity points."""
    import gr_lora_b200 as G
    from gr_lora_b200 import tx
    center = 868.1e6
    fs = 2e6
    for sf in (7, 8, 9):
        snr = SENSITIVITY[sf] + 1.5
        rng = np.random.default_rng(sf + 600)
        pays = [bytes(rng.integers(0, 256, 10, dtype=np.uint8)) for _ in range(5)]
        gen = make_dec(sf, 16)
        up = torch.from_numpy(tx.base_upchirp(sf, BW, fs).astype(np.complex64)).cuda()
        sps = 16 << sf
        n_items = int(len(pays) * (12 + G.tx_frame_symbols(10, sf, 4, False, True, False) + 8) * sps + 8 * sps) // 16 * 16
        cfo = [[float(rng.uniform(-0.5, 0.5) * BW / 4) for _ in pays]]
        out, placed = gen.synth_streams([pays], n_items, lead_symbols=2.37, gap_symbols=4.61, cfo_hz=cfo,
                                        noise_sigma=float(math.sqrt(10 ** (-(snr - 10 * math.log10(16)) / 10) / 2)), seed=sf, up_table_dev=up)
        torch.cuda.synchronize()
        gen.close()
        x = out[0].cpu().numpy()
        res = {}
        for decim in (1, 2):
            rx = G.lora_receiver(fs, center, [center], 125000, sf, False, 4, True, decimation=decim, sync="dechirp", quiet=True)
            rx.run(x)
            res[decim] = [bytes(f[18:]) for _, f in rx.frames]
        sent = [p for _, _, p in placed]
        print(f"SF{sf} at {snr:+.1f} dB: decimation 1 {len(res[1])}, decimation 2 {len(res[2])} of {len(sent)}")
        assert res[1] == res[2] == sent, (sf, res, sent)
