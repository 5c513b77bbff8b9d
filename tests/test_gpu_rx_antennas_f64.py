"""The several-antenna dechirp receiver's arithmetic on the device against float64 (tests/antenna_reference.py): the
synchroniser's window sums, energies and argmax per antenna (lora_b200_rs_window_dev, M = 1..4), the channel estimates,
weights and combined SNR and the assembled data windows of given frames (lora_b200_rs_frame_dev), the same quantities on
the frames lora_b200_receive_antennas publishes, and the receiver's invariance to the input's scale."""
import math

import numpy as np
import pytest

from antenna_common import BW, SENSITIVITY, CombinedReference, frame_rows, synth_antennas, tables
from antenna_reference import ENERGY_TOL, ChannelReference, assembly_windows, rs_sym, window_energy, window_sum

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


def gains_db(rng, m, spread):
    return 10 ** (rng.uniform(-spread, spread, m) / 20) * np.exp(2j * np.pi * rng.uniform(size=m))


# ---- window sums and argmax ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf", range(7, 13))
def test_window_sums_per_antenna_against_float64(torch, sf, osr):
    """M = 1..4 rows of at least 2^24 samples (noise at +10 dB, a frame at the end with per-antenna gains within +-10 dB and
    random phases), rows a multiple of sps apart (M = 1, 3) and not (M = 2, 4): at random unaligned positions on the frame
    and on noise, both chirps, CFOs within +-N/4 and the special bins, each antenna's binval within the window-sum bound
    and its energy within 1e-5, and the argmax of the combined spectrum inside antenna_common.CombinedReference's band."""
    sps, N = osr << sf, 1 << sf
    rng = np.random.default_rng(1000 + 10 * sf + osr)
    pay = bytes(rng.integers(0, 256, 8, dtype=np.uint8))
    F, _, L = frame_rows(sf, osr, pay, float(rng.uniform(-0.9, 0.9) * BW / 4), int(rng.integers(0, sps)), list(gains_db(rng, 4, 10)),
                         rr=sf > 10)
    L = F.shape[1]
    n = max(1 << 24, 2 * L) + 3
    down, up, _ = tables(sf, osr)
    dec = make_dec(sf, osr, sf > 10)
    g = torch.Generator(device="cuda").manual_seed(sf * 10 + osr)
    sigma = math.sqrt(10 ** (-(10.0 - 10 * math.log10(osr)) / 10) / 2)
    worst = {}
    for m in (1, 2, 3, 4):
        stride = (n + sps - 1) // sps * sps if m % 2 else n + 5
        rows = torch.randn(m, stride, dtype=torch.complex64, device="cuda", generator=g) * sigma
        rows[:, n - L: n] += torch.from_numpy(F[:m]).cuda()
        q = 48
        pos = np.concatenate([[0, n - sps], rng.integers(0, n - sps, q // 4 - 2), rng.integers(n - L, n - sps, q - q // 4)]).astype(np.int64)
        cfo = rng.uniform(-N / 4, N / 4, q).astype(np.float32)
        cfo[:8] = [0.0, 0.5, -0.5, 1.0, -3.0, N / 4, -N / 4, 7.25]
        special = [0, 1, -1, (0x1 * 8) % N, (0x2 * 8) % N, -N // 2, N // 2 - 1]
        bins = np.concatenate([np.resize(special, q // 2), rng.integers(-N // 2, N // 2, q - q // 2)]).astype(np.int32)
        upf = rng.integers(0, 2, q).astype(np.int32)
        out = torch.zeros(q * m, dtype=torch.complex64, device="cuda")
        en = torch.zeros(q * m, dtype=torch.float32, device="cuda")
        kb = torch.zeros(q, dtype=torch.int32, device="cuda")
        km = torch.zeros(q, dtype=torch.float32, device="cuda")
        dec.rs_window(rows, n, pos, cfo, upf, bins, out, en, kb, km, antennas=m, stride=stride)
        idx = torch.from_numpy(pos).cuda()[:, None] + torch.arange(sps, device="cuda")[None, :]
        W = rows[:, idx].cpu().numpy()                                        # [m, q, sps]
        del rows
        got, got_e = out.cpu().numpy().reshape(q, m), en.cpu().numpy().reshape(q, m)
        wr = 0.0
        for i in range(q):
            for a in range(m):
                X, tol = window_sum(W[a, i], up if upf[i] else down, pos[i], cfo[i], bins[i])
                wr = max(wr, abs(got[i, a] - X) / tol)
                assert abs(got[i, a] - X) <= tol, (m, i, a, int(pos[i]), float(cfo[i]), int(bins[i]), int(upf[i]), got[i, a], X, tol)
                e = window_energy(W[a, i])
                assert abs(got_e[i, a] - e) <= ENERGY_TOL * e, (m, i, a, got_e[i, a], e)
        kbh, kmh = kb.cpu().numpy(), km.cpu().numpy()
        for u in (0, 1):
            sel = upf == u
            CombinedReference(W[:, sel], sf, osr, chirp=up if u else down).check(kbh[sel], kmh[sel], f"SF{sf} fs/bw={osr} M={m} up={u}")
        worst[m] = wr
    print(f"SF{sf} fs/bw={osr}: worst window-sum err/bound " + ", ".join(f"M={m} {v:.3f}" for m, v in worst.items()))
    dec.close()


# ---- channel estimates, weights, SNR and assembly of given frames ----------------------------------------------------------------
LEVELS = {2: [10.0, 4.0], 3: [10.0, 4.0, -10.0], 4: [10.0, 4.0, -10.0, None]}     # noise 0, 6 and 20 dB apart, a noiseless row
PPMS = [0.0, 20.0, -20.0, 200.0, -200.0]


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("m", [2, 3, 4])
def test_channels_weights_snr_and_assembly_of_given_frames(torch, m, osr):
    """SF8 frames on M antennas with per-antenna noise 0, 6 and 20 dB apart (M = 4: one row noiseless, the floor), clock
    offsets 0, +-20 and +-200 ppm, one frame whose first preamble windows precede the row start: h, w, snr_db within the
    float64 bounds carried from the window sums, and data windows 0..5 within the assembly bound."""
    sf = 8
    sps, nb = osr << sf, 1 << sf
    rng = np.random.default_rng(50 * m + osr)
    frames, rows = [], []
    for k, ppm in enumerate(PPMS + [0.0]):
        cfo = float(np.float32(rng.uniform(-0.9, 0.9) * nb / 4))
        X, lead, _ = frame_rows(sf, osr, bytes(rng.integers(0, 256, 8, dtype=np.uint8)), cfo * BW / nb, int(rng.integers(0, sps)),
                                list(gains_db(rng, m, 3)), snr_db=LEVELS[m], seed=int(rng.integers(1 << 30)), sfo_ppm=ppm)
        if k == len(PPMS):                              # the row starts inside the preamble: windows 1 and 2 before it
            cut = lead + 2 * sps + sps // 3
            X, lead = X[:, cut:], lead - cut
        frames.append((lead, cfo, ppm))
        rows.append(X)
    n = max(X.shape[1] for X in rows)
    Y = np.zeros((m * len(rows), n), np.complex64)
    for g, X in enumerate(rows):
        Y[g * m: g * m + m, : X.shape[1]] = X
    nf, cnt = len(frames), 6
    dec = make_dec(sf, osr)
    yd = torch.from_numpy(Y).cuda()
    chan = torch.zeros((nf, 8), dtype=torch.complex64, device="cuda")
    snr = torch.zeros(nf, dtype=torch.float32, device="cuda")
    win = torch.zeros((nf, cnt, sps), dtype=torch.complex64, device="cuda")
    dec.rs_frame(yd, n, np.arange(nf), [f[0] for f in frames], [f[1] for f in frames], [f[2] for f in frames], 0, cnt, win, chan, snr,
                 antennas=m, stride=n)
    chan, snr, win = chan.cpu().numpy(), snr.cpu().numpy(), win.cpu().numpy()
    down = tables(sf, osr)[0]
    worst = dict(h=0.0, w_mag=0.0, w_phase=0.0, snr=0.0, asm=0.0)
    for g, (start, cfo, ppm) in enumerate(frames):
        Yg = Y[g * m: g * m + m].astype(np.complex128)
        ref = ChannelReference(Yg, n, start, cfo, ppm, down, osr)
        tag = f"M={m} fs/bw={osr} frame {g} ppm {ppm}"
        if g == len(PPMS):
            assert ref.nw == 4, ref.nw
        worst["h"] = max(worst["h"], ref.check_h(chan[g, :m], tag))
        wm, wp = ref.check_w(chan[g, 4: 4 + m], tag)
        worst["w_mag"], worst["w_phase"] = max(worst["w_mag"], wm), max(worst["w_phase"], wp)
        worst["snr"] = max(worst["snr"], ref.check_snr(float(snr[g]), tag))
        assert np.all(chan[g, m:4] == 0) and np.all(chan[g, 4 + m:] == 0)
        y, bound = assembly_windows(Y[g * m: g * m + m], n, sps, start, cfo, ppm, 0, cnt, chan[g, 4: 4 + m])
        err = np.abs(win[g] - y)
        assert np.all(err <= bound), (tag, float(np.max(err / np.maximum(bound, 1e-300))))
        worst["asm"] = max(worst["asm"], float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), 0.0))))
    print(f"M={m} fs/bw={osr}: worst err/bound " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
    dec.close()


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("m", [1, 2, 3, 4])
def test_assembly_past_two_to_the_24_against_float64(torch, m, osr):
    """Data windows of frames that start beyond 2^24 samples, clock offsets 0, +-20 and +-500 ppm, the last window crossing
    n_items: rs_assemble_kernel (M = 1) and rs_assemble_antennas_kernel (with the weights rs_channels gives) within the
    assembly bound, the samples past n_items 0."""
    sf, cnt = 8, 6
    sps = osr << sf
    rng = np.random.default_rng(70 * m + osr)
    base = (1 << 24) - 4 * sps
    ppms = [0.0, 20.0, -20.0, 500.0, -500.0]
    starts = [(1 << 24) + int(rng.integers(0, 1 << 20)) for _ in ppms]
    n = max(rs_sym(s, 12.25 + cnt - 1, sps, p) for s, p in zip(starts, ppms)) + sps // 2
    ng = len(ppms)
    R = (rng.standard_normal((ng * m, n - base)) + 1j * rng.standard_normal((ng * m, n - base))).astype(np.complex64)
    yd = torch.zeros((ng * m, n), dtype=torch.complex64, device="cuda")
    yd[:, base:] = torch.from_numpy(R).cuda()
    cfos = rng.uniform(-0.9, 0.9, ng).astype(np.float32) * ((1 << sf) / 4)
    chan = torch.zeros((ng, 8), dtype=torch.complex64, device="cuda")
    snr = torch.zeros(ng, dtype=torch.float32, device="cuda")
    win = torch.zeros((ng, cnt, sps), dtype=torch.complex64, device="cuda")
    dec = make_dec(sf, osr)
    dec.rs_frame(yd, n, np.arange(ng), starts, cfos, ppms, 0, cnt, win, chan if m > 1 else None, snr if m > 1 else None,
                 antennas=m, stride=n)
    chan, win = chan.cpu().numpy(), win.cpu().numpy()
    worst, crossed = 0.0, 0
    for g in range(ng):
        w = chan[g, 4: 4 + m] if m > 1 else np.ones(1, np.complex64)
        y, bound = assembly_windows(R[g * m: g * m + m], n, sps, starts[g], cfos[g], ppms[g], 0, cnt, w, base=base)
        err = np.abs(win[g] - y)
        assert np.all(err <= bound), (g, ppms[g], float(np.max(err / np.maximum(bound, 1e-300))))
        assert np.all(win[g][bound == 0] == 0)
        crossed += int(np.any(bound[-1] == 0))
        worst = max(worst, float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), 0.0))))
    assert crossed >= 1
    print(f"M={m} fs/bw={osr}: assembly past 2^24 worst err/bound {worst:.3f}")
    dec.close()


# ---- the published path ------------------------------------------------------------------------------------------------------------
def recovered_cfo_bins(cfo_hz, bin_hz):
    """rx_info's cfo_hz is the float32 product cfo_bins * bin_hz: the float32 nearest cfo_hz / bin_hz and its two neighbours,
    those of them that map back to cfo_hz exactly.  The product is not one to one (where c bin_hz crosses a power of two
    two neighbouring c can round to one product), so more than one may."""
    c = np.float32(float(cfo_hz) / float(bin_hz))
    cands = (np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf)))
    return [float(v) for v in cands if np.float32(v * np.float32(bin_hz)) == np.float32(cfo_hz)]


@pytest.mark.parametrize("m", [2, 3, 4])
def test_published_channels_and_snr_against_float64(torch, m):
    """receive(antennas=M), SF8 and SF10, antennas' noise 0, 6 and 20 dB apart (the fourth 3 dB below the first), the first
    antenna at +10 dB and at the sensitivity point: at each published frame's start, clock offset and CFO, rx_channels_last()
    and rx_info.snr_db within the float64 bounds; against the true combined SNR, 10 log10 sum_a |g_a|^2 / sigma_a^2, a mean
    error within 0.5 dB and every frame within 1.5 dB.  The CFO in bins is recovered from rx_info.cfo_hz; where two float32
    values map to it, the frame passes at either.  Every frame is published at +10 dB; at the sensitivity point the antenna
    20 dB noisier dilutes the unweighted power sums of the screen and the synchroniser (DESIGN section 5), and whatever is
    published is checked."""
    offs = [0.0, -6.0, -20.0, -3.0][:m]
    for sf in (8, 10):
        osr, n_rx = 8, 8
        sps, nb = osr << sf, 1 << sf
        bin_hz = np.float32(np.float32(osr * BW) / np.float32(sps))
        down = tables(sf, osr)[0]
        for top in (10.0, SENSITIVITY[sf]):
            rng = np.random.default_rng(sf * 100 + m + int(top))
            rows, truth = [], []
            for g in range(n_rx):
                gains = [1.0] + list(gains_db(rng, m - 1, 3))
                X, _, _ = frame_rows(sf, osr, bytes(rng.integers(0, 256, 8, dtype=np.uint8)), float(rng.uniform(-0.9, 0.9) * BW / 4),
                                     int(rng.integers(0, sps)), gains, snr_db=[top + o for o in offs], seed=int(rng.integers(1 << 30)))
                rows.append(X)
                s2 = np.array([10 ** (-(top + o) / 10) for o in offs])            # in 125 kHz, for a unit gain
                truth.append(10 * math.log10(np.sum(np.abs(gains) ** 2 / s2)))
            n = max(X.shape[1] for X in rows)
            Y = np.zeros((m * n_rx, n), np.complex64)
            for g, X in enumerate(rows):
                Y[m * g: m * g + m, : X.shape[1]] = X
            dec = make_dec(sf, osr, n_streams=m * n_rx, max_items_per_call=n)
            _, frames, info = dec.receive(Y, antennas=m)
            h = dec.rx_channels_last()
            dec.close()
            if top >= 10.0:
                assert len(frames) == n_rx, (sf, top, len(frames))
            err, inexact, twice, wh, ws = [], 0, 0, 0.0, 0.0
            for k, i in enumerate(info):
                g = int(i["stream"])
                cands = recovered_cfo_bins(i["cfo_hz"], bin_hz)
                inexact += not cands
                twice += len(cands) > 1
                tag = f"SF{sf} M={m} {top:+.1f} dB receiver {g}"
                fails = []
                for cfo in cands:
                    ref = ChannelReference(Y[m * g: m * g + m], n, int(i["start"]), cfo, float(i["sfo_ppm"]), down, osr)
                    try:
                        r = ref.check_h(h[k], tag), ref.check_snr(float(i["snr_db"]), tag)
                    except AssertionError as e:
                        fails.append(str(e))
                        continue
                    wh, ws = max(wh, r[0]), max(ws, r[1])
                    break
                else:
                    raise AssertionError(fails or f"{tag}: cfo_hz {float(i['cfo_hz'])} is no float32 cfo_bins times bin_hz")
                err.append(float(i["snr_db"]) - truth[g])
            err = np.array(err) if err else np.zeros(1)
            print(f"SF{sf} M={m} at {top:+.1f} dB: {len(frames)} of {n_rx} frames, cfo_bins not recovered on {inexact}, two candidates "
                  f"on {twice}; worst err/bound h {wh:.3f}, snr_db {ws:.3f}; SNR against the truth: mean {err.mean():+.3f} dB, max |error| "
                  f"{np.abs(err).max():.3f} dB")
            assert inexact == 0
            assert abs(err.mean()) <= 0.5 and np.abs(err).max() <= 1.5, (sf, top, err)


# ---- scale invariance ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 2, 4])
def test_receiver_is_invariant_to_the_input_scale(torch, m):
    """The input times 2^k, k = -24, -12, 12 and 15 (15: int16 full scale), hard, soft and soft with crc_list = 8: consumed,
    frame records and rx_info byte-identical, and h exactly 2^k times the unscaled call's."""
    sf, osr, ng = 8, 8, 6
    rng = np.random.default_rng(300 + m)
    pays = [[bytes(rng.integers(0, 256, 10, dtype=np.uint8))] for _ in range(ng)]
    import gr_lora_b200 as G
    n = int((12 + G.tx_frame_symbols(10, sf, 4, False, True, False)) * (osr << sf) + 10 * (osr << sf)) // 8 * 8
    x, _ = synth_antennas(torch, sf, osr, pays, n, SENSITIVITY[sf] + 1.0, gains_db(rng, ng * m, 6).reshape(ng, m), seed=400 + m)
    for mode in (dict(), dict(soft=True), dict(soft=True, crc_list=8)):
        dec = make_dec(sf, osr, n_streams=ng * m, max_items_per_call=n)
        c0, f0, i0 = dec.receive(x, n_items=n, antennas=m, **mode)
        h0 = dec.rx_channels_last()
        assert len(f0) >= ng - 1, (mode, len(f0))
        for k in (-24, -12, 12, 15):
            xs = x * (2.0 ** k)
            torch.cuda.synchronize()
            c, f, i = dec.receive(xs, n_items=n, antennas=m, **mode)
            h = dec.rx_channels_last()
            assert np.array_equal(c, c0) and f.tobytes() == f0.tobytes() and i.tobytes() == i0.tobytes(), (mode, k)
            assert np.array_equal(h, (h0.astype(np.complex128) * 2.0 ** k).astype(np.complex64)), (mode, k)
        dec.close()
