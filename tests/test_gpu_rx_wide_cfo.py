"""GPU: the dechirp receiver's coarse-offset search (lora_b200_rx_params.wide_cfo).  Off means off; a search no wider than
BW/4 gives the bytes of the receiver without it; the device matches the host emulation frame by frame on wide-offset
captures; frames 0.25..0.75 BW off carrier decode at the sensitivity point; a narrow-band (31.25 kHz) receiver follows +-20 ppm
crystals at 868.1 MHz; noise publishes nothing through the widest search; the window sums hold to float64 at the widest
offsets; argument errors launch nothing; lora_receiver passes the option through."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from antenna_common import BW, SENSITIVITY, frame_rows, tables
from antenna_reference import window_sum
from wide_cfo_common import dedup, receive_wide

pytestmark = pytest.mark.gpu

CARRIER = 868.1e6


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def make_dec(sf, osr=8, rr=False, bw=BW, **kw):
    import gr_lora_b200 as G
    return G.decoder(osr * bw, bw, sf, False, 4, True, rr, quiet=True, **kw)


def sigma_for(snr_db, osr=8):
    return float(np.sqrt(10 ** (-(snr_db - 10 * np.log10(osr)) / 10) / 2))


def frame_len(sf, plen, osr=8, rr=False):
    import gr_lora_b200 as G
    return (12 + G.tx_frame_symbols(plen, sf, 4, False, True, rr)) * (osr << sf) + (osr << sf) // 4


def synth(torch, sf, n_streams, snr_db, seed, cfo_lo, cfo_hi, osr=8, bw=BW, rr=None, plen=10, sfo_ppm=None):
    """One frame per stream with a CFO uniform in +-[cfo_lo, cfo_hi] BW (a random sign; with sfo_ppm, a per-frame crystal
    offset in ppm sets its CFO ppm * 868.1 Hz and its clock instead).  Returns (device rows, placed, cfo per stream, n_items)."""
    from gr_lora_b200 import tx
    rr = sf >= 11 if rr is None else rr
    rng = np.random.default_rng(seed)
    sps = osr << sf
    n_items = (frame_len(sf, plen, osr, rr) + 9 * sps) // 2 * 2
    pays = [[bytes(rng.integers(0, 256, plen, dtype=np.uint8))] for _ in range(n_streams)]
    kw = {}
    if sfo_ppm is None:
        cfo = [float(rng.choice((-1.0, 1.0)) * rng.uniform(cfo_lo, cfo_hi) * bw) for _ in range(n_streams)]
    else:
        ppm = [float(rng.uniform(-sfo_ppm, sfo_ppm)) for _ in range(n_streams)]
        cfo = [e * CARRIER * 1e-6 for e in ppm]
        kw["sfo_ppm"] = [[e] for e in ppm]
    gen = make_dec(sf, osr, rr, bw=bw)
    up = torch.from_numpy(tx.base_upchirp(sf, bw, osr * bw).astype(np.complex64)).cuda()
    out, placed = gen.synth_streams(pays, n_items, lead_symbols=float(rng.uniform(1.0, 3.0)), gap_symbols=4.0, cfo_hz=[[c] for c in cfo],
                                    noise_sigma=sigma_for(snr_db, osr), seed=seed, up_table_dev=up, **kw)
    torch.cuda.synchronize()
    gen.close()
    return out, placed, cfo, n_items


def decoded(frames, info, placed, cfo, tol_hz):
    """Per placed frame: decoded byte-exact with its CFO within tol_hz (rx_info)."""
    ok = []
    for s, _, p in placed:
        hit = False
        for r, i in zip(frames, info):
            if int(r["stream"]) == s and bytes(r["bytes"][18: int(r["len"])]) == p and abs(float(i["cfo_hz"]) - cfo[s]) <= tol_hz:
                hit = True
        ok.append(hit)
    return np.array(ok)


def records(frames, info, crc):
    return frames.tobytes(), info.tobytes(), np.asarray(crc).tobytes()


@pytest.mark.parametrize("sf,osr", [(7, 8), (10, 8), (8, 2)])
@pytest.mark.parametrize("soft", [False, True])
def test_search_within_bw4_is_byte_identical(torch, sf, osr, soft):
    """wide_cfo = 1 with max_cfo_hz <= BW/4 publishes the same frames, rx_info and CRC status bytes as wide_cfo = 0."""
    out, placed, _, n_items = synth(torch, sf, 48, SENSITIVITY[sf], 100 + sf, 0.0, 0.24, osr=osr)
    rx = make_dec(sf, osr, sf >= 11, n_streams=48, max_items_per_call=n_items)

    def run(**kw):
        _, f, i = rx.receive(out, n_items=n_items, soft=soft, **kw)
        return records(f, i, rx.frames_crc_last())

    base = run()
    assert len(base[0]) > 0
    assert run(wide_cfo=True, max_cfo_hz=BW / 4) == base
    assert run(wide_cfo=True, max_cfo_hz=0.2 * BW) == run(max_cfo_hz=0.2 * BW)


def _emulate_rows(host, sf, osr, max_bins, soft, m=1):
    def one(g):
        return receive_wide(host[g * m: g * m + m] if m > 1 else host[g], sf, osr, max_bins, soft=soft)
    with ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
        return list(ex.map(one, range(host.shape[0] // m)))


PARITY = [(7, 8, 1, 3.0), (10, 8, 1, 1.2), (12, 8, 1, 0.75), (7, 2, 1, 0.5), (10, 2, 1, 0.5), (7, 8, 2, 1.2), (10, 2, 2, 0.5)]


@pytest.mark.parametrize("sf,osr,m,max_bw", PARITY, ids=[f"sf{a}-osr{b}-m{c}-{d}bw" for a, b, c, d in PARITY])
@pytest.mark.parametrize("soft", [False, True])
def test_device_matches_emulation(torch, sf, osr, m, max_bw, soft):
    """Frames up to max_bw off carrier, 3 dB above the sensitivity point: every frame the device publishes is one the emulation
    publishes (its one-frame-per-preamble rule applied) -- start within one sample, CFO within 0.02 bin, the same payload -- and
    the emulation's frames are all published."""
    rr = sf >= 11
    N, sps = 1 << sf, osr << sf
    rng = np.random.default_rng(10 * sf + osr + m)
    n_groups = 8 if sf < 12 else 4
    X = []
    for g in range(n_groups):
        cfo = float(rng.choice((-1.0, 1.0)) * rng.uniform(0.25, max_bw - 0.02) * BW)
        snr = SENSITIVITY[sf] + 3.0
        rows, _, _ = frame_rows(sf, osr, bytes(rng.integers(0, 256, 10, dtype=np.uint8)), cfo, int(rng.integers(0, sps)),
                                   [1.0, 0.7 - 0.4j][:m], snr_db=[snr, snr + 2][:m], seed=int(rng.integers(1 << 30)), rr=rr)
        X.append(rows)
    n_items = max(x.shape[1] for x in X)
    host = np.zeros((n_groups * m, n_items), np.complex64)
    for g, rows in enumerate(X):
        host[g * m: g * m + m, : rows.shape[1]] = rows
    rx = make_dec(sf, osr, rr, n_streams=n_groups * m, max_items_per_call=n_items)
    _, frames, info = rx.receive(host, n_items=n_items, soft=soft, antennas=m, wide_cfo=True, max_cfo_hz=max_bw * BW)
    emu = _emulate_rows(host, sf, osr, max_bw * N, soft, m)
    bin_hz = BW / N
    for g in range(n_groups):
        want = [f for f in dedup(emu[g], sps) if f["status"] == 0 and f["start"] + frame_len(sf, 10, osr, rr) <= n_items]
        got = [(int(i["start"]), float(i["cfo_hz"]) / bin_hz, bytes(r["bytes"][18: int(r["len"])]))
               for r, i in zip(frames, info) if int(r["stream"]) == g]
        assert len(got) == len(want), (g, got, want)
        for (st, cf, pay), w in zip(got, want):
            assert abs(st - w["start"]) <= 1 and abs(cf - w["cfo"]) <= 0.02 and pay == w["payload"], (g, st, cf, w)
    assert len(frames) >= n_groups - 1


@pytest.mark.parametrize("sf", sorted(SENSITIVITY))
def test_sensitivity_with_offsets(torch, sf):
    """CFO uniform in +-[0.25, 0.75] BW at each SF's sensitivity point: >= 90 % of the frames decode byte-exact with wide_cfo
    (max_cfo_hz = 0.75 BW), each with its CFO within 1/8 bin.  Without it, none of the frames beyond 0.3 BW is received: no
    published frame carries such a frame's CFO."""
    ns = 48
    out, placed, cfo, n_items = synth(torch, sf, ns, SENSITIVITY[sf], 2000 + sf, 0.25, 0.75)
    rx = make_dec(sf, 8, sf >= 11, n_streams=ns, max_items_per_call=n_items)
    tol = BW / (1 << sf) / 8
    _, f, i = rx.receive(out, n_items=n_items, wide_cfo=True, max_cfo_hz=0.75 * BW)
    ok = decoded(f, i, placed, cfo, tol)
    assert ok.sum() >= 0.9 * len(placed), (sf, int(ok.sum()), len(placed))
    assert len(f) <= len(placed)
    _, f, i = rx.receive(out, n_items=n_items)
    assert np.all(np.abs(i["cfo_hz"]) <= BW / 4 + 1.0)
    far = np.array([abs(cfo[s]) > 0.3 * BW for s, _, _ in placed])
    assert not np.any(decoded(f, i, placed, cfo, 0.05 * BW)[far])


def test_narrow_band_crystals(torch):
    """A 31.25 kHz channel at 250 kS/s (fs/bw = 8), SF10, frames from +-20 ppm crystals at 868.1 MHz (up to 0.56 BW of CFO and
    the clock offset with it), 3 dB above the sensitivity point: with carrier_hz, wide_cfo and max_cfo_hz = 20 kHz every frame
    decodes; without wide_cfo those beyond BW/4 (7.8 kHz) are lost."""
    sf, bw, ns = 10, 31250.0, 32
    out, placed, cfo, n_items = synth(torch, sf, ns, SENSITIVITY[sf] + 3.0, 77, 0, 0, bw=bw, sfo_ppm=20.0)
    rx = make_dec(sf, 8, False, bw=bw, n_streams=ns, max_items_per_call=n_items)
    tol = bw / (1 << sf) / 8
    _, f, i = rx.receive(out, n_items=n_items, carrier_hz=CARRIER, wide_cfo=True, max_cfo_hz=20e3)
    assert decoded(f, i, placed, cfo, tol).all(), (decoded(f, i, placed, cfo, tol), cfo)
    _, f, i = rx.receive(out, n_items=n_items, carrier_hz=CARRIER)
    far = np.array([abs(cfo[s]) > bw / 4 + 500.0 for s, _, _ in placed])
    assert far.sum() >= 8
    assert not np.any(decoded(f, i, placed, cfo, 0.05 * bw)[far])


def test_noise_through_the_widest_search(torch):
    """64 streams x 2 s of pure noise at fs/bw = 8 through the search up to (fs - BW) / 2: nothing is published."""
    sf, ns, n_items = 7, 64, 2_000_000
    g = torch.Generator(device="cuda").manual_seed(3)
    noise = torch.randn((ns, n_items), dtype=torch.complex64, device="cuda", generator=g)
    rx = make_dec(sf, 8, n_streams=ns, max_items_per_call=n_items, max_frames_per_call=64)
    _, frames, _ = rx.receive(noise, n_items=n_items, wide_cfo=True, max_cfo_hz=3.5 * BW)
    assert len(frames) == 0


@pytest.mark.parametrize("sf,osr", [(7, 8), (10, 8), (12, 8), (9, 2)])
def test_window_sums_at_wide_offsets(torch, sf, osr):
    """lora_b200_rs_window_dev at |cfo_bins| up to (D - 1) N / 2 (and N where that is less): each binval within the float64
    window-sum bound."""
    sps, N = osr << sf, 1 << sf
    lim = max(N, (osr - 1) * N / 2)
    rng = np.random.default_rng(sf + osr)
    F, _, _ = frame_rows(sf, osr, b"window sums", float(rng.uniform(-3.0, 3.0) * BW) if osr == 8 else 0.4 * BW, 100, [1.0],
                         snr_db=10.0, rr=sf > 10)
    n = F.shape[1]
    down, up, _ = tables(sf, osr)
    dec = make_dec(sf, osr, sf > 10)
    rows = torch.from_numpy(F).cuda()
    q = 48
    pos = rng.integers(0, n - sps, q).astype(np.int64)
    cfo = rng.uniform(-lim, lim, q).astype(np.float32)
    cfo[:4] = [lim, -lim, lim - 0.5, -lim + 0.25]
    bins = rng.integers(-N // 2, N // 2, q).astype(np.int32)
    upf = rng.integers(0, 2, q).astype(np.int32)
    out = torch.zeros(q, dtype=torch.complex64, device="cuda")
    dec.rs_window(rows, n, pos, cfo, upf, bins, out, antennas=1, stride=n)
    got = out.cpu().numpy()
    for k in range(q):
        X, tol = window_sum(F[0, pos[k]: pos[k] + sps], up if upf[k] else down, pos[k], cfo[k], bins[k])
        assert abs(got[k] - X) <= tol, (k, float(cfo[k]), got[k], X, tol)


def test_argument_errors_launch_nothing(torch):
    import gr_lora_b200._native as N
    sf, n_items = 7, 1 << 16
    rx = make_dec(sf, 8, n_streams=2, max_items_per_call=n_items)
    x = torch.zeros((2, n_items), dtype=torch.complex64, device="cuda")
    rx.receive(x, n_items=n_items)
    before = rx.launch_count()
    for kw in (dict(wide_cfo=2), dict(wide_cfo=True), dict(wide_cfo=True, max_cfo_hz=-1.0), dict(wide_cfo=True, max_cfo_hz=float("nan")),
               dict(wide_cfo=True, max_cfo_hz=float("inf")), dict(wide_cfo=True, max_cfo_hz=3.5 * BW + 1.0)):
        with pytest.raises(N.LoraB200Error) as e:
            rx.receive(x, n_items=n_items, **kw)
        assert e.value.code == -1 and "wide_cfo" in str(e.value), (kw, str(e.value))
        assert rx.launch_count() == before, kw
    rx2 = make_dec(sf, 2, n_streams=2, max_items_per_call=n_items)
    with pytest.raises(N.LoraB200Error):
        rx2.receive(x, n_items=n_items, wide_cfo=True, max_cfo_hz=0.5 * BW + 1.0)
    rx2.receive(x, n_items=n_items, wide_cfo=True, max_cfo_hz=0.5 * BW)


def test_lora_receiver_passes_wide_cfo(torch):
    from gr_lora_b200.lora_receiver import lora_receiver
    sf = 8
    pay = b"lora receiver wide"
    X, _, _ = frame_rows(sf, 8, pay, 0.6 * BW, 123, [1.0], snr_db=5.0)
    host = np.concatenate([X[0], np.zeros(4 * (8 << sf), np.complex64)])
    got = {}
    for wide in (False, True):
        r = lora_receiver(1e6, CARRIER, [CARRIER], int(BW), sf, False, 4, True, disable_channelization=True, sync="dechirp",
                          wide_cfo=wide, max_cfo_hz=0.65 * BW if wide else 0.0, quiet=True)
        r.run(host)
        got[wide] = [f for _, f in r.frames]
    assert any(pay in bytes(f) for f in got[True]), got[True]
    assert not any(pay in bytes(f) for f in got[False])
    with pytest.raises(ValueError):
        lora_receiver(1e6, CARRIER, [CARRIER], int(BW), sf, False, 4, True, disable_channelization=True, wide_cfo=True, quiet=True)
