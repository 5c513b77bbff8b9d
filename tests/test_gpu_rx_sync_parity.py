"""The dechirp-synchronised receiver (lora_b200_receive) frame by frame against its host emulation (lb_emul_rx_receive_soft,
the same __host__ __device__ procedure with float64 window sums), run on every row with the decoder's own tables: start,
CFO, SNR, clock offset and payload of every published frame, hard and soft, with and without drift; the SNR estimate
against the truth; and the edges of the call's orchestration -- the per-call frame cap, header rounds over several batches,
staged and unstaged input, and a frame that ends exactly at n_items."""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from antenna_reference import ENERGY_TOL, window_energy, window_sum
from test_gpu_rx_sync import SENSITIVITY, check_exact, frame_len, make_dec, sigma_for

pytestmark = pytest.mark.gpu

BW, FS = 125000, 1e6
CARRIER = 868.1e6
CAP = 64                                              # synchronised frames the emulation reports per row


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
    f = L.lb_emul_rx_receive_soft
    f.restype = C.c_uint32
    f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int,
                  C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    return f


def dec_tables(dec):
    """The decoder's own down-chirp, up-chirp and twiddle tables (tables_export), so that K1's arithmetic is the same on both
    sides."""
    import gr_lora_b200 as G
    t = G.split_tables(dec.tables_export(), dec.sps)
    return tuple(np.ascontiguousarray(t[k]) for k in ("downchirp", "upchirp", "twiddles"))


def emulate(emul, host, sf, tabs, rows=None, sfo_ppm=0.0, carrier_hz=0.0, soft=False):
    """lb_emul_rx_receive_soft on each row of host [n_streams, n_items] (CR 4/8, explicit header, CRC, sync word 0x12,
    reduced rate at SF11/12), the rows in parallel (ctypes releases the GIL).  Returns {stream: [frame dicts]}."""
    down, up, tw = tabs
    rows = range(host.shape[0]) if rows is None else rows

    def one(s):
        x = np.ascontiguousarray(host[s], np.complex64)
        start, cfo, snr = np.zeros(CAP, np.int64), np.zeros(CAP, np.float32), np.zeros(CAP, np.float32)
        status, sfo = np.zeros(CAP, np.int32), np.zeros(CAP, np.float32)
        pay, ln = np.zeros((CAP, 256), np.uint8), np.zeros(CAP, np.uint32)
        n = emul(x.ctypes.data, x.size, down.ctypes.data, up.ctypes.data, tw.ctypes.data, sf, 4, 0, 1, int(sf > 10), 0x12, 0, 0,
                 float(sfo_ppm), float(carrier_hz), int(soft), start.ctypes.data, cfo.ctypes.data, snr.ctypes.data,
                 status.ctypes.data, sfo.ctypes.data, pay.ctypes.data, ln.ctypes.data, CAP)
        assert n < CAP
        return s, [dict(start=int(start[k]), cfo=float(cfo[k]), snr=float(snr[k]), status=int(status[k]), sfo=float(sfo[k]),
                        payload=bytes(pay[k, : ln[k]])) for k in range(n)]

    with ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
        return dict(ex.map(one, rows))


def dedup(frames, sps):
    """lora_b200_receive's rule for one stream's synchronised frames (lora_b200.cu, after the header round), restated: in
    order of start, a frame less than one symbol after the previous one belongs to its group, and a group keeps its best
    member -- a decodable header first, then the higher SNR.  The emulation reports status 0 (published), 1 (header
    checksum failed) or 2 (incomplete); the captures here hold every frame whole, so a status-2 entry is a preamble cut by
    the end of the row, which the device does not synchronise either, and is left out."""
    reps, prev = [], None
    for f in sorted((f for f in frames if f["status"] != 2), key=lambda f: f["start"]):
        if prev is not None and f["start"] - prev["start"] < sps:
            a = reps[-1]
            if (f["status"] == 0) > (a["status"] == 0) or ((f["status"] == 0) == (a["status"] == 0) and f["snr"] > a["snr"]):
                reps[-1] = f
        else:
            reps.append(f)
        prev = f
    return reps


def device_frames(frames, info, sf):
    """{stream: [frame dicts]} of one receive call, in the order published."""
    bin_hz = BW / (1 << sf)
    out = {}
    for r, i in zip(frames, info):
        out.setdefault(int(i["stream"]), []).append(dict(
            start=int(i["start"]), data_start=int(i["data_start"]), cfo=float(i["cfo_hz"]) / bin_hz, cfo_hz=float(i["cfo_hz"]),
            snr=float(i["snr_db"]), sfo=float(i["sfo_ppm"]), payload=bytes(r["bytes"][18: int(r["len"])])))
    return out


def data_start_of(start, sps, ppm):
    """rs_sym(start, 12.25, sps, ppm): the first sample of data symbol 0."""
    u = 12.25 * sps
    if ppm == 0.0:
        return start + int(u)
    v = u / (1.0 + 1e-6 * float(np.float32(ppm)))
    return start + int(np.floor(v + 0.5))


def synth(torch, sf, ns, per, plen, snr, seed, ppm=None, coupled=False, lead=2.0, gap=4.0, tail=6.0):
    """ns streams of per frames of plen random bytes, unit-amplitude tx.base_upchirp chirps (as test_gpu_rx_sync.synth),
    CFO within +-0.9 BW/4 per frame, random starts, AWGN for an SNR of snr in the 125 kHz band.  ppm: the transmitters'
    clock offset, one value for every frame; with coupled, every frame gets its own crystal offset within +-ppm that sets
    its clock offset and its CFO (ppm * 868.1 Hz).  Returns (device tensor, host copy, placed)."""
    from gr_lora_b200 import tx
    rr, sps = sf > 10, 8 << sf
    rng = np.random.default_rng(seed)
    pays = [[bytes(rng.integers(0, 256, plen, dtype=np.uint8)) for _ in range(per)] for _ in range(ns)]
    if coupled:
        ppms = [[float(rng.uniform(-ppm, ppm)) for _ in range(per)] for _ in range(ns)]
        cfo = [[p * CARRIER * 1e-6 for p in row] for row in ppms]
    else:
        ppms = 0.0 if ppm is None else ppm
        cfo = [[float(rng.uniform(-0.9, 0.9) * BW / 4) for _ in range(per)] for _ in range(ns)]
    flen = frame_len(sf, plen, rr=rr) * (1 + 50e-6 * bool(ppm))
    n_items = int((lead + 1) * sps + per * (flen + (gap + 1) * sps) + tail * sps) // 2 * 2
    gen = make_dec(sf, 4, False, True, rr)
    up = torch.from_numpy(tx.base_upchirp(sf).astype(np.complex64)).cuda()
    out, placed = gen.synth_streams(pays, n_items, lead_symbols=lead + float(rng.uniform(0, 1)), gap_symbols=gap + float(rng.uniform(0, 1)),
                                    cfo_hz=cfo, noise_sigma=sigma_for(snr), seed=seed, up_table_dev=up, sfo_ppm=ppms)
    torch.cuda.synchronize()
    gen.close()
    assert len(placed) == ns * per
    return out, out.cpu().numpy(), placed


def match(dev, emu, sps):
    """Pairs (device frame, emulated frame) whose starts lie within a symbol, and the frames of either side left over."""
    pairs, left = [], list(emu)
    only_dev = []
    for d in dev:
        k = next((k for k, e in enumerate(left) if abs(e["start"] - d["start"]) < sps), None)
        if k is None:
            only_dev.append(d)
        else:
            pairs.append((d, left.pop(k)))
    return pairs, only_dev, left


def check_exact_parity(dev, emu, sps, sf, streams, tag, sfo_ppm=0.0, carrier_hz=0.0):
    """The checks of a receive call against the emulation at high SNR: the same published frames per stream, start equal,
    data_start where the frame's clock offset places data symbol 0, |dCFO| <= 1e-3 bin, |dSNR| <= 0.1 dB, the same payload,
    the clock offset equal to the emulation's.  Returns the largest deviations (start, cfo, snr, sfo)."""
    worst = dict(start=0, cfo=0.0, snr=0.0, sfo=0.0)
    ppm_per_bin = 1e6 * (BW / (1 << sf)) / carrier_hz if carrier_hz else 0.0
    for s in streams:
        d = dev.get(s, [])
        e = [f for f in dedup(emu.get(s, []), sps) if f["status"] == 0]
        assert len(d) == len(e), (tag, s, [f["start"] for f in d], [(f["start"], f["status"]) for f in e])
        for a, b in zip(d, e):
            dcfo, dsnr = abs(a["cfo"] - b["cfo"]), abs(a["snr"] - b["snr"])
            worst["start"] = max(worst["start"], abs(a["start"] - b["start"]))
            worst["cfo"], worst["snr"] = max(worst["cfo"], dcfo), max(worst["snr"], dsnr)
            worst["sfo"] = max(worst["sfo"], abs(a["sfo"] - b["sfo"]))
            assert a["start"] == b["start"], (tag, s, a, b)
            assert a["data_start"] == data_start_of(a["start"], sps, a["sfo"]), (tag, s, a)
            assert dcfo <= 1e-3 and dsnr <= 0.1, (tag, s, a, b)
            assert a["payload"] == b["payload"], (tag, s, a, b)
            # the same clock offset: sfo_ppm + F ppm_per_bin on both sides, F within 1e-3 bin
            assert abs(a["sfo"] - b["sfo"]) <= 1e-3 * ppm_per_bin + 4e-7 * (abs(sfo_ppm) + abs(b["sfo"])) + 1e-9, (tag, s, a, b)
    return worst


def fmt(w):
    return f"start {w['start']} samples, CFO {w['cfo']:.2e} bin, SNR {w['snr']:.1e} dB, clock offset {w['sfo']:.2e} ppm"


# (sf, streams, frames per stream): the emulation's K1 on the CPU takes most of the time at SF11/12
SHAPES = {7: (24, 3), 8: (24, 3), 9: (16, 3), 10: (16, 2), 11: (8, 2), 12: (8, 2)}


# ---- the synchroniser's window sums ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("sf", range(7, 13))
def test_window_sums_against_float64(torch, sf):
    """RsDevOps::binval and ::energy, which every decision of the synchroniser is made of (float32 phases reduced from a
    float64 base, sincospif, the twiddle lookup tw[bin n mod sps], block sums), against float64 sums with the decoder's own
    chirp tables: windows of frames and of noise anywhere in a row of 2^24 samples, both chirps, CFOs within +-N/4 bins
    and bins 0, +-1, the sync-word bins, -N/2, N/2 - 1 and random ones.  The error is within 2.5e-7 plus the float32 phase
    rounding of a CFO of F bins, 2 pi (|F| + 1) 2^-25, times the window's sum of |x c| (an H100 stays below 1/10 of that);
    the energy within 1e-5 (antenna_reference.window_sum, which the several-antenna tests share)."""
    sps, N = 8 << sf, 1 << sf
    _, frames_row, _ = synth(torch, sf, 1, 2, 8, 10.0, seed=sf * 7 + 8)
    n = max(1 << 24, frames_row.shape[1])
    g = torch.Generator(device="cuda").manual_seed(sf)
    row = (torch.randn(n, dtype=torch.complex64, device="cuda", generator=g) * sigma_for(10.0) * np.sqrt(2)).contiguous()
    row[n - frames_row.shape[1]:] = torch.from_numpy(frames_row[0]).cuda()
    x = row.cpu().numpy()
    rng = np.random.default_rng(sf)
    m = 128
    pos = np.concatenate([[0, n - sps], rng.integers(0, n - sps, m // 4 - 2),
                          rng.integers(n - frames_row.shape[1], n - sps, m - m // 4)]).astype(np.int64)
    cfo = rng.uniform(-N / 4, N / 4, m).astype(np.float32)
    cfo[:8] = [0.0, 0.5, -0.5, 1.0, -3.0, N / 4, -N / 4, 7.25]
    special = [0, 1, -1, (0x1 * 8) % N, (0x2 * 8) % N, -N // 2, N // 2 - 1]
    bins = np.concatenate([np.resize(special, m // 2), rng.integers(-N // 2, N // 2, m - m // 2)]).astype(np.int32)
    up = rng.integers(0, 2, m).astype(np.int32)
    dec = make_dec(sf)
    down_t, up_t, _ = dec_tables(dec)
    out = torch.zeros(m, dtype=torch.complex64, device="cuda")
    en = torch.zeros(m, dtype=torch.float32, device="cuda")
    kb = torch.zeros(m, dtype=torch.int32, device="cuda")
    km = torch.zeros(m, dtype=torch.float32, device="cuda")
    dec.rs_window(row, n, pos, cfo, up, bins, out, en, kb, km)
    got, got_e = out.cpu().numpy(), en.cpu().numpy()
    worst = 0.0
    for i in range(m):
        w = x[pos[i]: pos[i] + sps]
        X, tol = window_sum(w, up_t if up[i] else down_t, pos[i], cfo[i], bins[i])
        worst = max(worst, abs(got[i] - X) / tol)
        assert abs(got[i] - X) <= tol, (i, int(pos[i]), float(cfo[i]), int(bins[i]), int(up[i]), got[i], X, tol)
        e = window_energy(w)
        assert abs(got_e[i] - e) <= ENERGY_TOL * e, (i, got_e[i], e)
    print(f"SF{sf}: window sums within {worst:.3f} of their tolerance")
    dec.close()


# ---- hard decisions, no clock offset ---------------------------------------------------------------------------
@pytest.mark.parametrize("sf", range(7, 13))
def test_hard_decisions_match_the_emulation_at_10db(torch, emul, sf):
    """+10 dB in band: every stream publishes the frames the emulation does after the device's deduplication, with equal
    start, data_start = start + 12.25 sps, CFO within 1e-3 bin, SNR within 0.1 dB, the same payloads, and the same count of
    failed headers."""
    sps, (ns, per) = 8 << sf, SHAPES[sf]
    out, host, placed = synth(torch, sf, ns, per, 8, 10.0, seed=sf * 7 + 1)
    rx = make_dec(sf, 4, False, True, sf > 10, n_streams=ns, max_items_per_call=host.shape[1])
    _, frames, info = rx.receive(out, n_items=host.shape[1])
    emu = emulate(emul, host, sf, dec_tables(rx))
    w = check_exact_parity(device_frames(frames, info, sf), emu, sps, sf, range(ns), f"SF{sf}")
    assert rx.header_drops == sum(f["status"] == 1 for s in emu for f in dedup(emu[s], sps))
    check_exact(placed, frames, ns)
    print(f"SF{sf} +10 dB, {len(frames)} frames: largest device - emulation: {fmt(w)}")
    rx.close()


@pytest.mark.parametrize("sf", range(7, 13))
def test_hard_decisions_match_the_emulation_near_sensitivity(torch, emul, sf):
    """1 dB above the sensitivity point: frames published on both sides agree -- start within one sample, CFO within 1/64
    bin, SNR within 0.25 dB, the same payload; at most one frame is published by one side only (a near-tie of the screen
    between the device's K1 kernels and the emulated K1 can change a candidate)."""
    sps, (ns, per) = 8 << sf, SHAPES[sf]
    out, host, _ = synth(torch, sf, 2 * ns, per if sf < 11 else 1, 8, SENSITIVITY[sf - 7][1] + 1.0, seed=sf * 7 + 2)
    rx = make_dec(sf, 4, False, True, sf > 10, n_streams=2 * ns, max_items_per_call=host.shape[1])
    _, frames, info = rx.receive(out, n_items=host.shape[1])
    emu = emulate(emul, host, sf, dec_tables(rx))
    dev = device_frames(frames, info, sf)
    single, both = 0, 0
    w = dict(start=0, cfo=0.0, snr=0.0, sfo=0.0)
    for s in range(2 * ns):
        pairs, od, oe = match(dev.get(s, []), [f for f in dedup(emu.get(s, []), sps) if f["status"] == 0], sps)
        single += len(od) + len(oe)
        for a, b in pairs:
            both += 1
            w["start"] = max(w["start"], abs(a["start"] - b["start"]))
            w["cfo"], w["snr"] = max(w["cfo"], abs(a["cfo"] - b["cfo"])), max(w["snr"], abs(a["snr"] - b["snr"]))
            assert abs(a["start"] - b["start"]) <= 1 and abs(a["cfo"] - b["cfo"]) <= 1 / 64 and abs(a["snr"] - b["snr"]) <= 0.25, (s, a, b)
            assert a["payload"] == b["payload"], (s, a, b)
    print(f"SF{sf} {SENSITIVITY[sf - 7][1] + 1.0:+.1f} dB, {both} frames on both sides, {single} on one: largest device - "
          f"emulation: {fmt(w)}")
    assert single <= 1 and both >= 0.8 * len(frames)
    rx.close()


# ---- drift ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sf", range(7, 13))
@pytest.mark.parametrize("mode", ["carrier", "sfo"])
def test_drift_matches_the_emulation(torch, emul, sf, mode):
    """The DRIFT = true synchroniser, +10 dB: with +-20 ppm crystals and carrier_hz = 868.1 MHz (each frame's clock offset
    follows its CFO), and with a clock offset of the same value for every frame given as sfo_ppm.  The checks of the
    undrifted case, data_start where rs_sym places data symbol 0, the clock offset the emulation's, and sfo_ppm =
    the float64 sfo_ppm + cfo_hz / carrier_hz 1e6 to float32 rounding."""
    sps, (ns, per) = 8 << sf, SHAPES[sf]
    ppm = 20.0 if mode == "carrier" else (60.0 if sf % 2 else -60.0)
    out, host, placed = synth(torch, sf, ns, per, 16, 10.0, seed=sf * 7 + 3 + len(mode), ppm=ppm, coupled=mode == "carrier")
    kw = dict(carrier_hz=CARRIER) if mode == "carrier" else dict(sfo_ppm=ppm)
    rx = make_dec(sf, 4, False, True, sf > 10, n_streams=ns, max_items_per_call=host.shape[1])
    _, frames, info = rx.receive(out, n_items=host.shape[1], **kw)
    emu = emulate(emul, host, sf, dec_tables(rx), **kw)
    w = check_exact_parity(device_frames(frames, info, sf), emu, sps, sf, range(ns), f"SF{sf} {mode}", sfo_ppm=kw.get("sfo_ppm", 0.0),
                           carrier_hz=kw.get("carrier_hz", 0.0))
    assert rx.header_drops == sum(f["status"] == 1 for s in emu for f in dedup(emu[s], sps))
    check_exact(placed, frames, ns)
    base = kw.get("sfo_ppm", 0.0)
    for i in info:
        want = base + (float(i["cfo_hz"]) / CARRIER * 1e6 if mode == "carrier" else 0.0)
        assert abs(float(i["sfo_ppm"]) - want) <= 4 * np.finfo(np.float32).eps * max(abs(want), abs(base), 1e-3), (i, want)
        assert float(i["sfo_ppm"]) != 0.0
    print(f"SF{sf} {mode}, {len(frames)} frames: largest device - emulation: {fmt(w)}")
    rx.close()


# ---- soft decisions ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sf", range(7, 13))
def test_soft_decisions_match_the_emulation_near_sensitivity(torch, emul, sf):
    """soft=True 1 dB above the sensitivity point against lb_emul_rx_receive_soft: identical payloads on every frame both
    sides publish, at most one frame published by one side only."""
    sps, (ns, per) = 8 << sf, SHAPES[sf]
    out, host, _ = synth(torch, sf, ns, per, 8, SENSITIVITY[sf - 7][1] + 1.0, seed=sf * 7 + 4)
    rx = make_dec(sf, 4, False, True, sf > 10, n_streams=ns, max_items_per_call=host.shape[1])
    _, frames, info = rx.receive(out, n_items=host.shape[1], soft=True)
    emu = emulate(emul, host, sf, dec_tables(rx), soft=True)
    dev = device_frames(frames, info, sf)
    single = both = 0
    for s in range(ns):
        pairs, od, oe = match(dev.get(s, []), [f for f in dedup(emu.get(s, []), sps) if f["status"] == 0], sps)
        single += len(od) + len(oe)
        for a, b in pairs:
            both += 1
            assert a["payload"] == b["payload"], (s, a, b)
    print(f"SF{sf} soft {SENSITIVITY[sf - 7][1] + 1.0:+.1f} dB: {both} frames on both sides, {single} on one")
    assert single <= 1 and both >= 0.8 * ns * per
    rx.close()


# ---- the SNR estimate against the truth --------------------------------------------------------------------------------
def loratap_snr_byte(snr_db):
    """K8's loratap SNR byte from a frame's estimate, in float32 as rs_frame_kernel and K8 compute it:
    (uint8)(int32)((double)(10 log10f(exp10f(snr_db / 10))) + 0.5)."""
    lin = max(np.float32(10.0) ** (np.float32(snr_db) / np.float32(10.0)), np.float32(1e-30))
    v = float(np.float32(10.0) * np.log10(np.float32(lin))) + 0.5
    return int(np.trunc(v)) & 0xFF, v


@pytest.mark.parametrize("sf", range(7, 13))
def test_snr_estimate_against_the_truth_on_the_device(torch, sf):
    """From the sensitivity point to +30 dB in band: the device's SNR estimate has a mean error within 0.5 dB and every
    frame is within 1.5 dB of the true SNR; each record's loratap SNR byte is K8's rounding of that frame's snr_db."""
    sps = 8 << sf
    s0 = SENSITIVITY[sf - 7][1]
    ns = 48 if sf < 11 else 24
    for k, snr in enumerate((s0, s0 + 3.0, s0 + 8.0, 10.0, 30.0)):
        out, host, placed = synth(torch, sf, ns, 1, 8, snr, seed=sf * 100 + k)
        rx = make_dec(sf, 4, False, True, sf > 10, n_streams=ns, max_items_per_call=host.shape[1])
        _, frames, info = rx.receive(out, n_items=host.shape[1])
        truth = {s: (st, p) for s, st, p in placed}
        err = []
        for r, i in zip(frames, info):
            st, p = truth[int(i["stream"])]
            if abs(int(i["start"]) - st) > 1 or bytes(r["bytes"][18: int(r["len"])]) != p:
                continue
            err.append(float(i["snr_db"]) - snr)
            b, v = loratap_snr_byte(float(i["snr_db"]))
            if abs(v - round(v)) > 1e-4:
                assert int(r["bytes"][13]) == b, (float(i["snr_db"]), int(r["bytes"][13]), b)
        err = np.array(err)
        assert err.size >= 0.8 * ns, (snr, err.size)
        print(f"SF{sf} at {snr:+.1f} dB on the device: {err.size} frames, SNR error mean {err.mean():+.3f} dB, max |error| "
              f"{np.abs(err).max():.3f} dB")
        assert abs(err.mean()) <= 0.5 and np.abs(err).max() <= 1.5, (snr, err)
        rx.close()


# ---- more preambles in a stream than max_frames_per_call -----------------------------------------------------------
def test_two_frames_per_call_under_the_consumed_rule(torch):
    """max_frames_per_call = 2, 16 streams of 7 frames: fed from consumed[s] on, each call holds a stream back from the
    third preamble it finds (rs_detect_stream's first_dropped); every frame is published exactly once, in order, with the
    absolute start, CFO and bytes of one call with max_frames_per_call = 16."""
    sf, ns, per = 7, 16, 7
    sps = 8 << sf
    out, host, placed = synth(torch, sf, ns, per, 8, 10.0, seed=71)
    n = host.shape[1]
    one = make_dec(sf, n_streams=ns, max_items_per_call=n, max_frames_per_call=16)
    _, f1, i1 = one.receive(out, n_items=n)
    check_exact(placed, f1, ns)
    want = {s: [(int(i["start"]), float(i["cfo_hz"]), bytes(r["bytes"][15: int(r["len"])])) for r, i in zip(f1, i1)
                if int(i["stream"]) == s] for s in range(ns)}
    rx = make_dec(sf, n_streams=ns, max_items_per_call=n, max_frames_per_call=2)
    rng = np.random.default_rng(72)
    sigma = sigma_for(10.0)
    pos = np.zeros(ns, np.int64)
    got = {s: [] for s in range(ns)}
    calls = 0
    while pos.min() < n and calls < 16:
        x = (sigma * (rng.standard_normal((ns, n)) + 1j * rng.standard_normal((ns, n)))).astype(np.complex64)
        for s in range(ns):                      # each row from its own consumed position, noise past the capture's end
            m = max(0, n - int(pos[s]))
            x[s, :m] = host[s, pos[s]: pos[s] + m]
        c, fr, inf = rx.receive(x)
        for r, i in zip(fr, inf):
            s = int(i["stream"])
            if int(i["start"]) + pos[s] < n:
                got[s].append((int(i["start"]) + int(pos[s]), float(i["cfo_hz"]), bytes(r["bytes"][15: int(r["len"])])))
        assert np.all(c > 0)
        pos += c
        calls += 1
    assert calls >= 4, calls                      # 7 frames, at most 2 per call
    bin_hz = BW / (1 << sf)
    for s in range(ns):
        assert [(a, b) for a, _, b in got[s]] == [(a, b) for a, _, b in want[s]], s
        assert all(abs(g[1] - w[1]) <= 1e-3 * bin_hz for g, w in zip(got[s], want[s])), (s, got[s], want[s])
    rx.close()
    one.close()


# ---- header rounds over more than one batch -----------------------------------------------------------------------
@pytest.mark.parametrize("sf,ns", [(12, 34), (11, 66)])
def test_header_round_over_several_batches(torch, emul, sf, ns):
    """More synchronised frames than one header-round batch holds (win_cap / 8 = 128 frames at SF12, 256 at SF11), so the
    header round and the payload round run in several batches: every placed payload is published once, and rx_info and
    payloads match the emulation on every 8th stream."""
    sps, per = 8 << sf, 4
    out, host, placed = synth(torch, sf, ns, per, 4, 10.0, seed=sf * 7 + 5, lead=1.0, gap=3.0, tail=4.0)
    assert len(placed) > (128 if sf == 12 else 256)
    rx = make_dec(sf, 4, False, True, True, n_streams=ns, max_items_per_call=host.shape[1])
    _, frames, info = rx.receive(out, n_items=host.shape[1])
    check_exact(placed, frames, ns)
    rows = list(range(0, ns, 8))
    emu = emulate(emul, host, sf, dec_tables(rx), rows=rows)
    w = check_exact_parity(device_frames(frames, info, sf), emu, sps, sf, rows, f"SF{sf}")
    print(f"SF{sf}, {len(frames)} frames in one call: largest device - emulation on every 8th stream: {fmt(w)}")
    rx.close()


# ---- staged and unstaged input ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("sf", [7, 10])
def test_four_input_paths_agree(torch, sf):
    """One set of samples through device rows whose stride is a multiple of sps (the screen reads them in place; the rows'
    padding is NaN), a stride that is not, a device pointer 8 bytes past a 16-byte boundary, and a host array: byte-identical
    frames, rx_info, consumed and header drops."""
    sps = 8 << sf
    ns = 8
    _, host, _ = synth(torch, sf, ns, 3, 8, 0.0, seed=sf * 7 + 6)
    n = host.shape[1]
    res = []

    def run(iq, **kw):
        rx = make_dec(sf, n_streams=ns, max_items_per_call=n)
        c, fr, inf = rx.receive(iq, **kw)
        res.append((c.tobytes(), fr.tobytes(), inf.tobytes(), rx.header_drops, len(fr)))
        rx.close()

    h = torch.from_numpy(host).cuda()
    s1 = (n + sps - 1) // sps * sps + sps
    a = torch.full((ns, s1), float("nan"), dtype=torch.complex64, device="cuda")
    a[:, :n] = h
    run(a, n_items=n, stride_items=s1)
    s2 = n + 3
    assert s2 % sps
    b = torch.full((ns, s2), float("nan"), dtype=torch.complex64, device="cuda")
    b[:, :n] = h
    run(b, n_items=n, stride_items=s2)
    flat = torch.zeros(ns * n + 2, dtype=torch.complex64, device="cuda")
    flat[1: 1 + ns * n] = h.reshape(-1)
    ptr = flat.data_ptr() + 8
    assert ptr % 16 == 8
    torch.cuda.synchronize()
    run(ptr, n_items=n, stride_items=n, host=0)
    run(host)
    assert res[0][4] >= 0.8 * 3 * ns
    assert all(r == res[0] for r in res[1:]), [r[3:] for r in res]


# ---- a frame whose last data window ends at n_items -------------------------------------------------------------
@pytest.mark.parametrize("sf", [8, 12])
def test_frame_ending_exactly_at_n_items(torch, sf):
    """The last data window ends exactly at n_items: the frame is published.  One sample less: it is not, consumed is at or
    before its start, and the call from consumed publishes it with the same absolute start."""
    import gr_lora_b200 as G
    sps, rr = 8 << sf, sf > 10
    out, host, placed = synth(torch, sf, 1, 1, 8, 20.0, seed=sf * 7 + 7)
    rx = make_dec(sf, 4, False, True, rr, n_streams=1, max_items_per_call=host.shape[1])
    _, f0, i0 = rx.receive(host)
    assert len(f0) == 1
    start = int(i0[0]["start"])
    end = start + int((12.25 + G.tx_frame_symbols(8, sf, 4, False, True, rr)) * sps)
    assert end <= host.shape[1]
    c, f1, i1 = rx.receive(host[:, :end])
    assert len(f1) == 1 and int(i1[0]["start"]) == start and f1.tobytes() == f0.tobytes()
    c, f2, _ = rx.receive(host[:, : end - 1])
    assert len(f2) == 0 and int(c[0]) <= start, (int(c[0]), start)
    c0 = int(c[0])
    _, f3, i3 = rx.receive(host[:, c0:])
    assert len(f3) == 1 and c0 + int(i3[0]["start"]) == start
    assert bytes(f3[0]["bytes"][15: int(f3[0]["len"])]) == bytes(f0[0]["bytes"][15: int(f0[0]["len"])])
    rx.close()
