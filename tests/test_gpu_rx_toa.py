"""The dechirp receiver's fine time of arrival on the device (lora_b200_rx_params.fine_toa, rs_toa_kernel): off means off,
the device against the float64 definition (tests/toa_reference.py) and against the host emulation, accuracy in noise,
chunked feeding, scaling and a bad value."""
import ctypes as C

import numpy as np
import pytest

from toa_reference import BW, NU_BOUND, SENSITIVITY, frame_rows, receive_toa, reference, rms, toa_bound

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def make_dec(sf, osr=8, **kw):
    import gr_lora_b200 as G
    if osr == 8:                                      # (the stream state machine's FFT demodulator exists at fs/bw = 8 only)
        kw["demod"] = "fft"
    return G.decoder(osr * BW, int(BW), sf, False, 4, True, sf > 10, quiet=True, **kw)


def streams(sf, osr, n_streams, snr_db, seed, frames_per_stream=2, ppm=0.0, cfo_frac=0.5):
    """n_streams rows, each with frames at random fractional delays and CFOs within cfo_frac N/4: (X [ns, n], truths)."""
    rng = np.random.default_rng(seed)
    rows, truths = [], []
    for s in range(n_streams):
        parts, tr, pos = [], [], 0
        for _ in range(frames_per_stream):
            X, t = frame_rows(sf, osr, float(rng.uniform(0, 1)), float(rng.uniform(-1, 1) * cfo_frac * (1 << sf) / 4), ppm=ppm,
                              snr_db=snr_db, seed=int(rng.integers(1 << 30)), lead_syms=int(rng.integers(1, 4)))
            parts.append(X[0])
            tr.append(pos + t)
            pos += X.shape[1]
        rows.append(np.concatenate(parts))
        truths.append(tr)
    n = max(r.size for r in rows)
    return np.ascontiguousarray(np.stack([np.pad(r, (0, n - r.size)) for r in rows])), truths


def test_off_means_off(torch):
    """fine_toa = 0 on a decoder that has had it on: frames, rx_info, consumed, CRC status and launches as a decoder that
    never had it, and no toa; fine_toa = 1: the same records, one launch more, one toa per frame."""
    sf, ns = 8, 16
    X, _ = streams(sf, 8, ns, 0.0, seed=1)
    n = X.shape[1]
    a = make_dec(sf, n_streams=ns, max_items_per_call=n)
    b = make_dec(sf, n_streams=ns, max_items_per_call=n)
    b.receive(X, fine_toa=True)
    runs = []
    for dec, opt in ((a, False), (b, False), (a, True)):
        l0 = dec.launch_count()
        c, f, i = dec.receive(X, fine_toa=opt)
        runs.append((c.tobytes(), f.tobytes(), i.tobytes(), dec.frames_crc_last().tobytes(), dec.launch_count() - l0,
                     dec.rx_toa_last(), len(f)))
    assert runs[0][:5] == runs[1][:5]
    assert runs[0][5].size == 0 and runs[1][5].size == 0
    assert runs[2][:4] == runs[0][:4] and runs[2][4] == runs[0][4] + 1
    assert runs[2][5].size == runs[2][6] > 0
    # a work call after a fine_toa call leaves no toa behind
    a.work_batch(X[:, : 16 << sf], callbacks=False)
    assert a.rx_toa_last().size == 0


def test_bad_value_before_any_launch(torch):
    import gr_lora_b200 as G
    from gr_lora_b200 import _native as N
    dec = make_dec(7, n_streams=1)
    x = np.zeros((1, 1 << 14), np.complex64)
    l0 = dec.launch_count()
    p = N.RxParams(fine_toa=2)
    consumed = (C.c_size_t * 1)()
    rc = dec._L.lora_b200_receive(dec._h, x.ctypes.data, x.shape[1], x.shape[1], 1, C.byref(p), consumed)
    assert rc == N.EINVAL and b"fine_toa" in N.lib().lora_b200_last_error()
    assert dec.launch_count() == l0
    assert G is not None


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf", range(7, 13))
def test_device_holds_the_definition(torch, sf, osr):
    """lora_b200_rs_toa_dev on frames past 2^24 samples into rows of M = 1..4 antennas of unequal gains, noisy, without and
    with +-20 ppm: nu_A, nu_B within NU_BOUND bins of the float64 reference, toa within osr NU_BOUND samples."""
    rng = np.random.default_rng(sf * 3 + osr)
    n, sps = 1 << sf, osr << sf
    gains = (1.0, 0.6j, -0.35 + 0.2j, 0.15)
    cases = [(1, 0.0), (2, 20.0), (3, -20.0), (4, 0.0)]
    base = 1 << 24
    dec = make_dec(sf, osr, n_streams=4)
    for m, ppm in cases:
        cfo = float(rng.uniform(-n / 4, n / 4))
        F, truth = frame_rows(sf, osr, float(rng.uniform(0, 1)), cfo, gains[:m], ppm=ppm, snr_db=SENSITIVITY[sf] + 6,
                              seed=int(rng.integers(1 << 30)))
        L = base + F.shape[1]
        rows = torch.zeros((m, L), dtype=torch.complex64, device="cuda")
        rows[:, base:] = torch.from_numpy(F).cuda()
        t = int(np.floor(truth)) + base + int(rng.integers(-osr // 2, osr // 2 + 1))
        da, db, dt = dec.rs_toa(rows, L, [0], [t], [cfo], [ppm], antennas=m, stride=L)
        ra, rb, rt = reference(F, sf, osr, t - base, cfo, ppm)
        assert abs(da[0] - ra) <= NU_BOUND and abs(db[0] - rb) <= NU_BOUND, (m, ppm, da, ra, db, rb)
        assert abs(dt[0] - base - rt) <= toa_bound(osr), (m, ppm, dt, rt)
        del rows
    assert sps


@pytest.mark.parametrize("soft,wide", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("sf,osr", [(7, 8), (9, 2)])
def test_device_matches_the_emulation(torch, sf, osr, soft, wide):
    """Each published frame's toa against lb_emul_rx_receive_toa's for the frame of the same start, hard and soft, with and
    without wide_cfo (max_cfo_hz = 0.4 BW at fs/bw = 8, 0.3 BW at 2)."""
    X, _ = streams(sf, osr, 4, SENSITIVITY[sf] + 8, seed=sf + osr, cfo_frac=0.9)
    max_cfo = (0.4 if osr == 8 else 0.3) * BW if wide else 0.0
    dec = make_dec(sf, osr, n_streams=4, max_items_per_call=X.shape[1])
    _, f, info = dec.receive(X, soft=soft, wide_cfo=wide, max_cfo_hz=max_cfo)
    toa = dec.rx_toa_last()
    assert toa.size == 0
    _, f, info = dec.receive(X, soft=soft, wide_cfo=wide, max_cfo_hz=max_cfo, fine_toa=True)
    toa = dec.rx_toa_last()
    assert toa.size == len(f) > 0
    n_bins = 1 << sf
    matched = 0
    for s in range(X.shape[0]):
        host = {e["start"]: e for e in receive_toa(X[s], sf, osr, soft=soft, max_cfo_bins=max_cfo / BW * n_bins if wide else 0.0)
                if e["status"] == 0}
        for k in np.nonzero(info["stream"] == s)[0]:
            e = host.get(int(info["start"][k]))
            if e is None:
                continue
            assert abs(toa[k] - e["toa"]) <= toa_bound(osr), (s, k, toa[k], e)
            matched += 1
    assert matched >= len(f) - 1, (matched, len(f))


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf", [7, 10, 12])
def test_accuracy_on_the_device(torch, sf, osr):
    """96 frames per point from the sensitivity point up: the RMS of toa - truth below that of start - truth, and at
    sensitivity + 20 dB within 0.01 chip.  Prints the figures DESIGN.md records."""
    for k, d in enumerate((0, 5, 10, 20)):
        X, truths = streams(sf, osr, 48, SENSITIVITY[sf] + d, seed=1000 * sf + 10 * osr + k)
        dec = make_dec(sf, osr, n_streams=48, max_items_per_call=X.shape[1], max_frames_per_call=4)
        _, f, info = dec.receive(X, fine_toa=True)
        toa = dec.rx_toa_last()
        et, es = [], []
        for j in range(len(f)):
            tr = np.array(truths[int(info["stream"][j])])
            i = int(np.argmin(np.abs(tr - float(info["start"][j]))))
            if abs(tr[i] - float(info["start"][j])) < osr * 4:
                et.append(toa[j] - tr[i])
                es.append(float(info["start"][j]) - tr[i])
        et, es = np.array(et), np.array(es)
        print(f"SF{sf} fs/bw={osr} SNR {SENSITIVITY[sf] + d:+.1f} dB: {et.size} frames, rms(toa-truth) {rms(et):.4f}, "
              f"bias {np.mean(et):+.4f}, rms(start-truth) {rms(es):.4f} samples")
        assert et.size >= 90, et.size
        assert rms(et) < rms(es)
        if d == 20:
            assert rms(et) <= 0.01 * osr


def test_chunked_feeding_and_scaling(torch):
    """A frame published after re-presentation from consumed has the toa - start of the one-call decode (bit for bit when
    the synchroniser's CFO and clock offset come out bit-identical, as they must for the same samples at another row
    offset to give the same window sums); input scaled by 2^+-12 gives bit-identical toa."""
    sf = 8
    X, _ = streams(sf, 8, 1, 3.0, seed=11, frames_per_stream=3)
    n = X.shape[1]
    dec = make_dec(sf, n_streams=1, max_items_per_call=n)
    _, f, info = dec.receive(X, fine_toa=True)
    toa = dec.rx_toa_last().copy()
    assert len(f) == 3
    one = {int(info["start"][k]): (toa[k] - float(info["start"][k]), float(info["cfo_hz"][k])) for k in range(3)}
    pos, seen, exact = 0, 0, 0
    while pos < n:
        c, fr, inf = dec.receive(X[:, pos: pos + n // 2], fine_toa=True)
        t = dec.rx_toa_last()
        for k in range(len(fr)):
            d0, cfo0 = one[pos + int(inf["start"][k])]
            d = t[k] - float(inf["start"][k])
            assert abs(d - d0) <= toa_bound(8)
            if float(inf["cfo_hz"][k]) == cfo0:
                assert d == d0
                exact += 1
            seen += 1
        if pos + n // 2 >= n:
            break
        assert c[0] > 0
        pos += int(c[0])
    assert seen == 3
    print(f"chunked: {exact} of {seen} frames with bit-identical CFO")
    for sc in (2.0 ** 12, 2.0 ** -12):
        _, f2, _ = dec.receive(X * np.float32(sc), fine_toa=True)
        assert f2.tobytes() == f.tobytes() and dec.rx_toa_last().tobytes() == toa.tobytes()
