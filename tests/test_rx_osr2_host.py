"""CPU: fs/bw = 2 through the host emulation -- k1_fft_kernel<SF, 2> and k1_llr_kernel<SF, 2> (the K1 phase functions at two
polyphase branches) against a float64 get_shift_fft, and the dechirp-synchronised receiver (lb_emul_rx_receive_osr) on frames
modulated at 250 kS/s."""
import numpy as np
import pytest

from gr_lora_b200 import tx
from k1_reference import check_k1
from osr2_common import BATCH, BW, CARRIER, FS, OSR, K1ReferenceOsr, check_llrs, frame_row, k1_batch, k1_emulate, llr_emulate, receive_emul, tables


@pytest.mark.parametrize("sf", range(7, 13))
def test_k1_emulation_against_float64(sf):
    """Every bin clean (a spread of bins at SF11/12), -3 dB, half a bin off frequency and pure noise: bins and magnitudes
    inside the float64 rounding band (tau criterion); tmp[N/2] is F[3N/2] + F[N/2]."""
    down, _, tw = tables(sf)
    x = k1_batch(sf, np.random.default_rng(sf))
    bins, mags = k1_emulate(x, sf)
    check_k1(bins, mags, None, sf, ref=K1ReferenceOsr(x, sf, down), what=f"k1<{sf}, 2>")
    n = 1 << sf
    clean = np.arange(n) if sf <= 10 else None
    if clean is not None:                                 # an up-chirp shifted by v dechirps to bin v
        assert np.array_equal(bins[:n], clean)


@pytest.mark.parametrize("sf", range(7, 13))
def test_k1_emulation_batch_sizes(sf):
    """Batches of G - 1, G, G + 1 and 2 G + 1 symbols (G the kernel's symbols per CTA batch): no symbol of a partial batch is
    lost or taken from its neighbour."""
    down, _, tw = tables(sf)
    g = BATCH[sf]
    rng = np.random.default_rng(50 + sf)
    sizes = [s for s in (g - 1, g, g + 1, 2 * g + 1) if s > 0]
    if sf >= 11:
        sizes = sizes[1:3]
    for s in sizes:
        vals = rng.integers(0, 1 << sf, s)
        x = (tx.modulate_shifts(vals, sf, BW, FS) + tx.awgn(s * (OSR << sf), 0.0, rng)).astype(np.complex64)
        bins, mags = k1_emulate(x, sf)
        check_k1(bins, mags, None, sf, ref=K1ReferenceOsr(x, sf, down), what=f"k1<{sf}, 2> batch {s}")
        assert np.array_equal(bins, vals), s


def test_quirk_bin_is_two_distinct_bins():
    """tmp[N/2] = F[3N/2] + F[N/2] at fs/bw = 2: a tone at F[N/2] alone reaches bin N/2 with its full magnitude."""
    sf = 8
    n, sps = 1 << sf, OSR << sf
    down, _, tw = tables(sf)
    y = np.exp(2j * np.pi * (n / 2) * np.arange(sps) / sps)          # F[N/2] after the dechirp
    x = (y / down.astype(np.complex128)).astype(np.complex64)
    bins, mags = k1_emulate(x, sf)
    ref = K1ReferenceOsr(x, sf, down)
    check_k1(bins, mags, None, sf, ref=ref)
    assert bins[0] == n // 2 and abs(mags[0] - sps) < 1e-3 * sps


@pytest.mark.parametrize("sf", range(7, 13))
@pytest.mark.parametrize("reduced", [0, 1])
def test_llr_emulation_against_float64(sf, reduced):
    """LLRs against the float64 max-log definition; their bins equal K1's at fs/bw = 2 bit for bit."""
    down, _, tw = tables(sf)
    x = k1_batch(sf, np.random.default_rng(10 * sf + reduced), n_clean=3 if sf < 11 else 1)
    llr, bins = llr_emulate(x, sf, reduced)
    check_llrs(llr, bins, K1ReferenceOsr(x, sf, down), sf, reduced, f"llr<{sf}, 2> reduced={reduced}")
    kb, _ = k1_emulate(x, sf)
    assert np.array_equal(bins, kb)


def test_osr_entry_points_refuse_other_rates():
    from osr2_common import emul
    x = np.zeros(4 << 7, np.complex64)
    down, _, tw = tables(7)
    b = np.zeros(1, np.uint32)
    m = np.zeros(1, np.float32)
    assert emul().lb_k1_emulate_osr(7, 4, x.ctypes.data, 1, down.ctypes.data, tw.ctypes.data, b.ctypes.data, m.ctypes.data) == -1


@pytest.mark.parametrize("sf", range(7, 13))
def test_receiver_recovers_start_cfo_and_payload(sf):
    """Clean frames at fs/bw = 2: start within one sample, CFO within 1/8 bin and the payload, for CFOs up to 0.9 BW/4 and
    start offsets across the symbol (odd offsets: half-chip timing)."""
    n, sps = 1 << sf, OSR << sf
    bin_hz = BW / n
    rng = np.random.default_rng(200 + sf)
    cfos = [0.0, 0.37, -5.5, 0.9 * n / 4, -0.9 * n / 4]
    offsets = [0, 1, sps // 2 + 1, sps - 1, int(rng.integers(0, sps))]
    if sf >= 11:
        cfos, offsets = cfos[::2], offsets[::2]
    pay = b"osr2" + bytes(rng.integers(0, 256, 6, dtype=np.uint8))
    for k, cfo in enumerate(cfos):
        x, start, _ = frame_row(sf, pay, cfo * bin_hz, offsets[k % len(offsets)])
        got = receive_emul(x, sf, rr=sf > 10)
        assert len(got) == 1, (cfo, got)
        g = got[0]
        assert abs(g["cfo"] - cfo) <= 1 / 8, (cfo, g)
        assert abs(g["start"] - start) <= 1, (cfo, g, start)
        assert g["status"] == 0 and g["payload"] == pay, (cfo, g)


@pytest.mark.parametrize("sf", [7, 8, 9])
@pytest.mark.parametrize("soft", [False, True])
def test_receiver_below_the_noise_floor(sf, soft):
    """Frames 3 dB above the sensitivity points the receiver reaches at fs/bw = 8 (SF7 -2, SF8 -5, SF9 -7.5 dB in 125 kHz),
    random CFO and start: decoded, hard and soft."""
    snr = {7: -2.0, 8: -5.0, 9: -7.5}[sf] + 3.0
    n, sps = 1 << sf, OSR << sf
    rng = np.random.default_rng(300 + sf)
    for k in range(3):
        pay = bytes(rng.integers(0, 256, 8, dtype=np.uint8))
        x, start, _ = frame_row(sf, pay, float(rng.uniform(-0.9, 0.9) * BW / 4), int(rng.integers(0, sps)), snr_db=snr, seed=k)
        got = [g for g in receive_emul(x, sf, soft=soft) if g["status"] == 0]
        assert len(got) == 1 and got[0]["payload"] == pay, (k, got)
        assert abs(got[0]["start"] - start) <= 1


def test_pure_noise_yields_no_frame():
    for sf in (7, 8):
        rng = np.random.default_rng(sf)
        m = 400 * (OSR << sf)
        x = (rng.standard_normal(m) + 1j * rng.standard_normal(m)).astype(np.complex64)
        assert [g for g in receive_emul(x, sf) if g["status"] == 0] == []


CASES = [(7, 20.0, True), (7, -200.0, False), (9, -20.0, True), (9, 200.0, False), (10, 20.0, True), (12, -20.0, True)]


@pytest.mark.parametrize("sf,ppm,coupled", CASES)
def test_drifted_frames_at_fs_bw_2(sf, ppm, coupled):
    """64-byte frames from a drifting transmitter at fs/bw = 2: start within one sample, CFO within 1/8 bin, the clock offset
    and the payload, through carrier_hz (a crystal offset on carrier and clock) or sfo_ppm."""
    rr = sf > 10
    n, sps = 1 << sf, OSR << sf
    bin_hz = BW / n
    rng = np.random.default_rng(sf * 1000 + int(ppm) + 7 * coupled)
    payload = bytes(rng.integers(0, 256, 64, dtype=np.uint8))
    cfo_hz = ppm * CARRIER * 1e-6 if coupled else float(rng.uniform(-0.5, 0.5) * BW / 4)
    x, start, _ = frame_row(sf, payload, cfo_hz, int(rng.integers(0, sps)), rr=rr, sfo_ppm=ppm)
    got = receive_emul(x, sf, rr=rr, **(dict(carrier_hz=CARRIER) if coupled else dict(sfo_ppm=ppm)))
    assert len(got) == 1, got
    g = got[0]
    assert abs(g["cfo"] - cfo_hz / bin_hz) <= 1 / 8, (g, cfo_hz / bin_hz)
    assert abs(g["start"] - start) <= 1, (g, start)
    tol = bin_hz / 8 / CARRIER * 1e6 if coupled else 1e-4
    assert abs(g["sfo"] - ppm) <= tol, (g["sfo"], ppm, tol)
    assert g["status"] == 0 and g["payload"] == payload, g
