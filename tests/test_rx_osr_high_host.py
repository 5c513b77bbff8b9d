"""CPU: fs/bw = 16 and 32 through the host emulation -- the shared-memory layout of k1_fft_kernel<SF, D>, the K1 and LLR phase
functions at 16 and 32 polyphase branches against a float64 get_shift_fft, and the dechirp-synchronised receiver on frames
modulated at 2 MS/s and 4 MS/s."""
import numpy as np
import pytest

from antenna_common import frame_rows, k1_batch, tables
from gr_lora_b200 import tx
from k1_reference import check_k1
from osr2_common import K1ReferenceOsr, check_llrs, emul
from osr_high_common import BW, RATES, SENSITIVITY, bank_multiplicity, batch, k1_emulate, llr_emulate, receive, smem_replay, split

CARRIER = 868.1e6


# ---- shared-memory layout ----------------------------------------------------------------------------------------------------
# worst bank multiplicity per phase.  Pass 0 and the combine are conflict-free at D = 2, 8 and 16; at D = 32 a pass-0 half-warp
# stores 16 branch pairs of one column at offsets 2 b SB, all of one parity, so it is 2-way whatever SB is.  The first
# in-place pass of a 512- or 1024-bin sub-problem (radix 8, stride SIG = 4 or 8) is 2-way at every D: a half-warp's 16 items
# are runs of SIG positions 8 SIG apart inside one branch, and the padding moves each run by SIG / 2 float2 only, so
# neighbouring runs share banks (SB plays no part; at 2048 bins a run is the whole half-warp).
def expected_multiplicity(sf, osr, phase):
    if phase == "pass0":
        return 2 if osr == 32 else 1
    if phase == "pass1":
        return 2 if min(1 << sf, 2048, 8192 // osr) in (512, 1024) else 1
    return 1


@pytest.mark.parametrize("osr", [2, 8, 16, 32])
@pytest.mark.parametrize("sf", range(7, 13))
def test_shared_memory_bank_multiplicity(sf, osr):
    acc = smem_replay(sf, osr)
    assert set(acc) >= {"pass0", "pass1", "combine"}
    for phase, a in acc.items():
        assert a.shape[1] == 256 and (a >= 0).any()
        assert bank_multiplicity(a) == expected_multiplicity(sf, osr, phase), (sf, osr, phase)


@pytest.mark.parametrize("osr", [2, 8, 16, 32])
@pytest.mark.parametrize("sf", [7, 10, 12])
def test_shared_memory_replay_covers_the_layout(sf, osr):
    """Pass 0 writes every position of every branch of every symbol of a batch once, and the combine reads each of them once."""
    acc = smem_replay(sf, osr)
    n = batch(sf, osr) * osr * min(1 << sf, 2048, 8192 // osr)
    for phase in ("pass0", "combine"):
        a = acc[phase][acc[phase] >= 0]
        assert a.size == n and np.unique(a).size == n, (sf, osr, phase)
    assert np.array_equal(np.unique(acc["pass0"][acc["pass0"] >= 0]), np.unique(acc["combine"][acc["combine"] >= 0]))


# ---- K1 and the LLR demodulator against float64 ----------------------------------------------------------------------------------
@pytest.mark.parametrize("osr", RATES)
@pytest.mark.parametrize("sf", range(7, 13))
def test_k1_emulation_against_float64(sf, osr):
    """Clean symbols (every bin up to SF9, a spread with the edges and N/2 +- 1 above), -3 dB, half a bin off and noise: bins and
    magnitudes inside the float64 rounding band; an up-chirp shifted by v dechirps to bin v."""
    down = tables(sf, osr)[0]
    rng = np.random.default_rng(100 * osr + sf)
    n = 1 << sf
    vals = np.arange(n) if sf <= 9 else np.unique(np.r_[0, 1, n // 2 - 1, n // 2, n // 2 + 1, n - 1, rng.integers(0, n, 6)])
    x = np.concatenate([tx.modulate_shifts(vals, sf, BW, osr * BW).reshape(-1, osr << sf), k1_batch(sf, osr, rng, n_clean=2)])
    x = np.ascontiguousarray(x, np.complex64)
    bins, mags = k1_emulate(x, sf, osr)
    check_k1(bins, mags, None, sf, ref=K1ReferenceOsr(x, sf, down, osr=osr), what=f"k1<{sf}, {osr}>")
    assert np.array_equal(bins[: vals.size], vals)


@pytest.mark.parametrize("osr", RATES)
@pytest.mark.parametrize("sf", [7, 9, 11])
def test_k1_emulation_batch_sizes(sf, osr):
    """Batches of G - 1 .. 2 G + 1 symbols (G symbols per CTA batch; split SFs too): no symbol is lost or taken from its
    neighbour."""
    down = tables(sf, osr)[0]
    g = batch(sf, osr)
    rng = np.random.default_rng(7 * osr + sf)
    for s in sorted({max(1, g - 1), g, g + 1, 2 * g + 1}):
        vals = rng.integers(0, 1 << sf, s)
        x = (tx.modulate_shifts(vals, sf, BW, osr * BW) + tx.awgn(s * (osr << sf), 0.0, rng)).astype(np.complex64)
        bins, mags = k1_emulate(x, sf, osr)
        check_k1(bins, mags, None, sf, ref=K1ReferenceOsr(x, sf, down, osr=osr), what=f"k1<{sf}, {osr}> batch {s}")
        assert np.array_equal(bins, vals), s


@pytest.mark.parametrize("osr", RATES)
def test_quirk_bin_is_two_distinct_bins(osr):
    """tmp[N/2] = F[sps - N/2] + F[N/2]: a tone at F[N/2] alone reaches bin N/2 with its full magnitude."""
    for sf in (7, 10):
        n, sps = 1 << sf, osr << sf
        down = tables(sf, osr)[0]
        y = np.exp(2j * np.pi * (n / 2) * np.arange(sps) / sps)
        x = (y / down.astype(np.complex128)).astype(np.complex64)
        bins, mags = k1_emulate(x, sf, osr)
        check_k1(bins, mags, None, sf, ref=K1ReferenceOsr(x, sf, down, osr=osr))
        assert bins[0] == n // 2 and abs(mags[0] - sps) < 1e-3 * sps


@pytest.mark.parametrize("osr", RATES)
@pytest.mark.parametrize("sf", range(7, 13))
def test_llr_emulation_against_float64(sf, osr):
    """LLRs against the float64 max-log definition, normal and reduced rate; their bins equal K1's bit for bit."""
    down = tables(sf, osr)[0]
    for reduced in (0, 1):
        x = np.ascontiguousarray(k1_batch(sf, osr, np.random.default_rng(10 * sf + reduced + osr), n_clean=2), np.complex64)
        llr, bins = llr_emulate(x, sf, osr, reduced)
        check_llrs(llr, bins, K1ReferenceOsr(x, sf, down, osr=osr), sf, reduced, f"llr<{sf}, {osr}> reduced={reduced}")
        kb, _ = k1_emulate(x, sf, osr)
        assert np.array_equal(bins, kb)


def test_split_follows_the_sub_problem_size():
    assert [split(sf, 16) for sf in range(7, 13)] == [1, 1, 1, 2, 4, 8]
    assert [split(sf, 32) for sf in range(7, 13)] == [1, 1, 2, 4, 8, 16]


def test_other_rates_are_refused():
    """fs/bw = 4 and 64 have no K1 kernels: the host entry points refuse them as before."""
    x = np.zeros(64 << 7, np.complex64)
    down, _, tw = tables(7, 8)
    b = np.zeros(1, np.uint32)
    m = np.zeros(1, np.float32)
    for osr in (4, 64):
        assert emul().lb_k1_emulate_osr(7, osr, x.ctypes.data, 1, down.ctypes.data, tw.ctypes.data, b.ctypes.data, m.ctypes.data) == -1
    from osr_high_common import _lib
    assert _lib().lb_k1_smem_replay(7, 4, None, None, 0) == -1


# ---- the emulated receiver -------------------------------------------------------------------------------------------------------
RX_SFS = [(sf, 16) for sf in (7, 8, 9, 10)] + [(sf, 32) for sf in (7, 8, 9)]


@pytest.mark.parametrize("sf,osr", RX_SFS)
def test_receiver_recovers_start_cfo_and_payload(sf, osr):
    """Clean frames: start within one sample, CFO within 1/8 bin and the payload, CFOs up to 0.9 BW/4, starts across the
    symbol."""
    n, sps = 1 << sf, osr << sf
    rng = np.random.default_rng(200 + sf + osr)
    pay = b"osr" + bytes(rng.integers(0, 256, 7, dtype=np.uint8))
    for cfo, off in [(0.37, 1), (0.9 * n / 4, sps // 2 + 3), (-0.9 * n / 4, int(rng.integers(0, sps)))]:
        X, start, _ = frame_rows(sf, osr, pay, cfo * BW / n, off, [1.0])
        got = receive(X[0], sf, osr)
        assert len(got) == 1, (cfo, got)
        g = got[0]
        assert abs(g["cfo"] - cfo) <= 1 / 8 and abs(g["start"] - start) <= 1, (cfo, g, start)
        assert g["status"] == 0 and g["payload"] == pay, (cfo, g)


@pytest.mark.parametrize("sf,osr", RX_SFS)
def test_receiver_near_sensitivity(sf, osr):
    """Frames 2 dB above the fs/bw = 8 sensitivity points, random CFO and start: decoded, hard and soft."""
    snr = SENSITIVITY[sf] + 2.0
    sps = osr << sf
    rng = np.random.default_rng(300 + sf + osr)
    pay = bytes(rng.integers(0, 256, 8, dtype=np.uint8))
    X, start, _ = frame_rows(sf, osr, pay, float(rng.uniform(-0.9, 0.9) * BW / 4), int(rng.integers(0, sps)), [1.0], snr_db=snr, seed=sf)
    for soft in (False, True):
        got = [g for g in receive(X[0], sf, osr, soft=soft) if g["status"] == 0]
        assert len(got) == 1 and got[0]["payload"] == pay, (soft, got)
        assert abs(got[0]["start"] - start) <= 1


@pytest.mark.parametrize("sf,osr,ppm", [(7, 16, 20.0), (9, 16, -20.0), (8, 32, 20.0)])
def test_drifted_frames_with_carrier(sf, osr, ppm):
    """A transmitter whose crystal is off by ppm on carrier and clock, found through carrier_hz: start, CFO, clock offset and
    payload."""
    n, sps = 1 << sf, osr << sf
    bin_hz = BW / n
    rng = np.random.default_rng(sf * 1000 + osr + int(ppm))
    pay = bytes(rng.integers(0, 256, 48, dtype=np.uint8))
    cfo_hz = ppm * CARRIER * 1e-6
    X, start, _ = frame_rows(sf, osr, pay, cfo_hz, int(rng.integers(0, sps)), [1.0], sfo_ppm=ppm)
    got = receive(X[0], sf, osr, carrier_hz=CARRIER)
    assert len(got) == 1, got
    g = got[0]
    assert abs(g["cfo"] - cfo_hz / bin_hz) <= 1 / 8 and abs(g["start"] - start) <= 1, (g, start)
    assert abs(g["sfo"] - ppm) <= bin_hz / 8 / CARRIER * 1e6
    assert g["status"] == 0 and g["payload"] == pay


@pytest.mark.parametrize("sf,osr", [(7, 16), (8, 16), (7, 32)])
def test_wide_cfo_beyond_the_fs_bw_8_band(sf, osr):
    """wide_cfo with max_cfo_hz = (fs - BW) / 2: frames at +-[4, 7] BW (D = 16) or +-[8, 15] BW (D = 32) -- beyond what fs/bw = 8
    samples -- decode with their CFO within 1/8 bin."""
    n, sps = 1 << sf, osr << sf
    lim = (osr - 1) * n / 2
    rng = np.random.default_rng(sf + 17 * osr)
    lo, hi = (4.0, 7.0) if osr == 16 else (8.0, 15.0)
    for k, sign in enumerate((1, -1)):
        cfo = sign * float(rng.uniform(lo, hi)) * n
        pay = bytes(rng.integers(0, 256, 8, dtype=np.uint8))
        X, start, _ = frame_rows(sf, osr, pay, cfo * BW / n, int(rng.integers(0, sps)), [1.0], snr_db=SENSITIVITY[sf] + 6.0, seed=k)
        got = [g for g in receive(X[0], sf, osr, max_cfo_bins=lim) if g["status"] == 0]
        assert len(got) == 1 and got[0]["payload"] == pay, (cfo / n, got)
        assert abs(got[0]["cfo"] - cfo) <= 1 / 8 and abs(got[0]["start"] - start) <= 1, (cfo, got[0], start)
