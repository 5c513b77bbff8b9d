"""CPU: the dechirp receiver's coarse-offset search (rx_params.wide_cfo) through the host emulation, lb_emul_rx_receive_wide:
frames up to 3 BW off carrier at fs/bw = 8 and BW/2 at fs/bw = 2 decode with their CFO to 1/8 bin, the receiver without the
search loses them, and a search no wider than BW/4 is exactly the receiver without it."""
import pytest

from antenna_common import frame_rows, receive_emul
from wide_cfo_common import BW, band_limit_bins, dedup, receive_wide, shifted_chirp, tables

PAY = b"wide carrier offset"
OFFSETS_8 = [s * v for v in (0.3, 0.49, 0.51, 0.74, 1.2, 3.0) for s in (1, -1)]
OFFSETS_2 = [s * v for v in (0.3, 0.45) for s in (1, -1)]


def _one(frames, lead, cfo_bw, sf, payload=PAY, osr=8):
    """The one frame the device would publish (its one-frame-per-preamble rule): at the frame start, CFO within 1/8 bin, the
    payload."""
    n = 1 << sf
    pub = [f for f in dedup(frames, osr * n) if f["status"] == 0]
    assert len(pub) == 1, frames
    f = pub[0]
    assert abs(f["start"] - lead) <= 1, (f["start"], lead)
    assert abs(f["cfo"] - cfo_bw * n) <= 0.125, (f["cfo"], cfo_bw * n)
    assert f["payload"] == payload


@pytest.mark.parametrize("sf", [7, 10])
@pytest.mark.parametrize("cfo_bw", OFFSETS_8)
def test_wide_offsets_decode_osr8(sf, cfo_bw):
    X, lead, _ = frame_rows(sf, 8, PAY, cfo_bw * BW, 29, [1.0], snr_db=15.0, seed=sf)
    _one(receive_wide(X[0], sf, 8, band_limit_bins(sf, 8)), lead, cfo_bw, sf)


@pytest.mark.parametrize("sf", [7, 10])
@pytest.mark.parametrize("cfo_bw", OFFSETS_2)
@pytest.mark.parametrize("soft", [False, True])
def test_wide_offsets_decode_osr2(sf, cfo_bw, soft):
    X, lead, _ = frame_rows(sf, 2, PAY, cfo_bw * BW, 3, [1.0], snr_db=15.0, seed=sf)
    _one(receive_wide(X[0], sf, 2, band_limit_bins(sf, 2), soft=soft), lead, cfo_bw, sf, osr=2)


@pytest.mark.parametrize("sf", [7, 10])
@pytest.mark.parametrize("cfo_bw", [v for v in OFFSETS_8 if abs(v) > 0.25])
def test_without_the_search_frames_beyond_bw4_are_lost(sf, cfo_bw):
    """The receiver without the search (and the search up to BW/4) does not receive these frames: whatever it publishes
    carries a CFO within +-BW/4, at least 0.05 BW from the frame's.  (Its dechirped windows do see a frame about N bins off
    carrier as one off by a timing shift, so such a frame can come out with an aliased CFO.)"""
    n = 1 << sf
    X, _, _ = frame_rows(sf, 8, PAY, cfo_bw * BW, 29, [1.0], snr_db=15.0, seed=sf)
    for frames in (receive_emul(X[0], sf, 8), receive_wide(X[0], sf, 8, n / 4)):
        for f in frames:
            assert abs(f["cfo"]) <= n / 4 and abs(f["cfo"] - cfo_bw * n) > 0.05 * n, f


@pytest.mark.parametrize("sf", [7, 9])
@pytest.mark.parametrize("cfo_bw", [0.245, 0.255, -0.245, -0.255, 0.745, -0.755, 1.245, -1.255])
@pytest.mark.parametrize("offset", [0, 300, 517])
def test_residual_near_a_quarter_band(sf, cfo_bw, offset):
    """CFOs whose residual lies near +-N/4 of a hypothesis, where the branches k = +-1 of the N/2 ambiguity decide, at
    several timings."""
    X, lead, _ = frame_rows(sf, 8, PAY, cfo_bw * BW, offset, [1.0], snr_db=15.0, seed=offset)
    _one(receive_wide(X[0], sf, 8, 1.5 * (1 << sf)), lead, cfo_bw, sf)


def _runs(bins, min_run=5):
    """Longest run of bins agreeing within +-1 (mod N unneeded: the test's bins sit away from the wrap)."""
    best = cur = 1
    for a, b in zip(bins[:-1], bins[1:]):
        cur = cur + 1 if abs(int(b) - int(a)) <= 1 else 1
        best = max(best, cur)
    return best >= min_run


def test_preamble_seen_in_two_hypotheses_gives_one_frame():
    """At 0.25 BW the preamble shows in the screens of c = 0 and c = 1 alike; one frame comes out."""
    from osr2_common import k1_emulate
    sf, osr = 7, 8
    sps = osr << sf
    X, lead, _ = frame_rows(sf, osr, PAY, 0.25 * BW, 0, [1.0], snr_db=None)
    x = X[0]
    tw = tables(sf, osr)[2]
    for c in (0, 1):
        n = x.size // sps
        bins, _ = k1_emulate(x[: n * sps], sf, osr=osr, chirp=shifted_chirp(sf, osr, c), tw=tw)
        assert _runs(bins[2:10]), (c, bins[:12])
    frames = receive_wide(x, sf, osr, 1.0 * (1 << sf))
    assert len(frames) == 1, frames
    _one(frames, lead, 0.25, sf)


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("soft", [False, True])
def test_search_within_bw4_is_the_receiver_without_it(osr, soft):
    """max_cfo_bins = N/4 (C = 0): the same frames, starts, CFOs, SNRs and payloads as the receiver without the search, on
    frames inside and outside BW/4 and on noise."""
    sf = 8
    for k, cfo_bw in enumerate((0.0, 0.1, -0.2, 0.3, 0.6)):
        X, _, _ = frame_rows(sf, osr, PAY, cfo_bw * BW, 11 * k, [1.0], snr_db=-3.0 if k % 2 else 10.0, seed=k)
        a = receive_emul(X[0], sf, osr, soft=soft)
        b = receive_wide(X[0], sf, osr, (1 << sf) / 4, soft=soft)
        for f in a:
            f.pop("h")
        assert a == b, (cfo_bw, a, b)


@pytest.mark.parametrize("sf", [7, 10])
@pytest.mark.parametrize("cfo_bw", [0.6, -1.2, 2.5])
@pytest.mark.parametrize("soft", [False, True])
def test_two_antennas_at_wide_offsets(sf, cfo_bw, soft):
    X, lead, _ = frame_rows(sf, 8, PAY, cfo_bw * BW, 41, [1.0, 0.6 - 0.5j], snr_db=[3.0, 6.0], seed=sf)
    _one(receive_wide(X, sf, 8, band_limit_bins(sf, 8), soft=soft), lead, cfo_bw, sf)


def test_clock_offset_follows_a_wide_cfo():
    """With carrier_hz, a frame 1.2 BW off carrier has its windows placed with the clock offset its CFO implies."""
    sf, carrier = 9, 868.1e6
    cfo = 1.2 * BW
    ppm = cfo / carrier * 1e6
    X, lead, _ = frame_rows(sf, 8, PAY * 4, cfo, 5, [1.0], snr_db=15.0, sfo_ppm=ppm)
    frames = receive_wide(X[0], sf, 8, band_limit_bins(sf, 8), carrier_hz=carrier)
    _one(frames, lead, 1.2, sf, PAY * 4)
    assert abs(frames[0]["sfo"] - ppm) < 0.05


def test_entry_point_refuses_out_of_band_search():
    sf = 7
    X, _, _ = frame_rows(sf, 8, PAY, 0.0, 0, [1.0], snr_db=None)
    assert receive_wide(X[0], sf, 8, band_limit_bins(sf, 8) + 1) == []
    assert receive_wide(X[0], sf, 2, band_limit_bins(sf, 2) + 1) == []
    assert receive_wide(X[0], sf, 8, 0.0) == []
