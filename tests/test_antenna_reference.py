"""CPU: the float64 references of the several-antenna receiver (tests/antenna_reference.py) -- they accept what the host
emulation (lb_emul_rx_receive_antennas) computes, they reject each wrong rule a kernel could plausibly follow, and on rows
of known gains and noise powers they give back the maximum-ratio weights and the combined SNR that physics predicts."""
import math

import numpy as np
import pytest

from antenna_common import BW, frame_rows, receive_emul, tables
from antenna_reference import ChannelReference, assembly_windows, rs_sym


def capture(sf, osr, m, snr_db, seed, sfo_ppm=0.0):
    """One frame on m antennas with random gains within +-6 dB and phases; per-antenna noise levels snr_db (a sequence, None =
    noiseless).  Returns (X, lead, gains, cfo_bins)."""
    rng = np.random.default_rng(seed)
    sps, nb = osr << sf, 1 << sf
    gains = 10 ** (rng.uniform(-6, 6, m) / 20) * np.exp(2j * np.pi * rng.uniform(size=m))
    cfo_bins = float(rng.uniform(-0.9, 0.9) * nb / 4)
    pay = bytes(rng.integers(0, 256, 8, dtype=np.uint8))
    X, lead, _ = frame_rows(sf, osr, pay, cfo_bins * BW / nb, int(rng.integers(0, sps)), list(gains), snr_db=snr_db,
                            seed=int(rng.integers(1 << 30)), sfo_ppm=sfo_ppm)
    return X, lead, gains, cfo_bins


def emulated_frame(X, sf, osr, sfo_ppm=0.0):
    got = [g for g in receive_emul(X, sf, osr, sfo_ppm=sfo_ppm) if g["status"] == 0]
    assert len(got) == 1, got
    return got[0]


# ---- the reference accepts the host emulation --------------------------------------------------------------------------------
@pytest.mark.parametrize("ppm", [0.0, 40.0])
@pytest.mark.parametrize("m", [2, 3, 4])
@pytest.mark.parametrize("osr", [8, 2])
def test_reference_accepts_the_host_emulation(osr, m, ppm):
    """SF8 at +10 dB per antenna (each antenna its own noise level, 0 to 12 dB apart), with and without a clock offset: the
    emulation's h and combined snr_db (rs_channels over float64 window sums, at the emulation's own start, cfo_bins and
    clock offset) lie within the reference's bounds."""
    sf = 8
    levels = [10.0, 4.0, -2.0, 7.0][:m]
    X, _, _, _ = capture(sf, osr, m, levels, seed=31 * m + osr + int(ppm), sfo_ppm=ppm)
    g = emulated_frame(X, sf, osr, sfo_ppm=ppm)
    assert g["sfo"] == np.float32(ppm)
    ref = ChannelReference(X, X.shape[1], g["start"], g["cfo"], g["sfo"], tables(sf, osr)[0], osr)
    ref.check_h(g["h"], "emulation")
    ref.check_snr(g["snr"], "emulation")


# ---- the reference rejects wrong quantities -------------------------------------------------------------------------------------
def test_reference_rejects_wrong_channel_rules():
    """On one emulated frame (SF8, M = 3, noise levels 0, 6 and 20 dB apart): h over windows 0..5, windows one sample late
    and F off by 1e-3 bin each fail the h check; weights without the noise normalisation and without the conjugate fail the
    weight check, which the reference's own weights in float32 pass."""
    sf, osr, m = 8, 8, 3
    X, _, _, _ = capture(sf, osr, m, [26.0, 20.0, 6.0], seed=5)
    g = emulated_frame(X, sf, osr)
    down = tables(sf, osr)[0]
    args = (X, X.shape[1], g["start"], g["cfo"], g["sfo"], down, osr)
    ref = ChannelReference(*args)
    ref.check_h(g["h"])
    for wrong in (ChannelReference(*args, windows=range(0, 6)),
                  ChannelReference(X, X.shape[1], g["start"] + 1, g["cfo"], g["sfo"], down, osr),
                  ChannelReference(X, X.shape[1], g["start"], float(np.float32(g["cfo"] + 1e-3)), g["sfo"], down, osr)):
        with pytest.raises(AssertionError):
            wrong.check_h(g["h"])
    ref.check_w(ref.w.astype(np.complex64))
    for wrong in (ChannelReference(*args, normalise=False).w, ChannelReference(*args, conj=False).w):
        with pytest.raises(AssertionError):
            ref.check_w(wrong.astype(np.complex64))


def test_assembly_bound_rejects_a_float32_phase():
    """Data windows of a frame starting past 2^24 samples: the float64 assembly reference in complex64 lies within its own
    bound, and the same windows with the de-rotation phase F n / sps formed and reduced in float32 do not."""
    sps, m = 256 * 8, 2
    start = (1 << 24) + 12345
    n_items = start + 20 * sps
    rng = np.random.default_rng(9)
    X = np.zeros((m, n_items), np.complex64)
    X[:, start:] = (rng.standard_normal((m, n_items - start)) + 1j * rng.standard_normal((m, n_items - start))).astype(np.complex64)
    w = np.array([0.6 + 0.2j, -0.3 + 0.7j], np.complex64)
    y, bound = assembly_windows(X, n_items, sps, start, 37.3125, 20.0, 0, 4, w)
    assert np.all(np.abs(y.astype(np.complex64) - y) <= bound)
    y32, _ = assembly_windows(X, n_items, sps, start, 37.3125, 20.0, 0, 4, w, phase32=True)
    assert np.mean(np.abs(y32 - y) > bound) > 0.5


# ---- physics anchor -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("osr", [8, 2])
def test_reference_weights_and_snr_against_known_gains_and_noise(osr):
    """Rows of known gains g_a and noise powers sigma_a^2, 0, 6 and 20 dB apart (SF9, the strongest at +30 dB in 125 kHz):
    the reference's weights meet maximum-ratio combining, w_a / w_0 = (conj(g_a) / sigma_a^2) / (conj(g_0) / sigma_0^2), to 3
    per cent, and its snr_db meets 10 log10 sum_a |g_a|^2 / sigma_a^2 (in 125 kHz) to 0.5 dB.  A noiseless row next to a noisy
    one: its noise power is the floor, 1e-6 of the strongest antenna's energy per sample, and carries the weights."""
    sf = 9
    levels = [30.0, 24.0, 10.0]
    X, lead, gains, cfo_bins = capture(sf, osr, 3, levels, seed=77 + osr)
    down = tables(sf, osr)[0]
    ref = ChannelReference(X, X.shape[1], lead, cfo_bins, 0.0, down, osr)
    s2 = np.array([10 ** (-(lv - 10 * math.log10(osr)) / 10) for lv in levels])      # per sample, for a unit gain
    mrc = np.conj(gains) / s2
    for a in (1, 2):
        r_ref, r_true = ref.w[a] / ref.w[0], mrc[a] / mrc[0]
        assert abs(r_ref / r_true - 1) <= 0.03, (a, r_ref, r_true)
    truth = 10 * math.log10(osr * np.sum(np.abs(gains) ** 2 / s2))
    assert abs(ref.snr_db - truth) <= 0.5, (ref.snr_db, truth)
    # the floor: one noiseless row beside one at +10 dB
    X, lead, gains, cfo_bins = capture(sf, osr, 2, [None, 10.0], seed=78 + osr)
    ref = ChannelReference(X, X.shape[1], lead, cfo_bins, 0.0, down, osr)
    emax = max(np.mean([np.sum(np.abs(X[a, p: p + down.size].astype(np.complex128)) ** 2) for p in
                        (rs_sym(lead, i, down.size, 0.0) for i in range(1, 7))]) / down.size for a in range(2))
    assert math.isclose(ref.s2[0], 1e-6 * emax, rel_tol=1e-12)
    assert ref.s2_lo[0] <= ref.s2[0] <= ref.s2_hi[0]
    assert abs(ref.w[0]) > 0.999 and abs(ref.w[1]) < 0.05
