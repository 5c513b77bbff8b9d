"""CPU: the dechirp receiver with several antennas per receiver through its host emulation (lb_emul_rx_receive_antennas):
M = 1 is the one-row receiver, the combined screen meets a float64 sum over antennas of |tmp_a|^2, and clean frames with
arbitrary per-antenna gains give back start, CFO, payload and the gains themselves."""
import numpy as np
import pytest

from antenna_common import BW, CombinedReference, frame_rows, k1_antennas_emulate, k1_batch, receive_emul

KEYS = ("start", "cfo", "snr", "status", "payload")


# ---- M = 1 is the one-row receiver; identical rows are one row ----------------------------------------------------------------
def existing_capture(sf, osr, pay, cfo_bins, offset, snr, seed):
    """The receiver tests' own captures: tests/test_rx_sync_host.py's one_frame at fs/bw = 8, tests/osr2_common.py's frame_row
    at fs/bw = 2."""
    if osr == 8:
        from test_rx_sync_host import one_frame
        return one_frame(sf, pay, cfo_bins, offset, snr_db=snr, seed=seed)[0]
    from osr2_common import frame_row
    return frame_row(sf, pay, cfo_bins * BW / (1 << sf), offset, snr_db=snr, seed=seed)[0]


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf", range(7, 13))
def test_one_antenna_is_the_one_row_receiver(sf, osr):
    """On the receiver tests' captures at +10 dB and 1 dB above the sensitivity point, hard and soft:
    lb_emul_rx_receive_antennas with M = 1 returns lb_emul_rx_receive_osr's frames (start, CFO, SNR, status, payload) exactly,
    and the same row given as M = 2 and M = 4 identical antennas (equal weights, every statistic scaled alike) gives the
    same starts, statuses and payloads, CFOs within 1e-3 bin and SNRs 10 log10 M dB higher within 0.1 dB (the one-row
    estimate is taken before the last CFO step, the combined one after it)."""
    rng = np.random.default_rng(10 * sf + osr)
    sps = osr << sf
    from antenna_common import SENSITIVITY
    for snr in ((10.0,) if sf >= 11 else (10.0, SENSITIVITY[sf] + 1.0)):
        pay = bytes(rng.integers(0, 256, 8, dtype=np.uint8))
        x = existing_capture(sf, osr, pay, float(rng.uniform(-0.9, 0.9) * (1 << sf) / 4), int(rng.integers(0, sps)), snr,
                             int(rng.integers(1 << 30)))
        for soft in ((False,) if sf >= 11 else (False, True)):
            one = receive_emul(x, sf, osr, soft=soft)
            ant = receive_emul(x[None, :], sf, osr, soft=soft)
            assert [{k: g[k] for k in KEYS} for g in ant] == [{k: g[k] for k in KEYS} for g in one], (snr, soft)
            if snr >= 10.0:
                assert [g["payload"] for g in one if g["status"] == 0] == [pay]
            for m in ((2,) if sf >= 11 else (2, 4)):
                rep = receive_emul(np.stack([x] * m), sf, osr, soft=soft)
                assert [(g["start"], g["status"], g["payload"]) for g in rep] == [(g["start"], g["status"], g["payload"]) for g in one]
                for a, b in zip(rep, one):
                    assert abs(a["cfo"] - b["cfo"]) <= 1e-3 and abs(a["snr"] - b["snr"] - 10 * np.log10(m)) <= 0.1, (m, a, b)


# ---- the combined screen against float64 -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf", range(7, 13))
def test_combined_screen_against_float64(sf, osr):
    """Every bin clean (a spread at SF11/12), -3 dB, half-bin and noise windows on M = 2, 3 and 4 antennas (2 and 3 at SF11/12), each antenna its own
    symbols and gain: bin and magnitude inside the band of the float64 sum_a |tmp_a|^2; the criterion fails when any one
    antenna is left out of the reference's sum."""
    rng = np.random.default_rng(100 * sf + osr)
    sps = osr << sf
    for m in ((2, 3) if sf >= 11 else (2, 3, 4)):
        batches = [k1_batch(sf, osr, np.random.default_rng(1000 * sf + 10 * osr + a), n_clean=24 if sf >= 11 else None)
                   for a in range(m)]
        n = min(b.shape[0] for b in batches)
        gains = np.exp(2j * np.pi * rng.uniform(size=m)) * 10 ** (rng.uniform(-3, 3, m) / 20)
        X = np.stack([g * b[:n] for g, b in zip(gains, batches)]).astype(np.complex64)
        bins, mags = k1_antennas_emulate(X.reshape(m, n * sps), sf, osr)
        ref = CombinedReference(X, sf, osr)
        ties = ref.check(bins, mags, f"SF{sf} fs/bw={osr} M={m}")
        assert ties < n // 4
        for drop in range(m):
            keep = [a for a in range(m) if a != drop]
            with pytest.raises(AssertionError):
                CombinedReference(X, sf, osr, antennas=keep).check(bins, mags)


# ---- clean frames with per-antenna gains ---------------------------------------------------------------------------------------------
CASES = {
    "opposite": lambda rng: [1.0, -1.0],                                            # one antenna at 180 degrees to the other
    "noise_only": lambda rng: [1.0, 1.0],                                           # antenna 1 carries noise only
    "weak": lambda rng: [np.exp(1j * rng.uniform(0, 2 * np.pi)), 0.1 * np.exp(1j * rng.uniform(0, 2 * np.pi))],   # -20 dB
    "four": lambda rng: list(10 ** (rng.uniform(-6, 6, 4) / 20) * np.exp(2j * np.pi * rng.uniform(size=4))),
}


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf", range(7, 13))
def test_clean_frames_with_antenna_gains(sf, osr):
    """M = 2 and 4 with arbitrary per-antenna gains and phases (one antenna at 180 degrees, one antenna noise only, one 20 dB
    weaker): start within one sample, CFO within 1/8 bin and the payload; at +10 dB the channel estimates' ratios and phase
    differences meet the true gains' to 0.5 dB and 5 degrees, for gains within 6 dB of each other (the 20 dB weaker antenna's
    estimate at +30 dB, which puts that antenna at +10 dB)."""
    rng = np.random.default_rng(7 * sf + osr)
    sps, nb = osr << sf, 1 << sf
    for case in CASES:
        gains = CASES[case](rng)
        noise_only = (1,) if case == "noise_only" else ()
        pay = bytes(rng.integers(0, 256, 6, dtype=np.uint8))
        cfo_bins = float(rng.uniform(-0.9, 0.9) * nb / 4)
        off = int(rng.integers(0, sps))
        for snr in (None, 10.0) + ((30.0,) if case == "weak" else ()):
            X, lead, _ = frame_rows(sf, osr, pay, cfo_bins * BW / nb, off, gains, snr_db=snr, seed=int(rng.integers(1 << 30)),
                                    noise_only=noise_only)
            got = [g for g in receive_emul(X, sf, osr) if g["status"] == 0]
            assert len(got) == 1, (case, snr, got)
            g = got[0]
            assert abs(g["start"] - lead) <= 1 and abs(g["cfo"] - cfo_bins) <= 1 / 8 and g["payload"] == pay, (case, snr, g, lead, cfo_bins)
            t = np.asarray(gains, np.complex128)
            if snr is None or noise_only or snr + 20 * np.log10(np.min(np.abs(t))) < 3.0:
                continue
            h = g["h"].astype(np.complex128)
            for a in range(1, len(gains)):
                r_est, r_true = h[a] / h[0], t[a] / t[0]
                assert abs(20 * np.log10(abs(r_est) / abs(r_true))) <= 0.5, (case, a, h, t)
                assert abs(np.degrees(np.angle(r_est / r_true))) <= 5.0, (case, a, h, t)
