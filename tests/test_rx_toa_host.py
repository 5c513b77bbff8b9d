"""CPU: the dechirp receiver's fine time of arrival (lora_b200_rx_params.fine_toa, rs_toa in csrc/rx_sync.cuh) through its
host emulation -- against the float64 restatement of its definition (tests/toa_reference.py) on given frames, the
restatement against known mistakes, clean frames over the whole timing and CFO range, and accuracy in noise end to end."""
import numpy as np
import pytest

from toa_reference import NU_BOUND, SENSITIVITY, emul_toa, frame_rows, half_width, receive_toa, reference, rms, toa_bound

GAINS = (1.0, 0.6j, -0.35 + 0.2j, 0.15)


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf", range(7, 13))
def test_emulation_holds_the_definition(sf, osr):
    """Given frames, noisy, on 1..4 antennas of unequal gains, without and with +-20 ppm clock offsets, and one whose first
    preamble windows precede the row start: the emulation's nu_A, nu_B within NU_BOUND bins of the float64 reference and
    toa within osr NU_BOUND samples."""
    rng = np.random.default_rng(sf * 10 + osr)
    n = 1 << sf
    cases = [(1, 0.0, 0), (2, 20.0, 0), (3, -20.0, 0), (4, 0.0, 0), (1, 20.0, 3)]
    for m, ppm, cut in cases:
        delay, cfo = float(rng.uniform(0, 1)), float(rng.uniform(-n / 4, n / 4))
        X, truth = frame_rows(sf, osr, delay, cfo, GAINS[:m], ppm=ppm, snr_db=SENSITIVITY[sf] + 6, seed=int(rng.integers(1 << 30)))
        t = int(np.floor(truth)) + int(rng.integers(-osr // 2, osr // 2 + 1))
        if cut:                                       # the row starts inside preamble window `cut`
            k = int(truth) + cut * (osr << sf) + 7
            X, t = np.ascontiguousarray(X[:, k:]), t - k
        ea, eb, et = emul_toa(X, sf, osr, [t], [cfo], [ppm])
        ra, rb, rt = reference(X, sf, osr, t, cfo, ppm)
        assert abs(ea[0] - ra) <= NU_BOUND and abs(eb[0] - rb) <= NU_BOUND, (m, ppm, cut, ea, ra, eb, rb)
        assert abs(et[0] - rt) <= toa_bound(osr), (m, ppm, cut, et, rt)


def test_reference_catches_mistakes():
    """Each restated mistake moves the reference's answer by more than the bound the tests hold the receiver to: a flipped
    sign, a missing rounding correction (+-20 ppm at SF12), the SFD windows left out (the CFO 0.05 bin off, as the
    synchroniser's estimate may be), and one antenna left out."""
    sf, osr = 12, 8
    for ppm in (20.0, -20.0):
        X, truth = frame_rows(sf, osr, 0.4, 7.3, ppm=ppm)
        t = int(truth) - 2
        good = reference(X, sf, osr, t, 7.3, ppm)[2]
        assert abs(good - truth) < 0.01
        assert abs(reference(X, sf, osr, t, 7.3, ppm, sign=-1)[2] - good) > 1.0
        assert abs(reference(X, sf, osr, t, 7.3, ppm, rounding=False)[2] - good) > 4 * toa_bound(osr)
    X, truth = frame_rows(7, osr, 0.4, 7.3)
    t = int(truth)
    good = reference(X, 7, osr, t, 7.35)[2]
    assert abs(good - truth) < 0.05
    assert abs(reference(X, 7, osr, t, 7.35, sfd=False)[2] - good) > 0.3
    X, truth = frame_rows(7, osr, 0.4, 7.3, (0.3, 1.0), snr_db=-2.0, seed=5)
    good = reference(X, 7, osr, t, 7.3)[2]
    assert abs(reference(X, 7, osr, t, 7.3, antennas=[0])[2] - good) > 2 * toa_bound(osr)


# the largest |toa - truth| on clean frames over eps in +-(osr / 2 + 1) samples and |CFO| <= N / 4, in samples: the bias of
# the windows' dechirped tones (the SFD's and the preamble's first samples belong to the symbol before) and the search
CLEAN_BOUND = {8: 0.02, 2: 0.01}


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf", [7, 10])
def test_clean_frames_over_the_range(sf, osr):
    n, W = 1 << sf, osr / 2 + 1
    errs = []
    for k, eps in enumerate(np.linspace(-W, W, 9)):
        for cfo in (-n / 4, -0.37 * n / 4, 0.0, 0.61 * n / 4, n / 4):
            X, truth = frame_rows(sf, osr, 0.5 + eps % 1.0, cfo)
            t = int(round(truth - eps))
            errs.append(emul_toa(X, sf, osr, [t], [cfo], [0.0])[2][0] - truth)
    assert np.max(np.abs(errs)) <= CLEAN_BOUND[osr], np.max(np.abs(errs))
    assert half_width(osr) * osr >= W        # (the search covers the range)


def accuracy(sf, osr, snr_db, n_frames, seed, ppm=0.0):
    """(toa - truth, start - truth) of the published frames of n_frames captures, each one frame at a random fractional
    delay, random CFO within N/8."""
    rng = np.random.default_rng(seed)
    e_toa, e_start = [], []
    for _ in range(n_frames):
        delay, cfo = float(rng.uniform(0, 1)), float(rng.uniform(-1, 1) * (1 << sf) / 8)
        X, truth = frame_rows(sf, osr, delay, cfo, ppm=ppm, snr_db=snr_db, seed=int(rng.integers(1 << 30)))
        pub = [f for f in receive_toa(X[0], sf, osr, sfo_ppm=ppm) if f["status"] == 0 and abs(f["start"] - truth) < osr << sf]
        for f in pub[:1]:
            e_toa.append(f["toa"] - truth)
            e_start.append(f["start"] - truth)
    return np.array(e_toa), np.array(e_start)


@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("sf", [7, 8, 9, 10])
def test_accuracy_in_noise(sf, osr):
    """96 frames per point: from the sensitivity point up, the fine estimate's RMS error below the integer start's, and at
    sensitivity + 20 dB within 0.01 chip (osr / 100 samples).  (SF11 and SF12, where the CPU emulation of the screen is
    slowest, are measured on the device, tests/test_gpu_rx_toa.py, and recorded in DESIGN.md.)"""
    for k, snr in enumerate((SENSITIVITY[sf], SENSITIVITY[sf] + 5, SENSITIVITY[sf] + 10, SENSITIVITY[sf] + 20)):
        et, es = accuracy(sf, osr, snr, 96, seed=100 * osr + k)
        assert et.size >= 80, et.size
        assert rms(et) < rms(es), (snr, rms(et), rms(es))
        if k == 3:
            assert rms(et) <= 0.01 * osr, rms(et)
