"""CPU: the float64 statistics of tests/rx_reference.py and their fp32 bounds.  The oracle's recorded metrics (fp32, running
sums, libm's atan2f) meet the criterion on every capture of tests/rx_steps_common.py; deliberately wrong statistics fail it;
and no step of those captures sits on a threshold, except the SYNC ties that DESIGN.md 3 documents -- so that what the GPU
tests require of the kernels there is a matter of arithmetic, not of luck."""
import math

import numpy as np
import pytest

import rx_reference as R
import rx_steps_common as S

CASES = S.cases()



@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_oracle_metrics_meet_the_criterion_and_no_step_is_near_a_threshold(oracle, case):
    c = case.cfg
    steps, _, _, _, _ = S.oracle_run(oracle, c, case.x)
    refs = R.walk(case.x, steps, c["sf"], c["fs"], implicit=c["implicit"])
    assert len(refs) == len(steps) > 0
    for i, (r, s) in enumerate(zip(refs, steps)):
        R.check_metric(r, s["metric"], int(s["consumed"]), what=f"{case.name} step {i}")
    near = [(i, r.near) for i, r in enumerate(refs) if r.near and r.near != "SYNC tie"]
    assert not near, f"{case.name}: steps on a threshold {near}: pick another seed"
    for r in refs:
        if r.sync is not None and r.sync.tie() and case.name not in S.FLAT_SYNC_PEAK:
            # the documented tie: the runner-up is the neighbouring sample
            assert abs(r.sync.runner_up - r.sync.best) == 1, (case.name, r.pos, r.sync.best, r.sync.runner_up)


def _window(oracle, sf, state, seed=3, snr=30.0):
    """(capture, position, oracle step) of the first step in `state` of a clean-ish frame"""
    c = S.cfg(sf)
    x = S.assemble([S.gap(c, 2.13), S.sig(S.frame(S.PAY, c)), S.gap(c, 3)], snr_db=snr, seed=seed)
    steps = S.oracle_run(oracle, c, x)[0]
    pos = 0
    for s in steps:
        if int(s["state"]) == state and pos > 0:
            return x, pos, s
        pos += int(s["consumed"])
    raise AssertionError("state not reached")


@pytest.mark.parametrize("sf", [7, 9])
@pytest.mark.parametrize("state", [R.DETECT, R.SYNC, R.FIND_SFD])
def test_a_metric_moved_by_1e_4_fails(oracle, sf, state):
    """1e-4 (relative for SYNC's correlation, which is of the order of the window length, absolute for the two normalised
    statistics) is more than any bound at these SFs, and less than every margin the existing 30-40 dB tests leave."""
    x, pos, s = _window(oracle, sf, state)
    ref = R.step_reference(x, pos, state, sf)
    m = float(s["metric"])
    assert R.check_metric(ref, m, int(s["consumed"])) < 1.0
    for sign in (1, -1):
        with pytest.raises(AssertionError):
            R.check_metric(ref, m * (1 + sign * 1e-4) if state == R.SYNC else m + sign * 1e-4, int(s["consumed"]))


@pytest.mark.parametrize("sf", [7, 9])
def test_a_pearson_correlation_over_one_entry_more_fails(oracle, sf):
    """sps instead of sps - 1 values (the last one is the repeated one, :243): the statistic moves by about 1 / (2 sps)"""
    x, pos, s = _window(oracle, sf, R.FIND_SFD)
    sps, down, _ = R.tables(sf)
    ref = R.step_reference(x, pos, R.FIND_SFD, sf)
    assert R.check_metric(ref, s["metric"], int(s["consumed"])) < 1.0
    with pytest.raises(AssertionError):
        R.check_metric(ref, np.float32(R.sfd64(x[pos:pos + sps], sps, down, entries=sps).value), int(s["consumed"]))


def test_the_table_mean_of_the_pearson_sum_is_redundant(oracle):
    """sum (f_i - fm)(g_i - gm) = sum (f_i - fm) g_i because sum (f_i - fm) = 0: a kernel that drops `- down_ifreq_avg` from
    its FIND_SFD sum computes the same statistic up to the rounding of its window mean, and no valid criterion can tell."""
    x, pos, _ = _window(oracle, 7, R.FIND_SFD)
    sps, down, _ = R.tables(7)
    a, b = R.sfd64(x[pos:pos + sps], sps, down), R.sfd64(x[pos:pos + sps], sps, down, center=False)
    assert abs(a.value - b.value) < 1e-12 and a.bound > 1e-7


@pytest.mark.parametrize("sf", [7, 11])
def test_an_autocorrelation_normalised_by_the_wrong_half_fails(oracle, sf):
    """|D| / e_a instead of |D| / sqrt(e_a e_b), on the window where the preamble begins (the halves' energies differ)"""
    c = S.cfg(sf)
    x = S.assemble([S.gap(c, 2.5), S.sig(S.frame(S.PAY, c)), S.gap(c, 3)], snr_db=20.0, seed=5)
    sps = S.sps_of(c)
    pos = 2 * sps
    st, ea, eb, _, _ = R.detect64(x[pos:pos + 2 * sps], sps)
    assert abs(ea - eb) > 0.1 * max(ea, eb)
    ref = R.StepRef(R.DETECT, pos, stat=st)
    good = oracle.Decoder(sf=sf).autocorr(x[pos:pos + 2 * sps])
    assert R.check_metric(ref, good, sps) < 1.0
    with pytest.raises(AssertionError):
        R.check_metric(ref, np.float32(st.value * math.sqrt(ea * eb) / ea), sps)


def test_silence_is_nan_and_a_number_there_fails():
    z = np.zeros(4096, np.complex64)
    ref = R.step_reference(z, 0, R.DETECT, 7)
    assert math.isnan(ref.stat.value) and R.check_metric(ref, math.nan, 1024) == 0.0
    with pytest.raises(AssertionError):
        R.check_metric(ref, 0.0, 1024)
    assert math.isnan(R.step_reference(z, 0, R.FIND_SFD, 7).stat.value)


def test_sync_lag_outside_the_band_fails(oracle):
    x, pos, s = _window(oracle, 8, R.SYNC)
    ref = R.step_reference(x, pos, R.SYNC, 8)
    lag = int(s["consumed"])
    assert ref.sync.admissible(lag)
    with pytest.raises(AssertionError):
        R.check_metric(ref, float(ref.sync.c[lag + 3]), lag + 3)


def test_bounds_are_what_the_docstring_derives():
    assert R.sum_bound(2.0, 1024, 1) == (6.0 * 32 + 1) * 2.0 ** -24 * 2.0
    assert R.EPS_F == 2 * 1.8 * 2.0 ** -22 + 3 * math.pi * 2.0 ** -24
    # a ramp's phase errors telescope: the bound of sum w_i f_i grows with the ramp's range, not with its length
    assert R.ifreq_bound(np.linspace(-1, 1, 4096), np.zeros(4096, bool)) < 20 * R.ifreq_bound(np.linspace(-1, 1, 16), np.zeros(16, bool))
    # a sample whose float64 phase step is within EPS_F of pi may unwrap either way in fp32
    x = np.array([1.0, -1.0 + 1e-9j, 1.0], np.complex64)
    f, amb = R.ifreq64(x)
    assert amb[0] and R.ifreq_bound(np.ones(3), amb) > 6.28
