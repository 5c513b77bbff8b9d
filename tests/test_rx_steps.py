"""CPU twins of tests/test_gpu_rx_steps.py: for every capture of tests/rx_steps_common.py the oracle alone must take the
branch the capture was built for, and the stream kernels' shared bookkeeping (rx_stream.cuh, run on the host) must replay
the oracle's steps to the oracle's next states, frames and printed lines."""
import pytest

import rx_steps_common as S

CASES = S.cases()


@pytest.fixture(scope="module")
def emul():
    return S.emul_lib()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_case_takes_its_branch_and_the_bookkeeping_replays_it(oracle, emul, case):
    steps, frames, consumed, final, out = S.oracle_run(oracle, case.cfg, case.x)
    assert len(steps) > 0 and consumed <= case.x.size
    if case.branch is not None:
        case.branch(steps, frames, final)
    S.assert_bookkeeping_replays(emul, case.cfg, steps, frames, final, out)


def test_ladder_loses_frames_at_the_bottom_and_decodes_at_the_top(oracle):
    """the ladder spans the gates: at 8 dB nothing is detected or the SFD search gives up, at 26 dB every SF publishes"""
    got = {}
    for case in S.cases("ladder"):
        snr = float(case.name.split("_")[2][:-2])
        got.setdefault(snr, []).append(len(S.oracle_run(oracle, case.cfg, case.x)[1]))
    assert not any(got[8.0]) and all(got[26.0])


def test_comparator_rules(oracle):
    """assert_steps_match on the oracle's own steps, and on edited copies: a consumed off by one outside SYNC, an
    uncompensated SYNC neighbour, a metric moved by 1e-4, one step more"""
    c = S.cfg(8)
    x = S.assemble([S.gap(c, 2.13), S.sig(S.frame(S.PAY, c)), S.gap(c, 3)], snr_db=30.0, seed=11)
    steps = S.oracle_run(oracle, c, x)[0]
    tr = [(int(s["state"]), int(s["consumed"]), int(s["bin"]), int(s["fine_sync"]), float(s["metric"])) for s in steps]
    worst = S.assert_steps_match(tr, steps, x, 8, "rx_stream_kernel")
    assert 0 < max(worst.values()) < 1
    k = next(i for i, t in enumerate(tr) if t[0] == 1)

    def edited(i, **kw):
        t = list(tr)
        d = dict(zip(("state", "consumed", "bin", "fine_sync", "metric"), t[i]))
        d.update(kw)
        t[i] = tuple(d.values())
        return t

    for bad, kernel in ((edited(k + 2, consumed=tr[k + 2][1] + 1), "rx_stream_kernel"),
                        (edited(k, consumed=tr[k][1] + 1), "rx_warp_kernel"),
                        (edited(k, consumed=tr[k][1] + 1), "rx_stream_kernel"),          # never pulled back: totals differ
                        (edited(0, metric=tr[0][4] + 1e-4), "rx_stream_kernel"),
                        (edited(k + 1, metric=tr[k + 1][4] - 1e-4), "rx_stream_kernel"),
                        (edited(len(tr) - 1, state=2), "rx_stream_kernel"),
                        (tr + [tr[-1]], "rx_stream_kernel"), (tr[:-1], "rx_stream_kernel")):
        with pytest.raises(AssertionError):
            S.assert_steps_match(bad, steps, x, 8, kernel)
