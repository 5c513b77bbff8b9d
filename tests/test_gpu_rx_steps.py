"""GPU: both stream state machines (rx_warp_kernel: SF7 at fs / bw = 8; rx_stream_kernel: everything else) held to the
oracle step by step off the happy path -- low SNR, failed SFDs, damaged and back-to-back frames, implicit headers, other
sample rates (the captures of tests/rx_steps_common.py, whose CPU twins are tests/test_rx_steps.py) -- with every recorded
metric against its float64 statistic (tests/rx_reference.py); the per-call limits; and many streams fed in chunks, each
at its own pace.  RX_STEPS_REPORT=<file> writes the worst err / bound per kernel and statistic as JSON."""
import json
import os

import numpy as np
import pytest

import rx_steps_common as S

pytestmark = pytest.mark.gpu
CASES = S.cases()


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    yield torch
    report = {"worst_err_over_bound": {f"{k} / {s}": v for (k, s), v in sorted(S.WORST.items())}, **S.COUNTS,
              "device": torch.cuda.get_device_name(0)}
    print("\nstate machine against float64:", json.dumps(report, indent=1))
    if os.environ.get("RX_STEPS_REPORT"):
        with open(os.environ["RX_STEPS_REPORT"], "w") as f:
            json.dump(report, f, indent=1)


def _tuples(steps):
    return [(int(s["state"]), int(s["consumed"]), int(s["bin"]), int(s["fine_sync"]), float(s["metric"])) for s in steps]


def _one_shot(c, x, demod, n_steps, **kw):
    dec = S.gpu_decoder(c, demod, trace_capacity=n_steps + 8, max_items_per_call=x.size, **kw)
    consumed = dec.work(x)
    got = dict(consumed=consumed, trace=dec.trace(), frames=[f for _, f in dec.frames], stdout=S.stdout_last(dec), state=dec.state())
    dec.close()
    return got


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_kernel_follows_the_oracle_step_by_step(torch, oracle, case):
    c = case.cfg
    for demod in S.demods_of(case):
        steps, frames, consumed, final, out = S.oracle_run(oracle, c, case.x, demod)
        got = _one_shot(c, case.x, demod, len(steps))
        try:
            S.assert_steps_match(got["trace"], steps, case.x, c["sf"], S.kernel_of(c), fs=c["fs"], implicit=c["implicit"],
                                 allow_open=case.name in S.FLAT_SYNC_PEAK)
        except S.DecisionOpen:
            continue                    # the kernel took another of the tied lags: nothing after that step is comparable
        assert got["frames"] == frames
        assert got["consumed"] == consumed and got["state"] == final
        assert got["stdout"] == S.published_stdout(out)


# ---- per-call limits ---------------------------------------------------------------------------------------------------
def _three_frames(sf):
    return [k for k in S.cases("back_to_back") if k.name == f"three_frames_gap_1_sf{sf}"][0]


@pytest.mark.parametrize("sf", [7, 9])
def test_one_frame_per_call_equals_one_shot(torch, oracle, sf):
    """max_frames_per_call = 1: every call stops after its frame, the caller re-presents from consumed; frames, total
    consumed, concatenated traces and the final state equal the one-shot run's and the oracle's"""
    case = _three_frames(sf)
    c, x = case.cfg, case.x
    steps, frames, consumed, final, out = S.oracle_run(oracle, c, x)
    assert len(frames) == 3
    dec = S.gpu_decoder(c, trace_capacity=len(steps) + 8, max_items_per_call=x.size, max_frames_per_call=1)
    pos, trace, text, calls = 0, [], "", 0
    while x.size - pos >= 2 * dec.sps:
        n = dec.work(x[pos:])
        trace += dec.trace()
        text += S.stdout_last(dec)
        calls += 1
        assert len(dec.frames) <= calls
        if n == 0:
            break
        pos += n
    assert calls == 4 and [f for _, f in dec.frames] == frames and pos == consumed and dec.state() == final
    assert text == S.published_stdout(out)
    S.assert_steps_match(trace, steps, x, sf, S.kernel_of(c))
    dec.close()


@pytest.mark.parametrize("sf", [7, 9])
def test_trace_capacity_smaller_than_the_steps(torch, oracle, sf):
    """lora_b200_trace_read with fewer records than steps: the first trace_capacity steps, the true count and
    LORA_B200_EOVERFLOW; frames and consumed are not affected"""
    import ctypes as C
    from gr_lora_b200 import _native as N
    case = _three_frames(sf)
    c, x = case.cfg, case.x
    steps, frames, consumed, _, _ = S.oracle_run(oracle, c, x)
    cap = 10
    dec = S.gpu_decoder(c, trace_capacity=cap, max_items_per_call=x.size)
    assert dec.work(x) == consumed and [f for _, f in dec.frames] == frames
    buf, n = (N.Step * 64)(), C.c_size_t(0)
    rc = dec._L.lora_b200_trace_read(dec._h, 0, buf, 64, C.byref(n))
    assert rc == N.EOVERFLOW and n.value == len(steps) > cap
    tr = dec.trace()
    assert len(tr) == cap
    S.assert_steps_match(tr + _tuples(steps[cap:]), steps, x, sf, S.kernel_of(c))
    dec.close()


# ---- many streams, fed in chunks ---------------------------------------------------------------------------------------
def _rows(sf, n_streams, seed):
    """n_streams captures of one SF, every stream its own payload, CR field in the header, lead and number of frames; stream 1
    is noise only and stream 2 true silence (where there are that many).  One decoder configuration (CR 4/8 payloads are
    announced by each frame's own header)."""
    c = S.cfg(sf, cr=4, crc=False)
    rng = np.random.default_rng(seed)
    caps = []
    for s in range(n_streams):
        if s == 1 and n_streams > 2:
            caps.append(S.assemble([S.noise(c, 30, -10.0)], snr_db=30.0, seed=seed + s))
        elif s == 2 and n_streams > 2:
            caps.append(np.zeros(25 * S.sps_of(c), np.complex64))
        else:
            cs = dict(c, cr=1 + (s % 4))
            parts = [S.gap(c, 2.0 + 0.37 * (s % 9))]
            for k in range(1 + s % 3 if sf < 12 else 1):
                parts += [S.sig(S.frame(bytes(rng.integers(0, 256, 2 + (s + k) % 7 if sf < 12 else 2, dtype=np.uint8)), cs)), S.gap(c, 1.5 + 0.5 * k)]
            caps.append(S.assemble(parts + [S.gap(c, 2.5)], snr_db=30.0, seed=seed + s))
    n = max(x.size for x in caps)
    rows = np.zeros((n_streams, n), np.complex64)
    for s, x in enumerate(caps):
        rows[s, :x.size] = x
    return c, rows


CHUNKED = [(7, 1, "gradient"), (7, 8, "gradient"), (7, 9, "fft"), (7, 10, "gradient"), (7, 11, "fft"), (7, 37, "gradient"),
           (9, 5, "gradient"), (9, 5, "fft"), (12, 5, "gradient")]


@pytest.mark.parametrize("sf,n_streams,demod", CHUNKED)
def test_many_streams_in_chunks_equal_one_shot_and_the_oracle(torch, oracle, sf, n_streams, demod):
    """Each stream advances by its own consumed while its neighbours -- other warps of one CTA in rx_warp_kernel -- sit in
    other states: per stream, frames, total consumed, the concatenated per-call traces and the final state equal the
    one-shot batch's and the oracle's, for chunks of 2.5, 7 and 40 symbols and a random size per call, from host and from
    device memory; two runs are identical."""
    c, rows = _rows(sf, n_streams, 8100 + 10 * sf + n_streams)
    sps, n = S.sps_of(c), rows.shape[1]
    want = [S.oracle_run(oracle, c, rows[s], demod) for s in range(n_streams)]
    cap = max(len(w[0]) for w in want) + 8
    kernel = S.kernel_of(c)

    def check(got, what):
        for s, (steps, frames, consumed, final, out) in enumerate(want):
            w = f"{what} stream {s}"
            S.assert_steps_match(got["trace"][s], steps, rows[s], sf, kernel)
            assert got["frames"][s] == frames, w
            assert got["consumed"][s] == consumed and got["state"][s] == final, w
            assert got["stdout"][s] == S.published_stdout(out), w

    dec = S.gpu_decoder(c, demod, n_streams=n_streams, trace_capacity=cap, max_items_per_call=n)
    consumed = dec.work_batch(rows)
    one = dict(trace=[dec.trace(s) for s in range(n_streams)], frames=[[f for st, f in dec.frames if st == s] for s in range(n_streams)],
               consumed=[int(v) for v in consumed], state=[dec.state(s) for s in range(n_streams)],
               stdout=[S.stdout_last(dec, s) for s in range(n_streams)])
    check(one, "one shot")
    assert sum(len(f) for f in one["frames"]) >= (n_streams + 1) // 2
    rng = np.random.default_rng(sf * 100 + n_streams)
    plans = [(int(2.5 * sps), None), (7 * sps, torch.device("cuda", 0)), (40 * sps, None), ((2 * sps, 12 * sps), torch.device("cuda", 0))]
    if sf == 12:
        plans = plans[:2]
    for chunk, device in plans:
        dec.reset()
        got = S.run_batch_chunked(dec, rows, chunk, device=device, rng=rng)
        check(got, f"chunks of {chunk}")
        assert repr(got["trace"]) == repr(one["trace"]) and got["frames"] == one["frames"]
    dec.reset()
    again = S.run_batch_chunked(dec, rows, int(2.5 * sps))
    dec.reset()
    first = S.run_batch_chunked(dec, rows, int(2.5 * sps))
    assert repr(again) == repr(first)
    dec.close()
