"""Captures off the happy path, the lockstep comparator of a device trace against the oracle's steps, and the run helpers
shared by tests/test_rx_steps.py (CPU: oracle alone) and tests/test_gpu_rx_steps.py (both stream kernels).  No torch."""
from __future__ import annotations

import ctypes as C
import functools
import math
from dataclasses import dataclass

import numpy as np

import rx_reference as R
from rx_reference import DECODE_HEADER, DECODE_PAYLOAD, DETECT, FIND_SFD, SYNC

BW = 125e3


# ---- captures ---------------------------------------------------------------------------------------------------------
def cfg(sf, cr=4, crc=True, implicit=False, fs=1e6):
    """decoder configuration of a case: reduced rate above SF10, as the reference's suites"""
    return dict(sf=sf, cr=cr, crc=crc, implicit=implicit, reduced_rate=sf > 10, fs=fs)


def sps_of(c):
    return int(c["fs"] / BW) << c["sf"]


def frame(payload, c, *, header=None, n_preamble=8, explicit=None):
    """One modulated frame (complex128, unit power) under configuration c.  header: the three bytes an explicit header
    carries instead of the true ones; explicit: override c's header mode (a frame of the other kind)."""
    from gr_lora_b200 import tx
    ex = (not c["implicit"]) if explicit is None else explicit
    fsy = tx.encode_frame(bytes(payload), c["sf"], c["cr"], explicit=ex, has_crc=c["crc"], reduced_rate=c["reduced_rate"], header=header)
    return tx.modulate_frame(fsy, c["sf"], fs=c["fs"], n_preamble=n_preamble, sync_word=0x78 if c["sf"] >= 11 else 0x12)


def upchirps(c, n):
    from gr_lora_b200 import tx
    return np.tile(tx.base_upchirp(c["sf"], fs=c["fs"]), n)


def half_wrap_chirps(c, n, early):
    """n periods of a frequency ramp like the up-chirp's, `early` samples ahead of the symbol grid, whose fall at the band
    edge is only half the band (the phase is the running sum of the decoder's own up-chirp instantaneous frequency, the
    values after the fall raised by half its range).  FIND_SFD sees another up-chirp in it (a fall of the whole band that
    far from the window's edge would push the Pearson correlation above -0.97 at SF7's 1024 samples: a cyclic shift of 5
    samples is the most a true up-chirp can show there), and the realignment's best lag is -early."""
    sps, _, up = R.tables(c["sf"], c["fs"])
    k = np.arange(n * sps)
    f = up[np.minimum((k + early) % sps, sps - 2)].copy()
    f[(k % sps) + early >= sps] += 0.5 * (up[sps - 2] - up[0])
    return np.exp(1j * np.concatenate([[0.0], np.cumsum(f)[:-1]]))


def data_start(c):
    """first sample of the first data symbol of a frame()"""
    return 12 * sps_of(c) + sps_of(c) // 4


# a capture is a list of parts (samples, noise): noise None = the capture's background noise, a number = noise of that
# power in dB relative to a unit-power signal, -inf = none at all (true silence: the reference then divides 0 by 0)
def sig(x):
    return (np.asarray(x, np.complex128), None)


def gap(c, symbols):
    return (np.zeros(int(symbols * sps_of(c)), np.complex128), None)


def noise(c, symbols, db):
    return (np.zeros(int(symbols * sps_of(c)), np.complex128), float(db))


def silence(c, symbols):
    return (np.zeros(int(symbols * sps_of(c)), np.complex128), -math.inf)


def assemble(parts, *, snr_db, seed, cfo_hz=0.0, fs=1e6):
    """Concatenate the parts, rotate by the CFO, add white noise (background at snr_db below a unit-power signal); cf32."""
    x = np.concatenate([p for p, _ in parts])
    if cfo_hz:
        x = x * np.exp(2j * np.pi * cfo_hz * np.arange(x.size) / fs)
    power = np.concatenate([np.full(p.size, 10.0 ** ((-snr_db if db is None else db) / 10.0)) for p, db in parts])
    rng = np.random.default_rng(seed)
    x = x + np.sqrt(power / 2.0) * (rng.standard_normal(x.size) + 1j * rng.standard_normal(x.size))
    return x.astype(np.complex64)


# ---- what a case must make the reference do ------------------------------------------------------------------------------
def states_of(steps):
    return "".join(str(int(s)) for s in steps["state"])


def lost_in_sfd(steps, frames, final):
    """>= 5 FIND_SFD steps and then DETECT again: corr_fails ran up to the fall-back (:808-813)"""
    assert "222222" in states_of(steps) and any(a == "2" and b == "0" for a, b in zip(states_of(steps), states_of(steps)[1:])), states_of(steps)


def realigned(steps, frames, final):
    """a FIND_SFD step that saw another up-chirp and moved the window (:801-803) by at least 2 decim samples: more than a
    search of half the reference's width (fine_sync(.., decim * 4): lags within +-(4 decim - 1)) could find"""
    got = [int(s["fine_sync"]) for s in steps if int(s["state"]) == FIND_SFD]
    assert max(abs(v) for v in got) >= 16, f"FIND_SFD corrections {sorted(set(got))}: none of 2 decim = 16 samples or more"


def n_frames(n):
    def check(steps, frames, final):
        assert len(frames) == n, f"{len(frames)} frames, want {n}"
    return check


def gate_fired(steps, frames, final):
    """the implicit header's energy gate ended a frame: a DECODE_PAYLOAD step without a bin (:861-864)"""
    assert any(int(s["state"]) == DECODE_PAYLOAD and int(s["bin"]) == -1 for s in steps), "no DECODE_PAYLOAD step with bin -1"


def silent_steps(steps, frames, final):
    assert np.isnan(steps["metric"][steps["state"] == DETECT]).any(), "no DETECT step on silence (0 / 0)"


def header_reads(cr=None, length=None):
    def check(steps, frames, final):
        assert frames, "no frame"
        f = frames[0]
        if cr is not None:
            assert f[16] >> 5 == cr, f"header CR {f[16] >> 5}, want {cr}"
        if length is not None:
            assert len(f) - 18 == length, f"payload of {len(f) - 18} bytes, want {length}"
    return check


def reaches(state):
    def check(steps, frames, final):
        assert (steps["state"] == state).any(), f"state {state} never entered: {states_of(steps)}"
    return check


def every(*checks):
    def check(steps, frames, final):
        for c in checks:
            c(steps, frames, final)
    return check


@dataclass
class Case:
    name: str
    cfg: dict
    build: object                       # () -> capture
    branch: object = None               # (oracle steps, frames, final state) -> None, asserts the branch the case exists for
    demods: tuple = ("gradient", "fft")

    @functools.cached_property
    def x(self):
        return self.build()


PAY = bytes.fromhex("c0ffee1234")


# Ladder captures whose first seed put a step on a threshold (at these SNRs SYNC's correlation peak is flat and two distant
# lags can tie within fp32 rounding): re-seeded until tests/test_rx_reference.py found no such step.
LADDER_RESEED = {"ladder_sf8_16dB_cfo-600_lead2.999": 1, "ladder_sf8_20dB_cfo-600_lead2.13": 2, "ladder_sf9_20dB_cfo0_lead2": 1,
                 "ladder_sf11_12dB_cfo0_lead2.999": 1, "ladder_sf11_20dB_cfo-600_lead2.13": 3}


def _ladder():
    """SF7..SF12 x 8..26 dB x CFO x lead: down to where the 0.90 / 0.96 / -0.97 gates fail and frames are lost"""
    out = []
    snrs, cfos, leads = (8.0, 12.0, 16.0, 20.0, 26.0), (0.0, -600.0, 900.0), (2.0, 2.13, 2.999)
    for sf in range(7, 13):
        c = cfg(sf, cr=4 if sf % 2 else 2)
        for i, snr in enumerate(snrs):
            for j in (range(3) if sf <= 10 else ((i + 1) % 3,)):
                cfo, lead = cfos[(i + j) % 3], leads[j]
                name = f"ladder_sf{sf}_{snr:g}dB_cfo{cfo:g}_lead{lead:g}"
                seed = 7000 + 100 * sf + 10 * i + j + 1000 * LADDER_RESEED.get(name, 0)
                out.append(Case(name, c,
                                functools.partial(lambda c, lead, snr, seed, cfo: assemble(
                                    [gap(c, lead), sig(frame(PAY[:3] + b"\x12\x34", c)), gap(c, 3)], snr_db=snr, seed=seed, cfo_hz=cfo),
                                    c, lead, snr, seed, cfo),
                                demods=("gradient", "fft") if j == i % 3 else ("gradient",)))
    return out


def _lost():
    out = []
    for sf in (7, 9, 12):
        c = cfg(sf)
        pre = lambda c=c, n=8: sig(upchirps(c, n))
        sync2 = lambda c=c: sig(frame(PAY, c)[8 * sps_of(c):10 * sps_of(c)])
        s = 7100 + sf
        out += [
            Case(f"lost_noise_sf{sf}", c, lambda c=c, pre=pre, s=s: assemble([gap(c, 2.3), pre(), noise(c, 9, 0.0), gap(c, 3)], snr_db=30.0, seed=s),
                 every(lost_in_sfd, n_frames(0)), ("gradient",)),
            Case(f"lost_silence_sf{sf}", c, lambda c=c, pre=pre, s=s: assemble([gap(c, 2.3), pre(), silence(c, 10)], snr_db=30.0, seed=s + 1),
                 every(lost_in_sfd, silent_steps, n_frames(0)), ("gradient",)),
            # a second transmitter's preamble, 18 (SF9) or 24 (SF12) samples early: beyond half of the +-31 samples the
            # realignment searches; at SF7 half_wrap_chirps, 18 samples early
            Case(f"lost_second_preamble_sf{sf}", c,
                 lambda c=c, pre=pre, s=s, sf=sf: assemble(
                     [gap(c, 2.6), pre()] + ([sig(half_wrap_chirps(c, 12, 18))] if sf == 7 else
                                             [sig(upchirps(c, 1)[:-(18 if sf == 9 else 24)]), pre(n=8 + 4 * (sf % 3))])
                     + [noise(c, 8, -3.0), gap(c, 3)], snr_db=40.0, seed=s + 2),
                 every(realigned, lost_in_sfd, n_frames(0)), ("gradient",)),
            Case(f"lost_cut_after_sync_word_sf{sf}", c, lambda c=c, pre=pre, sync2=sync2, s=s: assemble([gap(c, 2.1), pre(), sync2()], snr_db=30.0, seed=s + 3),
                 every(reaches(FIND_SFD), n_frames(0)), ("gradient",)),
        ]
    return out


def _damaged():
    from gr_lora_b200 import tx
    out = []
    pay16 = bytes(range(0x40, 0x50)) + b"\xab\xcd"
    for sf in (7, 9):
        c = cfg(sf)
        d0, sps = data_start(c), sps_of(c)
        for where, cut in (("header", d0 + int(3.5 * sps)), ("payload", d0 + 8 * sps + int(5.5 * sps))):
            for tail_name, tail in (("noise", noise(c, 30, 0.0)), ("silence", silence(c, 30))):
                out.append(Case(f"cut_in_{where}_then_{tail_name}_sf{sf}", c,
                                lambda c=c, cut=cut, tail=tail, sf=sf: assemble([gap(c, 2.4), sig(frame(pay16, c)[:cut]), tail, gap(c, 3)],
                                                                                 snr_db=32.0, seed=7200 + sf + cut % 89),
                                reaches(DECODE_HEADER if where == "header" else DECODE_PAYLOAD)))
    c = cfg(7)
    for cr in (5, 6, 7):
        out.append(Case(f"header_cr{cr}_sf7", c, lambda c=c, cr=cr: assemble(
            [gap(c, 2.2), sig(frame(pay16, c, header=tx.header_bytes(16, cr, 1))), gap(c, 5)], snr_db=34.0, seed=7300 + cr),
            every(n_frames(1), header_reads(cr=4, length=18))))
    for crc in (1, 0):
        # the header announces 255 (+ 2) bytes, the frame carries 18: the decoder reads on through 590 symbols of noise
        out.append(Case(f"header_length_255_crc{crc}_sf7", c, lambda c=c, crc=crc: assemble(
            [gap(c, 2.2), sig(frame(pay16, c, header=tx.header_bytes(255, 4, crc))), noise(c, 600, -6.0), gap(c, 3)], snr_db=34.0, seed=7310 + crc),
            every(n_frames(1), header_reads(length=255 + 2 * crc))))
    out.append(Case("header_length_0_sf7", c, lambda c=c: assemble(
        [gap(c, 2.2), sig(frame(pay16, c, header=tx.header_bytes(0, 4, 0))), gap(c, 5)], snr_db=34.0, seed=7320),
        header_reads(length=0)))
    ci = cfg(7, implicit=True)
    out.append(Case("explicit_decoder_implicit_frame_sf7", c, lambda c=c, ci=ci: assemble(
        [gap(c, 2.2), sig(frame(pay16, ci)), gap(c, 40)], snr_db=34.0, seed=7330), reaches(DECODE_PAYLOAD)))
    out.append(Case("implicit_decoder_explicit_frame_sf7", ci, lambda c=c, ci=ci: assemble(
        [gap(c, 2.2), sig(frame(pay16, c)), gap(c, 8)], snr_db=34.0, seed=7331), every(n_frames(1), gate_fired)))
    return out


def _implicit():
    out = []
    pay = bytes(range(0x30, 0x3c))
    for sf in (7, 10):
        c = cfg(sf, cr=1 if sf == 10 else 4, crc=False, implicit=True)
        s = 7400 + sf
        out += [
            Case(f"implicit_then_silence_sf{sf}", c, lambda c=c, s=s: assemble([gap(c, 2.5), sig(frame(pay, c)), silence(c, 6)], snr_db=30.0, seed=s),
                 every(gate_fired, n_frames(1))),
            Case(f"implicit_then_noise_3dB_below_sf{sf}", c,
                 lambda c=c, s=s: assemble([gap(c, 2.5), sig(frame(pay, c)), noise(c, 40, -3.0), gap(c, 4)], snr_db=30.0, seed=s + 1),
                 reaches(DECODE_PAYLOAD)),
            Case(f"implicit_then_noise_10dB_below_sf{sf}", c,
                 lambda c=c, s=s: assemble([gap(c, 2.5), sig(frame(pay, c)), noise(c, 12, -10.0), gap(c, 4)], snr_db=30.0, seed=s + 2),
                 every(gate_fired, n_frames(1))),
            Case(f"implicit_then_next_frame_sf{sf}", c,
                 lambda c=c, s=s: assemble([gap(c, 2.5), sig(frame(pay, c)), gap(c, 0.5), sig(frame(pay[::-1], c)), gap(c, 5)], snr_db=30.0, seed=s + 3),
                 reaches(DECODE_PAYLOAD)),
        ]
    return out


def _back_to_back():
    out = []
    c = cfg(7, cr=3)
    pays = [bytes([k] * 4) + b"\x01\x02" for k in (0x11, 0x5a, 0xe7)]
    for g in (0, 0.25, 1, 3):
        out.append(Case(f"three_frames_gap_{g:g}_sf7", c, lambda c=c, g=g: assemble(
            [gap(c, 2.7)] + [p for pay in pays for p in (sig(frame(pay, c)), gap(c, g))] + [gap(c, 4)], snr_db=32.0, seed=7500 + int(4 * g)),
            reaches(DECODE_PAYLOAD)))
    c9 = cfg(9, cr=1)
    out.append(Case("three_frames_gap_1_sf9", c9, lambda c=c9: assemble(
        [gap(c, 2.7)] + [p for pay in pays for p in (sig(frame(pay, c)), gap(c, 1))] + [gap(c, 4)], snr_db=32.0, seed=7510), reaches(DECODE_PAYLOAD)))
    sps = sps_of(c)
    for name, extra in (("at_last_symbol", 0), ("one_sample_short", -1), ("two_symbols_less_one_after", 2 * sps - 1)):
        def build(c=c, extra=extra):
            x = assemble([gap(c, 3.0), sig(frame(pays[0], c)), gap(c, 3)], snr_db=32.0, seed=7520)
            return x[:3 * sps_of(c) + frame(pays[0], c).size + extra]
        out.append(Case(f"capture_ends_{name}_sf7", c, build, reaches(DECODE_PAYLOAD)))
    return out


def _rates():
    out = []
    for fs in (500e3, 2e6):
        for sf in (8, 10, 12):
            c = cfg(sf, fs=fs)
            out.append(Case(f"fs{int(fs / 1e3)}k_sf{sf}", c, lambda c=c, fs=fs, sf=sf: assemble(
                [gap(c, 2.37), sig(frame(PAY[:2] + b"\x9a\xbc", c)), gap(c, 3)], snr_db=36.0, seed=7600 + sf + int(fs / 1e5), cfo_hz=150.0, fs=fs),
                n_frames(1), ("gradient",)))
    return out


GROUPS = {"ladder": _ladder, "lost": _lost, "damaged": _damaged, "implicit": _implicit, "back_to_back": _back_to_back, "rates": _rates}


@functools.lru_cache(maxsize=None)
def cases(group=None):
    if group is None:
        return tuple(c for g in GROUPS for c in cases(g))
    return tuple(GROUPS[group]())


# ---- runs ---------------------------------------------------------------------------------------------------------------
def oracle_run(O, c, x, demod="gradient"):
    """(steps, frames, consumed, final state, stdout) of the oracle over the capture"""
    d = O.Decoder(samp_rate=c["fs"], sf=c["sf"], implicit=c["implicit"], cr=c["cr"], crc=c["crc"], reduced_rate=c["reduced_rate"],
                  demod=O.DEMOD_FFT if demod == "fft" else O.DEMOD_GRADIENT)
    banner = d.stdout
    consumed, steps = d.run(x, max_steps=max(64, x.size // (sps_of(c) // 2)))
    return steps, d.frames(), consumed, d.state, d.stdout[len(banner):]


def published_stdout(out):
    """What of the oracle's stdout the library has delivered by the same sample: the reference prints a header's bytes as
    soon as the header block is decoded (:832) and the payload line when the frame completes (:872); the library delivers a
    frame's header bytes together with its payload line.  So a capture that ends inside a frame leaves the reference with
    a last, unterminated header print the library has not made yet."""
    return out[:out.rfind("\n") + 1]


def demods_of(case):
    """the demodulators a case runs: the FFT one exists at fs / bw = 8 only"""
    return tuple(d for d in case.demods if d == "gradient" or case.cfg["fs"] == 8 * BW)


def kernel_of(c):
    return "rx_warp_kernel" if c["sf"] == 7 and c["fs"] == 8 * BW else "rx_stream_kernel"


def gpu_decoder(c, demod="gradient", **kw):
    import gr_lora_b200 as G
    return G.decoder(c["fs"], int(BW), c["sf"], c["implicit"], c["cr"], c["crc"], c["reduced_rate"], False, quiet=True, demod=demod, **kw)


def stdout_last(dec, stream=0):
    buf = C.create_string_buffer(1 << 16)
    n = dec._L.lora_b200_stdout_last(dec._h, int(stream), buf, len(buf))
    return buf.value.decode(errors="replace") if n > 0 else ""


def near_threshold_steps(x, steps, c):
    """[(step index, which decision)] of the steps of a recorded run that are near a threshold (rx_reference)"""
    return [(i, r.near) for i, r in enumerate(R.walk(x, steps, c["sf"], c["fs"], implicit=c["implicit"])) if r.near]


# ---- the lockstep comparator ----------------------------------------------------------------------------------------------
class DecisionOpen(AssertionError):
    """assert_steps_match(allow_open=True): the device took another admissible lag than the oracle at a SYNC step whose
    lags tie within the fp32 bound; the steps up to it were compared, those after it cannot be"""


# At SF11 / SF12 and 16-20 dB the SYNC correlation's peak is flatter than the bound of a sum of 2^14 / 2^15 products: lags tens
# of samples apart tie within it under every seed tried.  No test may depend on which of them a kernel picks: the GPU test
# compares these captures with allow_open=True.
FLAT_SYNC_PEAK = {"ladder_sf11_16dB_cfo900_lead2", "ladder_sf12_16dB_cfo900_lead2", "ladder_sf12_20dB_cfo-600_lead2.13"}

WORST: dict = {}          # (kernel, statistic) -> worst err / bound seen by assert_steps_match in this process
COUNTS = {"steps": 0, "sync_ties": 0}
_STAT_NAME = {DETECT: "DETECT autocorrelation", SYNC: "SYNC correlation", FIND_SFD: "FIND_SFD Pearson"}


def assert_steps_match(trace, oracle_steps, x, sf, kernel, *, fs=1e6, implicit=False, allow_open=False):
    """Walk a device trace [(state, consumed, bin, fine_sync, metric)] and the oracle's steps of the same capture together.

    * the same number of steps; at every step the same state and bin;
    * consumed: rx_warp_kernel's is the oracle's at every step.  rx_stream_kernel may place a SYNC step one sample beside
      the oracle (two adjacent lags tie to fp32 rounding and its tree sum may pick the other); the following steps' fine
      sync must pull it back, so: the two window positions never differ by more than one sample, start to differ only at a
      SYNC step, and are equal at the end (identical totals).  (Not "only shrink afterwards": fine sync moves a window by
      whole samples from where it stands, so a device window one sample early can be left alone where the oracle's is
      moved back by two, and the two then stand one sample apart the other way -- SF11, CR 2-4 of the `short` suite.)
    * fine_sync: equal wherever consumed is equal, and otherwise differing by exactly what consumed differs by;
    * metric (DETECT, SYNC, FIND_SFD): within the derived bound of the float64 statistic at the DEVICE's own window, NaN
      where that is 0 / 0; at SYNC the reported lag must lie within the fp32 band of the float64 maximum; where both windows
      coincide, also within twice the bound of the oracle's metric.
    allow_open: at a SYNC step whose best lags tie within the bound (beyond the neighbouring sample), a device lag that is
    admissible but not the oracle's ends the comparison with DecisionOpen instead of failing it.
    A difference of state is reported with the step before it (whose decision it is): both metrics, the float64 value, its
    bound and whether that step is near a threshold.  Returns {statistic: worst err / bound}; WORST accumulates them."""
    n = min(len(trace), len(oracle_steps))
    pos_d = pos_o = 0
    thr = None
    sps = R.tables(sf, fs)[0]
    worst = {}
    prev = None
    for i in range(n):
        st_d, c_d, bin_d, fine_d, m_d = trace[i]
        o = oracle_steps[i]
        st_o, c_o, bin_o, fine_o, m_o = int(o["state"]), int(o["consumed"]), int(o["bin"]), int(o["fine_sync"]), float(o["metric"])
        what = f"{kernel} step {i} (state {st_d}, device sample {pos_d}, oracle sample {pos_o})"
        if st_d != st_o:
            raise AssertionError(f"{what}: device state {st_d}, oracle state {st_o}; decided by step {i - 1}: {prev}")
        ref = R.step_reference(x, pos_d, st_d, sf, fs, implicit=implicit, threshold=thr)
        if st_d == DETECT:
            _, _, eb, _, deb = R.detect64(x[pos_d:pos_d + 2 * sps], sps)
            thr = (eb / 2.0, deb / 2.0)
        q = R.check_metric(ref, m_d, c_d, what=what)
        if st_d in _STAT_NAME:
            worst[_STAT_NAME[st_d]] = max(worst.get(_STAT_NAME[st_d], 0.0), q)
            if pos_d == pos_o and not (math.isnan(m_d) and math.isnan(m_o)):
                b = ref.stat.bound if ref.stat else float(ref.sync.bound[min(max(c_d, 0), sps - 1)] + ref.sync.bound[min(max(c_o, 0), sps - 1)]) / 2
                same_lag = st_d != SYNC or c_d == c_o
                assert not same_lag or abs(m_d - m_o) <= 2 * b, f"{what}: metric {m_d!r}, oracle's {m_o!r}, more than 2 x {b:.3g} apart"
        v64 = ref.stat.value if ref.stat else (ref.sync.value if ref.sync else None)
        prev = (f"state {st_d}, device metric {m_d!r}, oracle metric {m_o!r}, float64 {v64!r}, "
                f"bound {ref.stat.bound if ref.stat else (float(ref.sync.bound[ref.sync.best]) if ref.sync else None)!r}, "
                f"near a threshold: {ref.near or 'no'}")
        assert bin_d == bin_o, f"{what}: bin {bin_d}, oracle {bin_o}"
        off_before = pos_d - pos_o
        if allow_open and st_d == SYNC and abs(c_d - c_o) > 1 and ref.near == "SYNC tie":
            raise DecisionOpen(f"{what}: lag {c_d}, oracle {c_o}, both within the fp32 band of the float64 maximum")
        if c_d != c_o:
            assert kernel != "rx_warp_kernel", f"{what}: consumed {c_d}, oracle {c_o} (rx_warp_kernel's must be the oracle's)"
            off_after = off_before + c_d - c_o
            if st_d == SYNC:
                assert off_before == 0 and abs(off_after) == 1, f"{what}: SYNC lag {c_d}, oracle {c_o}"
                COUNTS["sync_ties"] += 1
            else:
                assert off_before != 0, f"{what}: consumed {c_d}, oracle {c_o} from the same window"
                assert fine_d - fine_o == c_d - c_o, f"{what}: fine_sync {fine_d} / {fine_o} does not explain consumed {c_d} / {c_o}"
        else:
            assert fine_d == fine_o, f"{what}: fine_sync {fine_d}, oracle {fine_o}"
        pos_d += max(c_d, 0)
        pos_o += max(c_o, 0)
        assert abs(pos_d - pos_o) <= 1, f"{what}: windows {pos_d - pos_o} samples apart"
    assert len(trace) == len(oracle_steps), f"{kernel}: {len(trace)} steps, oracle {len(oracle_steps)}; last common step: {prev}"
    assert pos_d == pos_o, f"{kernel}: total consumed {pos_d}, oracle {pos_o}"
    COUNTS["steps"] += n
    for k, v in worst.items():
        WORST[(kernel, k)] = max(WORST.get((kernel, k), 0.0), v)
    return worst


# ---- many streams, fed in chunks ---------------------------------------------------------------------------------------
def run_batch_chunked(dec, rows, chunk_items, *, device=None, rng=None):
    """Feed rows [n_streams][n] to dec.work_batch the way a scheduler does, every stream at its own pace: each call presents
    the window [offset[s], offset[s] + items) of every stream, and every offset advances by that stream's own consumed.
    The rows are equally long (pad shorter captures: the padding is part of the row, in the one-shot run too).
    chunk_items: an int, or (lo, hi) for a size drawn per call from rng; items is that, cut to what is left of the
    shortest row still running so that no window reads past its row.  device: a torch device, to present device memory
    instead of host memory.

    work_batch takes one n_items for all streams, so a stream that has finished its row (fewer than 2 sps items left: the
    one-shot run stops there too) still has to be handed something while the others go on: it gets zeros, and whatever it
    does with them is dropped -- its consumed, trace, frames, stdout and state are recorded only from the calls in which
    its row was still running.  Returns a dict of per-stream lists: consumed, trace, frames, stdout, state."""
    rows = np.ascontiguousarray(rows, np.complex64)
    ns, n = rows.shape
    need = 2 * dec.sps
    off = np.zeros(ns, np.int64)
    out = dict(trace=[[] for _ in range(ns)], frames=[[] for _ in range(ns)], stdout=[""] * ns, state=[DETECT] * ns)
    while True:
        live = n - off >= need
        if not live.any():
            break
        chunk = int(chunk_items if np.isscalar(chunk_items) else rng.integers(chunk_items[0], chunk_items[1] + 1))
        items = max(need, int(min(chunk, (n - off)[live].min())))
        win = np.zeros((ns, items), np.complex64)
        for s in np.flatnonzero(live):
            win[s] = rows[s, off[s]:off[s] + items]
        n_before = len(dec.frames)
        if device is not None:
            import torch
            consumed = dec.work_batch(torch.from_numpy(win).to(device), n_items=items, stride_items=items, host=0)
        else:
            consumed = dec.work_batch(win)
        for s, blob in dec.frames[n_before:]:
            if live[s]:
                out["frames"][s].append(blob)
        for s in np.flatnonzero(live):
            out["trace"][s] += dec.trace(int(s))
            out["stdout"][s] += stdout_last(dec, int(s))
            out["state"][s] = dec.state(int(s))
            off[s] += int(consumed[s])
        if not consumed[live].any():
            break
    out["consumed"] = [int(v) for v in off]
    return out


# ---- the shared bookkeeping over recorded steps -------------------------------------------------------------------------
# lb::RxFrameRec (rx_stream.cuh)
FRAME_REC = np.dtype([("stream", "<u4"), ("seq", "<u4"), ("n_cw", "<u4"), ("cr", "<u4"), ("payload_length", "<u4"), ("snr", "<f4"),
                      ("phdr", "u1", 3), ("n_hdr_print", "u1"), ("hdr_print", "u1", 4), ("cw", "u1", 1024)])


def emul_lib():
    from gr_lora_b200 import build as B
    L = C.CDLL(str(B.build_host_emul()))
    L.lb_emul_decode.restype = C.c_uint32
    L.lb_emul_decode.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_uint32, C.c_void_p, C.c_uint32]
    L.lb_emul_rx_replay.restype = C.c_uint32
    L.lb_emul_rx_replay.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int, C.c_uint32, C.c_int, C.c_int,
                                    C.c_void_p, C.c_void_p, C.c_uint32]
    L.lb_emul_rx_frame_rec_size.restype = C.c_uint32
    assert L.lb_emul_rx_frame_rec_size() == FRAME_REC.itemsize
    return L


def assert_bookkeeping_replays(emul, c, steps, frames, final, stdout):
    """The stream kernels' scalar bookkeeping (rx_detect_commit .. rx_frame_record, rx_stream.cuh) run on the host over the
    oracle's steps (state, metric, bin): every next state, every frame's header and payload bytes (decoded as K8 does) and
    the printed lines must be the oracle's.  The SNR byte is not compared: the steps carry no energies."""
    states = np.ascontiguousarray(steps["state"])
    metrics = np.ascontiguousarray(steps["metric"])
    bins = np.ascontiguousarray(steps["bin"])
    nxt = np.empty(states.size, np.int32)
    recs = np.zeros(max(len(frames), 1) + 2, FRAME_REC)
    k = emul.lb_emul_rx_replay(states.ctypes.data, metrics.ctypes.data, bins.ctypes.data, states.size, c["sf"], int(c["implicit"]), c["cr"],
                               int(c["crc"]), int(c["reduced_rate"]), nxt.ctypes.data, recs.ctypes.data, len(recs))
    after = np.append(states[1:], final)
    replayed = nxt >= 0
    bad = np.flatnonzero(replayed & (nxt != after))
    assert bad.size == 0, f"step {bad[0]} (state {states[bad[0]]}, metric {metrics[bad[0]]!r}, bin {bins[bad[0]]}): next {nxt[bad[0]]}, oracle {after[bad[0]]}"
    assert k == len(frames), f"{k} frames replayed, oracle {len(frames)}"
    text = ""
    for r, f in zip(recs[:k], frames):
        cw = np.ascontiguousarray(r["cw"][:r["n_cw"]])
        dec = np.zeros(1024, np.uint8)
        m = emul.lb_emul_decode(cw.ctypes.data, int(r["n_cw"]), 0, int(r["cr"]), dec.ctypes.data, dec.size)
        plen = int(r["payload_length"])
        payload = bytes(dec[:min(m, plen)]) + bytes(max(0, plen - m))      # missing bytes read 0 (oracle D5)
        assert bytes(r["phdr"]) + payload == f[15:]
        hx = lambda v: "".join(f" {int(b):02x}" for b in v)
        text += hx(r["hdr_print"][:r["n_hdr_print"]]) + hx(payload) + " (" + "".join(chr(b) for b in payload if 32 <= b <= 126) + ")\n"
    assert published_stdout(stdout) == text
