"""Float64 statements of the statistics the stream state machines decide on, each with a derived fp32 bound (no torch;
imported by CPU and GPU tests).

Both stream kernels (rx_warp_kernel, rx_stream_kernel) and the oracle compute, from the window x[pos : pos + 2 sps] and the
decoder's own fp32 tables, in fp32 and each in its own summation order:

    DETECT    r = |sum a conj(b)| / sqrt(sum |a|^2 sum |b|^2), a = x[0:sps], b = x[sps:2 sps]      (decoder_impl.cc:340-366)
    FIND_SFD  c = Pearson correlation of ifreq(x[0:sps])[0:sps-1] with down_ifreq[0:sps-1]           (:283-298, :385-390)
    SYNC      c[lag] = sum_k ifreq(x[0:2 sps])[lag + k] up_ifreq[k], k < sps - 1, lag < sps; its maximum (:399-413)
    energy    e = sum |x[0:sps]|^2 against energy_threshold = (sum |b|^2 of the last DETECT window) / 2  (:861, :357)

Here they are evaluated in float64 (arg() by numpy's arctan2 on the fp32 samples, the reference's unwrap rule), together with
a bound on what an fp32 evaluation in ANY summation order may differ from the float64 value by.

The bound.  u = 2^-24.  An fp32 sum of n terms t_i, however it is ordered (running sum, lane-strided partial sums, a tree,
fused multiply-adds or not), makes at most n - 1 roundings, each at most u times a partial sum, and no partial sum exceeds
T = sum |t_i|.  Modelling the roundings as independent and zero-mean, Hoeffding's inequality bounds the accumulated error by
LAM sqrt(n) u T except with probability 2 exp(-LAM^2 / 2): 3e-8 per sum at LAM = 6, the value used.  (The worst-case bound
n u T is 7 to 40 times larger for n = 2^11 .. 2^16 and would let an error of 1e-4 pass at every SF.)  The `local` roundings
made on a term before it is added (the product, a subtraction) add local u T, worst case.  Hence

    sum_bound(T, n, local) = (LAM sqrt(n) + local) u T.

arg(): the kernels' lb_atan2f is within 1.8 ulp, libm's atan2f within 1 ulp; |arg| <= pi and ulp(pi) = 2^-22, so a phase is
off by at most EPS_PHI = 1.8 * 2^-22.  One value of the instantaneous frequency is a difference of two phases, unwrapped
(one rounding of a value below 2 pi when the correction is cast back to float) and subtracted (one rounding of a value of
at most pi): besides the two phase errors it carries EPS_SUB = (2 pi + pi) u of its own.  A statistic that is linear in
the instantaneous frequency with weights w, sum_i w_i f_i = sum_j phase_j (w_{j-1} - w_j), sees the phase errors
TELESCOPED: smooth weights (the ideal chirps' ramps) cancel them, and

    ifreq_bound(w) = EPS_PHI (|w_0| + sum_j |w_j - w_{j-1}| + |w_last|) + LAM EPS_SUB ||w||_2        (+ the unwraps, below)

(the phase errors worst case, the independent roundings of the subtractions by Hoeffding as above).  Where the float64
difference lies within EPS_F = 2 EPS_PHI + EPS_SUB of +-pi the fp32 evaluation may unwrap the other way: such a value may
differ by 2 pi, and the bounds carry 2 pi |w_i| for each of them.

The statistics' bounds follow by first-order propagation of those two sources; every formula is next to its code.
A step is NEAR A THRESHOLD when its float64 statistic lies within its bound of the constant it is compared with (0.90,
0.96, -0.97, the energy threshold) or, at SYNC, when the runner-up lag lies within the two lags' bounds of the best one:
there an fp32 evaluation may decide either way and no test may depend on the decision.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

U = 2.0 ** -24
LAM = 6.0
EPS_PHI = 1.8 * 2.0 ** -22
EPS_SUB = 3 * math.pi * U
EPS_F = 2 * EPS_PHI + EPS_SUB
DETECT_GATE, SFD_GATE, UP_AGAIN_GATE = 0.90, 0.96, -0.97

DETECT, SYNC, FIND_SFD, PAUSE, DECODE_HEADER, DECODE_PAYLOAD, STOP = range(7)


def sum_bound(T, n, local=1.0):
    """fp32 rounding of a sum of n terms with sum |t_i| = T in any order, `local` roundings per term before the add."""
    return (LAM * math.sqrt(n) + local) * U * T


_TABLES: dict = {}


def tables(sf: int, fs: float = 1e6):
    """(sps, down_ifreq, up_ifreq) of the decoder: the oracle's fp32 tables (tests/test_abi.py pins the library's to them
    bit for bit), as float64."""
    key = (sf, float(fs))
    if key not in _TABLES:
        from oracle import oracle as O
        d = O.Decoder(samp_rate=fs, sf=sf)
        _TABLES[key] = (d.sps, d.downchirp_ifreq.astype(np.float64), d.upchirp_ifreq.astype(np.float64))
    return _TABLES[key]


def ifreq64(x):
    """instantaneous_frequency (:224-244) of the fp32 samples x in float64: out[i] = unwrap(arg x[i+1] - arg x[i]), the last
    value repeats the one before it.  Also returns, per value, whether an fp32 evaluation may unwrap it the other way."""
    x = np.asarray(x, np.complex64)
    ph = np.arctan2(x.imag.astype(np.float64), x.real.astype(np.float64))
    d = np.diff(ph)
    d = np.where(d > math.pi, d - 2 * math.pi, d)
    d = np.where(d < -math.pi, d + 2 * math.pi, d)
    amb = math.pi - np.abs(d) <= EPS_F
    return np.append(d, d[-1]), np.append(amb, amb[-1])


def ifreq_bound(w, amb):
    """what sum_i w_i f_i may differ by between an fp32 instantaneous frequency and ifreq64 (module docstring)"""
    w = np.asarray(w, np.float64)
    tv = abs(w[0]) + float(np.sum(np.abs(np.diff(w)))) + abs(w[-1])
    return EPS_PHI * tv + LAM * EPS_SUB * float(np.sqrt(np.sum(w * w))) + 2 * math.pi * float(np.sum(np.abs(w)[amb]))


@dataclass
class Stat:
    value: float            # the float64 statistic (nan where the reference computes 0 / 0)
    bound: float            # what an fp32 evaluation may differ by

    def near(self, *gates) -> bool:
        return any(abs(self.value - g) <= self.bound for g in gates)


def detect64(w, sps):
    """DETECT on w = x[pos : pos + 2 sps]: (Stat of the autocorrelation, e_a, e_b, bound of e_a, bound of e_b).
    r = |D| / s with D = sum a conj(b), s = sqrt(e_a e_b):
      |dr| <= |dD| / s + r (de_a / (2 e_a) + de_b / (2 e_b)) + 6 u r
    (the last term: sqrt, two divisions, hypot), dRe D, dIm D, de from sum_bound over the 2 sps real products of each."""
    w = np.asarray(w, np.complex64).astype(np.complex128)
    a, b = w[:sps], w[sps:2 * sps]
    D = np.sum(a * np.conj(b))
    ea, eb = float(np.sum(a.real ** 2 + a.imag ** 2)), float(np.sum(b.real ** 2 + b.imag ** 2))
    n = 2 * sps
    dea, deb = sum_bound(ea, n), sum_bound(eb, n)
    if ea == 0.0 or eb == 0.0:
        return Stat(math.nan, 0.0), ea, eb, dea, deb
    s = math.sqrt(ea * eb)
    t_re = float(np.sum(np.abs(a.real * b.real) + np.abs(a.imag * b.imag)))
    t_im = float(np.sum(np.abs(a.imag * b.real) + np.abs(a.real * b.imag)))
    r = abs(D) / s
    bound = math.hypot(sum_bound(t_re, n), sum_bound(t_im, n)) / s + r * (dea / (2 * ea) + deb / (2 * eb)) + 6 * U * r
    return Stat(float(r), float(bound)), ea, eb, dea, deb


def sfd64(w, sps, down_ifreq, *, center=True, entries=None):
    """FIND_SFD on w = x[pos : pos + sps]: Stat of c = sum (f_i - fm)(g_i - gm) / (n sd_f sd_g), n = sps - 1, f = ifreq64(w),
    g = down_ifreq.  With F = (f - fm) / sd_f and G = (g - gm) / sd_g, dc/df_i = (G_i - c F_i) / (n sd_f), so
      |dc| <= ifreq_bound((G - c F) / (n sd_f))                                (arg() and unwrap)
            + sum_bound(sum |F_i G_i|, n, 4) / n                               (the sum of products; sub, sub, mul, div)
            + |c| (sum_bound(1, n, 3) / 2 + sum_bound(1, n, 3) / 2 + 4 u)      (sd_f, the table's fp32 sd_g, sqrt and divisions)
    The two means enter only through sum (g_i - gm) and sum (f_i - fm), zero to rounding: second order, not carried.
    center=False drops `- gm` -- which changes nothing: sum_i (f_i - fm) = 0, so sum (f_i - fm) g_i is the same sum; in fp32,
    where the window's mean is itself rounded, the two differ by rounding only.  entries: the number of values correlated
    instead of sps - 1 (a deliberately wrong statistic for the tests of the criterion)."""
    n = sps - 1 if entries is None else entries
    f, amb = ifreq64(np.asarray(w)[:sps])
    f, amb = f[:n], amb[:n]
    g = down_ifreq[:n]
    fm, gm = f.mean(), g.mean()
    sdf, sdg = math.sqrt(np.mean((f - fm) ** 2)), math.sqrt(np.mean((g - gm) ** 2))
    if sdf == 0.0 or not np.isfinite(sdf):
        return Stat(math.nan, 0.0)
    F, G = (f - fm) / sdf, (g - (gm if center else 0.0)) / sdg
    c = float(np.sum(F * G) / n)
    bound = (ifreq_bound((G - c * F) / (n * sdf), amb) + sum_bound(float(np.sum(np.abs(F * G))), n, 4) / n
             + abs(c) * (sum_bound(1.0, n, 3) + 4 * U))
    return Stat(c, float(bound))


def _xcorr(f, u, n_lags):
    """out[lag] = sum_k f[lag + k] u[k] for lag < n_lags, by FFT in float64 (error ~1e-16 |f| |u|: nothing next to fp32)"""
    m = 1 << int(math.ceil(math.log2(f.size + u.size)))
    return np.fft.irfft(np.fft.rfft(f, m) * np.conj(np.fft.rfft(u, m)), m)[:n_lags]


@dataclass
class Sync:
    c: np.ndarray           # float64 correlation of every lag
    bound: np.ndarray       # per lag
    best: int               # first maximal lag with c > 0 (0 with value 0 when there is none, as the reference's loop)
    runner_up: int          # the best lag other than `best`

    @property
    def value(self):
        return max(float(self.c[self.best]), 0.0)

    @property
    def gap(self):
        return float(self.c[self.best] - self.c[self.runner_up])

    def tie(self) -> bool:
        """may an fp32 evaluation pick another lag than `best`?"""
        return self.gap <= float(self.bound[self.best] + self.bound[self.runner_up])

    def admissible(self, lag) -> bool:
        return float(self.c[self.best] - self.c[lag]) <= float(self.bound[self.best] + self.bound[lag])


def sync64(w, sps, up_ifreq):
    """SYNC on w = x[pos : pos + 2 sps]: c[lag] = sum_{k < sps - 1} f[lag + k] up_ifreq[k], f = ifreq64(w).
      |dc[lag]| <= ifreq_bound(up) + sum_bound(sum_k |f[lag + k] up_k|, sps - 1, 1),
    the unwrap term of ifreq_bound per lag (2 pi |up_k| for every value of the lag's window that may unwrap the other way)"""
    f, amb = ifreq64(np.asarray(w)[:2 * sps])
    u = up_ifreq[:sps - 1]
    c = _xcorr(f, u, sps)
    bound = ifreq_bound(u, np.zeros(u.size, bool)) + sum_bound(_xcorr(np.abs(f), np.abs(u), sps), sps - 1, 1)
    if amb.any():
        bound = bound + 2 * math.pi * np.maximum(_xcorr(amb.astype(np.float64), np.abs(u), sps), 0.0)
    best = int(np.argmax(c)) if np.max(c) > 0 else 0
    masked = c.copy()
    masked[best] = -np.inf
    return Sync(c, bound, best, int(np.argmax(masked)))


def energy64(w, sps):
    """determine_energy (:368-375) of w = x[pos : pos + sps]: (e, bound)"""
    w = np.asarray(w, np.complex64)[:sps].astype(np.complex128)
    e = float(np.sum(w.real ** 2 + w.imag ** 2))
    return e, sum_bound(e, 2 * sps)


@dataclass
class StepRef:
    """The float64 view of one recorded step at window position pos."""
    state: int
    pos: int
    stat: Stat | None = None        # DETECT, FIND_SFD
    sync: Sync | None = None        # SYNC
    energy: tuple | None = None     # implicit DECODE_PAYLOAD: (e, bound, threshold, bound of the threshold)
    near: str = ""                  # which decision of this step an fp32 evaluation may take either way ("" = none)


def step_reference(x, pos, state, sf, fs=1e6, *, implicit=False, threshold=None):
    """StepRef of a step in `state` whose window starts at x[pos].  threshold = (energy_threshold, its bound) as the last
    DETECT step left it, for the implicit-header energy gate."""
    sps, down_if, up_if = tables(sf, fs)
    r = StepRef(state, pos)
    w = x[pos:pos + 2 * sps]
    if state == DETECT:
        r.stat = detect64(w, sps)[0]
        if r.stat.near(DETECT_GATE):
            r.near = "DETECT 0.90"
    elif state == FIND_SFD:
        r.stat = sfd64(w, sps, down_if)
        if r.stat.near(SFD_GATE):
            r.near = "FIND_SFD 0.96"
        elif r.stat.near(UP_AGAIN_GATE):
            r.near = "FIND_SFD -0.97"
    elif state == SYNC:
        r.sync = sync64(w, sps, up_if)
        if r.sync.tie():
            r.near = "SYNC tie"
    elif state == DECODE_PAYLOAD and implicit and threshold is not None:
        e, be = energy64(w, sps)
        r.energy = (e, be, threshold[0], threshold[1])
        if abs(e - threshold[0]) <= be + threshold[1]:
            r.near = "energy gate"
    return r


def walk(x, steps, sf, fs=1e6, *, implicit=False):
    """StepRef of every step of a recorded run (states and consumed of `steps`, a sequence of (state, consumed, ...) or the
    oracle's structured array) over the capture x, at the positions the run itself visited."""
    sps = tables(sf, fs)[0]
    out, pos, thr = [], 0, None
    for s in steps:
        state, consumed = int(s[0]), int(s[1])
        r = step_reference(x, pos, state, sf, fs, implicit=implicit, threshold=thr)
        if state == DETECT:
            _, _, eb, _, deb = detect64(x[pos:pos + 2 * sps], sps)
            thr = (eb / 2.0, deb / 2.0)
        out.append(r)
        pos += max(consumed, 0)
    return out


def check_metric(ref: StepRef, metric: float, consumed: int, *, scale=1.0, what="step"):
    """The recorded fp32 metric of a step against its float64 reference: returns err / bound (0 for steps without a
    statistic); raises AssertionError beyond `scale` bounds.  At SYNC `consumed` is the reported lag: it must be admissible
    (within the two lags' bounds of the float64 maximum) and the metric is that lag's correlation."""
    metric = float(metric)
    if ref.state in (DETECT, FIND_SFD):
        v, b = ref.stat.value, ref.stat.bound
        if math.isnan(v):
            assert math.isnan(metric), f"{what}: metric {metric!r} where the statistic is 0 / 0"
            return 0.0
    elif ref.state == SYNC:
        sy = ref.sync
        if sy.value == 0.0:                                   # no positive correlation: the loop never assigns
            assert metric == 0.0 and consumed == 0, f"{what}: SYNC without a positive correlation gave {metric!r} at {consumed}"
            return 0.0
        assert 0 <= consumed < sy.c.size and sy.admissible(consumed), (
            f"{what}: SYNC lag {consumed} (c64 {sy.c[consumed] if 0 <= consumed < sy.c.size else None!r}) is not within the fp32 "
            f"band of the float64 maximum at lag {sy.best} (c64 {sy.c[sy.best]!r}, bounds {sy.bound[sy.best]:.3g})")
        v, b = float(sy.c[consumed]), float(sy.bound[consumed])
    else:
        return 0.0
    err = abs(metric - v)
    assert err <= scale * b, (f"{what}: state {ref.state} at sample {ref.pos}: metric {metric!r}, float64 {v!r}, "
                              f"error {err:.3g} > {scale:g} x bound {b:.3g}")
    return err / b if b > 0 else 0.0
