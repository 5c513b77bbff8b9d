"""Float64 restatements of the dechirp receiver's window sums, of the several-antenna receiver's channel estimates, weights
and combined SNR, and of its assembled data windows -- from the documented rules (include/lora_b200.h, DESIGN section 5
"Several antennas"), not from rs_channels -- each with the error bound of the device's float32 arithmetic:

  window sums  X = sum_n x[pos + n] c[n] exp(-2 pi j (F (pos + n) + b n) / sps) within (2.5e-7 + 2 pi (|F| + 1) 2^-25)
               sum |x c| (float32 phases reduced from a float64 base, sincospif, block sums); energy within 1e-5
  channels     windows i = 1..6 at start + llround(i sps / (1 + 1e-6 ppm)), those outside the row skipped;
               h_a = mean_i X_a,i / ((1 + j) sps); px_a = sum_i |X_a,i|^2 / (2 nw sps), e_a = the mean window energy;
               s2_a = max((e_a - px_a) / (sps - 1), 1e-6 max_b e_b / sps, 1e-30); S_a = max((px_a - s2_a) / sps, 1e-30);
               w_a = conj(h_a) s2min / s2_a scaled to sum |w|^2 = 1; snr_db = 10 log10(decim sum_a S_a / s2_a).
               The window-sum and energy bounds are carried through each formula as intervals (max and the ratios are
               monotone).  At high SNR e - px cancels, so the interval on s2 -- and on w and snr_db -- widens there.
  assembly     y_k[n] = sum_a w_a x_a[ws_k + n] exp(-2 pi j F (ws_k + n) / sps), ws_k = start + llround((12.25 + first + k)
               sps / (1 + 1e-6 ppm)), 0 past n_items, within c 2^-24 sum_a |w_a| |x_a[ws_k + n]|."""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24                                        # float32 unit roundoff


# ---- window sums ----------------------------------------------------------------------------------------------------------
def window_sum(w, c, pos, cfo, b):
    """Bin b of the window w (complex, sps samples from row position pos) dechirped with the table c and de-rotated by cfo
    bins, in float64, and the bound of the device's float32 sum: 2.5e-7 (products and block sums) plus the float32 rounding
    of the phase of a CFO of F bins, 2 pi (|F| + 1) 2^-25, times sum |w c|."""
    sps = w.shape[-1]
    k = np.arange(sps)
    y = np.asarray(w, np.complex128) * np.asarray(c, np.complex128)
    ph = (float(cfo) * (int(pos) + k) + float(b) * k) / sps         # exact: F a float32, pos + k < 2^27, sps a power of 2
    ph -= np.floor(ph)
    X = np.sum(y * np.exp(-2j * np.pi * ph))
    return X, (2.5e-7 + 2 * np.pi * (abs(float(cfo)) + 1) * 2.0 ** -25) * np.sum(np.abs(y))


ENERGY_TOL = 1e-5                                     # relative, of sum |x|^2 over a window


def window_energy(w):
    return float(np.sum(np.abs(np.asarray(w, np.complex128)) ** 2))


# ---- window placement ------------------------------------------------------------------------------------------------------
def rs_sym(start, j, sps, ppm):
    """TX symbol position j of a frame at start with a clock offset of ppm (a float32): start + llround(j sps / (1 + 1e-6
    ppm)), start + j sps at ppm = 0."""
    u = j * sps
    if float(ppm) == 0.0:
        return int(start) + int(u)
    v = u / (1.0 + 1e-6 * float(np.float32(ppm)))
    return int(start) + int(math.floor(v + 0.5))      # (llround of a positive value)


def _lo(v):
    return v - 4 * U * abs(v)


def _hi(v):
    return v + 4 * U * abs(v)


# ---- channel estimates, weights, combined SNR -----------------------------------------------------------------------------
class ChannelReference:
    """The channel estimates, noise powers, weights and combined SNR of one frame at (start, cfo_bins, sfo_ppm) on the rows X
    [m, >= n_items] (antennas 0..m-1), with the down-chirp table `down` at fs/bw = decim.  `windows` and `conj` exist to
    show that the checks reject a wrong rule (windows 0..5, weights without the conjugate); `normalise = False` drops the
    noise normalisation of the weights."""

    def __init__(self, X, n_items, start, cfo_bins, sfo_ppm, down, decim, windows=range(1, 7), conj=True, normalise=True):
        m = X.shape[0]
        sps = down.size
        self.m, self.sps, self.decim = m, sps, decim
        F = float(np.float32(cfo_bins))
        Xs, ts, Es = [], [], []
        for i in windows:
            pos = rs_sym(start, i, sps, sfo_ppm)
            if pos < 0 or pos + sps > n_items:
                continue
            row = [window_sum(X[a, pos: pos + sps], down, pos, F, 0) for a in range(m)]
            Xs.append([r[0] for r in row])
            ts.append([r[1] for r in row])
            Es.append([window_energy(X[a, pos: pos + sps]) for a in range(m)])
        self.nw = nw = len(Xs)
        assert nw > 0, "no preamble window inside the row"
        Xs, ts, Es = np.array(Xs), np.array(ts), np.array(Es)          # [nw, m]
        aX = np.abs(Xs)
        # h: the mean peak over (1 + j) sps
        self.h = Xs.mean(axis=0) * (1 - 1j) / (2 * sps)
        self.rh = (ts.sum(axis=0) + 8 * U * aX.sum(axis=0)) / (nw * math.sqrt(2) * sps)
        # px, e and their intervals
        pk, pk_lo, pk_hi = (aX ** 2).sum(0), (np.maximum(aX - ts, 0) ** 2).sum(0), ((aX + ts) ** 2).sum(0)
        en, en_lo, en_hi = Es.sum(0), (Es * (1 - ENERGY_TOL)).sum(0), (Es * (1 + ENERGY_TOL)).sum(0)
        px, px_lo, px_hi = (v / (2 * nw * sps) for v in (pk, pk_lo * (1 - 8 * U), pk_hi * (1 + 8 * U)))
        e, e_lo, e_hi = (v / nw for v in (en, en_lo * (1 - 8 * U), en_hi * (1 + 8 * U)))
        emax, emax_lo, emax_hi = (np.max(v) / sps for v in (e, e_lo, e_hi))

        def s2_of(ev, pv, em, side):
            return np.array([max(side((ev[a] - pv[a]) / (sps - 1)), side(1e-6 * em), 1e-30) for a in range(m)])

        self.s2 = s2_of(e, px, emax, lambda v: v)
        self.s2_lo = s2_of(e_lo, px_hi, emax_lo, _lo)
        self.s2_hi = s2_of(e_hi, px_lo, emax_hi, _hi)
        S = np.maximum((px - self.s2) / sps, 1e-30)
        S_lo = np.maximum([_lo(v) for v in (px_lo - self.s2_hi) / sps], 1e-30)
        S_hi = np.maximum([_hi(v) for v in (px_hi - self.s2_lo) / sps], 1e-30)
        self.snr_db = 10 * math.log10(decim * np.sum(S / self.s2))
        self.snr_lo = 10 * math.log10(decim * np.sum(S_lo / self.s2_hi)) - 1e-4
        self.snr_hi = 10 * math.log10(decim * np.sum(S_hi / self.s2_lo)) + 1e-4
        # weights
        g = np.conj(self.h) if conj else self.h
        w = g * (self.s2.min() / self.s2 if normalise else 1.0)
        self.w = w / math.sqrt(np.sum(np.abs(w) ** 2))
        self.conj, self.normalise = conj, normalise

    def check_h(self, h, what=""):
        """|h_dev - h| within the carried bound, per antenna.  Returns the worst err/bound."""
        err = np.abs(np.asarray(h, np.complex128)[: self.m] - self.h)
        assert np.all(err <= self.rh), f"{what}: h {np.asarray(h)[: self.m]} against {self.h} +- {self.rh}"
        return float(np.max(err / self.rh))

    def check_snr(self, snr_db, what=""):
        """snr_db within [snr_lo, snr_hi].  Returns |snr_db - the interval's centre| over its half-width (1: at an end)."""
        assert self.snr_lo <= snr_db <= self.snr_hi, f"{what}: snr_db {snr_db} outside [{self.snr_lo}, {self.snr_hi}]"
        half = max((self.snr_hi - self.snr_lo) / 2, 1e-12)
        return float(abs(snr_db - (self.snr_lo + self.snr_hi) / 2) / half)

    def check_w(self, w, what=""):
        """sum |w|^2 = 1 to a few ulp, and every ratio w_a / w_r (r: the antenna of the largest reference weight) within its
        interval: |w_a / w_r| = |h_a| / |h_r| s2_r / s2_a with each factor's interval, the phase arg(conj(h_a) / conj(h_r))
        within the angles the bounds on h_a and h_r allow.  Returns the worst err/bound of the ratios (magnitude, phase)."""
        w = np.asarray(w, np.complex128)[: self.m]
        assert abs(np.sum(np.abs(w) ** 2) - 1) <= 8 * self.m * U, f"{what}: sum |w|^2 = {np.sum(np.abs(w) ** 2)!r}"
        r = int(np.argmax(np.abs(self.w)))
        ah = np.abs(self.h)
        worst_m = worst_p = 0.0
        for a in range(self.m):
            if a == r:
                continue
            lo = max(ah[a] - self.rh[a], 0) / (ah[r] + self.rh[r]) * self.s2_lo[r] / self.s2_hi[a] * (1 - 16 * U)
            hi = ((ah[a] + self.rh[a]) / max(ah[r] - self.rh[r], 1e-300) * self.s2_hi[r] / self.s2_lo[a] * (1 + 16 * U))
            got = abs(w[a]) / abs(w[r])
            want = ah[a] / ah[r] * self.s2[r] / self.s2[a]
            assert lo <= got <= hi, f"{what}: |w_{a} / w_{r}| = {got} outside [{lo}, {hi}] (float64 {want})"
            worst_m = max(worst_m, abs(got - want) / max(hi - want if got > want else want - lo, 1e-300))
            phi = sum(math.asin(min(1.0, self.rh[b] / ah[b])) if ah[b] > 0 else math.pi for b in (a, r)) + 16 * U
            ref = np.conj(self.h[a]) / np.conj(self.h[r])
            d = abs(np.angle(w[a] / w[r] / ref))
            assert d <= phi, f"{what}: arg(w_{a} / w_{r}) is {d:.3e} rad from arg(conj(h_{a}) / conj(h_{r})), bound {phi:.3e}"
            worst_p = max(worst_p, d / phi)
        return worst_m, worst_p


# ---- assembled data windows -------------------------------------------------------------------------------------------------
def assembly_c(m):
    """The constant of the assembly bound c 2^-24 sum_a |w_a| |x_a|: the float32 phase after the double reduction, within
    2^-25 revolutions (pi 2^-24 rad); sincospif within 1 ulp per component (< 2 2^-24 on the unit phasor); the complex FMA
    chain over m antennas, two roundings per component per step (3 2^-24 each in modulus); the final complex product, 3 more."""
    return math.pi + 2 + 3 * (m + 1)


def assembly_windows(X, n_items, sps, start, cfo_bins, sfo_ppm, first, cnt, w, phase32=False, base=0):
    """The data windows first .. first + cnt - 1 of a frame on the rows X [m, n_items - base] (row samples base ..
    n_items - 1) combined with the weights w (complex64; [1] for m = 1), in float64: y [cnt, sps] and the bound of each
    sample [cnt, sps].  phase32: the de-rotation phase F n / sps formed and reduced in float32 -- a wrong rule, to show
    that the bound rejects it."""
    m = X.shape[0]
    wv = np.asarray(w, np.complex64).astype(np.complex128)[:m]
    F = float(np.float32(cfo_bins))
    y = np.zeros((cnt, sps), np.complex128)
    bound = np.zeros((cnt, sps))
    for k in range(cnt):
        ws = rs_sym(start, 12.25 + first + k, sps, sfo_ppm)
        n = ws + np.arange(sps)
        ok = n < n_items
        nn = n[ok]
        xs = X[:, nn - base].astype(np.complex128)
        if phase32:
            t = (np.float32(F) / np.float32(sps)) * nn.astype(np.float32)
            t = (t - np.floor(t)).astype(np.float64)
        else:
            t = F * nn.astype(np.float64) / sps
            t -= np.floor(t)
        y[k, ok] = np.sum(wv[:, None] * xs, axis=0) * np.exp(-2j * np.pi * t)
        bound[k, ok] = assembly_c(m) * U * np.sum(np.abs(wv)[:, None] * np.abs(xs), axis=0)
    return y, bound
