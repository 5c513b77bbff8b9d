"""A float64 get_shift_fft and the criterion every K1 kernel is held to (no torch; imported by CPU and GPU tests).

For a symbol x of sps = 8N samples the reference dechirps in float64 with the decoder's fp32 down-chirp (y = x·c), takes
F = fft(y) in complex128, keeps tmp[0:N/2] = F[0:N/2] and tmp[N/2:N] = F[sps-N/2:sps], adds F[N/2] to tmp[N/2] (the
reference's quirk, lib/decoder_impl.cc:447-450) and returns m64 = |tmp|.  A kernel reports (bin b, magnitude mag); with

    tau = u · log2(sps) · (m64[b] + ||y||_2),   u = 2^-24

it must satisfy
    (A) m64[b] >= max(m64) - 2 tau   (so b is THE argmax whenever only one bin lies inside that band), and
    (M) |mag - m64[b]| <= tau.
tau bounds the rounding error of an fp32 FFT of log2(sps) butterfly levels applied to a vector of norm ||y||; on a clean
peak it is about 6e-7 of the peak.  Where two bins lie within 2 tau of each other (near ties) either may be reported.
"""
from __future__ import annotations

import math

import numpy as np

U_FP32 = 2.0 ** -24
CHUNK_BYTES = 64 << 20          # complex128 working set per chunk: a few hundred MB of host memory at most, even at SF12


def symbols_per_pass(sf: int, n_sms: int) -> int:
    """Symbols one grid pass of the DEFAULT K1 kernel of `sf` holds on a device with `n_sms` SMs (the launchers in
    k1_packed.cu, lora_b200.cu and k1_rows.cu): SF7 12 warps, SF8 6 groups, SF9 3 groups per CTA; SF10 and SF11 one
    symbol per CTA; SF12 one symbol per cluster of two CTAs.  One CTA (cluster) per SM."""
    return {7: 12 * n_sms, 8: 6 * n_sms, 9: 3 * n_sms, 10: n_sms, 11: n_sms, 12: n_sms // 2}[sf]


_CHIRPS: dict[int, np.ndarray] = {}


def downchirp(sf: int) -> np.ndarray:
    """The decoder's fp32 down-chirp (the oracle's table; tests/test_abi.py pins it bit-identical to the library's)."""
    if sf not in _CHIRPS:
        from oracle import oracle as O
        _CHIRPS[sf] = O.Decoder(sf=sf).downchirp
    return _CHIRPS[sf]


class K1Reference:
    """m64 [n, N] (float64 |tmp| of every kept bin) and ynorm [n] (||y||_2) of a batch of symbols."""

    def __init__(self, x: np.ndarray, sf: int, chirp: np.ndarray | None = None, *, quirk: bool = True):
        n_bins, sps = 1 << sf, 8 << sf
        x = np.asarray(x).reshape(-1, sps)
        c = (downchirp(sf) if chirp is None else chirp).astype(np.complex128)
        n = x.shape[0]
        self.sf, self.sps, self.n_bins = sf, sps, n_bins
        self.m64 = np.empty((n, n_bins), np.float64)
        self.ynorm = np.empty(n, np.float64)
        step = max(1, CHUNK_BYTES // (16 * sps))
        h = n_bins // 2
        for s in range(0, n, step):
            e = min(n, s + step)
            y = x[s:e].astype(np.complex128) * c
            self.ynorm[s:e] = np.sqrt(np.sum(y.real ** 2 + y.imag ** 2, axis=1))
            f = np.fft.fft(y, axis=1)
            tmp = np.concatenate([f[:, :h], f[:, sps - h:]], axis=1)
            if quirk:
                tmp[:, h] += f[:, h]
            self.m64[s:e] = np.abs(tmp)

    def __getitem__(self, sl: slice) -> "K1Reference":
        """The reference of a contiguous sub-batch (views, no copy)."""
        r = object.__new__(K1Reference)
        r.sf, r.sps, r.n_bins = self.sf, self.sps, self.n_bins
        r.m64, r.ynorm = self.m64[sl], self.ynorm[sl]
        return r

    def __len__(self) -> int:
        return self.m64.shape[0]

    def tau(self, mb: np.ndarray) -> np.ndarray:
        return U_FP32 * math.log2(self.sps) * (mb + self.ynorm)


def check_k1(bins, mags, x, sf: int, *, ref: K1Reference | None = None, what: str = "K1"):
    """Apply (A) to every symbol's bin and, unless `mags` is None, (M) to its magnitude.  `x` is the batch of IQ the
    kernel saw (or None when `ref` is given).  Returns (worst |mag - m64[b]| / tau, number of symbols whose (A) band held
    more than one bin).  Raises AssertionError naming the first offending symbols."""
    if ref is None:
        ref = K1Reference(x, sf)
    bins = np.asarray(bins).astype(np.int64).ravel()
    n = bins.size
    assert len(ref) == n, f"{what}: {n} bins for {len(ref)} symbols"
    if n == 0:
        return 0.0, 0
    m64 = ref.m64
    in_range = (bins >= 0) & (bins < ref.n_bins)
    b = np.where(in_range, bins, 0)
    rows = np.arange(n)
    mb = m64[rows, b]
    mx = m64.max(axis=1)
    tau = ref.tau(mb)
    band = np.sum(m64 >= (mx - 2.0 * tau)[:, None], axis=1)
    bad = ~in_range | ~(mb >= mx - 2.0 * tau)
    ratio = np.zeros(n)
    if mags is not None:
        mags = np.asarray(mags, np.float32).astype(np.float64).ravel()
        assert mags.size == n, f"{what}: {mags.size} magnitudes for {n} symbols"
        err = np.abs(mags - mb)
        bad |= ~(err <= tau)
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(tau > 0, err / np.where(tau > 0, tau, 1.0), np.where(err == 0, 0.0, np.inf))
    if bad.any():
        idx = np.flatnonzero(bad)
        lines = []
        for i in idx[:8]:
            lines.append(f"  symbol {i}: bin {bins[i]} (m64 {mb[i]:.9g}), argmax {int(np.argmax(m64[i]))} (m64 {mx[i]:.9g}), "
                         f"tau {tau[i]:.3g}" + (f", mag {mags[i]:.9g} (err/tau {ratio[i]:.3g})" if mags is not None else ""))
        raise AssertionError(f"{what}: {idx.size} of {n} symbols outside the float64 rounding band\n" + "\n".join(lines))
    return float(ratio.max()), int(np.sum(band > 1))
