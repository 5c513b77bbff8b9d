"""CPU: the float64 get_shift_fft of tests/k1_reference.py and its criterion.  The reference agrees with a direct DFT;
the fp32 oracle and every host emulation of the K1 kernels pass the criterion unchanged on clean, -15 dB and pure-noise
symbols at SF7-SF12; and outputs that are wrong by a little (one magnitude 1e-5 off, one noise bin moved by one, the
bin-N/2 quirk left out) fail it."""
import ctypes as C

import numpy as np
import pytest

from conftest import twiddle_table
from gr_lora_b200 import build as B, tx
from k1_reference import K1Reference, check_k1, downchirp


@pytest.fixture(scope="module")
def emul():
    L = C.CDLL(str(B.build_host_emul()))
    for f in ("lb_k1_emulate", "lb_k1_emulate_group", "lb_k1_emulate_rows"):
        getattr(L, f).argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.lb_k1_emulate_warp_sf7.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _inputs(sf, kind, n, seed):
    """clean / -15 dB symbols (edge values first) or complex Gaussian noise, complex64."""
    nb, sps = 1 << sf, 8 << sf
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return (rng.standard_normal(n * sps) + 1j * rng.standard_normal(n * sps)).astype(np.complex64)
    vals = rng.integers(0, nb, n)
    vals[:6] = [0, 1, nb // 2 - 1, nb // 2, nb // 2 + 1, nb - 1][:n]
    return tx.synth_symbols(vals, sf, snr_db=None if kind == "clean" else -15.0, seed=seed)


def test_reference_equals_direct_dft():
    """m64 against an O(sps) DFT with exactly reduced phase indices, at the bins where the decimation is easy to get
    wrong: 0, N/2 - 1, N/2 (= F[sps - N/2] + F[N/2]), N/2 + 1 (the wrap to F[sps - N/2 + 1]), N - 1 (F[sps - 1])."""
    for sf in (7, 9, 12):
        nb, sps = 1 << sf, 8 << sf
        x = _inputs(sf, "noise", 1, sf)[None, :]
        x[0] += tx.synth_symbols([nb // 2], sf)            # a peak at N/2 as well
        ref = K1Reference(x, sf)
        y = x[0].astype(np.complex128) * downchirp(sf).astype(np.complex128)
        n = np.arange(sps)

        def dft(k):
            return np.sum(y * np.exp(-2j * np.pi * ((k * n) % sps) / sps))

        for b in (0, 1, nb // 2 - 1, nb // 2, nb // 2 + 1, nb - 1):
            want = dft(b) if b < nb // 2 else dft(sps - nb + b)
            if b == nb // 2:
                want += dft(nb // 2)
            assert abs(ref.m64[0, b] - abs(want)) <= 1e-9 * np.linalg.norm(y) * np.sqrt(sps), (sf, b)
        assert int(np.argmax(ref.m64[0])) == nb // 2
        assert ref.ynorm[0] == pytest.approx(np.linalg.norm(y), rel=1e-12)


def _emulations(sf):
    out = [("generic", lambda L, *a: L.lb_k1_emulate(sf, *a))]
    if sf == 7:
        out.append(("warp7", lambda L, *a: L.lb_k1_emulate_warp_sf7(*a)))
    elif sf <= 10:
        out.append((f"group{sf}", lambda L, *a: L.lb_k1_emulate_group(sf, *a)))
    else:
        out.append((f"rows{sf}", lambda L, *a: L.lb_k1_emulate_rows(sf, *a)))
    return out


@pytest.mark.parametrize("sf", range(7, 13))
def test_oracle_and_host_emulations_within_the_band(emul, oracle, sf):
    """The fp32 oracle (worst err/tau measured 0.35) and every host emulation (0.56) stay inside the band; bins equal the
    float64 argmax wherever it is unique."""
    d = oracle.Decoder(sf=sf)
    chirp, tw = d.downchirp, twiddle_table(d.sps)
    n = {7: 48, 8: 32, 9: 24, 10: 16, 11: 10, 12: 8}[sf]
    for kind in ("clean", "m15db", "noise"):
        x = _inputs(sf, kind, n, 300 + sf)
        ref = K1Reference(x, sf)
        ob, om = d.demod_fft_batch(x)
        worst, _ = check_k1(ob, om, None, sf, ref=ref, what=f"oracle SF{sf} {kind}")
        assert worst < 0.75
        for name, fn in _emulations(sf):
            bins, mags = np.zeros(n, np.uint32), np.zeros(n, np.float32)
            rc = fn(emul, x.ctypes.data, n, chirp.ctypes.data, tw.ctypes.data, bins.ctypes.data, mags.ctypes.data)
            assert rc in (0, None)
            worst, _ = check_k1(bins, mags, None, sf, ref=ref, what=f"{name} SF{sf} {kind}")
            assert worst < 0.75, (name, kind, worst)
        if kind == "clean":
            assert np.array_equal(ob.astype(np.int64), np.argmax(ref.m64, axis=1))


@pytest.mark.parametrize("sf", [7, 11])
def test_negative_controls_fail(oracle, sf):
    nb = 1 << sf
    d = oracle.Decoder(sf=sf)
    # one magnitude of a clean symbol scaled by 1 + 1e-5: ~17 tau at a clean peak
    x = _inputs(sf, "clean", 8, 1)
    ref = K1Reference(x, sf)
    ob, om = d.demod_fft_batch(x)
    check_k1(ob, om, None, sf, ref=ref)
    bad = om.copy()
    bad[3] = np.float32(bad[3] * (1 + 1e-5))
    with pytest.raises(AssertionError, match="symbol 3"):
        check_k1(ob, bad, None, sf, ref=ref)
    # one bin of a noise symbol moved by +-1: the gap between the top two noise bins is many tau
    xn = _inputs(sf, "noise", 8, 2)
    refn = K1Reference(xn, sf)
    nbins, nm = d.demod_fft_batch(xn)
    check_k1(nbins, nm, None, sf, ref=refn)
    for delta in (1, -1):
        moved = nbins.astype(np.int64)
        moved[5] = (moved[5] + delta) % nb
        with pytest.raises(AssertionError, match="symbol 5"):
            check_k1(moved, None, None, sf, ref=refn)
    # the bin-N/2 quirk left out, on a symbol whose peak is bin N/2: the argmax and magnitude of that spectrum, and the
    # right bin with the magnitude of F[sps - N/2] alone
    xq = tx.synth_symbols([nb // 2, nb // 2 + 1, 7], sf, snr_db=10.0, seed=3)
    refq = K1Reference(xq, sf)
    noq = K1Reference(xq, sf, quirk=False)
    qb = np.argmax(noq.m64, axis=1)
    qm = noq.m64[np.arange(3), qb].astype(np.float32)
    check_k1(*d.demod_fft_batch(xq), None, sf, ref=refq)
    with pytest.raises(AssertionError, match="symbol 0"):
        check_k1(qb, qm, None, sf, ref=refq)
    with pytest.raises(AssertionError, match="symbol 0"):
        check_k1(np.array([nb // 2, nb // 2 + 1, 7]), noq.m64[:, [nb // 2, nb // 2 + 1, 7]].diagonal().astype(np.float32),
                 None, sf, ref=refq)


def test_flat_spectrum_and_silence():
    """A dechirped impulse (x[0] = 1 / c[0]) has equal magnitudes everywhere except bin N/2, which the quirk doubles;
    silence has all magnitudes 0 (any bin is inside the band there, the kernels' first-maximum rule is tested on the GPU)."""
    sf = 8
    nb, sps = 1 << sf, 8 << sf
    c = downchirp(sf)
    x = np.zeros((2, sps), np.complex64)
    x[0, 0] = np.complex64(1.0 / c[0].astype(np.complex128))
    ref = K1Reference(x, sf)
    assert int(np.argmax(ref.m64[0])) == nb // 2
    assert np.allclose(np.delete(ref.m64[0], nb // 2), 1.0, rtol=1e-6) and ref.m64[0, nb // 2] == pytest.approx(2.0, rel=1e-6)
    worst, ties = check_k1([nb // 2, 0], [np.float32(ref.m64[0, nb // 2]), 0.0], None, sf, ref=ref)
    assert worst < 0.1 and ties == 1
    with pytest.raises(AssertionError):
        check_k1([0, 0], None, None, sf, ref=ref)
