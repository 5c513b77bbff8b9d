"""GPU: every K1 kernel against the float64 get_shift_fft of tests/k1_reference.py, through the C ABI.

Every output goes through check_k1: the reported bin must lie within 2 tau of the float64 maximum and the magnitude
within tau of the float64 magnitude of that bin (tau = 2^-24 log2(sps) (m64[b] + ||y||), about 6e-7 of a clean peak).
  * every bin: one symbol per value 0..N-1 per SF, clean (bins exact), at -3 dB and with a half-bin frequency offset;
  * pure noise over more than two grid passes, a dechirped impulse (flat spectrum, bin N/2 doubled) and silence (bin 0);
  * batch sizes derived from the device's SM count around the symbols-per-pass count U of each default kernel, more than
    four passes with a ragged tail, and at SF12 every cluster getting exactly 1, 2, 3 symbols or a 1 / 2 mix: 64 untouched
    sentinels past the outputs, bins identical without magnitudes, two runs bit-identical, every symbol's result
    independent of the batch it was in;
  * input pointers 16 bytes and an odd number of symbols into a larger buffer, outputs at an odd element offset;
  * power-of-two amplitude scaling 2^-30 .. 2^30: bins identical, magnitudes scaled exactly.
The A/B kernels (LORA_B200_K1=generic, LORA_B200_K1_ROWS=0) are selected once per process, so the every-bin, noise and
batch-size cases run in a child process under each and its outputs are checked here against the same reference.

Each check prints one line `K1F64 kernel=... sf=... case=... worst=<err/tau> ties=<symbols with a near tie>`."""
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent
if __name__ == "__main__":                       # child process: the A/B kernels
    sys.path[:0] = [str(HERE.parent), str(HERE)]

from k1_reference import K1Reference, check_k1, downchirp, symbols_per_pass  # noqa: E402

pytestmark = pytest.mark.gpu

SFS = list(range(7, 13))
CHUNK_BYTES = 64 << 20
SENTINEL = 64
BIN_SENT = np.int32(-0x21524111)                 # 0xDEADBEEF
MAG_SENT = np.float32(-1234.5)
VARIANTS = ("clean", "m3db", "halfbin")
AB_KERNELS = {"generic": ("LORA_B200_K1", "generic", SFS), "rows0": ("LORA_B200_K1_ROWS", "0", [11, 12])}


# ---- inputs (deterministic, generated in chunks: SF12's every-bin batch is 1 GiB) ---------------------------------------
def every_bin_input(sf, variant):
    from gr_lora_b200 import tx
    nb, sps = 1 << sf, 8 << sf
    vals = np.arange(nb)
    x = np.empty((nb, sps), np.complex64)
    step = max(1, CHUNK_BYTES // (16 * sps))
    ramp = np.exp(1j * np.pi * np.arange(sps) / sps)           # half a bin (fs / (2 sps)) of frequency offset
    for s in range(0, nb, step):
        e = min(nb, s + step)
        y = tx.modulate_shifts(vals[s:e], sf).reshape(e - s, sps)
        if variant == "halfbin":
            y = y * ramp
        elif variant == "m3db":
            y = y + tx.awgn(y.size, -3.0, np.random.default_rng(1000 * sf + s)).reshape(y.shape)
        x[s:e] = y
    return vals, x.reshape(-1)


def noise_input(sf, n_sms):
    n = 2 * symbols_per_pass(sf, n_sms) + 5
    rng = np.random.default_rng(77 + sf)
    return (rng.standard_normal(n * (8 << sf)) + 1j * rng.standard_normal(n * (8 << sf))).astype(np.complex64)


def shape_counts(sf, n_sms):
    u = symbols_per_pass(sf, n_sms)
    ns = {1, 2, u - 1, u, u + 1, 2 * u - 1, 2 * u, 2 * u + 1, 4 * u + u // 2 + 3}
    if sf == 12:                                  # symbols per cluster: all 1 (u), all 2 (2u), all 3 (3u), a 1 / 2 mix
        ns |= {3 * u, u + u // 2}
    return sorted(k for k in ns if k >= 1)


def shape_pool(sf, n):
    """-3 dB symbols with the edge values first; every 7th symbol is noise only."""
    from gr_lora_b200 import tx
    nb, sps = 1 << sf, 8 << sf
    rng = np.random.default_rng(500 + sf)
    vals = rng.integers(0, nb, n)
    vals[:6] = [0, 1, nb // 2 - 1, nb // 2, nb // 2 + 1, nb - 1]
    x = np.empty((n, sps), np.complex64)
    step = max(1, CHUNK_BYTES // (16 * sps))
    for s in range(0, n, step):
        e = min(n, s + step)
        y = tx.synth_symbols(vals[s:e], sf, snr_db=-3.0, seed=600 + sf + s).reshape(e - s, sps)
        quiet = (np.arange(s, e) % 7) == 6
        y[quiet] = tx.awgn(int(quiet.sum()) * sps, 10.0, np.random.default_rng(s)).reshape(-1, sps)
        x[s:e] = y
    return x.reshape(-1)


# ---- running K1 through the C ABI -----------------------------------------------------------------------------------------
def run_k1(torch, dec, iq_ptr, n, with_mags=True, out_offset=0):
    """bins, mags of n symbols at iq_ptr; the outputs start out_offset elements into buffers that hold SENTINEL more
    elements past the n written ones, all of which must be left untouched."""
    tot = out_offset + n + SENTINEL
    bins = torch.full((tot,), int(BIN_SENT), dtype=torch.int32, device="cuda")
    mags = torch.full((tot,), float(MAG_SENT), dtype=torch.float32, device="cuda")
    dec.demod_fft(iq_ptr, n, bins[out_offset:].data_ptr(), mags[out_offset:].data_ptr() if with_mags else None,
                  torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    b, m = bins.cpu().numpy(), mags.cpu().numpy()
    outside = np.r_[0:out_offset, out_offset + n:tot]
    assert np.all(b[outside] == BIN_SENT), f"bins written outside [{out_offset}, {out_offset + n})"
    assert np.all(m[outside].view(np.int32) == MAG_SENT.view(np.int32)), f"mags written outside [{out_offset}, {out_offset + n})"
    b, m = b[out_offset:out_offset + n].view(np.uint32), m[out_offset:out_offset + n]
    if not with_mags:
        assert np.all(m.view(np.int32) == MAG_SENT.view(np.int32)), "mags written although none were passed"
        m = None
    return b, m


def run_shapes(torch, dec, sf, n_sms):
    """All batch sizes of shape_counts on the prefix of one pool; returns {n: (bins, mags)} after asserting sentinels,
    mags=None, two runs and independence of the batch."""
    ns = shape_counts(sf, n_sms)
    x = shape_pool(sf, ns[-1])
    iq = torch.from_numpy(x).cuda()
    out = {}
    for n in reversed(ns):
        b1, m1 = run_k1(torch, dec, iq.data_ptr(), n)
        b2, m2 = run_k1(torch, dec, iq.data_ptr(), n)
        b0, _ = run_k1(torch, dec, iq.data_ptr(), n, with_mags=False)
        assert np.array_equal(b1, b2) and np.array_equal(m1.view(np.int32), m2.view(np.int32)), f"SF{sf} n={n}: two runs differ"
        assert np.array_equal(b0, b1), f"SF{sf} n={n}: bins differ without magnitudes"
        if out:
            pb, pm = out[ns[-1]]
            assert np.array_equal(b1, pb[:n]) and np.array_equal(m1.view(np.int32), pm[:n].view(np.int32)), \
                f"SF{sf} n={n}: results differ from the same symbols in a batch of {ns[-1]}"
        out[n] = (b1, m1)
    return x, out


def new_decoder(sf):
    import gr_lora_b200 as G
    return G.decoder(1e6, 125000, sf, False, 4, True, demod="fft", quiet=True)


def sm_count(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def report(kernel, sf, case, stats):
    print(f"K1F64 kernel={kernel} sf={sf} case={case} worst={stats[0]:.3f} ties={stats[1]}")


# ---- the child process: every-bin, noise and batch-size outputs of an A/B kernel --------------------------------------------
def child_main(kind, out_path):
    import torch
    _, _, sfs = AB_KERNELS[kind]
    n_sms = sm_count(torch)
    res = {}
    for sf in sfs:
        dec = new_decoder(sf)
        for v in VARIANTS:
            _, x = every_bin_input(sf, v)
            iq = torch.from_numpy(x).cuda()
            res[f"{sf}/{v}/bins"], res[f"{sf}/{v}/mags"] = run_k1(torch, dec, iq.data_ptr(), x.size // (8 << sf))
            del iq
        x = noise_input(sf, n_sms)
        iq = torch.from_numpy(x).cuda()
        res[f"{sf}/noise/bins"], res[f"{sf}/noise/mags"] = run_k1(torch, dec, iq.data_ptr(), x.size // (8 << sf))
        del iq
        _, shapes = run_shapes(torch, dec, sf, n_sms)
        for n, (b, m) in shapes.items():
            res[f"{sf}/shape{n}/bins"], res[f"{sf}/shape{n}/mags"] = b, m
        dec.close()
    np.savez(out_path, **res)


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


@pytest.fixture(scope="module")
def ab_outputs():
    """kind -> outputs of the child process run under that kernel selection (run once, on first use)."""
    cache = {}
    tmp = tempfile.TemporaryDirectory(prefix="k1f64_")

    def get(kind):
        if kind not in cache:
            var, val, _ = AB_KERNELS[kind]
            path = os.path.join(tmp.name, f"{kind}.npz")
            env = dict(os.environ, **{var: val})
            p = subprocess.run([sys.executable, "-s", str(Path(__file__).resolve()), kind, path], env=env,
                               capture_output=True, text=True, timeout=1200)
            assert p.returncode == 0, f"child under {var}={val} failed:\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}"
            with np.load(path) as z:
                cache[kind] = {k: z[k] for k in z.files}
        return cache[kind]

    yield get
    tmp.cleanup()


_REF = {}


def cached_ref(key, make):
    """One (input, reference) pair at a time: consecutive tests of the same input share it."""
    if key not in _REF:
        _REF.clear()
        x = make()
        _REF[key] = (x, K1Reference(x[1] if isinstance(x, tuple) else x, key[0]))
    return _REF[key]


def _kernels(sf):
    return ["default"] + [k for k, (_, _, sfs) in AB_KERNELS.items() if sf in sfs]


@pytest.mark.parametrize("sf,variant,kernel", [(sf, v, k) for sf in SFS for v in VARIANTS for k in _kernels(sf)])
def test_every_bin(torch, ab_outputs, sf, variant, kernel):
    (vals, x), ref = cached_ref((sf, "every", variant), lambda: every_bin_input(sf, variant))
    nb = 1 << sf
    if kernel == "default":
        dec = new_decoder(sf)
        iq = torch.from_numpy(x).cuda()
        bins, mags = run_k1(torch, dec, iq.data_ptr(), nb)
        dec.close()
        del iq
    else:
        o = ab_outputs(kernel)
        bins, mags = o[f"{sf}/{variant}/bins"], o[f"{sf}/{variant}/mags"]
    report(kernel, sf, f"every-bin-{variant}", check_k1(bins, mags, None, sf, ref=ref, what=f"{kernel} SF{sf} {variant}"))
    if variant == "clean":
        assert np.array_equal(bins, vals.astype(np.uint32))
    if variant == "halfbin":                      # a genuine two-bin tie: the value or the one above it
        d = (bins.astype(np.int64) - vals) % nb
        assert np.all((d == 0) | (d == 1))


@pytest.mark.parametrize("sf,kernel", [(sf, k) for sf in SFS for k in _kernels(sf)])
def test_pure_noise(torch, ab_outputs, sf, kernel):
    n_sms = sm_count(torch)
    x, ref = cached_ref((sf, "noise", n_sms), lambda: noise_input(sf, n_sms))
    if kernel == "default":
        dec = new_decoder(sf)
        iq = torch.from_numpy(x).cuda()
        bins, mags = run_k1(torch, dec, iq.data_ptr(), x.size // (8 << sf))
        dec.close()
    else:
        o = ab_outputs(kernel)
        bins, mags = o[f"{sf}/noise/bins"], o[f"{sf}/noise/mags"]
    report(kernel, sf, "noise", check_k1(bins, mags, None, sf, ref=ref, what=f"{kernel} SF{sf} noise"))


@pytest.mark.parametrize("sf,kernel", [(sf, k) for sf in SFS for k in _kernels(sf)])
def test_batch_sizes_around_the_pass(torch, ab_outputs, sf, kernel):
    n_sms = sm_count(torch)
    ns = shape_counts(sf, n_sms)
    x, ref = cached_ref((sf, "shapes", n_sms), lambda: shape_pool(sf, ns[-1]))
    if kernel == "default":
        dec = new_decoder(sf)
        _, shapes = run_shapes(torch, dec, sf, n_sms)
        dec.close()
    else:
        o = ab_outputs(kernel)
        shapes = {n: (o[f"{sf}/shape{n}/bins"], o[f"{sf}/shape{n}/mags"]) for n in ns}
    assert sorted(shapes) == ns
    worst, ties = 0.0, 0
    for n in ns:
        w, t = check_k1(*shapes[n], None, sf, ref=ref[:n], what=f"{kernel} SF{sf} n={n}")
        worst, ties = max(worst, w), (t if n == ns[-1] else ties)
    report(kernel, sf, f"shapes(n={','.join(map(str, ns))})", (worst, ties))


@pytest.mark.parametrize("sf", SFS)
def test_flat_spectrum_and_silence(torch, sf):
    """x[0] = 1 / c[0], zeros elsewhere: the dechirped symbol is an impulse, every bin has the same magnitude except N/2,
    which the quirk doubles.  Silence: all magnitudes 0, the first maximum (bin 0) wins."""
    nb, sps = 1 << sf, 8 << sf
    c = downchirp(sf)
    x = np.zeros((4, sps), np.complex64)
    x[0, 0] = x[2, 0] = np.complex64(1.0 / c[0].astype(np.complex128))
    x = x.reshape(-1)
    dec = new_decoder(sf)
    iq = torch.from_numpy(x).cuda()
    bins, mags = run_k1(torch, dec, iq.data_ptr(), 4)
    dec.close()
    assert list(bins) == [nb // 2, 0, nb // 2, 0] and mags[1] == 0 and mags[3] == 0
    report("default", sf, "flat+silence", check_k1(bins, mags, x, sf))


@pytest.mark.parametrize("sf", SFS)
def test_pointer_offsets(torch, sf):
    """The input 16 bytes and an odd number of symbols into a larger buffer, the outputs at an odd element offset: the
    TMA bulk copies and SF12's tensor map take whatever 16-byte aligned base they are given."""
    sps = 8 << sf
    n = symbols_per_pass(sf, sm_count(torch)) + 5
    x = shape_pool(sf, n)
    dec = new_decoder(sf)
    iq = torch.from_numpy(x).cuda()
    want_b, want_m = run_k1(torch, dec, iq.data_ptr(), n)
    for lead in (2, 3 * sps):                     # 16 bytes; three whole symbols
        buf = torch.zeros(lead + x.size + sps, dtype=torch.complex64, device="cuda")
        buf[lead:lead + x.size] = iq
        for off in (0, 1, 3):
            b, m = run_k1(torch, dec, buf.data_ptr() + 8 * lead, n, out_offset=off)
            assert np.array_equal(b, want_b) and np.array_equal(m.view(np.int32), want_m.view(np.int32)), (lead, off)
    dec.close()
    check_k1(want_b, want_m, x, sf, what=f"SF{sf} pointer offsets")


@pytest.mark.parametrize("sf", SFS)
def test_power_of_two_scaling(torch, sf):
    """x * 2^k for k in -30..30: every fp32 operation of the kernels commutes with it exactly in that range (DESIGN 3
    states where the |.|^2 key would underflow or overflow), so bins are identical and magnitudes scale exactly."""
    n = 24
    x = shape_pool(sf, n)
    dec = new_decoder(sf)
    iq = torch.from_numpy(x).cuda()
    b0, m0 = run_k1(torch, dec, iq.data_ptr(), n)
    for k in (-30, -20, -11, -1, 1, 9, 20, 30):
        xs = (x * np.float32(2.0 ** k)).astype(np.complex64)
        assert np.array_equal(xs / np.float32(2.0 ** k), x)
        iq = torch.from_numpy(xs).cuda()
        b, m = run_k1(torch, dec, iq.data_ptr(), n)
        assert np.array_equal(b, b0), k
        assert np.array_equal(m, np.ldexp(m0, k)), (k, np.flatnonzero(m != np.ldexp(m0, k))[:4])
    dec.close()
    check_k1(b0, m0, x, sf, what=f"SF{sf} scaling")


if __name__ == "__main__":
    child_main(sys.argv[1], sys.argv[2])
