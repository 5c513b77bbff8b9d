"""GPU parity of the DEFAULT K1 kernels beyond one grid pass, through the C ABI.

The persistent kernels walk `grid x groups` symbols per pass and recycle their shared-memory ring slots, mbarrier
phases and (team kernels) exchange buffers + flags from the third pass on; a batch smaller than one pass never
exercises that.  Here every SF runs a ragged count of more than NSLOT + 2 passes with edge bins at -3 dB, twice back
to back (the second launch reuses every buffer), and must equal the oracle's get_shift_fft bit for bit.  Also: the
host-buffer pipeline across several 64 MiB chunks (two streams, one scratch per slot), two decoders of the same SF
running concurrently on two streams (the cross-CTA kernels are launched cooperatively: they must serialise, not
dead-lock), and two streams sharing ONE decoder."""
import time

import numpy as np
import pytest

from k1_reference import check_k1, symbols_per_pass

pytestmark = pytest.mark.gpu

# a ragged tail past four passes (more than NSLOT + 2 passes of the SF7-SF10 slot rings, more than two turns of the
# SF11 / SF12 row pools) of the default kernel's grid on the device's SMs
MULTIPASS_TAIL = {7: 7, 8: 7, 9: 7, 10: 315, 11: 15, 12: 35}


def multipass_n(torch, sf):
    return 4 * symbols_per_pass(sf, torch.cuda.get_device_properties(0).multi_processor_count) + MULTIPASS_TAIL[sf]


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _symbols(sf, n, seed, snr_db=-3.0):
    from gr_lora_b200 import tx
    nb = 1 << sf
    rng = np.random.default_rng(seed)
    vals = rng.integers(0, nb, n)
    vals[:6] = [0, 1, nb // 2 - 1, nb // 2, nb // 2 + 1, nb - 1]
    out = np.empty(n * (8 << sf), np.complex64)
    step = max(1, (64 << 20) // (16 * (8 << sf)))           # bound the complex128 temporaries of the modulator
    for s in range(0, n, step):
        e = min(n, s + step)
        out[s * (8 << sf): e * (8 << sf)] = tx.synth_symbols(vals[s:e], sf, snr_db=snr_db, seed=seed + 1 + s)
    return vals, out


def _wait(torch, seconds, what):
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream())
    t0 = time.time()
    while not ev.query():
        assert time.time() - t0 < seconds, f"device did not finish: {what}"
        time.sleep(0.005)


@pytest.mark.parametrize("sf", range(7, 13))
def test_default_kernel_multipass_ragged(torch, oracle, sf):
    import gr_lora_b200 as G
    n = multipass_n(torch, sf)
    vals, x = _symbols(sf, n, 4000 + sf)
    dec = G.decoder(1e6, 125000, sf, False, 4, True, demod="fft", quiet=True)
    iq = torch.from_numpy(x).cuda()
    ob, om = oracle.Decoder(sf=sf).demod_fft_batch(x)
    for rep in range(2):
        bins = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        mags = torch.zeros(n, dtype=torch.float32, device="cuda")
        dec.demod_fft(iq, n, bins, mags, torch.cuda.current_stream().cuda_stream)
        _wait(torch, 20.0, f"SF{sf} launch {rep}")
        gb = bins.cpu().numpy().astype(np.uint32)
        assert np.array_equal(gb, ob), (sf, rep, int(np.sum(gb != ob)), np.nonzero(gb != ob)[0][:8])
        if rep == 0:
            first = mags.cpu().numpy()
            check_k1(gb, first, x, sf, what=f"SF{sf} multipass")
        else:
            assert np.array_equal(mags.cpu().numpy().view(np.int32), first.view(np.int32))
    assert np.mean(ob == vals) == 1.0
    dec.close()


@pytest.mark.parametrize("sf,n", [(8, 9000), (11, 1100), (12, 601)])
def test_host_pipeline_multi_chunk(torch, oracle, sf, n):
    """lora_b200_demod_fft_host over more than two 64 MiB chunks (4096 / 512 / 256 symbols per chunk): both pipeline
    slots are reused, each with its own keys / exchange scratch; pageable and pinned host buffers."""
    import gr_lora_b200 as G
    vals, x = _symbols(sf, n, 5000 + sf, snr_db=0.0)
    dec = G.decoder(1e6, 125000, sf, False, 4, True, demod="fft", quiet=True)
    ob, om = oracle.Decoder(sf=sf).demod_fft_batch(x)
    bins = np.full(n, 0xFFFFFFFF, np.uint32)
    mags = np.zeros(n, np.float32)
    dec.demod_fft_host(x, bins, mags)                        # pageable: staged through the library's pinned chunks
    assert np.array_equal(bins, ob)
    check_k1(bins, mags, x, sf, what=f"SF{sf} host pipeline")
    hx = torch.from_numpy(x).pin_memory()
    hb = torch.full((n,), -1, dtype=torch.int32).pin_memory()
    for _ in range(2):
        hb.fill_(-1)
        dec.demod_fft_host((hx.data_ptr(), n), hb.numpy().view(np.uint32), None)
        assert np.array_equal(hb.numpy().view(np.uint32), ob)
    dec.close()


@pytest.mark.parametrize("sf", [11, 12])
def test_two_decoders_two_streams_concurrently(torch, oracle, sf):
    """Two decoders, two non-blocking streams, launches interleaved without synchronisation in between.  A kernel whose
    CTAs wait for each other must be co-resident as a whole (cooperative launch) or the two grids could each hold
    half of the SMs for ever."""
    import gr_lora_b200 as G
    n = multipass_n(torch, sf)
    vals, x = _symbols(sf, n, 6000 + sf)
    ob, _ = oracle.Decoder(sf=sf).demod_fft_batch(x)
    iq = torch.from_numpy(x).cuda()
    decs = [G.decoder(1e6, 125000, sf, False, 4, True, demod="fft", quiet=True) for _ in range(2)]
    streams = [torch.cuda.Stream() for _ in range(2)]
    bins = [torch.full((n,), -1, dtype=torch.int32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    for rep in range(3):
        for k in range(2):
            decs[k].demod_fft(iq, n, bins[k], None, streams[k].cuda_stream)
    t0 = time.time()
    while not all(s.query() for s in streams):
        assert time.time() - t0 < 30.0, "concurrent K1 launches did not finish"
        time.sleep(0.005)
    for k in range(2):
        assert np.array_equal(bins[k].cpu().numpy().astype(np.uint32), ob)
        decs[k].close()


@pytest.mark.parametrize("sf", [9, 12])
def test_one_decoder_two_streams(torch, oracle, sf):
    """The same decoder driven from two streams: the launches share the decoder's key / exchange scratch, so the
    library orders them (event wait) instead of letting the second launch's memset run under the first kernel."""
    import gr_lora_b200 as G
    n = multipass_n(torch, sf)
    xa = _symbols(sf, n, 7000 + sf)[1]
    xb = _symbols(sf, n, 7100 + sf)[1]
    o = oracle.Decoder(sf=sf)
    oa, ob = o.demod_fft_batch(xa)[0], o.demod_fft_batch(xb)[0]
    da, db = torch.from_numpy(xa).cuda(), torch.from_numpy(xb).cuda()
    dec = G.decoder(1e6, 125000, sf, False, 4, True, demod="fft", quiet=True)
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    ba = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    bb = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    for rep in range(3):
        dec.demod_fft(da, n, ba, None, s0.cuda_stream)
        dec.demod_fft(db, n, bb, None, s1.cuda_stream)
    t0 = time.time()
    while not (s0.query() and s1.query()):
        assert time.time() - t0 < 30.0, "launches did not finish"
        time.sleep(0.005)
    assert np.array_equal(ba.cpu().numpy().astype(np.uint32), oa)
    assert np.array_equal(bb.cpu().numpy().astype(np.uint32), ob)
    dec.close()
