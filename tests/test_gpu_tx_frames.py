"""The device frame encoder (lora_b200_tx_encode_dev) and frame modulator (lora_b200_tx_frames_dev) through the C ABI, against
the host encoder, modulator and channel of gr_lora_b200/tx.py, and through the receiver with every stream carrying its own
payloads."""
import ctypes as C

import numpy as np
import pytest

from gr_lora_b200 import _native as N

pytestmark = pytest.mark.gpu

SENTINEL = -1          # 0xFFFFFFFF in the int32 view of the shift buffer


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def make_dec(sf, cr=4, implicit=False, crc=True, rr=False, fs=1e6, **kw):
    import gr_lora_b200 as G
    return G.decoder(fs, 125000, sf, implicit, cr, crc, rr, quiet=True, **kw)


def encode_rows(torch, dec, payloads, rng, max_symbols):
    """tx_encode over `payloads` packed at unaligned offsets; returns the [n, max_symbols] shift rows (int64, host)."""
    offs, blob, pos = [], bytearray(b"\x5a"), 1
    for p in payloads:
        gap = int(rng.integers(0, 4))
        blob += b"\xa5" * gap
        pos += gap
        offs.append(pos)
        blob += p
        pos += len(p)
    pay = torch.from_numpy(np.frombuffer(bytes(blob), np.uint8).copy()).cuda()
    shifts = torch.full((len(payloads), max_symbols), SENTINEL, dtype=torch.int32, device="cuda")
    dec.tx_encode(pay, offs, [len(p) for p in payloads], shifts, max_symbols)
    torch.cuda.synchronize()
    return shifts, shifts.cpu().numpy().astype(np.int64)


@pytest.mark.parametrize("sf", range(7, 13))
def test_encoder_equals_host_encoder(torch, sf):
    """Every CR x header mode x CRC x reduced rate: one call of a few hundred frames of every short length and a random sweep
    to the maximum (random payloads, all-0x00, all-0xFF), payloads at unaligned offsets; untouched sentinels after each frame."""
    import gr_lora_b200 as G
    from gr_lora_b200 import tx
    for cr in (1, 2, 3, 4):
        for implicit in (False, True):
            for crc in (False, True):
                for rr in (False, True):
                    rng = np.random.default_rng(1000 * sf + 100 * cr + 8 * implicit + 4 * crc + 2 * rr)
                    lo, hi = (2 if crc and not implicit else 0), 255 + 2 * crc
                    lengths = list(range(lo, 21)) + rng.integers(21, hi + 1, 180).tolist() + [hi, hi]
                    pays = [bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in lengths]
                    pays += [bytes(hi), b"\xff" * hi, bytes(lo), b"\xff" * lo]
                    want = [tx.encode_frame(p, sf, cr, explicit=not implicit, has_crc=crc, reduced_rate=rr).shifts for p in pays]
                    max_symbols = max(len(w) for w in want) + 3
                    assert max(len(w) for w in want) == G.tx_frame_symbols(hi, sf, cr, implicit, crc, rr)
                    dec = make_dec(sf, cr, implicit, crc, rr)
                    _, got = encode_rows(torch, dec, pays, rng, max_symbols)
                    for f, w in enumerate(want):
                        assert got[f, : len(w)].tolist() == w, (sf, cr, implicit, crc, rr, len(pays[f]))
                        assert np.all(got[f, len(w):] == SENTINEL)
                    dec.close()


def test_encoder_refuses_bad_lengths_before_any_launch(torch):
    dec = make_dec(7, 4, False, True)
    pay = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    shifts = torch.full((4, 512), SENTINEL, dtype=torch.int32, device="cuda")
    L = N.lib()
    for lengths, max_symbols in (([6, 258], 512), ([6, 1], 512), ([6, 0], 512), ([6, 300], 512), ([6, 100], 20)):
        n0 = dec.launch_count()
        off = np.zeros(len(lengths), np.uint32)
        ln = np.array(lengths, np.uint32)
        rc = L.lora_b200_tx_encode_dev(dec._h, pay.data_ptr(), off.ctypes.data, ln.ctypes.data, len(lengths), shifts.data_ptr(),
                                       max_symbols, None)
        assert rc == N.EINVAL, (lengths, max_symbols)
        assert dec.launch_count() == n0
    torch.cuda.synchronize()
    assert bool((shifts == SENTINEL).all())
    implicit = make_dec(7, 4, True, True)                                   # implicit header: no length field, 0 and 1 are fine
    implicit.tx_encode(pay, [0, 0], [0, 1], shifts, 512)
    torch.cuda.synchronize()
    unsupported = make_dec(7, 0, False, True)                               # CR 4/4 has no interleaver block to encode
    with pytest.raises(N.LoraB200Error) as e:
        unsupported.tx_encode(pay, [0], [6], shifts, 512)
    assert e.value.code == N.EUNSUPPORTED


def assert_bits_equal(got, want):
    g, w = np.asarray(got).view(np.uint64), np.asarray(want).view(np.uint64)
    bad = np.flatnonzero(g != w)
    assert bad.size == 0, (bad.size, bad[:8].tolist(), np.asarray(got)[bad[:4]].tolist(), np.asarray(want)[bad[:4]].tolist())


def frames_array(dec, rows):
    """rows: (start, stream, n_symbols, cfo_hz, sync_word) -> TX_FRAME_DTYPE array."""
    fr = np.zeros(len(rows), dec.TX_FRAME_DTYPE)
    for f, (start, s, n, cfo, sw) in enumerate(rows):
        fr[f] = (start, s, n, cfo, sw, (0, 0, 0))
    return fr


def host_row(frames_host, starts, n_items, cfos=None, fs=1e6):
    """Reference row built from tx.modulate_frame outputs placed at `starts` (complex128 -> cf32 as tx.channel does it)."""
    x = np.zeros(n_items, np.complex128)
    for k, (f, s) in enumerate(zip(frames_host, starts)):
        v = 1.0 * np.asarray(f, np.complex128)          # tx.channel's amplitude scaling (it turns -0 imaginary parts into +0)
        if cfos is not None and cfos[k]:
            v = v * np.exp(2j * np.pi * cfos[k] * np.arange(s, s + v.size) / fs)
        x[s: s + v.size] = v
    return x.astype(np.complex64)


@pytest.mark.parametrize("sf,fs", [(7, 1e6), (8, 1e6), (9, 1e6), (10, 1e6), (11, 1e6), (12, 1e6), (9, 2e6)])
def test_frames_equal_host_channel(torch, sf, fs):
    """No noise, no CFO, the host's chirp table: row = tx.channel(...) zero-padded, bit for bit."""
    from gr_lora_b200 import tx
    rng = np.random.default_rng(sf * 10 + int(fs / 1e6))
    dec = make_dec(sf, 4, False, True, sf > 10, fs=fs)
    sps = dec.sps
    pays = [bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in (2, 9, 17)]
    sws = [0x12, 0x78, 0x12]
    enc = [tx.encode_frame(p, sf, 4, has_crc=True, reduced_rate=sf > 10) for p in pays]
    host = [tx.modulate_frame(e, sf, fs=fs, sync_word=sw) for e, sw in zip(enc, sws)]
    lead, gap, tail = 2.5, 3.25, 5.0
    want = tx.channel(host, sf=sf, fs=fs, snr_db=None, lead_symbols=lead, gap_symbols=gap, tail_symbols=tail)
    n_items = (want.size + 3 * sps) // 2 * 2
    starts, pos = [], int(lead * sps)
    for h in host:
        starts.append(pos)
        pos += h.size + int(gap * sps)
    max_symbols = max(len(e.shifts) for e in enc) + 1
    shifts, _ = encode_rows(torch, dec, pays, rng, max_symbols)
    rows = [(starts[k], 0, len(enc[k].shifts), 0.0, sws[k]) for k in range(3)]
    up = torch.from_numpy(tx.base_upchirp(sf, fs=fs).astype(np.complex64)).cuda()
    out = torch.full((1, n_items), float("nan"), dtype=torch.complex64, device="cuda")
    dec.tx_frames(frames_array(dec, rows), shifts, max_symbols, 1, n_items, out, up_table_dev=up)
    torch.cuda.synchronize()
    ref = np.zeros(n_items, np.complex64)
    ref[: want.size] = want
    assert_bits_equal(out.cpu().numpy()[0], ref)
    dec.close()


def test_frames_odd_starts_sparse_rows_any_order(torch):
    """Odd starts, adjacent frames, rows with 0, 1 and many frames: the same output for shuffled descriptors, and equal to
    the host modulator's frames placed at those starts."""
    from gr_lora_b200 import tx
    sf, ns = 8, 5
    rng = np.random.default_rng(99)
    dec = make_dec(sf, 2, False, False)
    sps = dec.sps
    n_items = 110 * sps
    rows, pays, placed = [], [], {s: [] for s in range(ns)}
    layout = {0: [], 1: [101], 2: [1, None, 7 * sps + 3], 3: [0], 4: [3, None]}     # None: right after the previous frame
    for s, starts in layout.items():
        pos = 0
        for st in starts:
            p = bytes(rng.integers(0, 256, int(rng.integers(0, 6)), dtype=np.uint8))
            e = tx.encode_frame(p, sf, 2, has_crc=False)
            start = pos if st is None else max(st, pos)
            rows.append((start, s, len(e.shifts), 0.0, 0x34))
            pays.append(p)
            h = tx.modulate_frame(e, sf, sync_word=0x34)
            placed[s].append((start, h))
            pos = start + h.size
    assert max(r[0] for r in rows if r[1] == 2) % 2 == 1
    max_symbols = max(r[2] for r in rows)
    shifts, _ = encode_rows(torch, dec, pays, rng, max_symbols)
    up = torch.from_numpy(tx.base_upchirp(sf).astype(np.complex64)).cuda()
    out = torch.empty((ns, n_items), dtype=torch.complex64, device="cuda")
    dec.tx_frames(frames_array(dec, rows), shifts, max_symbols, ns, n_items, out, up_table_dev=up)
    perm = rng.permutation(len(rows))
    out2 = torch.empty_like(out)
    dec.tx_frames(frames_array(dec, [rows[k] for k in perm]), shifts[torch.from_numpy(perm).cuda()].contiguous(), max_symbols, ns,
                  n_items, out2, up_table_dev=up)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert np.array_equal(got.view(np.uint64), out2.cpu().numpy().view(np.uint64))
    for s in range(ns):
        want = host_row([h for _, h in placed[s]], [st for st, _ in placed[s]], n_items)
        assert np.array_equal(got[s].view(np.uint64), want.view(np.uint64)), s
    assert not got[0].any()


def test_frames_refuse_bad_placement_before_any_launch(torch):
    dec = make_dec(7)
    sps = dec.sps
    n_sym = 20
    flen = (12 + n_sym) * sps + sps // 4
    shifts = torch.zeros((2, n_sym), dtype=torch.int32, device="cuda")
    out = torch.zeros((2, 4 * flen), dtype=torch.complex64, device="cuda")
    n_items = out.shape[1]
    good = [(0, 0, n_sym, 0.0, 0x12), (flen, 0, n_sym, 0.0, 0x12)]
    dec.tx_frames(frames_array(dec, good), shifts, n_sym, 2, n_items, out)          # adjacent is fine
    torch.cuda.synchronize()
    L = N.lib()
    bad = {
        "overlap": [(0, 1, n_sym, 0.0, 0x12), (flen - 1, 1, n_sym, 0.0, 0x12)],
        "overrun": [(n_items - flen + 1, 0, n_sym, 0.0, 0x12)],
        "stream": [(0, 2, n_sym, 0.0, 0x12)],
        "n_symbols": [(0, 0, n_sym + 1, 0.0, 0x12)],
    }
    for name, rows in bad.items():
        fr = frames_array(dec, rows)
        n0 = dec.launch_count()
        rc = L.lora_b200_tx_frames_dev(dec._h, None, C.cast(fr.ctypes.data, C.POINTER(N.TxFrame)), fr.size, shifts.data_ptr(), n_sym,
                                       0.0, 0, 2, n_items, out.data_ptr(), None)
        assert rc == N.EINVAL, name
        assert dec.launch_count() == n0, name


def test_frames_cfo_matches_host_channel(torch):
    """Per-frame CFO: each row within 2e-4 of tx.channel(..., cfo_hz=...) of its frame."""
    from gr_lora_b200 import tx
    sf = 9
    rng = np.random.default_rng(5)
    dec = make_dec(sf)
    sps = dec.sps
    cfos = [1234.5, -2718.0, 31.0]
    pays = [bytes(rng.integers(0, 256, 8, dtype=np.uint8)) for _ in cfos]
    enc = [tx.encode_frame(p, sf, 4) for p in pays]
    wants = [tx.channel([tx.modulate_frame(e, sf)], sf=sf, snr_db=None, lead_symbols=3.0, tail_symbols=2.0, cfo_hz=c)
             for e, c in zip(enc, cfos)]
    n_items = max(w.size for w in wants) // 2 * 2
    max_symbols = max(len(e.shifts) for e in enc)
    shifts, _ = encode_rows(torch, dec, pays, rng, max_symbols)
    rows = [(3 * sps, s, len(enc[s].shifts), cfos[s], 0x12) for s in range(len(cfos))]
    up = torch.from_numpy(tx.base_upchirp(sf).astype(np.complex64)).cuda()
    out = torch.empty((len(cfos), n_items), dtype=torch.complex64, device="cuda")
    dec.tx_frames(frames_array(dec, rows), shifts, max_symbols, len(cfos), n_items, out, up_table_dev=up)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for s, w in enumerate(wants):
        ref = np.zeros(n_items, np.complex64)
        ref[: min(n_items, w.size)] = w[:n_items]
        assert np.abs(got[s] - ref).max() < 2e-4, s


def test_frames_noise_is_tx_expand_noise(torch):
    """tx_frames(sigma, seed) == tx_expand(tx_frames(0), n_streams, sigma, seed) bit for bit (with CFO and odd starts);
    reproducible; another seed differs."""
    dec = make_dec(7)
    out0, placed = dec.synth_streams([[bytes([s, k, 3, 4]) for k in range(3)] for s in range(6)], 120 * dec.sps, lead_symbols=1.3,
                                     gap_symbols=0.77, cfo_hz=[[300.0 * s - 700.0 * k for k in range(3)] for s in range(6)])
    assert len(placed) >= 6 and any(st % 2 for _, st, _ in placed)
    ns, n_items = out0.shape
    sigma = 0.125
    a, _ = dec.synth_streams([[bytes([s, k, 3, 4]) for k in range(3)] for s in range(6)], n_items, lead_symbols=1.3, gap_symbols=0.77,
                             cfo_hz=[[300.0 * s - 700.0 * k for k in range(3)] for s in range(6)], noise_sigma=sigma, seed=11)
    b = torch.empty_like(a)
    dec.tx_expand(out0, ns, n_items, ns, b, noise_sigma=sigma, seed=11)
    c, _ = dec.synth_streams([[bytes([s, k, 3, 4]) for k in range(3)] for s in range(6)], n_items, lead_symbols=1.3, gap_symbols=0.77,
                             cfo_hz=[[300.0 * s - 700.0 * k for k in range(3)] for s in range(6)], noise_sigma=sigma, seed=11)
    e, _ = dec.synth_streams([[bytes([s, k, 3, 4]) for k in range(3)] for s in range(6)], n_items, lead_symbols=1.3, gap_symbols=0.77,
                             cfo_hz=[[300.0 * s - 700.0 * k for k in range(3)] for s in range(6)], noise_sigma=sigma, seed=12)
    torch.cuda.synchronize()
    assert torch.equal(torch.view_as_real(a), torch.view_as_real(b))
    assert torch.equal(torch.view_as_real(a), torch.view_as_real(c))
    assert not torch.equal(a, e)
    z = torch.view_as_real(a - out0).cpu().numpy().astype(np.float64)
    assert abs(z.std() - sigma) < 2e-3


def check_round_trip(dec, out, placed, n_streams, n_items):
    dec.work_batch(out, n_items=n_items, stride_items=n_items, host=0, callbacks=False)
    fr = dec.frames_last()
    want = {s: [] for s in range(n_streams)}
    for s, _, p in placed:
        want[s].append(p)
    got = {s: [] for s in range(n_streams)}
    for r in fr:
        got[int(r["stream"])].append(bytes(r["bytes"][18: int(r["len"])]))
    bad = [s for s in range(n_streams) if len(got[s]) != len(want[s]) or any(g[: len(w)] != w for g, w in zip(got[s], want[s]))]
    assert len(fr) == len(placed) and not bad, (len(fr), len(placed), bad[:8], [(got[s], want[s]) for s in bad[:2]])


def test_round_trip_every_stream_its_own_payloads(torch):
    """4096 SF7 streams x 256 symbol times, every frame a distinct payload, 35 dB: each placed frame is published on its own
    stream with its own payload, in order, and nothing else is published."""
    from gr_lora_b200 import tx
    sf, ns = 7, 4096
    sps = 8 << sf
    n_items = 256 * sps
    rng = np.random.default_rng(0x4C6F)
    pays = [[s.to_bytes(2, "little") + bytes([k]) + bytes(rng.integers(0, 256, 9, dtype=np.uint8)) for k in range(8)]
            for s in range(ns)]
    gen = make_dec(sf, 4, False, False)
    up = torch.from_numpy(tx.base_upchirp(sf).astype(np.complex64)).cuda()
    sigma = float(np.sqrt(10 ** (-3.5) / 2))
    out, placed = gen.synth_streams(pays, n_items, lead_symbols=2.5, noise_sigma=sigma, seed=3, up_table_dev=up)
    torch.cuda.synchronize()
    assert len({p for _, _, p in placed}) == len(placed) >= 4 * ns
    per_stream = max(sum(1 for s, _, _ in placed if s == t) for t in range(4))
    rx = make_dec(sf, 4, False, False, n_streams=ns, demod="fft", max_items_per_call=n_items, max_frames_per_call=per_stream + 2)
    check_round_trip(rx, out, placed, ns, n_items)


@pytest.mark.parametrize("sf", [8, 9, 10, 11, 12])
def test_round_trip_configurations(torch, sf):
    """SF8..SF12 x CR1..4, implicit and explicit header, CRC on and off, reduced rate above SF10: every stream publishes its
    own payloads.  Cases alternate between the gradient demodulator, with a per-frame CFO of 1-2.5 kHz, and the FFT
    demodulator without CFO (get_shift_fft has no CFO correction; a CFO of several bins moves its bins).  SF9 and SF10 run
    the FFT demodulator only: at CR 1-2 and 38 dB the gradient demodulator misreads an occasional header-block symbol there,
    on captures built by the host encoder and channel as well, which is a property of the receiver, not of this transmitter.
    """
    import gr_lora_b200 as G
    from gr_lora_b200 import tx
    rng = np.random.default_rng(sf)
    up = torch.from_numpy(tx.base_upchirp(sf).astype(np.complex64)).cuda()
    sigma = float(np.sqrt(10 ** (-3.8) / 2))
    k = 0
    for cr in (1, 2, 3, 4):
        for implicit in (False, True):
            for crc in (False, True):
                ns, plen = 4, 6 + 2 * crc
                pays = [[bytes([s, j]) + bytes(rng.integers(0, 256, plen - 2, dtype=np.uint8)) for j in range(2)] for s in range(ns)]
                demod = "fft" if (k % 2 or sf in (9, 10)) else "gradient"
                cfo = [[float(rng.uniform(1000.0, 2500.0)) if demod == "gradient" else 0.0 for _ in range(2)] for _ in range(ns)]
                gen = make_dec(sf, cr, implicit, crc, sf > 10)
                n_sym = G.tx_frame_symbols(plen, sf, cr, implicit, crc, sf > 10)
                n_items = (2 * (12 + n_sym + 5) + 6) * gen.sps
                out, placed = gen.synth_streams(pays, n_items, lead_symbols=2.6, gap_symbols=5.0, cfo_hz=cfo, noise_sigma=sigma,
                                                seed=k, sync_word=0x78 if sf >= 11 else 0x12, up_table_dev=up)
                torch.cuda.synchronize()
                assert len(placed) == 2 * ns
                rx = make_dec(sf, cr, implicit, crc, sf > 10, n_streams=ns, demod=demod,
                              max_items_per_call=n_items, max_frames_per_call=4)
                try:
                    check_round_trip(rx, out, placed, ns, n_items)
                except AssertionError as exc:
                    raise AssertionError((sf, cr, implicit, crc, demod, str(exc)[:300])) from None
                rx.close()
                gen.close()
                k += 1
