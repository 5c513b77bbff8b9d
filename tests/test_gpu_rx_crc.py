"""The payload CRC on the device paths: lora_b200_frames_crc_last after every entry point, and CRC-aided list decoding
(lora_b200_rx_params.crc_list, rs_crc_list_kernel) -- nothing changes with it off, the device follows the host emulation frame
by frame, it decodes at least the frames soft decisions decode, and wrong payloads it accepts stay within the false-accept
bound."""
import math

import numpy as np
import pytest

from antenna_common import BW, SENSITIVITY, synth_antennas
from conftest import FRAME_CASES, make_case_iq
from crc_common import BAD, OK, RECOVERED, receive_crc, with_crc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def make_dec(sf, osr=8, cr=4, rr=False, **kw):
    import gr_lora_b200 as G
    return G.decoder(osr * BW, BW, sf, False, cr, True, rr, quiet=True, **kw)


def n_items_for(sf, osr, n_bytes, rr, cr=4):
    import gr_lora_b200 as G
    sps = osr << sf
    return int((12 + G.tx_frame_symbols(n_bytes, sf, cr, False, True, rr)) * sps + sps // 4 + 9 * sps) // 8 * 8


def capture(torch, sf, osr, m, n_rx, snr, seed, cr=4, n_bytes=12, valid=True):
    """n_rx receivers x m antennas, one frame each (payload || CRC bytes, or random trailing bytes when not valid)."""
    rng = np.random.default_rng(seed)
    rr = sf > 10
    pays = []
    for _ in range(n_rx):
        p = bytes(rng.integers(0, 256, n_bytes, dtype=np.uint8))
        pays.append([with_crc(p, cr) if valid else p + bytes(rng.integers(0, 256, 2, dtype=np.uint8))])
    n = n_items_for(sf, osr, n_bytes + 2, rr, cr)
    gains = np.exp(2j * np.pi * rng.uniform(size=(n_rx, m)))
    x, placed = synth_antennas(torch, sf, osr, pays, n, snr, gains, seed, rr=rr, cr=cr)
    return x, n, placed


def rx(dec, x, n, m, **kw):
    before = dec.launch_count()
    c, frames, info = dec.receive(x, n_items=n, antennas=m, **kw)
    return dict(consumed=c.tobytes(), frames=frames.tobytes(), info=info.tobytes(), drops=dec.header_drops,
                launches=dec.launch_count() - before, crc=dec.frames_crc_last().tolist(), recs=frames)


# ---- with the option off nothing changes ------------------------------------------------------------------------------------
@pytest.mark.parametrize("osr", [8, 2])
@pytest.mark.parametrize("m", [1, 2])
@pytest.mark.parametrize("host", [False, True])
def test_option_off_changes_nothing(torch, osr, m, host):
    """crc_list = 0 twice and the field left out: byte-identical records, rx_info, consumed, header drops and launches, hard
    and soft, device and host input.  Soft with crc_list = 8 at +10 dB, where every frame checks: the same again, plus the
    one list kernel launch.  Hard decisions with crc_list > 0, and crc_list > 12, are refused before any launch."""
    from gr_lora_b200 import _native as N
    sf, n_rx = 8, 6
    x, n, placed = capture(torch, sf, osr, m, n_rx, 10.0, seed=osr * 10 + m)
    if host:
        x = x.cpu().numpy()
    dec = make_dec(sf, osr, n_streams=n_rx * m, max_items_per_call=n)
    for soft in (False, True):
        base = rx(dec, x, n, m, soft=soft)
        for kw in (dict(crc_list=0), dict()):
            r = rx(dec, x, n, m, soft=soft, **kw)
            assert {k: v for k, v in r.items() if k != "recs"} == {k: v for k, v in base.items() if k != "recs"}, (soft, kw)
        assert len(base["recs"]) == n_rx and base["crc"] == [OK] * n_rx
        if soft:
            r = rx(dec, x, n, m, soft=True, crc_list=8)
            assert (r["consumed"], r["frames"], r["info"], r["drops"], r["crc"]) == \
                   (base["consumed"], base["frames"], base["info"], base["drops"], base["crc"])
            assert r["launches"] == base["launches"] + 1
        before = dec.launch_count()
        for bad in ([dict(soft=False, crc_list=4)] if not soft else [dict(soft=True, crc_list=13)]):
            with pytest.raises(N.LoraB200Error) as e:
                dec.receive(x, n_items=n, antennas=m, **bad)
            assert e.value.code == N.EINVAL
        assert dec.launch_count() == before
    dec.close()


# ---- the status accessor ----------------------------------------------------------------------------------------------------
def test_status_after_work_batch_and_receive(torch):
    """work_batch on the README frame x 5: 5 x OK.  receive on frames with tx.crc_bytes: all OK; with random trailing bytes:
    BAD.  A decoder without frames: empty."""
    import gr_lora_b200 as G
    case = next(c for c in FRAME_CASES if c[0] == "readme_sf7_cr4")
    x, _, _ = make_case_iq(case, n_frames=5)
    d = G.decoder(1e6, BW, 7, False, 4, True, quiet=True, n_streams=1)
    assert len(d.frames_crc_last()) == 0
    d.work_batch(x[None, :], callbacks=False)
    assert len(d.frames_last()) == 5 and d.frames_crc_last().tolist() == [OK] * 5
    d.close()
    for valid in (True, False):
        x, n, placed = capture(torch, 9, 8, 1, 16, 5.0, seed=3 + valid, valid=valid)
        dec = make_dec(9, n_streams=16, max_items_per_call=n)
        _, frames, _ = dec.receive(x, n_items=n)
        assert len(frames) == 16
        assert dec.frames_crc_last().tolist() == [OK if valid else BAD] * 16
        dec.close()


def test_lora_receiver_drops_bad_crc_frames_when_asked(torch):
    import gr_lora_b200 as G
    rng = np.random.default_rng(9)
    good = with_crc(bytes(rng.integers(0, 256, 10, dtype=np.uint8)), 4)
    bad = good[:-1] + bytes([good[-1] ^ 1])
    from gr_lora_b200 import tx
    x = tx.channel([tx.modulate_frame(tx.encode_frame(p, 7, 4), 7) for p in (good, bad)], sf=7, snr_db=20.0, seed=1)
    for drop, want in ((False, [good, bad]), (True, [good])):
        r = G.lora_receiver(1e6, 868e6, [868e6], BW, 7, False, 4, True, disable_channelization=True, sync="dechirp", soft=True,
                            crc_list=4, drop_bad_crc=drop, quiet=True)
        got = []
        r.message_port_subscribe(lambda s, blob: got.append(bytes(blob[18:])))
        r.run(x)
        assert got == want
    with pytest.raises(ValueError):
        G.lora_receiver(1e6, 868e6, [868e6], BW, 7, False, 4, True, disable_channelization=True, drop_bad_crc=True)


# ---- device against the host emulation ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("sf,cr,osr,m", [(7, 1, 8, 1), (7, 4, 2, 2), (10, 1, 2, 1), (10, 4, 8, 2), (12, 1, 8, 2), (12, 4, 2, 1)])
def test_device_follows_the_host_emulation(torch, sf, cr, osr, m):
    """At 1.5 dB below the soft decoder's sensitivity point (per antenna, 3 dB lower with two): per frame the device's
    CRC status and payload equal the emulation's (frames matched by start within 2 samples), and two device runs are
    bit-identical."""
    n_rx = 8 if sf < 12 else 4
    snr = SENSITIVITY[sf] - 1.5 - (3.0 if m == 2 else 0.0)
    x, n, placed = capture(torch, sf, osr, m, n_rx, snr, seed=100 * sf + 10 * cr + osr + m, cr=cr)
    dec = make_dec(sf, osr, cr, sf > 10, n_streams=n_rx * m, max_items_per_call=n)
    a = rx(dec, x, n, m, soft=True, crc_list=8)
    b = rx(dec, x, n, m, soft=True, crc_list=8)
    assert (a["frames"], a["info"], a["crc"]) == (b["frames"], b["info"], b["crc"])
    _, _, info = dec.receive(x, n_items=n, antennas=m, soft=True, crc_list=8)
    X = x.cpu().numpy()
    dev = {}
    for r, i, s in zip(a["recs"], info, a["crc"]):
        dev.setdefault(int(r["stream"]), []).append((int(i["start"]), s, bytes(r["bytes"][18: int(r["len"])])))
    statuses = []
    for g in range(n_rx):
        host = [e for e in receive_crc(X[g * m: g * m + m, :n], sf, osr, crc_list=8, cr=cr) if e["status"] == 0]
        for start, s, pay in dev.get(g, []):
            h = [e for e in host if abs(e["start"] - start) <= 2]
            assert h, (g, start)
            assert (h[0]["crc"], h[0]["payload"]) == (s, pay), (g, start)
            statuses.append(s)
    print(f"SF{sf} CR 4/{4 + cr} fs/bw {osr} M {m} at {snr:+.1f} dB: statuses {sorted(statuses)}")
    dec.close()


# ---- sensitivity and false accepts ----------------------------------------------------------------------------------------------
def test_list_decoding_gains_and_false_accepts(torch):
    """CR 4/5 and 4/8 at SF7, SF10 and SF12, 96 frames: at the first SNR (0.5 dB steps down from the sensitivity point) where
    soft decisions lose 20-50 % of the frames, soft + crc_list = 8 decodes at least as many CRC-correct frames, and the frames
    reported OK are the same with and without the list.  Wrong payloads reported RECOVERED: a frame whose errors the list
    cannot fix passes some combination with probability about (2^8 - 1) / 2^16 = 0.39 %, so over all points at most
    1 + 3 x 0.0039 x (frames soft decisions lose) are allowed.  (Wrong payloads reported OK are the CRC's own blind spot --
    equal errors in payload[L-1] and c0 cancel -- and come from soft decisions alone; they are counted, not bounded.)"""
    K, n_frames = 8, 96
    bound = (2 ** K - 1) / 2 ** 16
    failing, wrong, wrong_ok, lines = 0, 0, 0, []
    for sf in (7, 10, 12):
        for cr in (1, 4):
            snr = SENSITIVITY[sf]
            for step in range(16):
                x, n, placed = capture(torch, sf, 8, 1, n_frames, snr, seed=7000 + 100 * sf + 10 * cr + step, cr=cr, n_bytes=16)
                sent = {(s, p) for s, _, p in placed}
                dec = make_dec(sf, 8, cr, sf > 10, n_streams=n_frames, max_items_per_call=n)
                res = {}
                for k in (0, K):
                    r = rx(dec, x, n, 1, soft=True, crc_list=k)
                    got = [((int(f["stream"]), bytes(f["bytes"][18: int(f["len"])])), s) for f, s in zip(r["recs"], r["crc"])]
                    res[k] = dict(good={g for g, s in got if s in (OK, RECOVERED)} & sent, ok={g for g, s in got if s == OK},
                                  wrong_rec={g for g, s in got if s == RECOVERED} - sent)
                dec.close()
                if len(res[0]["good"]) <= 0.8 * n_frames or step == 15:
                    break
                snr -= 0.5
            w_ok = len(res[0]["ok"] - sent)
            lines.append(f"SF{sf} CR 4/{4 + cr} at {snr:+.1f} dB: CRC-correct soft {len(res[0]['good'])}/{n_frames}, soft + list({K}) "
                         f"{len(res[K]['good'])}/{n_frames}, wrong RECOVERED {len(res[K]['wrong_rec'])}, wrong OK {w_ok}")
            assert len(res[0]["good"]) >= 0.5 * n_frames, lines[-1]
            assert len(res[K]["good"]) >= len(res[0]["good"]), lines[-1]
            assert res[K]["ok"] == res[0]["ok"], lines[-1]
            failing += n_frames - len(res[0]["good"])
            wrong += len(res[K]["wrong_rec"])
            wrong_ok += w_ok
    print("\n".join(lines))
    allowed = 1 + 3 * bound * failing
    print(f"wrong payloads RECOVERED {wrong}, expected {bound * failing:.3f} over {failing} failing frames, allowed {allowed:.2f}; "
          f"wrong payloads OK (soft decisions alone) {wrong_ok}")
    assert wrong <= math.floor(allowed)
