"""Time the device-side transmitter on one GPU (CUDA events, after warm-up) and print one JSON line.

  encode      lora_b200_tx_encode_dev: distinct 12-byte payloads -> chirp shifts, frames/s (SF7 and SF12, CR4/8)
  frames      lora_b200_tx_frames_dev against lora_b200_tx_expand_dev writing the same shape, GB/s written and the share of
              the 3 350 GB/s data-sheet HBM3 figure of the H100 SXM: [4096, 256 * sps] at SF7 (bench.py's e2e shape) and the
              config-4 shape (64 streams x 2 000 000 samples for each of SF7..SF12), with and without noise, and
              lora_b200_tx_frames_sfo_dev with every frame's clock off by +-20 ppm (tx_frames_sfo20)
  host        the path the tests and bench.py use today for the same kind of frames: tx.encode_frame + modulate_frame +
              channel on the host + the copy to the device, frames/s

The card's name and power limit are printed with the numbers: they are part of them.

    python tools/bench_tx.py [--iters 10] [--warmup 3] [--host-frames 256]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

HBM_GBS = 3350.0


def card(torch):
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # the numbers stay valid, the power limit is then unknown
        q = f"unknown ({exc})"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def timed(torch, fn, iters, warmup):
    """Mean seconds per call of fn() over `iters` calls between two CUDA events, after `warmup` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def layout(dec, n_streams, n_items, payload_len, lead=2.5, gap=4.0):
    """tx.channel's layout on every row: frame descriptors (start, stream, n_symbols) and the number of frames."""
    import gr_lora_b200 as G
    c = dec.cfg
    n_sym = G.tx_frame_symbols(payload_len, c.sf, c.cr, c.implicit, c.crc, c.reduced_rate)
    sps = dec.sps
    flen, g = (12 + n_sym) * sps + sps // 4, int(gap * sps)
    starts = []
    pos = int(lead * sps)
    while pos + flen + g <= n_items:
        starts.append(pos)
        pos += flen + g
    fr = np.zeros(n_streams * len(starts), dec.TX_FRAME_DTYPE)
    fr["stream"] = np.repeat(np.arange(n_streams), len(starts))
    fr["start"] = np.tile(np.array(starts, np.uint64), n_streams)
    fr["n_symbols"] = n_sym
    fr["sync_word"] = 0x78 if c.sf >= 11 else 0x12
    return fr, n_sym


def encode_inputs(torch, n_frames, payload_len, seed):
    rng = np.random.default_rng(seed)
    pay = torch.from_numpy(rng.integers(0, 256, n_frames * payload_len, dtype=np.uint8)).cuda()
    offsets = np.arange(n_frames, dtype=np.uint32) * payload_len
    lengths = np.full(n_frames, payload_len, np.uint32)
    return pay, offsets, lengths


def bench_encode(torch, G, sf, n_frames, args):
    dec = G.decoder(1e6, 125000, sf, False, 4, False, sf > 10, quiet=True)
    pay, off, ln = encode_inputs(torch, n_frames, 12, sf)
    n_sym = G.tx_frame_symbols(12, sf, 4, False, False, sf > 10)
    shifts = torch.empty((n_frames, n_sym), dtype=torch.int32, device="cuda")
    t = timed(torch, lambda: dec.tx_encode(pay, off, ln, shifts, n_sym, torch.cuda.current_stream().cuda_stream), args.iters, args.warmup)
    dec.close()
    return {"sf": sf, "frames": n_frames, "payload_bytes": 12, "s_per_call": t, "frames_per_s": n_frames / t}


def bench_shape(torch, G, sf, n_streams, n_items, args, payload_len=12):
    """tx_frames and tx_expand (k = 32 base rows, as bench.py's e2e) writing [n_streams, n_items], alternated per sigma."""
    from gr_lora_b200 import tx
    dec = G.decoder(1e6, 125000, sf, False, 4, False, sf > 10, quiet=True)
    st = torch.cuda.current_stream().cuda_stream
    fr, n_sym = layout(dec, n_streams, n_items, payload_len)
    pay, off, ln = encode_inputs(torch, len(fr), payload_len, 100 + sf)
    shifts = torch.empty((max(len(fr), 1), n_sym), dtype=torch.int32, device="cuda")
    dec.tx_encode(pay, off, ln, shifts, n_sym, st)
    up = torch.from_numpy(tx.base_upchirp(sf).astype(np.complex64)).cuda()
    out = torch.empty((n_streams, n_items), dtype=torch.complex64, device="cuda")
    k = min(32, n_streams)
    base = torch.empty((k, n_items), dtype=torch.complex64, device="cuda")
    dec.tx_frames(fr[fr["stream"] < k], shifts, n_sym, k, n_items, base, up_table_dev=up, cuda_stream=st)
    nbytes = n_streams * n_items * 8
    ppm = np.where(np.arange(len(fr)) % 2 == 0, 20.0, -20.0).astype(np.float32)
    res = {"sf": sf, "streams": n_streams, "items": n_items, "frames": len(fr), "bytes_written": nbytes}
    for sigma in (0.0, float(np.sqrt(10 ** -3.5 / 2))):
        tag = "noise" if sigma else "clean"
        run_f = lambda: dec.tx_frames(fr, shifts, n_sym, n_streams, n_items, out, noise_sigma=sigma, seed=1, up_table_dev=up, cuda_stream=st)
        run_e = lambda: dec.tx_expand(base, k, n_items, n_streams, out, noise_sigma=sigma, seed=1, cuda_stream=st)
        # every frame from a transmitter whose clock is off by +-20 ppm (tx_frames_sfo: the phase law at fractional times)
        run_d = lambda: dec.tx_frames(fr, shifts, n_sym, n_streams, n_items, out, noise_sigma=sigma, seed=1, up_table_dev=up,
                                      cuda_stream=st, sfo_ppm=ppm)
        tf, te, td = [], [], []
        for _ in range(2):                                 # alternate the kernels
            tf.append(timed(torch, run_f, args.iters, args.warmup))
            te.append(timed(torch, run_e, args.iters, args.warmup))
            td.append(timed(torch, run_d, args.iters, args.warmup))
        tf, te, td = min(tf), min(te), min(td)
        res[tag] = {"tx_frames_s": tf, "tx_frames_gbs": nbytes / tf / 1e9, "tx_frames_share_of_hbm": nbytes / tf / 1e9 / HBM_GBS,
                    "tx_frames_sfo20_s": td, "tx_frames_sfo20_gbs": nbytes / td / 1e9,
                    "tx_expand_s": te, "tx_expand_gbs": nbytes / te / 1e9, "tx_expand_share_of_hbm": nbytes / te / 1e9 / HBM_GBS}
    t_enc = timed(torch, lambda: dec.tx_encode(pay, off, ln, shifts, n_sym, st), args.iters, args.warmup)
    res["encode_plus_frames_frames_per_s"] = len(fr) / (t_enc + res["noise"]["tx_frames_s"])
    del out, base
    dec.close()
    torch.cuda.empty_cache()
    return res


def bench_host(torch, n_frames, args):
    """tx.encode_frame + modulate_frame + channel per frame on the host (each stream its own payloads), then H2D."""
    from gr_lora_b200 import tx
    sf, sps = 7, 8 << 7
    rng = np.random.default_rng(7)
    pays = [bytes(rng.integers(0, 256, 12, dtype=np.uint8)) for _ in range(n_frames)]
    per_row = 4
    n_items = 256 * sps
    t0 = time.perf_counter()
    rows = []
    for r in range(0, n_frames, per_row):
        frames = [tx.modulate_frame(tx.encode_frame(p, sf, 4, has_crc=False), sf) for p in pays[r: r + per_row]]
        x = tx.channel(frames, sf=sf, snr_db=35.0, seed=r, lead_symbols=2.5)
        row = np.zeros(n_items, np.complex64)
        row[: min(n_items, x.size)] = x[:n_items]
        rows.append(row)
    dev = torch.from_numpy(np.stack(rows)).cuda()
    torch.cuda.synchronize()
    t = time.perf_counter() - t0
    del dev
    return {"frames": n_frames, "rows": len(rows), "s": t, "frames_per_s": n_frames / t,
            "path": "tx.encode_frame + modulate_frame + channel (numpy, one process) + H2D"}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-frames", type=int, default=256)
    ap.add_argument("--e2e-streams", type=int, default=4096)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_tx.py needs a CUDA device")
    import gr_lora_b200 as G
    out = {"card": card(torch), "hbm_datasheet_gbs": HBM_GBS}
    out["encode"] = [bench_encode(torch, G, sf, 1 << 16, args) for sf in (7, 12)]
    out["e2e_shape"] = bench_shape(torch, G, 7, args.e2e_streams, 256 * (8 << 7), args)
    out["config4_shape"] = [bench_shape(torch, G, sf, 64, 2_000_000, args, payload_len={7: 16, 8: 16, 9: 16, 10: 16, 11: 8, 12: 4}[sf])
                            for sf in range(7, 13)]
    out["host"] = bench_host(torch, args.host_frames, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
