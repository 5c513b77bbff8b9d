"""Measure the dechirp receiver's fine time of arrival (lora_b200_rx_params.fine_toa) on the GPU and print one JSON line:
  * accuracy: per SF, fs/bw and SNR (the SF's sensitivity point and 5, 10, 20 dB above), RMS and bias of toa - truth next to
    start - truth (rx_info.start, the integer start) over --frames frames, each at a random fractional delay (tx.modulate_frame
    delay=) with a random CFO within +-BW/8;
  * timing: the 384-stream SF7 x 2 s call (1 MS/s, frames 3 dB above the sensitivity point) with fine_toa on and off,
    alternating call by call, wall time per call (median, min, max of --repeats each), with the card's name and power limit
    read in the same run.
Usage: python tools/bench_rx_toa.py [--frames 96] [--sfs 7 10 12] [--repeats 10]"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

BW = 125e3
SENSITIVITY = {7: -2.0, 8: -5.0, 9: -7.5, 10: -10.0, 11: -12.5, 12: -15.0}


def rows(sf, osr, n_streams, per_stream, snr_db, rng):
    """n_streams rows of per_stream frames at fractional delays: (X [ns, n] complex64, truth per stream)."""
    from gr_lora_b200 import tx
    sps = osr << sf
    out, truths = [], []
    for _ in range(n_streams):
        parts, tr, pos = [], [], 0
        for _ in range(per_stream):
            delay, cfo = float(rng.uniform(0, 1)), float(rng.uniform(-1, 1) * (1 << sf) / 8)
            f = tx.modulate_frame(tx.encode_frame(b"fine toa", sf, 4, reduced_rate=sf > 10), sf, fs=osr * BW, delay=delay)
            lead = int(rng.integers(1, 4)) * sps
            s = np.zeros(lead + f.size + 3 * sps, np.complex128)
            s[lead: lead + f.size] = f
            parts.append(s * np.exp(2j * np.pi * cfo * (pos + np.arange(s.size)) / sps))
            tr.append(pos + lead + delay)
            pos += s.size
        out.append(np.concatenate(parts))
        truths.append(tr)
    n = max(r.size for r in out)
    X = np.stack([np.pad(r, (0, n - r.size)) for r in out])
    X += tx.awgn(X.size, snr_db - 10 * np.log10(osr), rng).reshape(X.shape)
    return X.astype(np.complex64), truths


def accuracy(sf, osr, snr_db, n_frames, seed):
    import gr_lora_b200 as G
    rng = np.random.default_rng(seed)
    ns = n_frames // 2
    X, truths = rows(sf, osr, ns, 2, snr_db, rng)
    dec = G.decoder(osr * BW, int(BW), sf, False, 4, True, sf > 10, quiet=True, n_streams=ns, max_items_per_call=X.shape[1])
    _, frames, info = dec.receive(X, fine_toa=True)
    toa = dec.rx_toa_last()
    et, es = [], []
    for k in range(len(frames)):
        tr = np.array(truths[int(info["stream"][k])])
        i = int(np.argmin(np.abs(tr - float(info["start"][k]))))
        if abs(tr[i] - float(info["start"][k])) < 4 * osr:
            et.append(toa[k] - tr[i])
            es.append(float(info["start"][k]) - tr[i])
    dec.close()
    et, es = np.array(et), np.array(es)
    r = lambda e: float(np.sqrt(np.mean(e * e))) if e.size else None
    return {"snr_db": snr_db, "frames": int(et.size), "of": 2 * ns, "toa_rms": r(et), "toa_bias": float(np.mean(et)) if et.size else None,
            "start_rms": r(es), "start_bias": float(np.mean(es)) if es.size else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=96, help="frames per accuracy point")
    ap.add_argument("--sfs", type=int, nargs="*", default=[7, 10, 12], help="SFs of the accuracy table (none: timing only)")
    ap.add_argument("--repeats", type=int, default=10, help="timed calls per mode")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_rx_toa.py needs a CUDA device")
    res = {"gpu": torch.cuda.get_device_name(0)}
    try:
        res["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        res["power_limit_w"] = "unknown"
    acc = {}
    for sf in a.sfs:
        for osr in (8, 2):
            acc[f"sf{sf}_osr{osr}"] = [accuracy(sf, osr, SENSITIVITY[sf] + d, a.frames, seed=sf * 100 + osr * 10 + k)
                                       for k, d in enumerate((0, 5, 10, 20))]
    res["accuracy_samples"] = acc
    # the 384-stream SF7 x 2 s call, fine_toa on and off alternating
    import bench_rx_sync as B
    out, placed, n_items = B.capture(torch, 7, 384, 40, SENSITIVITY[7] + 3.0, seed=4, n_items=2_000_000)
    rx = B.dec(7, False, n_streams=384, max_items_per_call=n_items, max_frames_per_call=64)
    times = {"on": [], "off": []}
    n_pub = {}
    for opt in (True, False):                      # warm-up of both modes
        _, f, _ = rx.receive(out, n_items=n_items, fine_toa=opt)
        n_pub["on" if opt else "off"] = len(f)
    for _ in range(a.repeats):
        for opt in (True, False):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rx.receive(out, n_items=n_items, fine_toa=opt)
            torch.cuda.synchronize()
            times["on" if opt else "off"].append(1e3 * (time.perf_counter() - t0))
    res["config4_frames_placed"] = len(placed)
    res["config4_frames_published"] = n_pub
    for m, t in times.items():
        res[f"config4_ms_{m}"] = {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
