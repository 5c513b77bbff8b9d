"""The dechirp receiver with 1, 2 and 4 antennas per receiver (lora_b200_receive_antennas).

  sensitivity: frames decoded per SF and per-antenna SNR, in white noise (independent noise per antenna, random relative
               phase) and in Rayleigh fading (an independent complex-Gaussian gain of mean power 1 per frame and antenna),
               hard and soft, --runs runs x --frames frames per point
  timing:      the config-4 shape (--streams SF7 receivers x 2 s at +1 dB per antenna) with M = 1, 2 and 4 antennas per
               receiver, calls alternating between the M values: call time (CUDA events) and stage device times
               (torch.profiler)

    python tools/bench_rx_diversity.py --what timing --reps 5
    python tools/bench_rx_diversity.py --what sensitivity --sfs 7 9 12 --runs 3 --frames 96
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from antenna_common import BW, SENSITIVITY, rayleigh, synth_antennas  # noqa: E402


def n_items_for(G, sf, n_bytes, rr):
    sps = 8 << sf
    return int((12 + G.tx_frame_symbols(n_bytes, sf, 4, False, True, rr)) * sps + sps // 4 + 9 * sps) // 8 * 8


def sensitivity(torch, G, sfs, runs, n_frames, offsets):
    out = []
    for sf in sfs:
        rr = sf >= 11
        n = n_items_for(G, sf, 10, rr)
        for fading in (False, True):
            for off in offsets:
                snr = SENSITIVITY[sf] + off
                for m in (1, 2, 4):
                    for soft in (False, True):
                        ok = 0
                        for run in range(runs):
                            seed = 1000 * sf + 100 * run + 10 * m + int(fading)
                            rng = np.random.default_rng(seed)
                            gains = rayleigh(rng, (n_frames, m)) if fading else np.exp(2j * np.pi * rng.uniform(size=(n_frames, m)))
                            pays = [[bytes(rng.integers(0, 256, 10, dtype=np.uint8))] for _ in range(n_frames)]
                            x, placed = synth_antennas(torch, sf, 8, pays, n, snr, gains, seed, rr=rr)
                            rx = G.decoder(8 * BW, BW, sf, False, 4, True, rr, quiet=True, n_streams=n_frames * m, max_items_per_call=n)
                            _, frames, _ = rx.receive(x, n_items=n, soft=soft, antennas=m)
                            sent = {(s, p) for s, _, p in placed}
                            ok += len({(int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in frames} & sent)
                            rx.close()
                        rec = dict(sf=sf, channel="rayleigh" if fading else "white", snr_db=snr, antennas=m, soft=soft,
                                   decoded=ok, sent=runs * n_frames)
                        print(json.dumps(rec), flush=True)
                        out.append(rec)
    return out


def timing(torch, G, n_streams, reps):
    sf, fs, n = 7, 1e6, 1953 * 1024                         # 2 s, whole windows: no staging copy
    rng = np.random.default_rng(4)
    sps = 8 << sf
    per = int((12 + G.tx_frame_symbols(10, sf, 4, False, True, False)) * sps + 4 * sps)
    n_pay = max(1, (n - 3 * sps) // per - 1)
    # one capture of n_streams receivers x 4 antennas; M = 2 and M = 1 take the first antennas of each receiver (copies)
    pays = [[bytes(rng.integers(0, 256, 10, dtype=np.uint8)) for _ in range(n_pay)] for _ in range(n_streams)]
    gains = np.exp(2j * np.pi * rng.uniform(size=(n_streams, 4)))
    x4, placed = synth_antennas(torch, sf, 8, pays, n, 1.0, gains, 50)
    sent = {(s, p) for s, _, p in placed}
    caps = {4: x4}
    for m in (2, 1):
        caps[m] = x4.view(n_streams, 4, n)[:, :m, :].reshape(n_streams * m, n).contiguous()
    torch.cuda.synchronize()                          # (receive reads device input on its own stream)
    caps = {m: (caps[m], sent) for m in (1, 2, 4)}
    decs = {}
    for m in caps:
        decs[m] = G.decoder(fs, BW, sf, False, 4, True, False, quiet=True, n_streams=n_streams * m, max_items_per_call=n,
                            max_frames_per_call=n_pay + 2)
        decs[m].receive(caps[m][0], n_items=n, antennas=m)                  # warm-up
    times = {m: [] for m in caps}
    decoded = {}
    for _ in range(reps):
        for m in caps:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            _, frames, _ = decs[m].receive(caps[m][0], n_items=n, antennas=m)
            e1.record()
            torch.cuda.synchronize()
            times[m].append(e0.elapsed_time(e1))
            decoded[m] = len({(int(r["stream"]), bytes(r["bytes"][18: int(r["len"])])) for r in frames} & caps[m][1])
    stages = {}
    from torch.profiler import ProfilerActivity, profile
    for m in caps:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            decs[m].receive(caps[m][0], n_items=n, antennas=m)
            torch.cuda.synchronize()
        agg = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA":
                name = ev.name.split("<")[0].split("(")[0].replace("void ", "").replace("lb::", "")
                agg[name] = agg.get(name, 0.0) + ev.device_time_total / 1e3
        stages[m] = {k: round(v, 3) for k, v in sorted(agg.items(), key=lambda kv: -kv[1])}
    for m in caps:
        rec = dict(antennas=m, receivers=n_streams, rows=n_streams * m, call_ms_median=float(np.median(times[m])),
                   call_ms=[round(t, 2) for t in times[m]], frames_decoded=decoded[m], frames_sent=len(caps[m][1]),
                   stage_ms=stages[m])
        print(json.dumps(rec), flush=True)
    for d in decs.values():
        d.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--what", choices=["timing", "sensitivity"], default="timing")
    ap.add_argument("--streams", type=int, default=384)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sfs", type=int, nargs="+", default=list(range(7, 13)))
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--frames", type=int, default=96)
    ap.add_argument("--offsets", type=float, nargs="+", default=[-3.0, 0.0, 3.0], help="per-antenna SNR relative to the sensitivity point")
    a = ap.parse_args()
    import torch
    import gr_lora_b200 as G
    print(json.dumps(dict(device=torch.cuda.get_device_name(0))), flush=True)
    if a.what == "timing":
        timing(torch, G, a.streams, a.reps)
    else:
        sensitivity(torch, G, a.sfs, a.runs, a.frames, a.offsets)


if __name__ == "__main__":
    main()
