"""The payload CRC and CRC-aided list decoding of the dechirp receiver (lora_b200_rx_params.crc_list).

  sensitivity: frames whose payload is the one sent and whose CRC checks, hard / soft / soft + list (K = 4, 8, 12), per SF at
               CR 4/5 and 4/8 and per SNR, --runs runs x --frames frames per point (one frame of --bytes bytes + CRC per
               stream); and the payloads reported OK or RECOVERED that were not sent, against (2^K - 1) / 2^16 x the frames
               whose CRC soft decisions alone leave failing
  timing:      the config-4 shape (--streams SF7 streams x 2 s at --snr dB) with crc_list = 0 and 8, the two alternating from
               call to call: call time (CUDA events, median of --reps), and in a separate profiled call the device time of
               every stage (torch.profiler), rs_crc_list_kernel's included

    python tools/bench_rx_crc.py --what timing --reps 5
    python tools/bench_rx_crc.py --what timing --snr -4 --reps 5
    python tools/bench_rx_crc.py --what sensitivity --sfs 7 10 12 --runs 3 --frames 96
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

from antenna_common import BW, SENSITIVITY, synth_antennas  # noqa: E402

CRC_OK, CRC_BAD, CRC_RECOVERED = 1, 2, 3


def n_items_for(G, sf, n_bytes, rr, cr):
    sps = 8 << sf
    return int((12 + G.tx_frame_symbols(n_bytes, sf, cr, False, True, rr)) * sps + sps // 4 + 9 * sps) // 8 * 8


def sensitivity(torch, G, sfs, runs, n_frames, n_bytes, offsets):
    from gr_lora_b200 import tx
    out = []
    for sf in sfs:
        rr = sf >= 11
        for cr in (1, 4):
            n = n_items_for(G, sf, n_bytes + 2, rr, cr)
            for off in offsets:
                snr = SENSITIVITY[sf] + off
                tot = {}
                for run in range(runs):
                    seed = 10000 * sf + 1000 * cr + 100 * run + int(10 * (off + 10))
                    rng = np.random.default_rng(seed)
                    pays = []
                    for _ in range(n_frames):
                        p = bytes(rng.integers(0, 256, n_bytes, dtype=np.uint8))
                        pays.append([p + tx.crc_bytes(p, cr)])
                    x, placed = synth_antennas(torch, sf, 8, pays, n, snr, np.ones((n_frames, 1)), seed, rr=rr, cr=cr)
                    sent = {(s, p) for s, _, p in placed}
                    dec = G.decoder(8 * BW, BW, sf, False, cr, True, rr, quiet=True, n_streams=n_frames, max_items_per_call=n)
                    for mode, soft, k in (("hard", False, 0), ("soft", True, 0), ("list4", True, 4), ("list8", True, 8),
                                          ("list12", True, 12)):
                        _, frames, _ = dec.receive(x, n_items=n, soft=soft, crc_list=k)
                        st = dec.frames_crc_last()
                        got = [((int(f["stream"]), bytes(f["bytes"][18: int(f["len"])])), int(s)) for f, s in zip(frames, st)]
                        good = {g for g, s in got if s in (CRC_OK, CRC_RECOVERED)}
                        t = tot.setdefault(mode, dict(decoded=0, wrong_accepted=0, recovered=0))
                        t["decoded"] += len(good & sent)
                        t["wrong_accepted"] += len(good - sent)
                        t["recovered"] += sum(1 for _, s in got if s == CRC_RECOVERED)
                    dec.close()
                sent_n = runs * n_frames
                failing = sent_n - tot["soft"]["decoded"]
                for mode, t in tot.items():
                    rec = dict(sf=sf, cr=f"4/{4 + cr}", snr_db=snr, mode=mode, sent=sent_n, **t)
                    if mode.startswith("list"):
                        k = int(mode[4:])
                        rec["false_accept_bound"] = round((2 ** k - 1) / 2 ** 16 * failing, 4)
                    print(json.dumps(rec), flush=True)
                    out.append(rec)
    return out


def timing(torch, G, n_streams, reps, snr):
    sf, fs, n = 7, 1e6, 1953 * 1024                         # 2 s, whole windows: no staging copy
    from gr_lora_b200 import tx
    rng = np.random.default_rng(4)
    sps = 8 << sf
    per = int((12 + G.tx_frame_symbols(12, sf, 4, False, True, False)) * sps + 4 * sps)
    n_pay = max(1, (n - 3 * sps) // per - 1)
    pays = []
    for _ in range(n_streams):
        row = []
        for _ in range(n_pay):
            p = bytes(rng.integers(0, 256, 10, dtype=np.uint8))
            row.append(p + tx.crc_bytes(p, 4))
        pays.append(row)
    x, placed = synth_antennas(torch, sf, 8, pays, n, snr, np.ones((n_streams, 1)), 50)
    sent = {(s, p) for s, _, p in placed}
    decs = {k: G.decoder(fs, BW, sf, False, 4, True, False, quiet=True, n_streams=n_streams, max_items_per_call=n,
                         max_frames_per_call=n_pay + 2) for k in (0, 8)}
    for k, d in decs.items():
        d.receive(x, n_items=n, soft=True, crc_list=k)          # warm-up
    times = {k: [] for k in decs}
    res = {}
    for _ in range(reps):
        for k, d in decs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            _, frames, _ = d.receive(x, n_items=n, soft=True, crc_list=k)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
            st = d.frames_crc_last()
            good = {(int(f["stream"]), bytes(f["bytes"][18: int(f["len"])])) for f, s in zip(frames, st) if s in (CRC_OK, CRC_RECOVERED)}
            res[k] = dict(published=len(frames), crc_correct=len(good & sent), bad=int(np.sum(st == CRC_BAD)),
                          recovered=int(np.sum(st == CRC_RECOVERED)))
    from torch.profiler import ProfilerActivity, profile
    stages = {}
    for k, d in decs.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            d.receive(x, n_items=n, soft=True, crc_list=k)
            torch.cuda.synchronize()
        agg = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA":
                name = ev.name.split("<")[0].split("(")[0].replace("void ", "").replace("lb::", "")
                agg[name] = agg.get(name, 0.0) + ev.device_time_total / 1e3
        stages[k] = {name: round(v, 3) for name, v in sorted(agg.items(), key=lambda kv: -kv[1])}
    for k in decs:
        rec = dict(crc_list=k, streams=n_streams, snr_db=snr, call_ms_median=float(np.median(times[k])),
                   call_ms=[round(t, 2) for t in times[k]], frames_sent=len(sent), **res[k], stage_ms=stages[k])
        print(json.dumps(rec), flush=True)
    for d in decs.values():
        d.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--what", choices=["timing", "sensitivity"], default="timing")
    ap.add_argument("--streams", type=int, default=384)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--snr", type=float, default=1.0, help="timing: SNR in 125 kHz")
    ap.add_argument("--sfs", type=int, nargs="+", default=[7, 10, 12])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--frames", type=int, default=96)
    ap.add_argument("--bytes", type=int, default=16, help="payload bytes per frame, without the CRC")
    ap.add_argument("--offsets", type=float, nargs="+", default=[-2.5, -1.5], help="SNR relative to the sensitivity point")
    a = ap.parse_args()
    import torch
    import gr_lora_b200 as G
    print(json.dumps(dict(device=torch.cuda.get_device_name(0))), flush=True)
    if a.what == "timing":
        timing(torch, G, a.streams, a.reps, a.snr)
    else:
        sensitivity(torch, G, a.sfs, a.runs, a.frames, a.bytes, a.offsets)


if __name__ == "__main__":
    main()
