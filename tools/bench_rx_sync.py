"""Measure the dechirp-synchronised receiver (lora_b200_receive) on the GPU and print one JSON line:
  * sensitivity: per SF, the share of frames decoded byte-exact at SNRs around its sensitivity point (CR 4/8, explicit header,
    random CFO within +-0.9 BW/4, random starts; --runs captures of 96 frames per point, or 32 with --quick), next to the
    genie-timing symbol error rate of K1 at the same SNR;
  * stages: device time per stage of a call (torch.profiler; median, min and max over --repeats profiled calls): screen (the
    K1 launches before detection), detect, sync, assemble + K1 (data windows), integer chain (header, frame records, K8);
  * realtime: 384 SF7 streams x 2 s (1 MS/s) with frames, wall time per call (median of repeats) and the real-time factor.
With --ppm P every frame comes from a crystal off by a per-frame offset uniform in +-P ppm at 868.1 MHz, which sets both its
CFO (ppm * 868.1 Hz, in place of the random CFO) and its clock (tx_frames_sfo); every sensitivity point and the real-time
shape are then measured both with carrier_hz = 868.1e6 (the clock offset follows each frame's CFO) and without.  P above
about 36 puts the CFO beyond BW/4.
With --soft every capture is decoded with hard and with soft decisions (lora_b200_rx_params.soft), alternating; each SF's
points gain two SNRs 1.5 and 3 dB below its lowest, and the stages gain the soft-decision kernels (LLR demodulator time is
part of assemble + K1).
With --osr 2 the sensitivity curve is measured at fs/bw = 2 (250 kS/s, the generic K1 and LLR kernels at D = 2), and the
real-time shape is decoded at fs/bw = 8 and at fs/bw = 2 (the same payloads, CFOs and layout, synthesised at each rate),
alternating call by call; its results carry the suffix _osr8 / _osr2.  --osr 16 and --osr 32 do the same at 2 MS/s and 4 MS/s
(the real-time shape has 192 streams at fs/bw = 32: about 12 GB of cf32 either way), and --all-rates times the shape at
fs/bw = 2, 8, 16 and 32 in one run.
With --cfo-range LO HI every frame's CFO is uniform in +-[LO, HI] BW (a random sign), and every capture is decoded with the
coarse-offset search (lora_b200_rx_params.wide_cfo, max_cfo_hz = --max-cfo, default HI, in BW) and without it, alternating;
results carry the suffix _wide / _off.
Usage: python tools/bench_rx_sync.py [--quick] [--ppm P | --soft | --cfo-range LO HI [--max-cfo M]] [--osr 2|16|32] [--all-rates]"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

BW, FS = 125000, 1e6
CARRIER = 868.1e6
POINTS = {7: (-5.0, -3.5, -2.0, 0.0), 8: (-8.0, -6.5, -5.0, -3.0), 9: (-10.5, -9.0, -7.5, -5.5), 10: (-13.0, -11.5, -10.0, -8.0),
          11: (-15.5, -14.0, -12.5, -10.5), 12: (-18.0, -16.5, -15.0, -13.0)}


def sigma_for(snr_db):
    return float(np.sqrt(10 ** (-(snr_db - 10 * np.log10(FS / BW)) / 10) / 2))


def set_osr(osr):
    """fs = osr * BW for every capture and decoder made after the call"""
    global FS
    FS = float(osr * BW)


def dec(sf, rr, **kw):
    import gr_lora_b200 as G
    if FS == 8 * BW:                                 # (the stream state machine's FFT demodulator exists at fs/bw = 8 only)
        kw["demod"] = "fft"
    return G.decoder(FS, BW, sf, False, 4, True, rr, quiet=True, **kw)


CFO_RANGE = None                                     # (lo, hi) in BW: --cfo-range


def capture(torch, sf, n_streams, per_stream, snr, seed, n_items=None, plen=10, ppm=0.0):
    import gr_lora_b200 as G
    from gr_lora_b200 import tx
    rr = sf >= 11
    rng = np.random.default_rng(seed)
    sps = int(FS / BW) << sf
    flen = (12 + G.tx_frame_symbols(plen, sf, 4, False, True, rr)) * sps + sps // 4
    if n_items is None:
        n_items = per_stream * (flen + 5 * sps) + 8 * sps
    pays = [[bytes(rng.integers(0, 256, plen, dtype=np.uint8)) for _ in range(per_stream)] for _ in range(n_streams)]
    cfo = [[float(rng.uniform(-0.9, 0.9) * BW / 4) for _ in p] for p in pays]
    if CFO_RANGE:
        lo, hi = CFO_RANGE
        cfo = [[float(rng.choice((-1.0, 1.0)) * rng.uniform(lo, hi) * BW) for _ in p] for p in pays]
    kw = {}
    if ppm:                                          # a crystal off by e ppm: CFO e * 868.1 Hz, clock off by e ppm
        sfo = [[float(rng.uniform(-ppm, ppm)) for _ in p] for p in pays]
        cfo = [[e * CARRIER * 1e-6 for e in es] for es in sfo]
        kw["sfo_ppm"] = sfo
    gen = dec(sf, rr)
    up = torch.from_numpy(tx.base_upchirp(sf, BW, FS).astype(np.complex64)).cuda()
    out, placed = gen.synth_streams(pays, n_items, lead_symbols=float(rng.uniform(1, 3)), gap_symbols=4.3, cfo_hz=cfo,
                                    noise_sigma=sigma_for(snr), seed=seed, up_table_dev=up, **kw)
    torch.cuda.synchronize()
    return out, placed, n_items


def decoded(frames, placed):
    got = {}
    for r in frames:
        got.setdefault(int(r["stream"]), []).append(bytes(r["bytes"][18: int(r["len"])]))
    return sum(1 for s, _, p in placed if p in got.get(s, []))


def genie_ser(torch, sf, snr, n=2048, seed=1):
    """K1 on aligned symbols with known timing and no CFO (the demodulator's own limit)."""
    from gr_lora_b200 import tx
    d = dec(sf, False)
    rng = np.random.default_rng(seed)
    vals = torch.from_numpy(rng.integers(0, 1 << sf, n).astype(np.int32)).cuda()
    x = torch.empty(n * (int(FS / BW) << sf), dtype=torch.complex64, device="cuda")
    up = torch.from_numpy(tx.base_upchirp(sf, BW, FS).astype(np.complex64)).cuda()
    d.tx_symbols(vals, x, n, noise_sigma=sigma_for(snr), seed=seed, up_table_dev=up)
    bins = torch.empty(n, dtype=torch.int32, device="cuda")
    d.demod_fft(x, n, bins)
    torch.cuda.synchronize()
    return float((bins != vals).float().mean().item())


def stages(torch, rx, out, n_items, **kw):
    from torch.profiler import ProfilerActivity, profile
    rx.receive(out, n_items=n_items, **kw)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rx.receive(out, n_items=n_items, **kw)
        torch.cuda.synchronize()
    ev = sorted([e for e in prof.events() if e.device_type.name == "CUDA"], key=lambda e: e.time_range.start)
    t = {"screen": 0.0, "detect": 0.0, "sync": 0.0, "assemble_k1": 0.0, "soft_decisions": 0.0, "integer_chain": 0.0, "copies": 0.0}
    seen_detect = False
    for e in ev:
        name, us = e.name, e.time_range.elapsed_us()
        if "rs_detect" in name:
            t["detect"] += us
            seen_detect = True
        elif "rs_sync" in name:
            t["sync"] += us
        elif "rs_soft" in name:
            t["soft_decisions"] += us
        elif "rs_header" in name or "rs_frame" in name or "k8_frames" in name:
            t["integer_chain"] += us
        elif "Memcpy" in name or "Memset" in name or "memcpy" in name or "memset" in name:
            t["copies"] += us
        elif not seen_detect:
            t["screen"] += us
        else:
            t["assemble_k1"] += us
    return {k: round(v / 1e3, 3) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="fewer frames per point")
    ap.add_argument("--repeats", type=int, default=5, help="timed calls of the real-time shape, and profiled calls")
    ap.add_argument("--runs", type=int, default=3, help="independent captures (seeds) per sensitivity point")
    ap.add_argument("--ppm", type=float, default=0.0, help="per-frame crystal offset uniform in +-PPM at 868.1 MHz (0: none)")
    ap.add_argument("--soft", action="store_true", help="decode every capture with hard and with soft decisions, alternating, "
                    "at two more SNRs 1.5 and 3 dB below each SF's lowest point")
    ap.add_argument("--osr", type=int, default=8, choices=(8, 2, 16, 32), help="fs/bw of the sensitivity curve; another "
                    "than 8 also times the real-time shape at fs/bw = 8 against it")
    ap.add_argument("--all-rates", action="store_true", help="time the real-time shape at fs/bw = 2, 8, 16 and 32, alternating "
                    "(192 streams at 32, 384 below)")
    ap.add_argument("--cfo-range", type=float, nargs=2, metavar=("LO", "HI"), help="CFO uniform in +-[LO, HI] BW; decode with "
                    "and without wide_cfo, alternating")
    ap.add_argument("--max-cfo", type=float, default=None, help="max_cfo_hz of the wide_cfo decodes, in BW (default: HI)")
    a = ap.parse_args()
    set_osr(a.osr)
    global CFO_RANGE
    CFO_RANGE = tuple(a.cfo_range) if a.cfo_range else None
    if CFO_RANGE and (a.soft or a.ppm):
        raise SystemExit("--cfo-range compares two modes of its own: give it without --soft and --ppm")
    if a.soft and a.ppm:
        raise SystemExit("--soft and --ppm each compare two modes: give one of them")
    if abs(a.ppm) * CARRIER * 1e-6 > BW / 4:
        raise SystemExit(f"--ppm {a.ppm}: a CFO of {a.ppm * CARRIER * 1e-6:.0f} Hz is beyond BW/4")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_rx_sync.py needs a CUDA device")
    res = {"gpu": torch.cuda.get_device_name(0)}
    try:
        import subprocess
        res["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        res["power_limit_w"] = "unknown"
    ns = 32 if a.quick else 96
    res["ppm"] = a.ppm
    # with --ppm, every measurement with the clock offset following the CFO ("tracked") and without ("fixed")
    # with --soft, every measurement with hard and with soft decisions
    modes = ({"tracked": dict(carrier_hz=CARRIER), "fixed": dict(carrier_hz=0.0)} if a.ppm else
             {"hard": dict(soft=False), "soft": dict(soft=True)} if a.soft else
             {"wide": dict(wide_cfo=True, max_cfo_hz=(a.max_cfo or CFO_RANGE[1]) * BW), "off": {}} if CFO_RANGE else {"": {}})
    if CFO_RANGE:
        res["cfo_range_bw"], res["max_cfo_bw"] = list(CFO_RANGE), a.max_cfo or CFO_RANGE[1]
    res["soft"] = a.soft
    if a.osr != 8:
        res["osr"] = a.osr
    curve = {}
    for sf, pts in (POINTS.items() if a.runs > 0 else ()):
        rr = sf >= 11
        row = []
        if a.soft:
            pts = list(pts) + [min(pts) - 1.5, min(pts) - 3.0]
        for snr in pts:
            oks, n = {m: [] for m in modes}, 0
            for r in range(a.runs):
                out, placed, n_items = capture(torch, sf, ns, 1, snr, seed=sf * 100 + int(snr * 10) % 97 + 7919 * r, ppm=a.ppm)
                rx = dec(sf, rr, n_streams=ns, max_items_per_call=n_items)
                for m, kw in modes.items():
                    _, frames, _ = rx.receive(out, n_items=n_items, **kw)
                    oks[m].append(decoded(frames, placed))
                n = len(placed)
                rx.close()
                del out
            pt = {"snr_db": snr, "frames_per_run": n}
            for m in modes:
                pt["ok_per_run" + (m and "_" + m)] = oks[m]
                pt["frames_ok" + (m and "_" + m)] = sum(oks[m]) / (n * a.runs)
            pt.update({"genie_ser": genie_ser(torch, sf, snr), "genie_symbols": 2048})
            row.append(pt)
        curve[f"sf{sf}"] = row
    res["sensitivity"] = curve
    # config-4 shape: 384 SF7 streams x 2 s, frames 3 dB above the sensitivity point; with --osr 2 the same frames at both
    # rates, the calls alternating between them
    rates = [2, 8, 16, 32] if a.all_rates else [8, a.osr] if a.osr != 8 else [8]
    sfx = (lambda d: f"_osr{d}") if len(rates) > 1 else (lambda d: "")
    n_str = {d: 192 if d == 32 else 384 for d in rates}       # about 12 GB of cf32 at fs/bw = 16 and 32
    shape = {}
    for d in rates:
        set_osr(d)
        out, placed, n_items = capture(torch, 7, n_str[d], 40, 1.0, seed=4, n_items=int(2 * FS), ppm=a.ppm)
        rx = dec(7, False, n_streams=n_str[d], max_items_per_call=n_items, max_frames_per_call=64)
        shape[d] = (out, placed, n_items, rx, FS)
        for m, kw in modes.items():
            runs = [stages(torch, rx, out, n_items, **kw) for _ in range(a.repeats)]
            res["stages_ms" + (m and "_" + m) + sfx(d)] = {
                k: {"median": float(np.median([r[k] for r in runs])), "min": min(r[k] for r in runs), "max": max(r[k] for r in runs)}
                for k in runs[0]}
    times = {(m, d): [] for m in modes for d in rates}
    for _ in range(a.repeats):                       # the modes (and rates) alternate, so that all see the same conditions
        for d in rates:
            out, placed, n_items, rx, fs = shape[d]
            for m, kw in modes.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                _, frames, _ = rx.receive(out, n_items=n_items, **kw)
                times[m, d].append(time.perf_counter() - t0)
                med = float(np.median(times[m, d]))
                res["realtime" + (m and "_" + m) + sfx(d)] = {
                    "streams": n_str[d], "seconds_per_stream": n_items / fs, "frames_placed": len(placed),
                    "frames_decoded": decoded(frames, placed), "call_s_median": round(med, 4), "call_s_min": round(min(times[m, d]), 4),
                    "call_s_max": round(max(times[m, d]), 4), "realtime_factor": round(n_str[d] * n_items / fs / med, 1)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
