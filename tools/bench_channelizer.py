#!/usr/bin/env python3
"""Throughput of the GPU channelizer (SURVEY.md 8f N1): wideband 10 MS/s -> 64 channels at 1 MS/s
(the front half of BASELINE.json configs[3]) and the reference's own use (1 MS/s, one channel, D = 1).
Prints one JSON object.  Algorithmic work per launch: 8*ntaps flop per (channel, output) and
8*n_in + 8*C*n_out bytes."""
import json
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def run(torch, G, fs, decim, n_channels, seconds):
    center = 868e6
    offs = (np.arange(n_channels) - (n_channels - 1) / 2.0) * (fs / (n_channels + 1))
    ch = G.channelizer(fs, center, [center + f for f in offs], 125000, decim)
    n_in = int(seconds * fs) // decim * decim
    x = torch.randn(n_in, dtype=torch.complex64, device="cuda")
    n_out = n_in // decim
    out = torch.empty((n_channels, n_out), dtype=torch.complex64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for _ in range(2):
        ch.work_dev(x, n_in, out, n_out, st)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 5
    e0.record()
    for _ in range(reps):
        ch.work_dev(x, n_in, out, n_out, st)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    flop = 8.0 * ch.ntaps * n_channels * n_out
    byts = 8.0 * n_in + 8.0 * n_channels * n_out
    r = {"fs": fs, "decimation": decim, "channels": n_channels, "ntaps": ch.ntaps, "n_in": n_in, "ms": ms,
         "input_msamples_per_s": n_in / ms / 1e3, "realtime_factor": (n_in / fs) / (ms * 1e-3),
         "tflops_fp32": flop / ms / 1e9, "gbs_algorithmic": byts / ms / 1e6}
    ch.close()
    return r


def main():
    import torch
    import gr_lora_b200 as G
    out = {"wideband_10MSps_64ch": run(torch, G, 10e6, 10, 64, 1.0),
           "reference_use_1MSps_1ch": run(torch, G, 1e6, 1, 1, 4.0),
           "note": "fp32 CUDA-core FIR bank; H100 SXM data-sheet fp32 peak 67 TFLOP/s"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
