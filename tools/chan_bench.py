"""Throughput of the wideband channelizer (lcs_chan_*) and of a wideband sweep built on it.

For each decimation D (default 16 and 32: 30.72 and 61.44 Msps) every 100 kHz raster channel in the band is channelized
from a synthetic ci16 recording (complex noise, 2 LTE carriers).  One JSON line per D reports:
  - the channelizer's device time per 80 ms of input (CUDA events around each launch, lcs_chan_timing_read), the input
    rate it sustains in Msamp/s and the real-time factor (80 ms / device time), over --reps pushes of 80 ms each into
    device memory (a continuing stream), and the host clock around each push;
  - a wideband sweep end to end (auto gain + channelize into device memory + lcs_sweep_search_cu8_device), against
    lcs_sweep_search_cu8 on the same channelized bytes from host memory;
  - the card name and power limit, read in the same run.

With --fs-in FS:FMT ... (e.g. 2.4e6:cu8 20e6:cs8 25e6:ci16) it first reports the same device time per 80 ms and
real-time factor for the resampling channelizer (lcs_chan_create_rational) at each rate and sample format, every raster
channel, then the --d runs as usual.

Usage: python tools/chan_bench.py [--d 16 32] [--reps 10] [--fs-in FS:FMT ...]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "lte-cell-scanner_b200"))
sys.path.insert(0, os.path.join(ROOT, "track_oracle"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import lcs_b200 as L  # noqa: E402
import lte_dl_synth as S  # noqa: E402

N_CAP = 153600
FC_IN = 739e6


def recording(D, n, rng):
    """Complex noise over the band plus two LTE carriers (one cell each) at about a third of the band either side."""
    fs_in = D * 1.92e6
    off = round(fs_in / 6 / 100e3) * 100e3
    cells = [dict(n_id_cell=277, n_ports=2, cp_type=1, n_rb_dl=25, phich_duration=1, phich_resource=3, t0=1234.0, sfn0=0),
             dict(n_id_cell=100, n_ports=1, cp_type=1, n_rb_dl=50, phich_duration=1, phich_resource=2, t0=9000.0, sfn0=0)]
    iq =S.synth_wide_ci16(n, fs_in, FC_IN, [(FC_IN - off, [cells[0]], 1.0), (FC_IN + off, [cells[1]], 1.0)], snr_db=10,
                           seed=D, scale=2048.0)
    return iq, [FC_IN - off, FC_IN + off]


def run(D, reps, ctx):
    import torch
    fs_in = D * 1.92e6
    edge = fs_in / 2 - 960e3
    fcs = FC_IN + 100e3 * np.arange(-int(edge // 100e3), int(edge // 100e3) + 1)
    h = L.chan_design_taps(fs_in)
    M = (h.size - 1) // 2
    n = 153599 * D + M + 1                  # 153 600 outputs per channel: one 80 ms capture buffer
    iq, carriers = recording(D, n, np.random.default_rng(D))
    n80 = N_CAP * D                         # 80 ms of input
    out = torch.empty((fcs.size, N_CAP + 1, 2), dtype=torch.uint8, device="cuda")
    # device time per 80 ms: a continuing stream, one 80 ms push after another
    ch = L.Channelizer(ctx, fs_in, FC_IN, fcs)
    ch.auto_gain(iq)
    ch.push_ci16_device(iq[:n80], out)      # warm-up
    ch.timing_read()
    host = []
    for r in range(reps):
        t0 = time.perf_counter()
        ch.push_ci16_device(iq[:n80], out)
        host.append(time.perf_counter() - t0)
    kernel_ms, launches = ch.timing_read()
    ch.close()
    per80 = kernel_ms / reps
    # wideband sweep end to end vs the host-input sweep on the same bytes
    sw = L.Sweep(ctx, N_CAP)
    f_set = L.f_search_set(fcs[0], 120.0)
    dev = torch.empty((fcs.size, N_CAP, 2), dtype=torch.uint8, device="cuda")
    e2e, e2e_cells = [], None
    for r in range(3):                      # the first call builds the sweep's plans and warms up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ch = L.Channelizer(ctx, fs_in, FC_IN, fcs)
        ch.auto_gain(iq)
        ch.push_ci16_device(iq, dev)
        per_ch = sw.search_cu8_device(dev, fcs, f_set, max_cells=16)
        e2e.append(time.perf_counter() - t0)
        ch.close()
        e2e_cells = sorted({c.n_id_cell() for c in L.dedup([c for cs in per_ch for c in cs])})
    host_bytes = dev.cpu().numpy()
    hs = []
    for r in range(3):
        t0 = time.perf_counter()
        sw.search_cu8(host_bytes, fcs, f_set, max_cells=16)
        hs.append(time.perf_counter() - t0)
    sw.close()
    return {
        "D": D, "fs_in_msps": fs_in / 1e6, "channels": int(fcs.size), "taps": int(h.size),
        "chan_kernel_ms_per_80ms": per80,
        "chan_launches_per_push": launches / reps,
        "chan_input_msamp_s": n80 / (per80 / 1e3) / 1e6,
        "chan_realtime_factor": 80.0 / per80,
        "chan_push_ms_mean": 1e3 * float(np.mean(host)),
        "wideband_sweep_e2e_ms": 1e3 * float(np.min(e2e[1:])),
        "wideband_sweep_cells": e2e_cells,
        "host_input_sweep_ms": 1e3 * float(np.min(hs[1:])),
        "carriers_mhz": [c / 1e6 for c in carriers],
    }


def run_rational(fs_in, fmt, reps, ctx):
    """Device time per 80 ms of a continuing stream of fs_in fmt samples, every raster channel, into device memory."""
    import torch
    edge = fs_in / 2 - 960e3
    fcs = FC_IN + 100e3 * np.arange(-int(edge // 100e3), int(edge // 100e3) + 1)
    up, down, h = L.chan_design_rational(fs_in)
    n80 = N_CAP * down // up                # 80 ms of input
    off = round(fs_in / 6 / 100e3) * 100e3
    cell = dict(n_id_cell=277, n_ports=2, cp_type=1, n_rb_dl=6, phich_duration=1, phich_resource=3, t0=1234.0, sfn0=0)
    iq16 = S.synth_wide_ci16(n80, fs_in, FC_IN, [(FC_IN - off, [cell], 1.0)], snr_db=10, seed=1, scale=2048.0)
    if fmt == "cf32":
        iq = (iq16 / 32768).astype(np.float32)
    elif fmt in ("cs8", "cu8"):
        v = np.clip(np.round(iq16 * (20 / np.sqrt(np.mean(iq16.astype(np.float64) ** 2)))), -127, 127)
        iq = v.astype(np.int8) if fmt == "cs8" else (v + 127).astype(np.uint8)
    else:
        iq = iq16
    out = torch.empty((fcs.size, N_CAP + 1, 2), dtype=torch.uint8, device="cuda")
    ch = L.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt=fmt)
    ch.auto_gain(iq)
    ch.push_device(iq, out)                 # warm-up
    ch.timing_read()
    host = []
    for r in range(reps):
        t0 = time.perf_counter()
        ch.push_device(iq, out)
        host.append(time.perf_counter() - t0)
    kernel_ms, launches = ch.timing_read()
    ch.close()
    per80 = kernel_ms / reps
    taps_per_out = -(-h.size // up)
    return {
        "fs_in_msps": fs_in / 1e6, "format": fmt, "up": up, "down": down, "channels": int(fcs.size), "taps": int(h.size),
        "taps_per_output": taps_per_out,
        "chan_kernel_ms_per_80ms": per80,
        "chan_launches_per_push": launches / reps,
        "chan_input_msamp_s": n80 / (per80 / 1e3) / 1e6,
        "chan_realtime_factor": 80.0 / per80,
        "chan_tflops": 8.0 * taps_per_out * N_CAP * fcs.size / (per80 / 1e3) / 1e12,
        "chan_push_ms_mean": 1e3 * float(np.mean(host)),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d", type=int, nargs="+", default=[16, 32])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--fs-in", nargs="*", default=[], metavar="FS:FMT")
    a = ap.parse_args()
    ctx = L.Context(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    for spec in a.fs_in:
        fs, fmt = spec.split(":")
        r = run_rational(float(fs), fmt, a.reps, ctx)
        r["gpu"] = q[0] if q else "unknown"
        print(json.dumps(r), flush=True)
    for D in a.d:
        r = run(D, a.reps, ctx)
        r["gpu"] = q[0] if q else "unknown"
        print(json.dumps(r), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
