"""Throughput of the Welch spectrum (lcs_psd_*, DESIGN.md section 4.8) on wideband recordings.

For each configuration (default 30.72 Msps ci16, 61.44 Msps ci16 and 122.88 Msps cs8, each at N = 4096 and 65 536) a
synthetic recording of 80 ms (complex noise and tones) is pushed from host memory --reps times as one continuing stream,
after a warm-up push.  One JSON line per configuration reports:
  - device time per second of recording (CUDA events around the kernels of each launch chunk, lcs_psd_timing_read) and the
    real-time factor (recording time / device time), with the host clock per push beside it;
  - the achieved FLOP rate, counting 5 N log2 N per segment;
  - the achieved byte rate, counting the input once plus the |X|^2 scratch written and read once (4 + 4 bytes per bin
    and segment); for N > 4096 the four-step intermediate (8 bytes written and read per point) is reported separately;
  - the lower bounds from the H100 SXM data sheet (3.35 TB/s HBM3, 67 TFLOP/s FP32) for those counts, and which is larger;
  - the card name, power limit and SM clocks, read in the same run.

Usage: python tools/psd_bench.py [--reps 10] [--config FS:FMT:N ...]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "lte-cell-scanner_b200"))

import lcs_b200 as L  # noqa: E402

HBM_BPS, FP32_FLOPS = 3.35e12, 67e12
CONFIGS = ["30.72e6:ci16:4096", "30.72e6:ci16:65536", "61.44e6:ci16:4096", "61.44e6:ci16:65536",
           "122.88e6:cs8:4096", "122.88e6:cs8:65536"]


def recording(fs, fmt, n, rng):
    """Complex noise at a tenth of full scale and three tones, in the format's [n][2] dtype."""
    m = np.arange(n)
    x = 0.1 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    for f, a in ((0.11 * fs, 0.3), (-0.27 * fs, 0.05), (0.4 * fs, 0.01)):
        x += a * np.exp(2j * np.pi * f / fs * m)
    if fmt == "cf32":
        return np.stack([x.real, x.imag], axis=1).astype(np.float32)
    scale, off, lo, hi, dt = {"ci16": (32768, 0, -32768, 32767, np.int16), "cs8": (128, 0, -128, 127, np.int8),
                              "cu8": (128, 127, 0, 255, np.uint8)}[fmt]
    return np.clip(np.round(np.stack([x.real, x.imag], axis=1) * scale) + off, lo, hi).astype(dt)


def run(fs, fmt, N, reps, ctx):
    n = int(round(0.08 * fs))                      # 80 ms per push
    iq = recording(fs, fmt, n, np.random.default_rng(N))
    sp = L.Spectrum(ctx, fs, fmt, N)
    sp.push(iq)                                    # warm-up
    sp.read()
    sp.timing_read()
    wall = []
    for _ in range(reps):
        t = time.perf_counter()
        sp.push(iq)
        wall.append(time.perf_counter() - t)
    ms, launches = sp.timing_read()
    _, _, S = sp.read()
    sp.close()
    seconds = reps * n / fs
    esz = {"ci16": 4, "cs8": 2, "cu8": 2, "cf32": 8}[fmt]
    flops = 5.0 * N * math.log2(N) * S
    bytes_ = reps * n * esz + S * N * 8.0
    extra = S * N * 16.0 if N > 4096 else 0.0
    t = ms / 1e3
    t_hbm, t_fp32 = bytes_ / HBM_BPS, flops / FP32_FLOPS
    return {
        "fs_in": fs, "format": fmt, "nfft": N, "segments": S, "launches": launches, "recording_s": seconds,
        "device_ms_per_s": ms / seconds, "real_time": seconds / t,
        "host_ms_per_push": 1e3 * float(np.median(wall)), "push_ms_recording": 80.0,
        "gflops": flops / t / 1e9, "gbytes_per_s": bytes_ / t / 1e9, "fourstep_gbytes_per_s": extra / t / 1e9,
        "bound_hbm_ms_per_s": 1e3 * t_hbm / seconds, "bound_fp32_ms_per_s": 1e3 * t_fp32 / seconds,
        "larger_bound": "hbm" if t_hbm > t_fp32 else "fp32",
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--config", nargs="*", default=CONFIGS, metavar="FS:FMT:N")
    a = ap.parse_args()
    ctx = L.Context(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    for spec in a.config:
        fs, fmt, N = spec.split(":")
        r = run(float(fs), fmt, int(N), a.reps, ctx)
        r["gpu"] = q[0] if q else "unknown"
        print(json.dumps(r), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
