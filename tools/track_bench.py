"""Throughput of the device cell tracker (lcs_track_*): 64 channels x 4 two-port cells, synthetic, 10 s of stream
pushed as 1 s pushes after a warm-up push.  Prints one JSON line: stream seconds per wall second (the real-time
multiple), the kernel time per push (CUDA events around each launch, lcs_track_timing_read), the whole push (a host
clock around lcs_track_push_cu8, which includes the host staging and the copy to the device), the cells' lock state at
the end (live, MIB failures 0) and the card name and power limit read in the same run.

Each channel's 1 s of synthetic stream is pushed again and again.  That is seamless for the tracker: 1 s is 100 frames,
a multiple of the 40 ms PBCH period, so the SFN alignment of the MIB windows carries on, and the carrier rotation at
f_true = 2000 Hz is a whole number of turns per second.  Only the sample-clock offset of f_true makes the frame start
step by 1.92e6 * 2000 / 739e6 = 0.005 samples at each repetition.

Usage: python tools/track_bench.py [--channels 64] [--cells 4] [--seconds 10]
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

FS = 1.92e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=64)
    ap.add_argument("--cells", type=int, default=4)
    ap.add_argument("--seconds", type=int, default=10)
    a = ap.parse_args()
    n = int(FS)
    rng = np.random.default_rng(1)
    # one second of synthetic stream per channel, pushed repeatedly (the tracker's state carries across pushes)
    fcs = 739e6 + 1e6 * np.arange(a.channels)
    base = []
    cells = []
    for ch in range(min(a.channels, 4)):
        ds = [dict(n_id_cell=int(i), n_ports=2, cp_type=1, n_rb_dl=25, phich_duration=1, phich_resource=3,
                   t0=float(rng.uniform(0, 19000)), sfn0=0) for i in rng.choice(504, size=a.cells, replace=False)]
        base.append(S.synth_cu8(n, ds, f_true=2000.0, fc=fcs[ch], snr_db=10, seed=ch))
        cells.append(ds)
    iq = np.stack([base[c % len(base)] for c in range(a.channels)])
    ctx = L.Context(0)
    tr = L.Tracker(ctx, fcs, 2000.0, max_cells=a.cells)
    for ch in range(a.channels):
        for d in cells[ch % len(base)]:
            c = L.new_cell(n_id_1=d["n_id_cell"] // 3, n_id_2=d["n_id_cell"] % 3, cp_type=1, n_ports=2, n_rb_dl=25,
                           phich_duration=1, phich_resource=3)
            tr.add_cell(ch, c, d["t0"] - 2)
    tr.push_cu8(iq)                                   # warm-up: module load, first allocation
    tr.timing_read()
    wall = time.perf_counter()
    host = []
    for s in range(a.seconds):
        t0 = time.perf_counter()
        tr.push_cu8(iq)
        host.append(time.perf_counter() - t0)
    wall = time.perf_counter() - wall
    kernel_ms, launches = tr.timing_read()
    res = [c for ch in range(a.channels) for c in tr.read(ch)]
    locked = sum(1 for c in res if not c["dropped"] and c["mib_decode_failures"] == 0 and c["mib_successes"] > 0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print(json.dumps({
        "workload": "%d channels x %d two-port cells, %d x 1 s pushes" % (a.channels, a.cells, a.seconds),
        "realtime_multiple": a.seconds / wall,
        "kernel_ms_per_push": kernel_ms / launches,
        "push_ms_mean": 1e3 * float(np.mean(host)),
        "push_ms_min": 1e3 * float(np.min(host)),
        "cells_locked_at_end": locked,
        "mib_attempts": int(sum(c["mib_attempts"] for c in res)),
        "mib_successes": int(sum(c["mib_successes"] for c in res)),
        "cells_dropped": sum(1 for c in res if c["dropped"]),
        "cells": a.channels * a.cells,
        "gpu": q[0] if q else "unknown",
    }))
    tr.close()
    ctx.close()


if __name__ == "__main__":
    main()
