"""Cost of the per-cell RSRP / RSRQ / SINR measurement (lcs_meas_cells, DESIGN.md section 4.9), next to the search's.

A few synthetic 80 ms cu8 capture buffers (each with one or two cells) are tiled to --channels channels in device memory.
The batched search (lcs_sweep_search_cu8_device) finds the cells of every channel; then all of them are measured, read in
place, in one call, --reps times after a warm-up call.  One JSON line reports:
  - the measurement's device time per cell (CUDA events around its two launches, lcs_meas_timing_read) and its host clock
    per call, beside the search's host clock per found cell (the search's call ends in a synchronise);
  - the bytes the two kernels need per cell (capture samples read, the 854 x 72 grid written, and the grid's CRS and
    RSSI resource elements read back), the achieved byte rate and the lower bound at 3.35 TB/s (H100 SXM data sheet);
  - the card name, power limit and SM clocks, read in the same run.

With --carrier it times the full-carrier measurement (lcs_carrier_cells, DESIGN.md section 4.10) instead: a synthetic
30.72 Msps ci16 recording with three 50-RB carriers of eight cells each, read in place from device memory, every cell
measured --copies times in one call.  One JSON line reports the device time per cell (lcs_carrier_timing_read), the bytes
the two kernels need per cell (the CRS windows' samples read, the 12 R grid columns of those windows written, and the CRS
pairs and RSSI columns read back), the achieved byte rate, the lower bound at 3.35 TB/s, and the card, read in the same
run.

With --cir it times the power delay profile (lcs_cir_cells, DESIGN.md section 4.11) on the same recording and cells in
the same way: one JSON line with the device time per cell (lcs_cir_timing_read), the complex multiply-adds of the delay
transform per cell (2 R CRS x 320 taps for every CRS symbol of every port), their FP64 rate, and the card, read in the
same run.

With --pcfich it times the CFI decoder (lcs_pcfich_cells, DESIGN.md section 4.12) on the same recording and cells in
the same way: one JSON line with the device time per cell (lcs_pcfich_timing_read), the launches and the card, read in
the same run.

With --pdcch it times the common-search-space DCI decoder (lcs_pdcch_cells, DESIGN.md section 4.13) on the same
recording and cells in the same way (PHICH duration normal, N_g = 1): one JSON line with the device time per cell
(lcs_pdcch_timing_read), the launches and the card, read in the same run.

With --sib1 it times the SIB1 decoder (lcs_sib1_cells, DESIGN.md section 4.14) on the same recording and cells in the
same way, each cell also sending a 1A-scheduled SIB1 of 328 bits on 6 PRBs in its SIB1 occasions (lte_dl_synth's "sib1"
key): one JSON line with the device time per cell (lcs_sib1_timing_read), the occasions decoded and passing CRC, the
launches and the card, and a split of the device time per cell by kernel from torch.profiler in a separate call.

Usage: python tools/meas_bench.py [--channels 64] [--reps 20]
       python tools/meas_bench.py --carrier [--copies 8] [--reps 20]
       python tools/meas_bench.py --cir [--copies 8] [--reps 20]
       python tools/meas_bench.py --pcfich [--copies 8] [--reps 20]
       python tools/meas_bench.py --sib1 [--copies 8] [--reps 20]
       python tools/meas_bench.py --pdcch [--copies 8] [--reps 20]
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

import lcs_b200 as L  # noqa: E402
import lte_dl_synth as S  # noqa: E402

HBM_BPS = 3.35e12
FC = 739e6


def cell(nid, ports, cp, t0, scale=1.0):
    g = [1.0, 0.8 * np.exp(0.7j), 0.9 * np.exp(-1.1j), 0.7 * np.exp(2.2j)]
    return dict(n_id_cell=nid, n_ports=ports, cp_type=cp, n_rb_dl=50, phich_duration=1, phich_resource=2, t0=t0, sfn0=7,
                gains=[scale * v for v in g])


BUFFERS = [[cell(137, 2, 1, 1234.0)], [cell(52, 4, 2, 7000.0)], [cell(277, 2, 1, 3000.0), cell(271, 1, 1, 15000.0, 0.6)],
           [cell(100, 1, 1, 500.0)]]


def cell_bytes(c):
    """Bytes the two kernels move for one cell: the samples of its 122-slot grid (cu8), the grid written and read back
    at its CRS pairs and RSSI symbols (complex double)."""
    n_symb = 7 if c.cp_type == 1 else 6
    n_ofdm = 122 * n_symb
    pairs = sum([2880, 2880, 1440, 1440][:c.n_ports])
    return n_ofdm * 128 * 2 + n_ofdm * 72 * 16 + 2 * pairs * 16 + 244 * 72 * 16


def gpu_name():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def carrier_bytes(c, D, esz=4):
    """Bytes the two carrier kernels move for one cell: its CRS windows' N = 128 D samples, the 12 R grid columns of each
    written (float2), and read back at the CRS pairs (two REs each) and the RSSI columns of the port-0 CRS symbols."""
    R, nw = c.n_rb_dl, 3 if c.n_ports == 4 else 2
    n_win = 122 * nw
    pairs = sum([480 * R, 480 * R, 240 * R, 240 * R][:c.n_ports])
    return n_win * 128 * D * esz + n_win * 12 * R * 8 + 2 * pairs * 8 + 244 * 12 * R * 8


def cir_macs(c):
    """Complex multiply-adds of cir_kernel's transform for one cell: 2 R CRS times 320 taps in each of the 244 symbols of
    ports 0 and 1 and the 122 of ports 2 and 3."""
    return sum([244, 244, 122, 122][:c.n_ports]) * 2 * c.n_rb_dl * 320


def carrier_main(a):
    import torch
    D, fs_in = 16, 16 * 1.92e6
    carriers, cells = [], []
    for j, off in enumerate((-10_000_000, 0, 10_000_000)):
        cs = []
        for i in range(8):
            c = cell(3 * (8 * j + i) + i % 3, (1, 2, 4)[i % 3], 1 + (i % 4 == 3), 1000 + 517 * i)
            c["n_rb_dl"] = 50
            if a.sib1:
                c.update(cfi=(3,), sib1=dict(format="1A", L=8, cce=0, riv=50 * 5 + 6 * i, mcs=10, tpc=0,
                                             tb=bytes((17 * i + b) % 256 for b in range(41))))
            cs.append(c)
        carriers.append((FC + off, cs))
        for c in cs:
            cells.append(L.new_cell(fc_requested=FC + off, fc_programmed=FC + off, n_id_1=c["n_id_cell"] // 3,
                                    n_id_2=c["n_id_cell"] % 3, cp_type=c["cp_type"], n_ports=c["n_ports"],
                                    frame_start=float(c["t0"]), freq_superfine=0.0, n_rb_dl=50, phich_duration=1,
                                    phich_resource=2 if a.sib1 else 3, sfn=c["sfn0"]))
    x, _ = S.synth_wide_full(D * (5000 + 122 * 960 + 400), fs_in, FC, carriers, 30.0, 0)
    iq = S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    cells = cells * a.copies
    ctx = L.Context(0)
    d_iq = torch.from_numpy(iq).cuda()
    name = "sib1" if a.sib1 else "pdcch" if a.pdcch else "pcfich" if a.pcfich else "cir" if a.cir else "carrier"
    m = {"carrier": L.CarrierMeasure, "cir": L.CellImpulse, "pcfich": L.ControlFormat, "pdcch": L.ControlChannel,
         "sib1": L.SystemInfo}[name](ctx)
    m.measure(d_iq, "ci16", fs_in, FC, cells, 1.92e6)              # warm-up
    m.timing_read()
    wall = []
    for _ in range(a.reps):
        t = time.perf_counter()
        m.measure(d_iq, "ci16", fs_in, FC, cells, 1.92e6)
        wall.append(time.perf_counter() - t)
    ms, launches = m.timing_read()
    n = len(cells)
    split = None
    if name == "sib1":
        out = m.measure(d_iq, "ci16", fs_in, FC, cells, 1.92e6)
        split = kernel_split(lambda: m.measure(d_iq, "ci16", fs_in, FC, cells, 1.92e6), n)
    m.close()
    dev_s = ms / 1e3 / a.reps
    rec = {name: True, "fs_in": fs_in, "cells": n, "reps": a.reps, "launches": launches,
           name + "_device_us_per_cell": 1e6 * dev_s / n, name + "_host_us_per_cell": 1e6 * float(np.median(wall)) / n}
    if name == "carrier":
        bytes_ = sum(carrier_bytes(c, D) for c in cells)
        rec.update(carrier_bytes_per_cell=bytes_ / n, carrier_gbytes_per_s=bytes_ / dev_s / 1e9,
                   bound_hbm_us_per_cell=1e6 * bytes_ / HBM_BPS / n)
    if name == "cir":
        macs = sum(cir_macs(c) for c in cells)
        rec.update(cir_cmacs_per_cell=macs / n, cir_fp64_tflops=8 * macs / dev_s / 1e12)
    if split is not None:
        rec.update(sib1_occasions_found=int(out["n_found"].sum()), sib1_occasions_crc_ok=int(out["n_crc_ok"].sum()),
                   sib1_occasions=3 * n, kernel_us_per_cell=split)
    rec["gpu"] = gpu_name()
    print(json.dumps(rec), flush=True)
    ctx.close()


def kernel_split(call, n):
    """Device time per cell of each kernel of one call(), from torch.profiler with CUDA activities (a run of its own)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = ev.cuda_time_total
        for k in ("carrier_grid_kernel", "pcfich_kernel", "pdcch_kernel", "pdsch_kernel", "turbo_kernel"):
            if k in ev.key and us > 0:
                split[k] = split.get(k, 0.0) + us / n
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--carrier", action="store_true", help="time lcs_carrier_cells instead")
    ap.add_argument("--cir", action="store_true", help="time lcs_cir_cells instead")
    ap.add_argument("--pcfich", action="store_true", help="time lcs_pcfich_cells instead")
    ap.add_argument("--pdcch", action="store_true", help="time lcs_pdcch_cells instead")
    ap.add_argument("--sib1", action="store_true", help="time lcs_sib1_cells instead")
    ap.add_argument("--copies", type=int, default=8, help="with --carrier, --cir, --pcfich, --pdcch or --sib1: how often each of "
                    "the 24 cells is measured per call")
    a = ap.parse_args()
    if a.carrier or a.cir or a.pcfich or a.pdcch or a.sib1:
        return carrier_main(a)
    import torch
    bufs = [S.synth_cu8(153600, cs, fc=FC, snr_db=12.0, seed=i) for i, cs in enumerate(BUFFERS)]
    iq = np.stack([bufs[c % len(bufs)] for c in range(a.channels)])
    ctx = L.Context(0)
    d_iq = torch.from_numpy(iq).cuda()
    fcs = np.full(a.channels, FC)
    f_set = L.f_search_set(FC, 20.0)
    sw = L.Sweep(ctx)
    sw.search_cu8_device(d_iq, fcs, f_set)                       # warm-up
    t = time.perf_counter()
    found = sw.search_cu8_device(d_iq, fcs, f_set)
    search_s = time.perf_counter() - t
    sw.close()
    cells = [c for row in found for c in row]
    ch = [i for i, row in enumerate(found) for _ in row]
    m = L.CellMeasure(ctx)
    m.measure(d_iq, cells, ch)                                    # warm-up
    m.timing_read()
    wall = []
    for _ in range(a.reps):
        t = time.perf_counter()
        m.measure(d_iq, cells, ch)
        wall.append(time.perf_counter() - t)
    ms, launches = m.timing_read()
    m.close()
    n = len(cells)
    dev_s = ms / 1e3 / a.reps
    bytes_ = sum(cell_bytes(c) for c in cells)
    print(json.dumps({
        "channels": a.channels, "cells": n, "reps": a.reps, "launches": launches,
        "meas_device_us_per_cell": 1e6 * dev_s / n, "meas_host_us_per_cell": 1e6 * float(np.median(wall)) / n,
        "search_host_us_per_cell": 1e6 * search_s / n, "search_host_ms": 1e3 * search_s,
        "meas_bytes_per_cell": bytes_ / n, "meas_gbytes_per_s": bytes_ / dev_s / 1e9,
        "bound_hbm_us_per_cell": 1e6 * bytes_ / HBM_BPS / n, "gpu": gpu_name(),
    }), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
