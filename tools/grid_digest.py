"""Bit-exact fingerprint of the five modules on the whole-carrier grid (lcs_carrier_cells, lcs_cir_cells, lcs_pcfich_cells,
lcs_pdcch_cells and lcs_sib1_cells): per module one SHA-256 over the record bytes of every call, with the kernels the
calls launched and the count its timing_read reports, then the status and message of one rejected call.

The GPU tests compare against float64 restatements within an FP32 tolerance, so they cannot show that a change left every
byte alone; two builds that print the same lines here computed the same thing.  The calls run on seeded lte_dl_synth
recordings: every IQ format and every D from 2 to 32, host and device input, 1, 2 and 4 ports in both CPs, cells sending
a CFI schedule and planted common-search-space DCIs, single-cell calls, and one 40-cell call of two chunks.  lcs_sib1_cells
runs the same calls with an SFN given to each cell, then the planted-SIB1 recordings of tests/test_sib1_gpu.py.

Usage: python tools/grid_digest.py        (needs an H100; a minute or so)
"""
import ctypes as C
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "lte-cell-scanner_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import lcs_b200 as L  # noqa: E402
from test_carrier_meas_host import FS, S, found, n_samples  # noqa: E402
from test_pdcch_host import pdcch_cell, plant  # noqa: E402

FC_IN = 739e6
MODULES = [("carrier", L.CarrierMeasure), ("cir", L.CellImpulse), ("pcfich", L.ControlFormat), ("pdcch", L.ControlChannel)]
# one cell per recording: (D, fmt, on_device, n_ports, cp_type, R, carrier offset in Hz, phich_duration, phich_resource,
# cfi schedule)
SINGLE = [(2, "ci16", False, 1, 1, 6, 200_000, 1, 1, (3,)), (4, "cs8", True, 2, 2, 15, -1_000_000, 2, 2, (3, 2)),
          (8, "cu8", False, 4, 1, 25, 3_000_000, 1, 3, (2, 3)), (16, "cf32", True, 2, 1, 50, -5_000_000, 1, 4, (3,)),
          (32, "ci16", True, 4, 2, 100, 12_000_000, 2, 1, (1, 2, 3)), (16, "cu8", True, 1, 2, 75, 0, 1, 2, (3,)),
          (8, "cs8", False, 2, 1, 50, 1_500_000, 2, 3, (2,)), (4, "cf32", False, 4, 2, 25, -600_000, 1, 4, (3, 2))]


def found_cell(c, fc):
    d = found(c, fc)
    d.update(phich_duration=c["phich_duration"], phich_resource=c["phich_resource"])
    return L.new_cell(**d)


def recording(carriers, n, D, fmt, seed):
    x, _ = S.synth_wide_full(n, D * FS, FC_IN, carriers, 30.0, seed)
    return S.quantise(x, fmt, 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))


def calls():
    """Every call: (iq, fmt, D, cells)."""
    import torch
    out = []
    for k, (D, fmt, dev, P, cp, R, off, dur, res, cfi) in enumerate(SINGLE):
        nid = 137 if cp == 1 else 52
        sched, _ = plant(R, cfi, P, cp, dur, res, nid)
        c = pdcch_cell(nid, P, cp, R, sched, cfi, dur, res, fill=D, paths=[(0.0, 1.0), (0.8e-6, 0.5 * np.exp(1j))])
        iq = recording([(FC_IN + off, [c])], n_samples(D), D, fmt, seed=k)
        out.append((torch.from_numpy(iq).cuda() if dev else iq, fmt, D, [found_cell(c, FC_IN + off)]))
    carriers, cells = [], []                     # 40 cells on five 25-RB carriers
    for j, off in enumerate((-10_500_000, -4_500_000, 0, 4_500_000, 10_500_000)):
        cs = []
        for i in range(8):
            nid, P, cp, dur, res = 3 * (8 * j + i) + i % 3, (1, 2, 4)[i % 3], 1 + (i % 4 == 3), 1 + i % 2, 1 + (i + j) % 4
            sched, _ = plant(25, (3, 2, 3), P, cp, dur, res, nid, seed=i)
            c = pdcch_cell(nid, P, cp, 25, sched, (3, 2, 3), dur, res, t0=1000 + 517 * i)
            c["gains"] = [g * (0.3 + 0.1 * (nid % 7)) for g in c["gains"]]
            cs.append(c)
            cells.append(found_cell(c, FC_IN + off))
        carriers.append((FC_IN + off, cs))
    iq = recording(carriers, n_samples(16, 5000), 16, "ci16", seed=11)
    out.append((iq, "ci16", 16, cells))
    dev = torch.from_numpy(iq).cuda()
    out += [(dev, "ci16", 16, [cells[i]]) for i in (0, 13, 39)]
    return out


def sib1_calls(todo):
    """The calls of calls() with an SFN for each cell, then one call per planted-SIB1 case of test_sib1_gpu."""
    import torch
    from test_sib1_gpu import CASES, case_cell
    out = []
    for iq, fmt, D, cells in todo:
        cs = []
        for k, c in enumerate(cells):
            x = L.Cell()
            C.memmove(C.byref(x), C.byref(c), C.sizeof(L.Cell))
            x.sfn = (37 * k + D) % 1024
            cs.append(x)
        out.append((iq, fmt, D, cs))
    for k, case in enumerate(CASES):
        D, fmt, dev, off = case[0], case[1], case[2], case[6]
        c, d = case_cell(case)
        iq = recording([(FC_IN + off, [c])], n_samples(D), D, fmt, seed=100 + k)
        out.append((torch.from_numpy(iq).cuda() if dev else iq, fmt, D, [L.new_cell(**d)]))
    return out


def digest(ctx, name, cls, todo):
    m = cls(ctx)
    h = hashlib.sha256()
    n0 = ctx.launches
    for iq, fmt, D, cells in todo:
        h.update(m.measure(iq, fmt, D * FS, FC_IN, cells, FS).tobytes())
    launches = ctx.launches - n0
    print("%-8s %s  launches %d  timed %d" % (name, h.hexdigest(), launches, m.timing_read()[1]), flush=True)
    iq, fmt, D, cells = todo[2]
    bad = L.Cell()
    C.memmove(C.byref(bad), C.byref(cells[0]), C.sizeof(L.Cell))
    bad.n_ports = 3
    try:
        m.measure(iq, fmt, D * FS, FC_IN, [cells[0], bad], FS)
        print("%-8s rejected: nothing" % name, flush=True)
    except L.LcsError as e:
        print("%-8s rejected: %s" % (name, e), flush=True)
    m.close()


def main():
    todo = calls()
    ctx = L.Context(0)
    for name, cls in MODULES:
        digest(ctx, name, cls, todo)
    digest(ctx, "sib1", L.SystemInfo, sib1_calls(todo))
    ctx.close()


if __name__ == "__main__":
    main()
