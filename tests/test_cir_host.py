"""The power delay profile's contract (DESIGN.md section 4.11, include/lcs_cir.h) restated in float64 numpy on the grid of
test_carrier_meas_host, checked against the paths planted by lte_dl_synth's full-bandwidth generator; the binding of
liblcs_cir.so; the kernels' resources; and the CLI's --cir argument errors (no device is touched)."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

from test_spectrum_host import exported
from test_channelizer_host import cellsearch
from test_carrier_meas_host import (FS, GAINS, N_SLOT, S, carrier_grid, found, measure_carrier, n_samples,
                                    offset_scenario, OFFSET, synth_cell, window_starts)

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
TAPS, TAP0, RANGE_DB = 320, 64, 20.0
T_S = 1 / 30.72e6
TAU = (np.arange(TAPS) - TAP0) * T_S


# ---- the contract, restated -------------------------------------------------------------------------------------------------
def cir_stats(pdp):
    """Rule 5 on one port's pdp [TAPS]: (peak_delay, first_delay, mean_delay, rms_spread, n_taps, K as a bool mask)."""
    js = int(np.argmax(pdp))
    k = pdp >= pdp[js] * 10 ** (-RANGE_DB / 10)
    ext = np.concatenate([[-np.inf], pdp, [-np.inf]])
    local = (ext[1:-1] >= ext[:-2]) & (ext[1:-1] >= ext[2:])
    jf = int(np.flatnonzero(k & local)[0])
    delta = 0.0
    if 0 < jf < TAPS - 1:
        pm, p0, pp = pdp[jf - 1], pdp[jf], pdp[jf + 1]
        den = pm - 2 * p0 + pp
        if den != 0:
            delta = float(np.clip((pm - pp) / (2 * den), -0.5, 0.5))
    w = pdp[k]
    mean = np.sum(w * TAU[k]) / np.sum(w)
    rms = np.sqrt(np.sum(w * (TAU[k] - mean) ** 2) / np.sum(w))
    return TAU[js], TAU[jf] + delta * T_S, mean, rms, int(k.sum()), k


def measure_cir(Y, n_id_cell, cp_type, n_ports, R, t_frame):
    """One lcs_cir_meas as a dict (rules 1-7), from the grid Y [n_ofdm][12 R]; t_frame = D frame_start / fs_in."""
    n_symb = 7 if cp_type == 1 else 6
    rs = S.crs_full(n_id_cell, cp_type, R)
    _, shift = S.O.rs_dl(n_id_cell, cp_type)
    m = np.arange(2 * R)
    w = np.sin(np.pi * (m + 0.5) / (2 * R)) ** 2
    b = S.subcarriers(R)
    nan4 = lambda: np.full(4, np.nan)
    out = dict(pdp=np.full((4, TAPS), np.nan), t=np.full((4, TAPS), np.nan), floor=nan4(), peak_delay=nan4(), first_delay=nan4(), mean_delay=nan4(),
               rms_spread=nan4(), n_pairs=np.zeros(4, int), n_taps=np.zeros(4, int))
    for p in range(n_ports):
        syms = [0, n_symb - 3] if p < 2 else [1]
        c = np.zeros((N_SLOT, len(syms), TAPS), complex)
        for t in range(N_SLOT):
            for i, s in enumerate(syms):
                cols = 6 * m + int(shift[(t % 20) * n_symb + s, p])
                h = Y[t * n_symb + s, cols] * np.conj(rs[t % 20, s])
                c[t, i] = (w * h) @ np.exp(2j * np.pi * np.outer(b[cols], np.arange(TAPS) - TAP0) / 2048)
        ca, cb = c[:-2].reshape(-1, TAPS), c[2:].reshape(-1, TAPS)
        s_ = np.abs(np.mean(ca * np.conj(cb), axis=0))
        t_ = np.mean((np.abs(ca) ** 2 + np.abs(cb) ** 2) / 2, axis=0)
        out["pdp"][p] = s_ / (128 * R * R)
        out["t"][p] = t_ / (128 * R * R)                # T_j in pdp's units (not a field of lcs_cir_meas)
        out["floor"][p] = np.mean((t_ - s_) / (128 * R * R))
        st = cir_stats(out["pdp"][p])
        for key, v in zip(("peak_delay", "first_delay", "mean_delay", "rms_spread", "n_taps"), st):
            out[key][p] = v
        out["n_pairs"][p] = ca.shape[0]
    out["frame_arrival"] = t_frame + out["first_delay"][0]
    return out


def measure(oracle, x, fs_in, fc_in, d, fs_programmed=FS):
    """measure_cir of the oracle-style cell dict d in the recording x, with the carrier restatement's rsrp beside it."""
    D = int(round(fs_in / FS))
    cell = oracle.new_cell(**d)
    Y = carrier_grid(x, fs_in, fc_in, cell, window_starts(oracle, cell, x.size, D, fs_programmed), fs_programmed)
    m = measure_cir(Y, cell.n_id_cell(), cell.cp_type, cell.n_ports, cell.n_rb_dl, D * d["frame_start"] / fs_in)
    m["rsrp"] = measure_carrier(Y, cell.n_id_cell(), cell.cp_type, cell.n_ports, cell.n_rb_dl)["rsrp"]
    return m


# ---- planted paths ---------------------------------------------------------------------------------------------------------
D_OF_R = {6: 2, 15: 2, 25: 4, 50: 8, 75: 8, 100: 16}     # the smallest D with 6 R < 64 D


@functools.lru_cache(maxsize=None)
def case(R, paths=((0.0, 1.0),), n_ports=1, cp=1, seed=0, snr_db=30.0, dt=0.0, load=1.0):
    """(restatement, cell dict) of one cell with the given paths, measured with frame_start = t0 + dt."""
    D = D_OF_R[R]
    cell = synth_cell(137 if cp == 1 else 52, n_ports, cp, R, paths=[tuple(p) for p in paths], load=load)
    x, _ = S.synth_wide_full(n_samples(D), D * FS, 739e6, [(739e6, [cell])], snr_db, seed)
    d = found(cell, 739e6)
    d["frame_start"] += dt
    import lcs_oracle
    return measure(lcs_oracle, x, D * FS, 739e6, d), d


def spread(paths):
    p = np.abs([g for _, g in paths]) ** 2
    t = np.array([d for d, _ in paths])
    mu = np.sum(p * t) / p.sum()
    return mu, np.sqrt(np.sum(p * (t - mu) ** 2) / p.sum())


# Tolerances: about twice the largest error over seeds 0-7 (error_spread), which was
#   a single path's pdp peak against the carrier's rsrp: 0.10 % (R = 6) ... 0.02 % (R = 100); first_delay of a path on a
#   tap: 0.0125 T_s; a path 0.37 T_s off the grid: 0.036 T_s; two paths' rms_spread against the analytic: 1.2 %.
TOL_PEAK = 0.002
TOL_FIRST = 0.025 * T_S
TOL_OFFGRID = 0.075 * T_S
TOL_SPREAD = 0.025


@pytest.mark.parametrize("R", sorted(D_OF_R))
def test_single_path_peaks_on_its_tap_with_the_carrier_rsrp(oracle, R):
    m, _ = case(R)
    assert m["pdp"][0].argmax() == TAP0 and m["peak_delay"][0] == 0.0
    assert abs(m["pdp"][0, TAP0] / m["rsrp"][0] - 1) < TOL_PEAK, (m["pdp"][0, TAP0], m["rsrp"][0])
    assert abs(m["first_delay"][0]) < TOL_FIRST
    assert abs(m["mean_delay"][0]) < TOL_FIRST
    assert list(m["n_pairs"]) == [240, 0, 0, 0] and np.all(np.isnan(m["pdp"][1:]))
    # the main lobe of the taper: 2 bins of 1 / (2 R 90 kHz) either side
    lobe = 2 * 30.72e6 / (2 * R * 90e3)
    assert m["n_taps"][0] <= 2 * lobe + 1 and m["rms_spread"][0] < lobe * T_S
    assert 0 < m["floor"][0] < 1e-2 * m["pdp"][0, TAP0]


def test_frame_start_moves_first_delay_but_not_frame_arrival(oracle):
    a, da = case(50)
    b, db = case(50, dt=-2.25)
    assert abs((b["first_delay"][0] - a["first_delay"][0]) - 2.25 / FS) < TOL_OFFGRID
    assert abs(b["frame_arrival"] - a["frame_arrival"]) < TOL_OFFGRID
    assert abs(a["frame_arrival"] - da["frame_start"] / FS) < TOL_FIRST


def test_off_grid_delay(oracle):
    d = 0.37 * T_S
    m, _ = case(100, paths=((d, 1.0),))
    assert m["pdp"][0].argmax() == TAP0
    assert abs(m["first_delay"][0] - d) < TOL_OFFGRID, m["first_delay"][0] / T_S


@pytest.mark.parametrize("R,paths", [
    (25, ((0.0, 0.5), (1.5e-6, 1.0))),
    (50, ((0.0, 0.5 * np.exp(1j)), (1.0e-6, 1.0))),
    (100, ((0.2e-6, 0.5), (0.9e-6, 1.0 * np.exp(-2j)), (2.1e-6, 0.6))),
], ids=["25rb-2path", "50rb-2path", "100rb-3path"])
def test_first_path_is_the_earlier_weaker_one(oracle, R, paths):
    """The first path is 6 dB below the strongest; first_delay finds it, peak_delay the strongest, and mean_delay and
    rms_spread follow the paths' powers (for two paths rms_spread = sqrt(p1 p2) / (p1 + p2) Delta)."""
    m, _ = case(R, paths=paths)
    assert abs(m["first_delay"][0] - paths[0][0]) < TOL_FIRST + 0.05 * T_S, m["first_delay"][0] / T_S
    assert abs(m["peak_delay"][0] - paths[1][0]) <= T_S / 2
    mu, sd = spread(paths)
    if len(paths) == 2:
        p1, p2 = np.abs(paths[0][1]) ** 2, np.abs(paths[1][1]) ** 2
        assert np.isclose(sd, np.sqrt(p1 * p2) / (p1 + p2) * (paths[1][0] - paths[0][0]))
    assert abs(m["mean_delay"][0] - mu) < TOL_SPREAD * sd
    assert abs(m["rms_spread"][0] / sd - 1) < TOL_SPREAD, (m["rms_spread"][0], sd)


def test_extended_cp_path_at_7us(oracle):
    paths = ((0.0, 1.0), (7e-6, 0.8))
    m, _ = case(50, paths=paths, n_ports=2, cp=2)
    j7 = TAP0 + int(round(7e-6 / T_S))
    for p in range(2):
        assert m["pdp"][p].argmax() == TAP0
        assert abs(np.argmax(m["pdp"][p, TAP0 + 100:]) + TAP0 + 100 - j7) <= 1
        mu, sd = spread(paths)
        assert abs(m["mean_delay"][p] - mu) < TOL_SPREAD * sd and abs(m["rms_spread"][p] / sd - 1) < TOL_SPREAD


def test_clock_offset_cell_arrives_at_its_frame_start(oracle):
    """The clock-offset case of the carrier test (25 ppm fast clock, carrier 1737.5 Hz off, fractional frame start): a
    single path on tap 0, and frame_arrival at the frame start in the recording's samples."""
    x, d, _ = offset_scenario(0)
    D = OFFSET["D"]
    m = measure(oracle, x, D * FS, 739e6, d)
    tol = 0.05 * T_S                            # twice the 0.027 T_s the case gives
    for p in range(2):
        assert m["pdp"][p].argmax() == TAP0 and abs(m["first_delay"][p]) < tol, m["first_delay"][p] / T_S
        assert abs(m["pdp"][p, TAP0] / m["rsrp"][p] - 1) < TOL_PEAK
    assert abs(m["frame_arrival"] - d["frame_start"] / FS) < tol


def two_cells(seed=0):
    a = synth_cell(137, 2, 1, 50, t0=1234, load=0.1)
    b = synth_cell(100, 1, 1, 50, t0=5000, load=0.1, paths=[(0.0, 0.7)])
    x, _ = S.synth_wide_full(n_samples(8, 5000), 8 * FS, 739e6, [(740e6, [a, b])], 30.0, seed)
    return x, found(a, 740e6), found(b, 740e6)


def test_two_cells_on_one_carrier_give_their_timing_offset(oracle):
    x, da, db = two_cells()
    ma, mb = (measure(oracle, x, 8 * FS, 739e6, d) for d in (da, db))
    assert abs((mb["frame_arrival"] - ma["frame_arrival"]) - (5000 - 1234) / FS) < TOL_FIRST


@pytest.mark.parametrize("n_ports", [1, 2, 4])
def test_port_gains(oracle, n_ports):
    m, _ = case(25, n_ports=n_ports)
    want = S.AMP ** 2 * np.abs(np.asarray(GAINS[:n_ports])) ** 2 / 128
    assert np.all(np.abs(m["pdp"][:n_ports, TAP0] / want - 1) < TOL_PEAK + 0.02), m["pdp"][:n_ports, TAP0] / want
    assert list(m["n_pairs"]) == [240, 240, 120, 120][:n_ports] + [0] * (4 - n_ports)
    assert np.all(np.isnan(m["pdp"][n_ports:])) and np.all(np.isnan(m["first_delay"][n_ports:]))


def test_noise_stays_out_of_the_range_at_10_db(oracle):
    """At 10 dB SNR per RE only taps of the planted paths' main lobes enter K."""
    R, paths = 50, ((0.0, 1.0), (1.2e-6, 0.6))
    lobe = 2 * 30.72e6 / (2 * R * 90e3)
    for seed in range(2):
        m, _ = case(R, paths=paths, seed=seed, snr_db=10.0)
        k = np.flatnonzero(cir_stats(m["pdp"][0])[5])
        near = np.min([np.abs(k - (TAP0 + d / T_S)) for d, _ in paths], axis=0)
        assert np.all(near <= lobe), (seed, k)
        assert m["floor"][0] > 0


def error_spread(seeds=range(8)):
    """The largest errors over `seeds` that TOL_* were set from."""
    e = {}
    for s in seeds:
        for R in sorted(D_OF_R):
            m, _ = case(R, seed=s)
            e["peak%d" % R] = max(e.get("peak%d" % R, 0), abs(m["pdp"][0, TAP0] / m["rsrp"][0] - 1))
            e["first"] = max(e.get("first", 0), abs(m["first_delay"][0]) / T_S)
        m, _ = case(100, paths=((0.37 * T_S, 1.0),), seed=s)
        e["offgrid"] = max(e.get("offgrid", 0), abs(m["first_delay"][0] / T_S - 0.37))
        paths = ((0.0, 0.5), (1.5e-6, 1.0))
        m, _ = case(25, paths=paths, seed=s)
        e["spread"] = max(e.get("spread", 0), abs(m["rms_spread"][0] / spread(paths)[1] - 1))
    return e


# ---- the kernels' resources -----------------------------------------------------------------------------------------------------
def test_cir_kernels_compile_without_spills(tmp_path):
    """Every kernel of cir.cu compiles for sm_90a with no stack frame and no spills (DESIGN.md section 4.11)."""
    csrc = os.path.join(ROOT, "lte-cell-scanner_b200", "csrc")
    r = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c", os.path.join(csrc, "cir.cu"), "-o",
                        str(tmp_path / "cir.o")], capture_output=True, text=True, check=True)
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 5 and len(frames) == 5, r.stderr            # the grid kernel in four formats, the transform
    assert sum("carrier_grid_kernel" in e for e in entries) == 4 and sum("cir_kernel" in e for e in entries) == 1
    assert all(f == ("0", "0", "0") for f in frames), r.stderr


# ---- binding -------------------------------------------------------------------------------------------------------------------
LAYOUT_DRIVER = r"""
#include <stddef.h>
#include <stdio.h>
#include "lcs_cir.h"
#define F(f) printf(#f " %zu\n", offsetof(lcs_cir_meas, f));
int main(void) {
  printf("size %zu\n", sizeof(lcs_cir_meas));
  F(pdp) F(floor) F(peak_delay) F(first_delay) F(mean_delay) F(rms_spread) F(frame_arrival) F(n_pairs) F(n_taps)
  printf("consts %d %d %d %.17g\n", LCS_CIR_CHUNK, LCS_CIR_LAUNCHES_PER_CHUNK, LCS_CIR_TAPS, LCS_CIR_RANGE_DB);
  return 0;
}
"""


def test_cir_prototypes_cover_header_and_library(lcs, tmp_path):
    """liblcs_cir.so exports exactly the four functions of include/lcs_cir.h, all bound with the header's prototypes;
    the other four libraries export none of them.  CIR_MEAS has the C layout."""
    header = re.sub(r"/\*.*?\*/", " ", open(lcs.CIR_HEADER).read(), flags=re.S)
    names = set(re.findall(r"\b(lcs_\w+)\s*\(", header))
    assert names == {"lcs_cir_create", "lcs_cir_destroy", "lcs_cir_cells", "lcs_cir_timing_read"}
    assert set(lcs.prototypes(lcs.CIR_HEADER)) == names
    assert exported(lcs.CIR_LIB_PATH) == names
    for other in (lcs.LIB_PATH, lcs.MEAS_LIB_PATH, lcs.PSD_LIB_PATH, lcs.CARRIER_LIB_PATH):
        assert not exported(other) & names
    l = lcs.cir_lib()
    V, I, U, D = C.c_void_p, C.c_int, C.c_uint32, C.c_double
    assert l.lcs_cir_cells.argtypes == [V, V, I, I, C.c_uint64, D, D, V, U, D, V]
    assert l.lcs_cir_create.argtypes == [V, V]
    assert l.lcs_cir_timing_read.argtypes == [V, V, V]
    assert l.lcs_cir_destroy.restype is None
    src = tmp_path / "layout.c"
    src.write_text(LAYOUT_DRIVER)
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = dict(line.split(" ", 1) for line in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(got["size"]) == lcs.CIR_MEAS.itemsize
    for f in lcs.CIR_MEAS.names:
        assert int(got[f]) == lcs.CIR_MEAS.fields[f][1], f
    chunk, launches, taps, range_db = got["consts"].split()
    assert (int(chunk), int(launches), int(taps), float(range_db)) == (lcs.CIR_CHUNK, 2, lcs.CIR_TAPS, RANGE_DB)
    assert np.array_equal(lcs.cir_delays(), TAU)


# ---- CLI argument errors with --cir (no device is touched) --------------------------------------------------------------------
def test_cli_cir_argument_errors(lcs, tmp_path):
    f = str(tmp_path / "rec.ci16")
    np.zeros((1000, 2), np.int16).tofile(f)
    wide = ["--wideband", f, "--fc-in", "739e6", "-s", "739e6"]
    cases = [
        (["-s", "739e6", "-l", "-d", str(tmp_path), "--cir"], "--cir needs --wideband"),
        (wide + ["--fs-in", "7.68e6", "--cir-csv", str(tmp_path / "c.csv")], "--cir-csv needs --cir"),
        (["--wideband", f, "--fc-in", "739e6", "--fs-in", "10e6", "--spectrum", str(tmp_path / "p.csv"), "--cir"],
         "--cir needs a search (-s)"),
        (wide + ["--fs-in", "11.52e6", "--cir"], "--cir needs --fs-in = D * 1.92 MHz"),
        (wide + ["--fs-in", "10e6", "--resample", "--cir"], "--cir needs --fs-in = D * 1.92 MHz"),
        (wide + ["--fs-in", "7.68e6", "--cir"], "holds 1000 ci16 samples"),
    ]
    for args, msg in cases:
        out = cellsearch(*args)
        assert out.returncode != 0 and msg in out.stderr, (args, out.stderr)
        assert "lcs_ctx_create" not in out.stderr
