"""The PCFICH decoder's contract (DESIGN.md section 4.12, include/lcs_pcfich.h) restated in float64 numpy on the grid of
test_carrier_meas_host, checked against CFI schedules planted by lte_dl_synth's full-bandwidth generator; its tables
against 36.211 / 36.212; the binding of liblcs_pcfich.so; the kernels' resources; and the CLI's --cfi argument errors (no
device is touched)."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

from test_spectrum_host import exported
from test_channelizer_host import cellsearch
from test_carrier_meas_host import FS, OFFSET, S, carrier_grid, found, n_samples, synth_cell, window_starts

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
N_SF = 61
RBS = (6, 15, 25, 50, 75, 100)
SCHED = (1, 2, 3, 3, 1, 2, 2, 3, 1)       # nine long, so every subframe number sees every CFI


# ---- the contract, restated -------------------------------------------------------------------------------------------------
def codeword(k):
    """cw_k of rule 5: 0 where b mod 3 = k - 1, else 1."""
    return (np.arange(32) % 3 != k - 1).astype(int)


def reg_columns(n_id, R):
    """Rule 2: the grid column of each of the 16 PCFICH REs."""
    cols = []
    for i in range(4):
        start = (6 * (n_id % (2 * R)) + 6 * (i * R // 2)) % (12 * R)
        cols += [k for k in range(start, start + 6) if k % 3 != n_id % 3]
    return np.array(cols)


def scrambling(n_id, sf):
    """c_b, b < 32, of subframe number sf (rule 5)."""
    return S.O.lte_pn((sf + 1) * (2 * n_id + 1) * 2 ** 9 + n_id, 32).astype(int)


def pcfich_grid(oracle, x, fs_in, fc_in, d, fs_programmed=FS):
    """Y [61][nw][12 R]: symbol 0 (and 1 for four ports) of every even slot of the grid of the found-cell dict d."""
    D = int(round(fs_in / FS))
    cell = oracle.new_cell(**d)
    n_symb = 7 if d["cp_type"] == 1 else 6
    ts = window_starts(oracle, cell, x.size, D, fs_programmed)
    syms = (0, 1) if d["n_ports"] == 4 else (0,)
    rows = [2 * s * n_symb + w for s in range(N_SF) for w in syms]
    Y = carrier_grid(x, fs_in, fc_in, cell, ts[rows], fs_programmed)
    return Y.reshape(N_SF, len(syms), -1)


def measure_pcfich(Y, n_id, cp_type, n_ports, R):
    """One lcs_pcfich_meas as a dict (rules 1-6) from pcfich_grid's Y, with the equalised symbols `xhat` [61][16] and
    `sens` [61][16] beside it: |d xhat_n| <= delta sens_n to first order when every grid element errs by at most delta."""
    n_symb = 7 if cp_type == 1 else 6
    rs = S.crs_full(n_id, cp_type, R)
    _, shift = S.O.rs_dl(n_id, cp_type)
    k = reg_columns(n_id, R)
    cw = np.array([codeword(c) for c in (1, 2, 3)])
    out = dict(metric=np.zeros((N_SF, 3)), sinr=np.zeros(N_SF), cfi=np.zeros(N_SF, int), xhat=np.zeros((N_SF, 16), complex),
               sens=np.zeros((N_SF, 16)))
    for s in range(N_SF):
        sl = (2 * s) % 20

        def hhat(p):
            sym = 0 if p < 2 else 1
            sh = int(shift[sl * n_symb + sym, p])
            cols = 6 * np.arange(2 * R) + sh
            h = Y[s, sym, cols] * np.conj(rs[sl, sym])
            return np.interp(k, cols, h.real) + 1j * np.interp(k, cols, h.imag)

        y = Y[s, 0, k]
        if n_ports == 1:
            h = hhat(0)
            xh = y / h
            sens = (1 + np.abs(xh)) / np.abs(h)
        else:
            xh, sens = np.zeros(16, complex), np.zeros(16)
            hp = [hhat(p) for p in range(n_ports)]
            for j in range(8):
                a, b = (0, 1) if n_ports == 2 else ((0, 2) if j % 2 == 0 else (1, 3))
                ha, hb = hp[a][2 * j:2 * j + 2].mean(), hp[b][2 * j:2 * j + 2].mean()
                g = abs(ha) ** 2 + abs(hb) ** 2
                y0, y1 = y[2 * j], y[2 * j + 1]
                xh[2 * j] = np.sqrt(2) * (np.conj(ha) * y0 + hb * np.conj(y1)) / g
                xh[2 * j + 1] = np.sqrt(2) * (np.conj(ha) * y1 - hb * np.conj(y0)) / g
                hs = abs(ha) + abs(hb)
                for n in (2 * j, 2 * j + 1):
                    sens[n] = (np.sqrt(2) * (abs(y0) + abs(y1) + hs) + 2 * abs(xh[n]) * hs) / g
        soft = np.stack([xh.real, xh.imag], axis=1).reshape(-1)
        c = scrambling(n_id, s % 10)
        met = np.sqrt(2) / 32 * ((soft * (1 - 2 * c))[None, :] * (1 - 2 * cw)).sum(axis=1)
        best = int(np.argmax(met))
        e = cw[best] ^ c
        xref = ((1 - 2 * e[0::2]) + 1j * (1 - 2 * e[1::2])) / np.sqrt(2)
        err = np.sum(np.abs(xh - xref) ** 2)
        out["metric"][s], out["cfi"][s], out["xhat"][s], out["sens"][s] = met, best + 1, xh, sens
        out["sinr"][s] = 16 / err if err > 0 else np.inf
    out["count"] = np.array([0] + [int(np.sum(out["cfi"] == c)) for c in (1, 2, 3)])
    out["cfi_mode"] = int(np.argmax(out["count"][1:])) + 1
    out["n_ctrl_symbols"] = out["cfi_mode"] + (R <= 10)
    out["n_subframes"] = N_SF
    return out


def measure(oracle, x, fs_in, fc_in, d, fs_programmed=FS):
    """measure_pcfich of the found-cell dict d in the recording x."""
    Y = pcfich_grid(oracle, x, fs_in, fc_in, d, fs_programmed)
    return measure_pcfich(Y, d["n_id_1"] * 3 + d["n_id_2"], d["cp_type"], d["n_ports"], d["n_rb_dl"])


def planted(n=N_SF, sched=SCHED):
    return np.array([sched[s % len(sched)] for s in range(n)])


# ---- tables --------------------------------------------------------------------------------------------------------------------
def test_codewords_are_those_of_36212():
    """36.212 Table 5.3.4-1, written out."""
    table = {1: "01101101101101101101101101101101", 2: "10110110110110110110110110110110",
             3: "11011011011011011011011011011011"}
    for k, bits in table.items():
        assert list(codeword(k)) == [int(b) for b in bits], k


@pytest.mark.parametrize("R", RBS)
def test_reg_positions(R):
    """16 distinct columns inside the carrier, none on a CRS of port 0 or 1 (columns 6 m + (N_ID + 3 v) mod 6), in four
    REGs of 6 that start on a multiple of 6; the generator plants the PCFICH on the same columns."""
    for n_id in range(0, 504, 5):
        k = reg_columns(n_id, R)
        assert k.size == 16 and len(set(k)) == 16 and k.min() >= 0 and k.max() < 12 * R, (n_id, k)
        crs = {6 * m + (n_id + 3 * v) % 6 for m in range(2 * R) for v in (0, 1)}
        assert not crs & set(k), n_id
        assert all(len({c // 6 for c in k[4 * i:4 * i + 4]}) == 1 for i in range(4)), n_id
        assert np.array_equal(k, S.pcfich_res(n_id, R))
    assert list(reg_columns(0, 6)[::4]) == [1, 19, 37, 55]       # k bar = 0: REGs at 0, 18, 36, 54


def gold(c_init, n):
    """36.211 7.2 from the recursions, independently of lte_pn."""
    nc = 1600
    x1 = np.zeros(nc + n + 31, int)
    x2 = np.zeros(nc + n + 31, int)
    x1[0] = 1
    x2[:31] = [(c_init >> i) & 1 for i in range(31)]
    for i in range(nc + n):
        x1[i + 31] = (x1[i + 3] + x1[i]) % 2
        x2[i + 31] = (x2[i + 3] + x2[i + 2] + x2[i + 1] + x2[i]) % 2
    return (x1[nc:nc + n] + x2[nc:nc + n]) % 2


def test_scrambling_words():
    for n_id in (0, 1, 137, 277, 503):
        for sf in range(10):
            c_init = (sf + 1) * (2 * n_id + 1) * 512 + n_id
            assert np.array_equal(scrambling(n_id, sf), gold(c_init, 32)), (n_id, sf)


# ---- planted CFI schedules ------------------------------------------------------------------------------------------------------
D_OF_R = {6: 2, 15: 2, 25: 4, 50: 8, 75: 8, 100: 16}     # the smallest D with 6 R < 64 D


@functools.lru_cache(maxsize=None)
def case(R, n_ports=1, cp=1, seed=0, snr_db=30.0, paths=None, nid=None):
    """(restatement, cell dict) of one cell sending SCHED."""
    import lcs_oracle
    D = D_OF_R[R]
    kw = dict(cfi=SCHED)
    if paths:
        kw["paths"] = [tuple(p) for p in paths]
    cell = synth_cell((137 if cp == 1 else 52) if nid is None else nid, n_ports, cp, R, **kw)
    x, _ = S.synth_wide_full(n_samples(D), D * FS, 739e6, [(739e6, [cell])], snr_db, seed)
    d = found(cell, 739e6)
    return measure(lcs_oracle, x, D * FS, 739e6, d), d


def assert_decodes(m, R, what):
    want = planted()
    assert np.array_equal(m["cfi"], want), (what, np.flatnonzero(m["cfi"] != want))
    count = [int(np.sum(want == c)) for c in (1, 2, 3)]
    assert list(m["count"]) == [0] + count == [0, 20, 21, 20], what              # SCHED over 61 subframes
    assert m["cfi_mode"] == 2 and m["n_ctrl_symbols"] == 2 + (R <= 10) and m["n_subframes"] == N_SF, what


@pytest.mark.parametrize("R", RBS)
def test_every_bandwidth_decodes(oracle, R):
    m, _ = case(R)
    assert_decodes(m, R, R)
    assert np.all(np.abs(m["metric"][np.arange(N_SF), m["cfi"] - 1] - 1) < 0.1)
    assert np.all(10 * np.log10(m["sinr"]) > 20)


@pytest.mark.parametrize("n_ports,cp,R", [(1, 2, 25), (2, 1, 25), (2, 2, 15), (4, 1, 50), (4, 2, 6)])
def test_ports_and_cyclic_prefix(oracle, n_ports, cp, R):
    """Unequal port gains (those of test_carrier_meas_host.GAINS) over 1, 2 and 4 ports, in both CPs."""
    m, _ = case(R, n_ports=n_ports, cp=cp)
    assert_decodes(m, R, (n_ports, cp, R))
    assert np.all(10 * np.log10(m["sinr"]) > 20)


def test_two_path_channel_inside_the_cp(oracle):
    m, _ = case(50, n_ports=2, paths=((0.0, 1.0), (1.5e-6, 0.6 * np.exp(1j))))
    assert_decodes(m, 50, "two paths")
    assert np.all(10 * np.log10(m["sinr"]) > 15)


def test_clock_offset_cell(oracle):
    """The clock-offset case of the carrier test (25 ppm fast clock, carrier 1737.5 Hz off, fractional frame start)."""
    o = OFFSET
    cell = synth_cell(137, 2, 1, 25, t0=o["t0"], cfi=SCHED)
    x, _ = S.synth_wide_offset(o["D"] * (1300 + 122 * 960 + 400), o["D"] * FS, 739e6, o["fc_c"], cell, o["clock_ratio"],
                               o["f_res"], 30.0, 0)
    d = found(cell, o["fc_c"])
    d.update(fc_programmed=(o["fc_c"] - o["f_res"]) / o["clock_ratio"], freq=o["f_res"], freq_fine=o["f_res"],
             freq_superfine=o["f_res"], frame_start=o["t0"] * o["clock_ratio"])
    m = measure(oracle, x, o["D"] * FS, 739e6, d)
    assert_decodes(m, 25, "clock offset")


@pytest.mark.parametrize("n_ports", [1, 2, 4])
def test_every_subframe_decodes_at_5_db(oracle, n_ports):
    m, _ = case(25, n_ports=n_ports, snr_db=5.0, seed=3)
    assert_decodes(m, 25, n_ports)


def test_a_cell_without_cfi_is_unchanged():
    """The generator draws no random numbers for the PCFICH, and a cell without "cfi" gives the same recording."""
    a, b = synth_cell(137, 2, 1, 6), synth_cell(137, 2, 1, 6, cfi=SCHED)
    xa, _ = S.synth_wide_full(n_samples(2), 2 * FS, 739e6, [(739e6, [a])], 30.0, 5)
    xb, _ = S.synth_wide_full(n_samples(2), 2 * FS, 739e6, [(739e6, [b])], 30.0, 5)
    assert not np.array_equal(xa, xb)
    ga, _ = S._grid_full(a, 7, np.random.default_rng(1))
    gb, _ = S._grid_full(b, 7, np.random.default_rng(1))
    k = S.pcfich_res(137, 6)
    sym0 = np.zeros(ga.shape[1], bool)
    sym0[::14] = True
    other = np.ones(ga.shape[2], bool)
    other[k] = False
    assert np.array_equal(ga[:, ~sym0], gb[:, ~sym0]) and np.array_equal(ga[:, sym0][:, :, other], gb[:, sym0][:, :, other])


# ---- the kernels' resources -----------------------------------------------------------------------------------------------------
def test_pcfich_kernels_compile_without_spills(tmp_path):
    """Every kernel of pcfich.cu compiles for sm_90a with no stack frame and no spills (DESIGN.md section 4.12)."""
    csrc = os.path.join(ROOT, "lte-cell-scanner_b200", "csrc")
    r = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c", os.path.join(csrc, "pcfich.cu"), "-o",
                        str(tmp_path / "pcfich.o")], capture_output=True, text=True, check=True)
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 5 and len(frames) == 5, r.stderr            # the grid kernel in four formats, the decoder
    assert sum("carrier_grid_kernel" in e for e in entries) == 4 and sum("pcfich_kernel" in e for e in entries) == 1
    assert all(f == ("0", "0", "0") for f in frames), r.stderr


# ---- binding -------------------------------------------------------------------------------------------------------------------
LAYOUT_DRIVER = r"""
#include <stddef.h>
#include <stdio.h>
#include "lcs_pcfich.h"
#define F(f) printf(#f " %zu\n", offsetof(lcs_pcfich_meas, f));
int main(void) {
  printf("size %zu\n", sizeof(lcs_pcfich_meas));
  F(metric) F(sinr) F(cfi) F(count) F(cfi_mode) F(n_ctrl_symbols) F(n_subframes)
  printf("consts %d %d %d\n", LCS_PCFICH_CHUNK, LCS_PCFICH_LAUNCHES_PER_CHUNK, LCS_PCFICH_SUBFRAMES);
  return 0;
}
"""


def test_pcfich_prototypes_cover_header_and_library(lcs, tmp_path):
    """liblcs_pcfich.so exports exactly the four functions of include/lcs_pcfich.h, all bound with the header's
    prototypes; the other libraries export none of them.  PCFICH_MEAS has the C layout."""
    header = re.sub(r"/\*.*?\*/", " ", open(lcs.PCFICH_HEADER).read(), flags=re.S)
    names = set(re.findall(r"\b(lcs_\w+)\s*\(", header))
    assert names == {"lcs_pcfich_create", "lcs_pcfich_destroy", "lcs_pcfich_cells", "lcs_pcfich_timing_read"}
    assert set(lcs.prototypes(lcs.PCFICH_HEADER)) == names
    assert exported(lcs.PCFICH_LIB_PATH) == names
    for other in (lcs.LIB_PATH, lcs.MEAS_LIB_PATH, lcs.PSD_LIB_PATH, lcs.CARRIER_LIB_PATH, lcs.CIR_LIB_PATH):
        assert not exported(other) & names
    l = lcs.pcfich_lib()
    V, I, U, D = C.c_void_p, C.c_int, C.c_uint32, C.c_double
    assert l.lcs_pcfich_cells.argtypes == [V, V, I, I, C.c_uint64, D, D, V, U, D, V]
    assert l.lcs_pcfich_create.argtypes == [V, V]
    assert l.lcs_pcfich_timing_read.argtypes == [V, V, V]
    assert l.lcs_pcfich_destroy.restype is None
    src = tmp_path / "layout.c"
    src.write_text(LAYOUT_DRIVER)
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = dict(line.split(" ", 1) for line in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(got["size"]) == lcs.PCFICH_MEAS.itemsize
    for f in lcs.PCFICH_MEAS.names:
        assert int(got[f]) == lcs.PCFICH_MEAS.fields[f][1], f
    chunk, launches, n_sf = got["consts"].split()
    assert (int(chunk), int(launches), int(n_sf)) == (lcs.PCFICH_CHUNK, 2, lcs.PCFICH_SUBFRAMES) == (32, 2, N_SF)


# ---- CLI argument errors with --cfi (no device is touched) --------------------------------------------------------------------
def test_cli_cfi_argument_errors(lcs, tmp_path):
    f = str(tmp_path / "rec.ci16")
    np.zeros((1000, 2), np.int16).tofile(f)
    wide = ["--wideband", f, "--fc-in", "739e6", "-s", "739e6"]
    cases = [
        (["-s", "739e6", "-l", "-d", str(tmp_path), "--cfi"], "--cfi needs --wideband"),
        (wide + ["--fs-in", "7.68e6", "--cfi-csv", str(tmp_path / "c.csv")], "--cfi-csv needs --cfi"),
        (["--wideband", f, "--fc-in", "739e6", "--fs-in", "10e6", "--spectrum", str(tmp_path / "p.csv"), "--cfi"],
         "--cfi needs a search (-s)"),
        (wide + ["--fs-in", "11.52e6", "--cfi"], "--cfi needs --fs-in = D * 1.92 MHz"),
        (wide + ["--fs-in", "10e6", "--resample", "--cfi"], "--cfi needs --fs-in = D * 1.92 MHz"),
        (wide + ["--fs-in", "7.68e6", "--cfi"], "holds 1000 ci16 samples"),
    ]
    for args, msg in cases:
        out = cellsearch(*args)
        assert out.returncode != 0 and msg in out.stderr, (args, out.stderr)
        assert "lcs_ctx_create" not in out.stderr
