"""The full-carrier measurement's contract (DESIGN.md section 4.10, include/lcs_carrier.h) restated in float64 numpy, checked
against the truth planted by lte_dl_synth's full-bandwidth generator; RsDl's full-band CRS; the binding of
liblcs_carrier.so; and the CLI's --measure-carrier argument errors (no device is touched)."""
import ctypes as C
import functools
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from test_spectrum_host import exported
from test_channelizer_host import cellsearch
from test_cell_meas_host import measure_grid

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "track_oracle"))
import lte_dl_synth as S  # noqa: E402

FS = 1.92e6
GAINS = [1.0, 0.8 * np.exp(0.7j), 0.9 * np.exp(-1.1j), 0.7 * np.exp(2.2j)]   # lte_dl_synth's default port gains
N_SLOT = 122


# ---- the contract, restated -------------------------------------------------------------------------------------------------
def window_starts(oracle, cell, n_in, D, fs_programmed=FS):
    """loc_t: the oracle's extract_tfg timestamps for a copy of `cell` (an oracle Cell) with freq_fine = freq_superfine."""
    g = oracle.new_cell(**{k: getattr(cell, k) for k, _ in oracle.Cell._fields_})
    g.freq_fine = cell.freq_superfine
    _, ts = oracle.extract_tfg(g, np.zeros(n_in // D + 256, complex), cell.fc_requested, cell.fc_programmed, fs_programmed)
    return ts


def carrier_grid(x, fs_in, fc_in, cell, ts, fs_programmed=FS, foc_sign=1, late_sign=1):
    """Y [n_ofdm][12 R] (rules 2-4) of the recording x (complex, full-scale units).  foc_sign / late_sign = -1 turn the
    FOC rotation or the lateness ramp the wrong way (to show that a test depends on them)."""
    D = int(round(fs_in / FS))
    N, fs, R = 128 * D, int(round(fs_in)), cell.n_rb_dl
    delta = int(round(cell.fc_requested - fc_in))
    kf = (cell.fc_requested - cell.freq_superfine) / cell.fc_programmed
    kappa = -2 * np.pi * cell.freq_superfine / (D * fs_programmed * kf)
    q = np.rint(D * ts).astype(np.int64)
    late = q - D * ts
    assert q.min() >= 0 and q.max() + N <= x.size
    m = q[:, None] + np.arange(N)
    p = ((m % fs) * (delta % fs)) % fs
    X = np.fft.fft(x[m] * np.exp(-2j * np.pi * p / fs) * np.exp(foc_sign * 1j * kappa * m), axis=1)
    b = S.subcarriers(R)
    return np.sqrt(128) / N * X[:, b % N] * np.exp(-late_sign * 2j * np.pi * late[:, None] * b / N)


def measure_carrier(Y, n_id_cell, cp_type, n_ports, R):
    """One lcs_carrier_meas as a dict (rules 6-7), from the grid Y [n_ofdm][12 R]."""
    n_symb = 7 if cp_type == 1 else 6
    rs = S.crs_full(n_id_cell, cp_type, R)
    _, shift = S.O.rs_dl(n_id_cell, cp_type)
    nan4 = lambda: np.full(4, np.nan)
    m = dict(rsrp=nan4(), noise=nan4(), sinr=nan4(), n_pairs=np.zeros(4, int), rb_rsrp=np.full((4, 100), np.nan),
             rb_noise=np.full((4, 100), np.nan), rb_rssi=np.full(100, np.nan), n_rb=R)
    cols = 6 * np.arange(2 * R)
    for p in range(n_ports):
        ha, hb = [], []
        for t in range(N_SLOT - 2):
            for s in ([0, n_symb - 3] if p < 2 else [1]):
                for h, tt in ((ha, t), (hb, t + 2)):
                    sh = int(shift[(tt % 20) * n_symb + s, p])
                    h.append(Y[tt * n_symb + s, cols + sh] * np.conj(rs[tt % 20, s]))
        ha, hb = np.array(ha), np.array(hb)                            # [terms][2R]
        c = (ha * np.conj(hb)).reshape(len(ha), R, 2).sum(axis=(0, 2))
        t2 = ((np.abs(ha) ** 2 + np.abs(hb) ** 2) / 2).reshape(len(ha), R, 2).sum(axis=(0, 2))
        n = 2 * len(ha)
        s_rb = np.abs(c / n)
        m["rb_rsrp"][p, :R], m["rb_noise"][p, :R] = s_rb / 128, (t2 / n - s_rb) / 128
        s, t = np.abs(c.sum() / (n * R)), t2.sum() / (n * R)
        m["rsrp"][p], m["noise"][p] = s / 128, (t - s) / 128
        m["sinr"][p] = s / (t - s) if t > s else np.inf
        m["n_pairs"][p] = n * R
    rows = [r for r in range(N_SLOT * n_symb) if r % n_symb in (0, n_symb - 3)]
    e = np.abs(Y[rows]) ** 2
    m["rb_rssi"][:R] = e.reshape(len(rows), R, 12).sum(axis=2).mean(axis=0) / 128
    m["rssi"] = e.sum(axis=1).mean() / 128
    m["rsrq"] = R * m["rsrp"][0] / m["rssi"]
    return m


def measure(oracle, x, fs_in, fc_in, cell, fs_programmed=FS, **signs):
    D = int(round(fs_in / FS))
    Y = carrier_grid(x, fs_in, fc_in, cell, window_starts(oracle, cell, x.size, D, fs_programmed), fs_programmed, **signs)
    return measure_carrier(Y, cell.n_id_cell(), cell.cp_type, cell.n_ports, cell.n_rb_dl)


# ---- synthetic carriers with planted truth ----------------------------------------------------------------------------------
def synth_cell(nid, n_ports, cp, R, t0=1234, **kw):
    return dict(n_id_cell=nid, n_ports=n_ports, cp_type=cp, n_rb_dl=R, phich_duration=1, phich_resource=1, t0=t0, sfn0=0,
                gains=list(GAINS), **kw)


def found(d, fc):
    """The oracle-style cell dict the search would return for synth cell d on carrier fc (nominal clock)."""
    return dict(fc_requested=fc, fc_programmed=fc, n_id_1=d["n_id_cell"] // 3, n_id_2=d["n_id_cell"] % 3,
                cp_type=d["cp_type"], n_ports=d["n_ports"], frame_start=float(d["t0"]), freq=0.0, freq_fine=0.0,
                freq_superfine=0.0, n_rb_dl=d["n_rb_dl"])


def n_samples(D, t0=1234):
    return D * (t0 + N_SLOT * 960 + 400)


def scenario(cell, D, fc_off=0, seed=0, snr_db=30.0, fc_in=739e6):
    """(x, oracle-style cell dict, received grid) of one cell on a carrier fc_off Hz from the recording's centre."""
    fs_in = D * FS
    x, grids = S.synth_wide_full(n_samples(D, cell["t0"]), fs_in, fc_in, [(fc_in + fc_off, [cell])], snr_db, seed)
    return x, found(cell, fc_in + fc_off), grids[0]


def noise_per_re(snr_db):
    return S.AMP ** 2 / 10 ** (snr_db / 10)


def planted_rssi(grid, cp_type, R, snr_db):
    """RSSI x 128 of the received grid: the mean over the port-0 CRS symbols of its 12 R REs' power, plus the noise."""
    n_symb = 7 if cp_type == 1 else 6
    rows = [r for r in range(N_SLOT * n_symb) if r % n_symb in (0, n_symb - 3)]
    return np.mean(np.sum(np.abs(grid[rows]) ** 2, axis=1)) + 12 * R * noise_per_re(snr_db)


# (n_ports, cp_type, R, D, load)
FLAT = {"1port_6rb": (1, 1, 6, 2, 1.0), "2port_25rb": (2, 1, 25, 4, 0.5), "4port_50rb": (4, 1, 50, 8, 1.0),
        "2port_ext_100rb": (2, 2, 100, 16, 0.25), "4port_ext_25rb": (4, 2, 25, 8, 1.0), "1port_100rb": (1, 1, 100, 32, 1.0)}

# Relative tolerances of (S per RB, S of the carrier, RSRQ) against the planted truth at 30 dB SNR: about twice the largest
# error over seeds 0-3 of each FLAT case (tolerance_spread), which was
#   1port_6rb 0.40 / 0.071 / 0.052 %, 2port_25rb 0.73 / 0.070 / 0.034 %, 4port_50rb 1.32 / 0.075 / 0.055 %,
#   2port_ext_100rb 0.87 / 0.052 / 0.036 %, 4port_ext_25rb 1.34 / 0.127 / 0.096 %, 1port_100rb 0.72 / 0.046 / 0.039 %.
# An RB has 480 pairs per port 0/1 and 240 per port 2/3, so the four-port cases spread most.
TOL_RB, TOL_S, TOL_RSRQ = 0.03, 0.003, 0.002


def flat_case(name, seed):
    P, cp, R, D, load = FLAT[name]
    cell = synth_cell(137 if cp == 1 else 52, P, cp, R, load=load)
    x, d, grid = scenario(cell, D, seed=seed)
    return x, d, grid, D


def flat_errors(oracle, name, seed):
    x, d, grid, D = flat_case(name, seed)
    P, cp, R = d["n_ports"], d["cp_type"], d["n_rb_dl"]
    m = measure(oracle, x, D * FS, 739e6, oracle.new_cell(**d))
    s_true = S.AMP ** 2 * np.abs(np.asarray(GAINS[:P])) ** 2
    rsrq_true = R * s_true[0] / planted_rssi(grid, cp, R, 30.0)
    return m, (np.abs(m["rb_rsrp"][:P, :R] * 128 / s_true[:, None] - 1).max(),
               np.abs(m["rsrp"][:P] * 128 / s_true - 1).max(), abs(m["rsrq"] / rsrq_true - 1))


@pytest.mark.parametrize("name", sorted(FLAT))
def test_flat_channel_matches_planted_powers(oracle, name):
    m, (e_rb, e_s, e_q) = flat_errors(oracle, name, 0)
    assert e_rb < TOL_RB and e_s < TOL_S and e_q < TOL_RSRQ, (name, e_rb, e_s, e_q)
    P, R = FLAT[name][0], FLAT[name][2]
    assert list(m["n_pairs"]) == [480 * R, 480 * R, 240 * R, 240 * R][:P] + [0] * (4 - P)
    assert np.all(np.isnan(m["rsrp"][P:])) and np.all(np.isnan(m["rb_rsrp"][:, R:])) and np.all(np.isnan(m["rb_rssi"][R:]))
    assert np.all(np.isnan(m["rb_rsrp"][P:])) and np.all(np.isnan(m["rb_noise"][P:]))
    assert np.allclose(m["rsrp"][:P], m["rb_rsrp"][:P, :R].mean(axis=1), rtol=1e-2)
    assert np.isclose(m["rssi"], m["rb_rssi"][:R].sum(), rtol=1e-12)


def test_two_path_channel_shapes_rb_rsrp(oracle):
    """A 2-path channel: each RB's RSRP follows the RB's mean |H(f)|^2 over its CRS subcarriers, across a fade of more than
    10 dB."""
    paths = [(0.0, 1.0), (1.3e-6, 0.8 * np.exp(1.0j))]
    cell = synth_cell(137, 2, 1, 50, paths=paths)
    x, d, _ = scenario(cell, 8, fc_off=1_000_000, seed=1)
    m = measure(oracle, x, 8 * FS, 739e6, oracle.new_cell(**d))
    h2 = np.abs(S.channel_response(paths, S.subcarriers(50) * 15e3)) ** 2
    crs = [137 % 6, 137 % 6 + 6, (137 + 3) % 6, (137 + 3) % 6 + 6]   # port 0's CRS columns of an RB (symbols 0 and 4)
    want = S.AMP ** 2 * np.abs(GAINS[0]) ** 2 * h2.reshape(50, 12)[:, crs].mean(axis=1) / 128
    assert want.max() / want.min() > 10
    err = np.abs(m["rb_rsrp"][0, :50] / want - 1)
    assert err.max() < 0.025, err.max()         # largest over seeds 0-3: 1.2 %


def test_partial_band_interferer_raises_only_its_rbs(oracle):
    lo, hi = 10, 16
    cell = synth_cell(137, 1, 1, 25, interferer=(lo, hi, 0.1))
    x, d, _ = scenario(cell, 4, seed=2, snr_db=25.0)
    m = measure(oracle, x, 4 * FS, 739e6, oracle.new_cell(**d))
    n = m["rb_noise"][0, :25] * 128
    base, extra = noise_per_re(25.0), 0.1 * S.AMP ** 2
    inside = np.arange(25)[(np.arange(25) >= lo) & (np.arange(25) < hi)]
    outside = np.setdiff1d(np.arange(25), inside)
    # largest over seeds 0-3: 12.2 % inside, 14.4 % outside (one RB's noise is a difference of two near-equal sums)
    assert np.all(np.abs(n[inside] / (base + extra) - 1) < 0.25), n[inside] / (base + extra)
    assert np.all(np.abs(n[outside] / base - 1) < 0.3), n[outside] / base
    assert n[inside].min() > 5 * n[outside].max()


def test_six_rbs_equal_the_six_rb_restatement(oracle):
    """For R = 6 the carrier grid holds the 6-RB grid's 72 subcarriers, and the two estimators agree on it."""
    cell = synth_cell(137, 4, 1, 6)
    x, d, _ = scenario(cell, 2, fc_off=300_000, seed=3)
    c = oracle.new_cell(**d)
    Y = carrier_grid(x, 2 * FS, 739e6, c, window_starts(oracle, c, x.size, 2))
    a = measure_carrier(Y, c.n_id_cell(), 1, 4, 6)
    b = measure_grid(oracle, Y, c.n_id_cell(), 1, 4)
    for k in ("rsrp", "noise", "sinr", "rssi"):
        assert np.allclose(a[k], b[k], rtol=1e-12, equal_nan=True), k
    assert np.isclose(a["rsrq"], b["rsrq"], rtol=1e-12)
    assert list(a["n_pairs"]) == [2880, 2880, 1440, 1440]


# A receiver whose sample clock is 25 ppm fast, a carrier 1737.5 Hz off after the nominal mixer, fc_programmed !=
# fc_requested and a fractional frame start: the FOC rotation (kappa != 0) and every window's lateness ramp matter.
OFFSET = dict(D=4, fc_c=739e6 + 1.2e6, clock_ratio=1 + 25e-6, f_res=1737.5, t0=1234.37)


@functools.lru_cache(maxsize=None)
def offset_scenario(seed):
    """(x, oracle-style cell dict, received grid) of a 25-RB two-port cell at 7.68 Msps with the clock offset of OFFSET,
    by direct evaluation."""
    o = OFFSET
    cell = synth_cell(137, 2, 1, 25, t0=o["t0"])
    x, Y = S.synth_wide_offset(o["D"] * (1300 + N_SLOT * 960 + 400), o["D"] * FS, 739e6, o["fc_c"], cell, o["clock_ratio"],
                               o["f_res"], 30.0, seed)
    d = found(cell, o["fc_c"])
    d.update(fc_programmed=(o["fc_c"] - o["f_res"]) / o["clock_ratio"], freq=o["f_res"], freq_fine=o["f_res"],
             freq_superfine=o["f_res"], frame_start=o["t0"] * o["clock_ratio"])
    return x, d, Y


def test_clock_offset_matches_planted_powers(oracle):
    """Over seeds 0-2 the largest errors were 0.59 % per RB, 0.14 % over the carrier and 0.04 % in RSRQ: inside the
    FLAT tolerances.  Turning the FOC rotation or the lateness ramp the wrong way breaks them, so the case checks both."""
    x, d, Y = offset_scenario(0)
    c = oracle.new_cell(**d)
    D = OFFSET["D"]
    late = np.rint(D * window_starts(oracle, c, x.size, D)) - D * window_starts(oracle, c, x.size, D)
    assert np.abs(late).max() > 0.4 and d["fc_programmed"] != d["fc_requested"] and d["frame_start"] % 1
    s_true = S.AMP ** 2 * np.abs(np.asarray(GAINS[:2])) ** 2

    def errors(m):
        return (np.abs(m["rb_rsrp"][:2, :25] * 128 / s_true[:, None] - 1).max(), np.abs(m["rsrp"][:2] * 128 / s_true - 1).max(),
                abs(m["rsrq"] / (25 * s_true[0] / planted_rssi(Y, 1, 25, 30.0)) - 1))

    e_rb, e_s, e_q = errors(measure(oracle, x, D * FS, 739e6, c))
    assert e_rb < TOL_RB and e_s < TOL_S and e_q < TOL_RSRQ, (e_rb, e_s, e_q)
    for signs in (dict(foc_sign=-1), dict(late_sign=-1)):
        e_rb, e_s, _ = errors(measure(oracle, x, D * FS, 739e6, c, **signs))
        assert e_rb > 2 * TOL_RB and e_s > 5 * TOL_S, (signs, e_rb, e_s)


def tolerance_spread(oracle, seeds=range(4)):
    """{case: largest relative error of (S per RB, S, RSRQ) over `seeds`}: how TOL_RB, TOL_S and TOL_RSRQ were set."""
    return {name: np.max([flat_errors(oracle, name, s)[1] for s in seeds], axis=0) for name in FLAT}


# ---- RsDl's full-band CRS -----------------------------------------------------------------------------------------------------
RSDL_DRIVER = r"""
#include <cstdio>
#include "chain_host.hpp"
int main() {
  const int rbs[] = {6, 15, 25, 50, 75, 100};
  for (int cp = 1; cp <= 2; cp++)
    for (int nid : {0, 137, 503})
      for (int R : rbs) {
        const lcs::RsDl a = R == 6 ? lcs::RsDl(nid, cp) : lcs::RsDl(nid, cp, R);
        for (int slot = 0; slot < 20; slot++)
          for (int sym : {0, 1, a.n_symb - 3}) {
            const lcs::cd* r = a.get(slot, sym);
            for (int m = 0; m < 2 * R; m++) std::printf("%d %d %d %d %d %d %.17g %.17g\n", cp, nid, R, slot, sym, m, r[m].real(), r[m].imag());
          }
      }
}
"""


def test_rsdl_full_band_crs(lcs, tmp_path):
    """RsDl(n_id_cell, cp, R) holds r(110 - R + m) for every m < 2R; its default (R = 6) is the oracle's 6-RB table, and
    the centre 12 of every R are that table too."""
    src = tmp_path / "rsdl.cpp"
    src.write_text(RSDL_DRIVER)
    exe = str(tmp_path / "rsdl")
    csrc = os.path.join(ROOT, "lte-cell-scanner_b200", "csrc")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + csrc, "-I/usr/local/cuda/include", str(src), "-o", exe,
                           "-L" + os.path.dirname(lcs.LIB_PATH), "-llcs_b200", "-Wl,-rpath," + os.path.dirname(lcs.LIB_PATH),
                           "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])
    rows = np.loadtxt(subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines())
    for cp in (1, 2):
        n_symb = 7 if cp == 1 else 6
        for nid in (0, 137, 503):
            rs6, _ = S.O.rs_dl(nid, cp)
            for R in (6, 15, 25, 50, 75, 100):
                sel = rows[(rows[:, 0] == cp) & (rows[:, 1] == nid) & (rows[:, 2] == R)]
                got = (sel[:, 6] + 1j * sel[:, 7]).reshape(20, 3, 2 * R)
                full = S.crs_full(nid, cp, R)[:, [0, 1, n_symb - 3]]
                assert np.array_equal(got, full), (cp, nid, R)
                centre = got[:, :, R - 6:R + 6]
                want = rs6.reshape(20, n_symb, 12)[:, [0, 1, n_symb - 3]]
                assert np.array_equal(centre, want), (cp, nid, R)


# ---- host planning of many cells under AddressSanitizer ----------------------------------------------------------------------
PLAN_DRIVER = r"""
#include <cstdio>
#include <cstdlib>
#include "carrier_plan.hpp"
int main(int argc, char** argv) {
  using namespace lcs::carrier;
  const int rbs[] = {6, 15, 25, 50, 75, 100}, Ds[] = {2, 4, 8, 16, 32}, ports[] = {1, 2, 4};
  std::vector<CellPlan> plans;                     // every plan kept, as lcs_carrier_cells keeps them
  int ok = 0, bad = 0;
  for (int D : Ds)
    for (int R : rbs)
      for (int cp = 1; cp <= 2; cp++)
        for (int P : ports)
          for (int v = 0; v < 3; v++) {
            lcs_cell c;
            lcs_cell_init(&c);
            c.cp_type = cp; c.n_id_1 = 45; c.n_id_2 = 2; c.n_ports = P; c.n_rb_dl = R;
            c.fc_requested = 739e6 + 100000.0 * v; c.fc_programmed = c.fc_requested - 7.0 * v;
            c.freq_superfine = 300.0 * v - 250.0; c.frame_start = 1000.25 + 4321.5 * v;
            CellPlan p;
            const std::string why = plan_cell(c, (uint64_t)D * 130000, D, D * 1.92e6, 739e6, 1.92e6, p);
            if (why.empty()) {
              ok++;
              for (size_t i = 1; i < p.q.size(); i++) if (p.q[i] <= p.q[i - 1]) return 3;
              for (double l : p.late) if (l < -0.5 || l > 0.5) return 4;
            } else {
              bad++;
            }
            plans.push_back(p);
          }
  std::printf("%d %d\n", ok, bad);
  lcs_cell c;                                      // the cell of argv: its windows
  lcs_cell_init(&c);
  c.cp_type = 1; c.n_id_1 = 45; c.n_id_2 = 2; c.n_ports = 2; c.n_rb_dl = 25;
  c.fc_requested = std::atof(argv[1]); c.fc_programmed = std::atof(argv[2]); c.freq_superfine = std::atof(argv[3]);
  c.frame_start = std::atof(argv[4]);
  CellPlan p;
  if (!plan_cell(c, std::atoll(argv[5]), 4, 4 * 1.92e6, 739e6, 1.92e6, p).empty()) return 5;
  for (size_t i = 0; i < p.q.size(); i++) std::printf("%lld %.17g\n", p.q[i], p.late[i]);
  return 0;
}
"""


def test_plan_many_cells_under_asan(lcs, oracle, tmp_path):
    """plan_cell, built with AddressSanitizer, lays out 540 cells of every rate, bandwidth, CP and port count, keeping
    every plan, without a stray access; the windows it gives a clock-offset cell are rint(D loc_t) of the oracle's
    extract_tfg timestamps, with their lateness."""
    csrc = os.path.join(ROOT, "lte-cell-scanner_b200", "csrc")
    libdir = os.path.dirname(lcs.LIB_PATH)
    src = tmp_path / "plan.cpp"
    src.write_text(PLAN_DRIVER)
    exe = str(tmp_path / "plan")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address", "-fno-omit-frame-pointer", "-I" + csrc,
                           "-I/usr/local/cuda/include", str(src), os.path.join(csrc, "carrier_plan.cpp"), "-o", exe,
                           "-L" + libdir, "-llcs_b200", "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64",
                           "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])
    x, d, _ = offset_scenario(0)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1")
    r = subprocess.run([exe, repr(d["fc_requested"]), repr(d["fc_programmed"]), repr(d["freq_superfine"]),
                        repr(d["frame_start"]), str(x.size)], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = r.stdout.splitlines()
    ok, bad = map(int, lines[0].split())
    # measurable: 6R < 64D, and every raster offset (0, 100, 200 kHz) inside the band
    want = sum(3 * 2 * 3 for D in (2, 4, 8, 16, 32) for R in (6, 15, 25, 50, 75, 100)
               if 6 * R < 64 * D and 200000 + 90000 * R <= D * FS / 2)
    assert (ok, ok + bad) == (want, 540)
    got = np.array([[float(v) for v in line.split()] for line in lines[1:]])
    ts = window_starts(oracle, oracle.new_cell(**d), x.size, 4)
    rows = [t for t in range(ts.size) if t % 7 in (0, 4)]
    q = np.rint(4 * ts[rows])
    assert np.array_equal(got[:, 0], q) and np.allclose(got[:, 1], q - 4 * ts[rows], atol=1e-9)


# ---- the kernels' resources -----------------------------------------------------------------------------------------------------
def test_carrier_kernels_compile_without_spills(tmp_path):
    """Every kernel of carrier.cu compiles for sm_90a with no stack frame and no spills (DESIGN.md section 4.10)."""
    csrc = os.path.join(ROOT, "lte-cell-scanner_b200", "csrc")
    r = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c", os.path.join(csrc, "carrier.cu"), "-o",
                        str(tmp_path / "carrier.o")], capture_output=True, text=True, check=True)
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 5 and len(frames) == 5, r.stderr            # the grid kernel in four formats, the measurement
    assert sum("carrier_grid_kernel" in e for e in entries) == 4 and sum("carrier_meas_kernel" in e for e in entries) == 1
    assert all(f == ("0", "0", "0") for f in frames), r.stderr


# ---- binding -------------------------------------------------------------------------------------------------------------------
LAYOUT_DRIVER = r"""
#include <stddef.h>
#include <stdio.h>
#include "lcs_carrier.h"
#define F(f) printf(#f " %zu\n", offsetof(lcs_carrier_meas, f));
int main(void) {
  printf("size %zu\n", sizeof(lcs_carrier_meas));
  F(rsrp) F(noise) F(sinr) F(rssi) F(rsrq) F(rb_rsrp) F(rb_noise) F(rb_rssi) F(n_pairs) F(n_rb)
  printf("chunk %d %d\n", LCS_CARRIER_CHUNK, LCS_CARRIER_LAUNCHES_PER_CHUNK);
  return 0;
}
"""


def test_carrier_prototypes_cover_header_and_library(lcs, tmp_path):
    """liblcs_carrier.so exports exactly the four functions of include/lcs_carrier.h, all bound with the header's
    prototypes; liblcs_b200.so, liblcs_meas.so and liblcs_psd.so export none of them.  CARRIER_MEAS has the C layout."""
    header = re.sub(r"/\*.*?\*/", " ", open(lcs.CARRIER_HEADER).read(), flags=re.S)
    names = set(re.findall(r"\b(lcs_\w+)\s*\(", header))
    assert names == {"lcs_carrier_create", "lcs_carrier_destroy", "lcs_carrier_cells", "lcs_carrier_timing_read"}
    assert set(lcs.prototypes(lcs.CARRIER_HEADER)) == names
    assert exported(lcs.CARRIER_LIB_PATH) == names
    for other in (lcs.LIB_PATH, lcs.MEAS_LIB_PATH, lcs.PSD_LIB_PATH):
        assert not exported(other) & names
    l = lcs.carrier_lib()
    V, I, U, D = C.c_void_p, C.c_int, C.c_uint32, C.c_double
    assert l.lcs_carrier_cells.argtypes == [V, V, I, I, C.c_uint64, D, D, V, U, D, V]
    assert l.lcs_carrier_create.argtypes == [V, V]
    assert l.lcs_carrier_timing_read.argtypes == [V, V, V]
    assert l.lcs_carrier_destroy.restype is None
    src = tmp_path / "layout.c"
    src.write_text(LAYOUT_DRIVER)
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = dict(line.split(" ", 1) for line in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(got["size"]) == lcs.CARRIER_MEAS.itemsize
    for f in lcs.CARRIER_MEAS.names:
        assert int(got[f]) == lcs.CARRIER_MEAS.fields[f][1], f
    assert got["chunk"] == "%d 2" % lcs.CARRIER_CHUNK


# ---- CLI argument errors with --measure-carrier (no device is touched) -----------------------------------------------------
def test_cli_measure_carrier_argument_errors(lcs, tmp_path):
    f = str(tmp_path / "rec.ci16")
    np.zeros((1000, 2), np.int16).tofile(f)
    wide = ["--wideband", f, "--fc-in", "739e6", "-s", "739e6"]
    cases = [
        (["-s", "739e6", "-l", "-d", str(tmp_path), "--measure-carrier"], "--measure-carrier needs --wideband"),
        (wide + ["--fs-in", "7.68e6", "--carrier-csv", str(tmp_path / "c.csv")], "--carrier-csv needs --measure-carrier"),
        (["--wideband", f, "--fc-in", "739e6", "--fs-in", "10e6", "--spectrum", str(tmp_path / "p.csv"), "--measure-carrier"],
         "--measure-carrier needs a search (-s)"),
        (wide + ["--fs-in", "11.52e6", "--measure-carrier"], "--measure-carrier needs --fs-in = D * 1.92 MHz"),
        (wide + ["--fs-in", "10e6", "--resample", "--measure-carrier"], "--measure-carrier needs --fs-in = D * 1.92 MHz"),
        (wide + ["--fs-in", "7.68e6", "--measure-carrier"], "holds 1000 ci16 samples"),
    ]
    for args, msg in cases:
        out = cellsearch(*args)
        assert out.returncode != 0 and msg in out.stderr, (args, out.stderr)
        assert "lcs_ctx_create" not in out.stderr
