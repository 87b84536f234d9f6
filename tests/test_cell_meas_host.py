"""The per-cell measurement's contract (DESIGN.md section 4.9, include/lcs_meas.h) restated in float64 numpy on the oracle's
extract_tfg grid, checked against the powers planted in synthetic signals; the binding of liblcs_meas.so; and the CLI's
--measure argument errors (no device is touched)."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

from test_spectrum_host import exported
from test_channelizer_host import cellsearch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "track_oracle"))
import lte_dl_synth as S  # noqa: E402

FC = 739e6
FS = 1.92e6
QUANT = 2 * (1 / 128) ** 2 / 12          # cu8 rounding noise per complex sample (1/128 steps in I and Q)
GAINS = [1.0, 0.8 * np.exp(0.7j), 0.9 * np.exp(-1.1j), 0.7 * np.exp(2.2j)]   # lte_dl_synth's default port gains


# ---- the contract, restated -------------------------------------------------------------------------------------------------
def grid_of(oracle, cell, capbuf, fs_programmed=FS):
    """Y: the oracle's extract_tfg grid of a copy of `cell` (an oracle Cell) whose freq_fine is its freq_superfine."""
    g = oracle.new_cell(**{k: getattr(cell, k) for k, _ in oracle.Cell._fields_})
    g.freq_fine = cell.freq_superfine
    Y, _ = oracle.extract_tfg(g, capbuf, cell.fc_requested, cell.fc_programmed, fs_programmed)
    return Y


def crs_pairs(oracle, Y, n_id_cell, cp_type, port):
    """(h_a, h_b): h = Y conj(r) at every CRS RE of `port` and at the RE of the same port, symbol and subcarrier two slots
    later, for every such pair inside the grid."""
    n_symb = 7 if cp_type == 1 else 6
    n_slot = Y.shape[0] // n_symb
    rs, shift = oracle.rs_dl(n_id_cell, cp_type)
    syms = [0, n_symb - 3] if port < 2 else [1]
    ha, hb = [], []
    for t in range(n_slot - 2):
        for s in syms:
            for h, tt in ((ha, t), (hb, t + 2)):
                row = (tt % 20) * n_symb + s
                idx = int(shift[row, port]) + 6 * np.arange(12)
                h.append(Y[tt * n_symb + s, idx] * np.conj(rs[row]))
    return np.concatenate(ha), np.concatenate(hb)


def measure_grid(oracle, Y, n_id_cell, cp_type, n_ports):
    """One lcs_cell_meas as a dict, from the grid Y."""
    m = dict(rsrp=np.full(4, np.nan), noise=np.full(4, np.nan), sinr=np.full(4, np.nan), n_pairs=np.zeros(4, int))
    for p in range(n_ports):
        ha, hb = crs_pairs(oracle, Y, n_id_cell, cp_type, p)
        c = np.mean(ha * np.conj(hb))
        t = np.mean((np.abs(ha) ** 2 + np.abs(hb) ** 2) / 2)
        s = np.abs(c)
        m["rsrp"][p], m["noise"][p] = s / 128, (t - s) / 128
        m["sinr"][p] = s / (t - s) if t - s > 0 else np.inf
        m["n_pairs"][p] = ha.size
    n_symb = 7 if cp_type == 1 else 6
    rows = [r for r in range(Y.shape[0]) if r % n_symb in (0, n_symb - 3)]
    m["rssi"] = np.mean(np.sum(np.abs(Y[rows]) ** 2, axis=1) / 128)
    m["rsrq"] = 6 * m["rsrp"][0] / m["rssi"]
    return m


def measure(oracle, capbuf, cell, fs_programmed=FS):
    return measure_grid(oracle, grid_of(oracle, cell, capbuf, fs_programmed), cell.n_id_cell(), cell.cp_type, cell.n_ports)


# ---- synthetic scenarios with planted powers --------------------------------------------------------------------------------
def synth_cell(nid, n_ports, cp, scale=1.0, t0=1234.0):
    return dict(n_id_cell=nid, n_ports=n_ports, cp_type=cp, n_rb_dl=6, phich_duration=1, phich_resource=1, t0=t0, sfn0=0,
                gains=[scale * g for g in GAINS])


# name: (cells, f_true, error of freq_superfine, snr_db)
SCENARIOS = {
    "1port": ([synth_cell(137, 1, 1)], 0.0, 0.0, 10.0),
    "2port": ([synth_cell(137, 2, 1)], 0.0, 0.0, 10.0),
    "4port": ([synth_cell(137, 4, 1)], 0.0, 0.0, 10.0),
    "2port_extended": ([synth_cell(52, 2, 2)], 0.0, 0.0, 10.0),
    "4port_extended": ([synth_cell(52, 4, 2)], 0.0, 0.0, 10.0),
    "residual_offset": ([synth_cell(137, 2, 1)], 3000.0, 40.0, 10.0),          # 40 Hz left after freq_superfine
    "cochannel_other_mod3": ([synth_cell(100, 2, 1), synth_cell(101, 2, 1, 0.5)], 0.0, 0.0, 15.0),
    "cochannel_equal_mod3": ([synth_cell(100, 2, 1), synth_cell(106, 2, 1, 0.5)], 0.0, 0.0, 15.0),
}


def scenario(name, seed, n_cap=153600):
    """(cu8, oracle-style cell dicts with the planted truth)."""
    cells, f_true, err, snr = SCENARIOS[name]
    cu8 = S.synth_cu8(n_cap, cells, f_true=f_true, fc=FC, snr_db=snr, seed=seed)
    k = (FC - f_true) / FC
    found = []
    for c in cells:
        found.append(dict(fc_requested=FC, fc_programmed=FC, n_id_1=c["n_id_cell"] // 3, n_id_2=c["n_id_cell"] % 3,
                          cp_type=c["cp_type"], n_ports=c["n_ports"], frame_start=c["t0"] * k, freq=f_true,
                          freq_fine=f_true, freq_superfine=f_true + err, n_rb_dl=6))
    return cu8, found


def truth(name):
    """Per cell: S_p, N_p (in |Y|^2 units, i.e. x 128 of the outputs) and the RSSI sum over 72 REs, from the planted
    channel gains, snr_db, cu8 quantisation and the co-channel cell's REs that land on this cell's CRS."""
    cells, _, _, snr = SCENARIOS[name]
    a2 = S.AMP ** 2
    noise = a2 / 10 ** (snr / 10) + QUANT
    out = []
    for i, c in enumerate(cells):
        g = np.abs(np.asarray(c["gains"])) ** 2
        s = a2 * g[:c["n_ports"]]
        n = np.full(c["n_ports"], noise)
        for j, o in enumerate(cells):
            if j == i:
                continue
            go = np.abs(np.asarray(o["gains"])) ** 2
            if o["n_id_cell"] % 6 == c["n_id_cell"] % 6:
                n = n + a2 * go[:c["n_ports"]]          # the same ports' CRS on the same REs
            else:
                n = n + a2 * go[0]                      # data (port 0) on this cell's CRS REs
        rssi = 72 * noise + a2 * (60 * g[0] + 12 * g[1] if c["n_ports"] > 1 else 72 * g[0])
        for j, o in enumerate(cells):
            if j != i:
                go = np.abs(np.asarray(o["gains"])) ** 2
                rssi += a2 * (60 * go[0] + 12 * go[1])
        out.append(dict(S=s, N=n, rssi=rssi))
    return out


def oracle_cell(oracle, d):
    return oracle.new_cell(**d)


# Relative tolerances (S_p, N_p, RSSI) of the restatement against the planted truth: about twice the largest error seen
# over seeds 0-7 of each scenario, which was
#   1port 1.0 / 3.5 / 0.7 %, 2port 1.7 / 4.9 / 0.8 %, 4port 3.4 / 6.5 / 0.9 %, 2port_extended 1.4 / 4.5 / 1.3 %,
#   4port_extended 4.4 / 6.1 / 1.6 %, residual_offset 2.0 / 4.6 / 0.7 %, cochannel_other_mod3 22 / 3.9 / 1.5 %,
#   cochannel_equal_mod3 20 / 3.7 / 1.5 %.
# The co-channel S error is the weaker cell's, at an SINR of about -6 dB; 1440 pairs (ports 2 and 3) spread more than 2880.
TOL = {"1port": (0.03, 0.08, 0.02), "2port": (0.04, 0.10, 0.02), "4port": (0.07, 0.13, 0.02),
       "2port_extended": (0.03, 0.09, 0.03), "4port_extended": (0.09, 0.12, 0.035), "residual_offset": (0.04, 0.09, 0.02),
       "cochannel_other_mod3": (0.43, 0.08, 0.03), "cochannel_equal_mod3": (0.40, 0.08, 0.03)}


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_restatement_matches_planted_powers(oracle, name):
    for seed in (0, 1):
        cu8, found = scenario(name, seed)
        cap = S.to_c128(cu8)
        for d, tr in zip(found, truth(name)):
            m = measure(oracle, cap, oracle_cell(oracle, d))
            P = d["n_ports"]
            TOL_S, TOL_N, TOL_RSSI = TOL[name]
            assert np.all(np.abs(m["rsrp"][:P] * 128 / tr["S"] - 1) < TOL_S), (name, seed, m["rsrp"] * 128, tr["S"])
            assert np.all(np.abs(m["noise"][:P] * 128 / tr["N"] - 1) < TOL_N), (name, seed, m["noise"] * 128, tr["N"])
            assert abs(m["rssi"] * 128 / tr["rssi"] - 1) < TOL_RSSI, (name, seed, m["rssi"] * 128, tr["rssi"])
            assert np.all(np.isnan(m["rsrp"][P:])) and np.all(np.isnan(m["sinr"][P:])) and not m["n_pairs"][P:].any()
            assert list(m["n_pairs"][:P]) == [2880, 2880, 1440, 1440][:P]
            assert np.allclose(m["sinr"][:P], m["rsrp"][:P] / m["noise"][:P], rtol=1e-12)
            assert m["rsrq"] == 6 * m["rsrp"][0] / m["rssi"]


def test_cochannel_cells_are_told_apart(oracle):
    """Two cells on one carrier: the RSRP of each is its own (a factor 4 apart as planted), while the carrier's power, and
    so the RSSI, is shared."""
    for name in ("cochannel_other_mod3", "cochannel_equal_mod3"):
        cu8, found = scenario(name, 3)
        cap = S.to_c128(cu8)
        a, b = (measure(oracle, cap, oracle_cell(oracle, d)) for d in found)
        assert abs(a["rsrp"][0] / b["rsrp"][0] / 4 - 1) < 2 * TOL[name][0]
        assert abs(a["rssi"] / b["rssi"] - 1) < 0.01


def test_restatement_is_blind_to_a_common_phase(oracle):
    cu8, found = scenario("2port", 5)
    cell = oracle_cell(oracle, found[0])
    Y = grid_of(oracle, cell, S.to_c128(cu8))
    a = measure_grid(oracle, Y, cell.n_id_cell(), 1, 2)
    b = measure_grid(oracle, Y * np.exp(0.9j), cell.n_id_cell(), 1, 2)
    for k in ("rsrp", "noise", "sinr"):
        assert np.allclose(a[k][:2], b[k][:2], rtol=1e-12)


def tolerance_spread(oracle, seeds=range(8)):
    """{scenario: largest relative error of (S_p, N_p, RSSI) against the truth over `seeds`}: how TOL was set."""
    worst = {}
    for name in SCENARIOS:
        w = np.zeros(3)
        for seed in seeds:
            cu8, found = scenario(name, seed)
            cap = S.to_c128(cu8)
            for d, tr in zip(found, truth(name)):
                m = measure(oracle, cap, oracle_cell(oracle, d))
                P = d["n_ports"]
                w = np.maximum(w, [np.abs(m["rsrp"][:P] * 128 / tr["S"] - 1).max(),
                                   np.abs(m["noise"][:P] * 128 / tr["N"] - 1).max(), abs(m["rssi"] * 128 / tr["rssi"] - 1)])
        worst[name] = w
    return worst


# ---- binding -------------------------------------------------------------------------------------------------------------------
def test_meas_prototypes_cover_header_and_library(lcs):
    """liblcs_meas.so exports exactly the four functions of include/lcs_meas.h, all bound with the header's prototypes;
    liblcs_b200.so exports none of them."""
    header = re.sub(r"/\*.*?\*/", " ", open(lcs.MEAS_HEADER).read(), flags=re.S)
    names = set(re.findall(r"\b(lcs_\w+)\s*\(", header))
    assert names == {"lcs_meas_create", "lcs_meas_destroy", "lcs_meas_cells", "lcs_meas_timing_read"}
    assert set(lcs.prototypes(lcs.MEAS_HEADER)) == names
    assert exported(lcs.MEAS_LIB_PATH) == names
    assert not exported(lcs.LIB_PATH) & names
    l = lcs.meas_lib()
    V, I, U = C.c_void_p, C.c_int, C.c_uint32
    assert l.lcs_meas_cells.argtypes == [V, V, I, I, U, U, V, V, U, C.c_double, V]
    assert l.lcs_meas_create.argtypes == [V, V]
    assert l.lcs_meas_timing_read.argtypes == [V, V, V]
    assert l.lcs_meas_destroy.restype is None
    assert lcs.CELL_MEAS.itemsize == 128            # sizeof(lcs_cell_meas): 14 doubles and 4 uint32


# ---- CLI argument errors with --measure (no device is touched) ------------------------------------------------------------
def test_cli_measure_argument_errors(lcs, tmp_path):
    f = str(tmp_path / "rec.ci16")
    np.zeros((1000, 2), np.int16).tofile(f)
    cases = [
        (["--measure"], "must specify a start frequency"),
        (["-s", "739e6", "--measure"], "live capture / recording needs an rtl-sdr dongle"),
        (["--wideband", f, "--fc-in", "739e6", "--fs-in", "10e6", "--spectrum", str(tmp_path / "p.csv"), "--measure"],
         "--measure needs a search (-s)"),
        (["-s", "739e6", "-l", "-d", str(tmp_path), "--measure"], "cannot read"),
    ]
    for args, msg in cases:
        out = cellsearch(*args)
        assert out.returncode != 0 and msg in out.stderr, (args, out.stderr)
        assert "lcs_ctx_create" not in out.stderr
