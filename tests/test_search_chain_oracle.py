"""The oracle's cell-search chain (oracle.cell_search_one) off the nominal clock, against the truth planted in synthetic
captures (track_oracle/lte_dl_synth.synth_cu8, whose LO and sample clock share one oscillator).  The GPU suite
(test_search_chain_gpu.py) takes this oracle as its yardstick on the same scenarios; this file checks the yardstick."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "track_oracle"))
import lte_dl_synth as S  # noqa: E402

FC = 739e6

CASES = {
    # 4-port extended CP, slow clock, fc_programmed 3 kHz below fc
    "ext_cp_4port": (dict(n_id_cell=301, n_ports=4, cp_type=2, n_rb_dl=25, phich_duration=2, phich_resource=4, t0=12345.0,
                          sfn0=7), 41000.0, FC - 3000.0, 1.92e6 * (1 - 60e-6), 153600),
    # 100 PSS positions per peak
    "long_capture": (dict(n_id_cell=55, n_ports=1, cp_type=1, n_rb_dl=100, phich_duration=1, phich_resource=1, t0=500.0,
                          sfn0=1000), 12000.0, FC, 1.92e6 * (1 + 10e-6), 960000),
    # 2-port normal CP, fast clock, peak away from the start of the half frame
    "normal_cp_2port": (dict(n_id_cell=137, n_ports=2, cp_type=1, n_rb_dl=50, phich_duration=1, phich_resource=2, t0=3333.0,
                             sfn0=100), -22000.0, FC, 1.92e6 * (1 + 40e-6), 153600),
}


def capture(cell, f_true, fcp, fs, n):
    return S.to_c128(S.synth_cu8(n, [cell], f_true=f_true, fc=FC, fc_programmed=fcp, fs_programmed=fs, snr_db=5.0, seed=3))


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_decodes_the_planted_cell(oracle, name):
    cell, f_true, fcp, fs, n = CASES[name]
    cap = capture(cell, f_true, fcp, fs, n)
    cells, peaks = oracle.cell_search_one(cap, f_true + 5000.0 * np.arange(-2, 3), FC, fcp, fs)
    assert len(cells) == 1
    c = cells[0]
    assert c.n_id_cell() == cell["n_id_cell"] and c.cp_type == cell["cp_type"] and c.n_ports == cell["n_ports"]
    assert (c.n_rb_dl, c.phich_duration, c.phich_resource) == (cell["n_rb_dl"], cell["phich_duration"], cell["phich_resource"])
    assert c.sfn == cell["sfn0"]
    assert abs(c.freq_superfine - f_true) < 5.0
    # the frame starts 2 samples before t0 in the searcher's convention (2-sample DFT offset), on the capture's own clock
    k = (FC - f_true) / fcp
    assert abs(c.frame_start - (cell["t0"] - 2) * (fs / 1.92e6 * k)) < 1.0


def test_oracle_frame_start_from_the_unshifted_peak(oracle):
    """A peak at ind < 153 has its PSS positions moved one half frame on (searcher.cpp:549-563), but frame_start is derived
    from the unshifted ind (searcher.cpp:735): it comes out half a frame late and the MIB cannot be decoded.  The GPU chain
    reproduces this."""
    cell = dict(n_id_cell=137, n_ports=2, cp_type=1, n_rb_dl=50, phich_duration=1, phich_resource=2, t0=8900.0, sfn0=100)
    f_true, fs = -22000.0, 1.92e6 * (1 + 40e-6)
    cap = capture(cell, f_true, FC, fs, 153600)
    cells, peaks = oracle.cell_search_one(cap, f_true + 5000.0 * np.arange(-2, 3), FC, FC, fs)
    assert cells == []
    assert peaks[0].ind < 153 and peaks[0].n_id_2 == 2
    o, _ = oracle.sss_detect(peaks[0], cap, 3.0, FC, FC, fs)
    assert o.n_id_cell() == 137 and o.cp_type == 1
    assert abs(o.frame_start - 18499.28) < 0.01
    k = (FC - peaks[0].freq) / FC
    half = 9600 * (fs / 1.92e6) * k * k
    assert abs(o.frame_start - half - (cell["t0"] - 2) * (fs / 1.92e6 * k)) < 1.0
