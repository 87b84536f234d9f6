"""The host path every module on the whole-carrier grid shares (carrier_grid.cuh's grid_cells): for lcs_carrier_cells,
lcs_cir_cells, lcs_pcfich_cells and lcs_pdcch_cells, every invalid argument returns LCS_ERR_ARG, launches nothing and
names the function (and the cell at fault), and a valid call launches its kernels."""
import numpy as np
import pytest

from test_carrier_meas_gpu import FC_IN
from test_carrier_meas_host import FS, found, n_samples, synth_cell
from test_pdcch_gpu import found_pdcch

pytestmark = pytest.mark.gpu

# module: (handle class, library, record dtype, launches per chunk)
MODULES = {
    "carrier": ("CarrierMeasure", "carrier_lib", "CARRIER_MEAS", 2),
    "cir": ("CellImpulse", "cir_lib", "CIR_MEAS", 2),
    "pcfich": ("ControlFormat", "pcfich_lib", "PCFICH_MEAS", 2),
    "pdcch": ("ControlChannel", "pdcch_lib", "PDCCH_MEAS", 3),
}


@pytest.mark.parametrize("module", list(MODULES))
def test_invalid_arguments_launch_nothing(lcs, module):
    cls, lib_fn, dtype, launches = MODULES[module]
    D = 8
    cell = synth_cell(137, 2, 1, 25)
    d = found_pdcch(cell, FC_IN + 1e6) if module == "pdcch" else found(cell, FC_IN + 1e6)
    n = n_samples(D)
    iq = np.zeros((n, 2), np.int16)
    ctx = lcs.Context(0)
    h = getattr(lcs, cls)(ctx)
    fn = getattr(getattr(lcs, lib_fn)(), "lcs_%s_cells" % module)
    good = lcs.new_cell(**d)
    out = np.zeros(2, getattr(lcs, dtype))

    def call(cells, iq_ptr=iq.ctypes.data, fmt=lcs.IQ_CI16, n_in=n, fs_in=D * FS, fc_in=FC_IN, fs_prog=FS, out_ptr=out.ctypes.data,
             on_device=0, n_cells=None):
        arr = (lcs.Cell * len(cells))(*cells) if cells else None
        return fn(h._h, iq_ptr, fmt, on_device, n_in, fs_in, fc_in, arr, len(cells) if n_cells is None else n_cells, fs_prog,
                  out_ptr)

    def bad(**kw):
        c = lcs.new_cell(**d)
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    cases = {
        "null iq": dict(cells=[good], iq_ptr=None), "null out": dict(cells=[good], out_ptr=None),
        "null cells": dict(cells=[], n_cells=1), "format c128": dict(cells=[good], fmt=lcs.IQ_C128),
        "format 9": dict(cells=[good], fmt=9), "n_in 0": dict(cells=[good], n_in=0),
        "rate 10 Msps": dict(cells=[good], fs_in=10e6), "rate D=3": dict(cells=[good], fs_in=3 * FS),
        "rate D=64": dict(cells=[good], fs_in=64 * FS), "fc_in nan": dict(cells=[good], fc_in=float("nan")),
        "fs_programmed 0": dict(cells=[good], fs_prog=0.0), "unaligned device iq": dict(cells=[good], on_device=1, iq_ptr=8 * 1024 + 4),
        "cp_type": dict(cells=[good, bad(cp_type=0)]), "n_id_1": dict(cells=[good, bad(n_id_1=168)]),
        "n_id_2": dict(cells=[bad(n_id_2=3)]), "n_ports 3": dict(cells=[bad(n_ports=3)]),
        "n_rb_dl 20": dict(cells=[bad(n_rb_dl=20)]), "frame_start nan": dict(cells=[bad(frame_start=float("nan"))]),
        "freq_superfine inf": dict(cells=[bad(freq_superfine=float("inf"))]), "fc_programmed 0": dict(cells=[bad(fc_programmed=0.0)]),
        "fractional delta": dict(cells=[bad(fc_requested=FC_IN + 1e6 + 0.5)]),
        "window before the recording": dict(cells=[bad(frame_start=-400.0)]),
        "window past the recording": dict(cells=[good], n_in=n - 500 * D),
        "too wide for D": dict(cells=[bad(n_rb_dl=50)], fs_in=4 * FS),
        "outside the band": dict(cells=[bad(fc_requested=FC_IN + 6e6, fc_programmed=FC_IN + 6e6)]),
    }
    assert len(cases) == 25
    if module == "pdcch":
        cases.update({
            "phich_duration 0": dict(cells=[good, bad(phich_duration=0)]), "phich_duration 3": dict(cells=[bad(phich_duration=3)]),
            "phich_resource 0": dict(cells=[bad(phich_resource=0)]), "phich_resource 5": dict(cells=[good, bad(phich_resource=5)]),
        })
    for what, kw in cases.items():
        n0 = ctx.launches
        assert call(**kw) == 1, what                      # LCS_ERR_ARG
        assert ctx.launches == n0, what
        msg = lcs.lib().lcs_last_error(ctx._h).decode()
        assert msg.startswith("lcs_%s_cells: " % module), (what, msg)
        if what.startswith("phich"):
            assert ("cell 1: " if len(kw["cells"]) == 2 else "cell 0: ") + what.split()[0] in msg, msg
    n0 = ctx.launches
    assert call([good, good]) == 0 and ctx.launches - n0 == launches
    h.close()
    ctx.close()
