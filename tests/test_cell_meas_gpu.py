"""lcs_meas on the H100 (DESIGN.md section 4.9): every field of every cell equal to the float64 restatement of
test_cell_meas_host to 1e-9 in all input formats, from host and device memory, many channels and cells per call and a
real capture; two launches per call; argument errors before any launch; and `CellSearch_b200 --wideband --measure` end to
end against the planted power."""
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from test_cell_meas_host import FS, S, TOL, measure, scenario

pytestmark = pytest.mark.gpu

FIELDS = ("rsrp", "noise", "sinr", "rssi", "rsrq")


def check_equal(dev, ref, rtol=1e-9):
    """Every field of one device record against the restatement's dict: NaN where it is NaN, 1e-9 relative elsewhere."""
    for k in FIELDS:
        a, b = np.atleast_1d(dev[k]).astype(np.float64), np.atleast_1d(ref[k]).astype(np.float64)
        assert np.array_equal(np.isnan(a), np.isnan(b)), (k, a, b)
        ok = ~np.isnan(b)
        assert np.all(np.abs(a[ok] - b[ok]) <= rtol * np.abs(b[ok])), (k, a, b)
    assert list(dev["n_pairs"]) == list(ref["n_pairs"])


@pytest.fixture(scope="module")
def channels(oracle):
    """Three 80 ms cu8 capture buffers [3][153600][2] (2 ports; 4 ports, extended CP; two co-channel cells with equal
    PCI mod 3), their cells and channels, and the restatement of every cell."""
    bufs, cells, ch = [], [], []
    for c, name in enumerate(("2port", "4port_extended", "cochannel_equal_mod3")):
        cu8, found = scenario(name, 11 + c)
        bufs.append(cu8)
        for d in found:
            cells.append(oracle.new_cell(**d))
            ch.append(c)
    cu8 = np.stack(bufs)
    ref = [measure(oracle, S.to_c128(cu8[c]), cell) for cell, c in zip(cells, ch)]
    return cu8, cells, np.array(ch), ref


def as_format(cu8, fmt):
    v = (cu8.astype(np.float64) - 127) / 128                     # exact in float32 too
    return {"cu8": cu8, "cf32": v.astype(np.float32), "c128": v}[fmt]


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("fmt", ["cu8", "cf32", "c128"])
def test_device_matches_restatement(lcs, ctx, channels, fmt, where):
    import torch
    cu8, cells, ch, ref = channels
    iq = as_format(cu8, fmt)
    if where == "device":
        iq = torch.from_numpy(iq).cuda()
    m = lcs.CellMeasure(ctx)
    out = m.measure(iq, cells, ch, FS, fmt)
    m.close()
    assert out.shape == (len(cells),)
    for d, r in zip(out, ref):
        check_equal(d, r)


def test_many_channels_and_cells_in_one_call(lcs, ctx, channels):
    """The same cells repeated over 24 channels in one call: each equals its own restatement, whatever its neighbours,
    and the call costs two launches."""
    cu8, cells, ch, ref = channels
    reps = 8
    iq = np.concatenate([cu8] * reps)
    all_cells = cells * reps
    all_ch = np.concatenate([ch + 3 * r for r in range(reps)])
    m = lcs.CellMeasure(ctx)
    m.timing_read()
    before = ctx.launches
    out = m.measure(iq, all_cells, all_ch, FS, "cu8")
    assert ctx.launches - before == 2
    ms, launches = m.timing_read()
    assert launches == 2 and ms > 0
    m.close()
    for i, d in enumerate(out):
        check_equal(d, ref[i % len(cells)])
        j = i % len(cells)
        assert out[i:i + 1].tobytes() == out[j:j + 1].tobytes()          # bitwise: a fixed summation order per cell


def test_capbuf_0000_cells_differ(lcs, ctx, oracle, capbuf0000):
    """The recording's two cells share 739 MHz; each gets its own RSRP, equal to the restatement."""
    fc = capbuf0000["fc"]
    cells, _ = ctx.cell_search(capbuf0000["capbuf"], lcs.f_search_set(fc, 120.0), fc, fc, FS)
    assert sorted(c.n_id_cell() for c in cells) == [271, 277]
    m = lcs.CellMeasure(ctx)
    out = m.measure(capbuf0000["cu8"], cells, None, FS, "cu8")
    out128 = m.measure(capbuf0000["capbuf"], cells, None, FS, "c128")
    m.close()
    for d, d2, c in zip(out, out128, cells):
        r = measure(oracle, capbuf0000["capbuf"], c)
        check_equal(d, r)
        check_equal(d2, r)
        assert np.all(d["rsrp"][:c.n_ports] > 0)
    assert abs(10 * np.log10(out[0]["rsrp"][0] / out[1]["rsrp"][0])) > 1.0


def test_timing_reports_two_launches_per_call(lcs, ctx, channels):
    cu8, cells, ch, _ = channels
    m = lcs.CellMeasure(ctx)
    for k in (1, 3):
        for _ in range(k):
            m.measure(cu8, cells, ch, FS, "cu8")
        ms, launches = m.timing_read()
        assert launches == 2 * k and ms > 0
    m.measure(cu8, [], None, FS, "cu8")                        # no cells: nothing launched
    assert m.timing_read() == (0.0, 0)
    m.close()


def test_invalid_arguments_launch_nothing(lcs, ctx, channels):
    import torch
    cu8, cells, ch, _ = channels
    l = lcs.meas_lib()
    m = lcs.CellMeasure(ctx)
    out = np.zeros(len(cells), lcs.CELL_MEAS)
    good = dict(iq=cu8.ctypes.data, fmt=lcs.IQ_CU8, dev=0, n_ch=3, n_cap=cu8.shape[1], ch=np.ascontiguousarray(ch, np.uint32),
                fs=FS, out=out.ctypes.data)

    def call(cells_=None, **kw):
        a = dict(good, **kw)
        cs = cells if cells_ is None else cells_
        arr = (lcs.Cell * len(cs))(*[lcs._copy(c) if isinstance(c, lcs.Cell) else lcs.new_cell(**c.as_dict()) for c in cs])
        return l.lcs_meas_cells(m._h, a["iq"], a["fmt"], a["dev"], a["n_ch"], a["n_cap"], arr, a["ch"].ctypes.data,
                                len(cs), a["fs"], a["out"])

    def with_cell(**kw):
        c = [lcs.new_cell(**x.as_dict()) for x in cells]
        for k, v in kw.items():
            setattr(c[1], k, v)
        return c

    d_iq = torch.from_numpy(cu8).cuda()
    assert call() == 0
    before = ctx.launches
    bad = [
        dict(iq=None), dict(out=None), dict(fmt=lcs.IQ_CI16), dict(fmt=lcs.IQ_CS8), dict(fmt=7), dict(n_ch=0),
        dict(n_cap=0), dict(fs=0.0), dict(fs=float("nan")), dict(ch=np.ascontiguousarray(ch + 1, np.uint32)),
        dict(n_ch=2), dict(n_cap=100000), dict(dev=1, iq=d_iq.data_ptr() + 2),
        dict(cells_=with_cell(cp_type=0)), dict(cells_=with_cell(cp_type=3)), dict(cells_=with_cell(n_ports=3)),
        dict(cells_=with_cell(n_ports=0)), dict(cells_=with_cell(n_ports=-1)), dict(cells_=with_cell(frame_start=np.nan)),
        dict(cells_=with_cell(freq_superfine=np.inf)), dict(cells_=with_cell(n_id_1=-1)), dict(cells_=with_cell(n_id_2=3)),
        dict(cells_=with_cell(fc_requested=np.nan)), dict(cells_=with_cell(frame_start=1e6)),
        dict(cells_=with_cell(frame_start=-50000.0)),
    ]
    for kw in bad:
        assert call(**kw) == 1, (kw, lcs.lib().lcs_last_error(ctx._h))
        assert ctx.launches == before, kw
    assert l.lcs_meas_cells(m._h, cu8.ctypes.data, lcs.IQ_CU8, 0, 3, cu8.shape[1], None, None, 2, FS, None) == 1
    assert l.lcs_meas_cells(None, cu8.ctypes.data, lcs.IQ_CU8, 0, 3, cu8.shape[1], None, None, 0, FS, None) == 1
    assert l.lcs_meas_timing_read(m._h, None, None) == 1
    assert ctx.launches == before
    assert m.timing_read()[1] == 2                               # only the good call
    m.close()


def table_rows(stdout):
    """The cell table's rows as lists of fields."""
    lines = stdout.splitlines()
    i = next(k for k, s in enumerate(lines) if s.startswith("CID A"))
    return [s.split() for s in lines[i + 1:] if re.match(r"^\s*\d+\s+\d\s", s)]


def test_cli_wideband_measure(lcs, ctx, tmp_path):
    """`CellSearch_b200 --wideband --measure` on a 7.68 Msps recording of two carriers: each cell's RSRP is the power
    planted on its port-0 CRS in the recording's dBFS, and every other column equals the run without --measure."""
    host = os.path.join(ROOT, "lte-cell-scanner_b200", "host")
    subprocess.check_call(["make", "-C", host, "-s"])
    fs_in, fc_in, D, scale = 7.68e6, 739e6, 4, 4096.0
    n = 153599 * D + lcs.chan_design_taps(fs_in).size // 2 + 1
    a = dict(n_id_cell=211, n_ports=2, cp_type=1, n_rb_dl=75, phich_duration=1, phich_resource=3, t0=3000.0, sfn0=12)
    b = dict(n_id_cell=58, n_ports=1, cp_type=1, n_rb_dl=25, phich_duration=1, phich_resource=1, t0=9000.0, sfn0=3)
    rel = {211: 1.0, 58: 0.25}
    path = str(tmp_path / "wide.ci16")
    S.synth_wide_ci16(n, fs_in, fc_in, [(fc_in + 1.5e6, [a], rel[211]), (fc_in - 2.0e6, [b], rel[58])], f_true=2000.0,
                      snr_db=15, seed=43).tofile(path)
    args = [os.path.join(host, "CellSearch_b200"), "--wideband", path, "--fs-in", "7.68e6", "--fc-in", "739e6",
            "-s", "736.2e6", "-e", "741.8e6", "-p", "15"]
    plain = subprocess.run(args, capture_output=True, text=True, timeout=300)
    meas = subprocess.run(args + ["--measure"], capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0 and meas.returncode == 0, plain.stderr + meas.stderr
    assert "RSRP[dBFS] RSRQ[dB] SINR[dB]" in meas.stdout and "RSRP" not in plain.stdout
    p_rows, m_rows = table_rows(plain.stdout), table_rows(meas.stdout)
    assert sorted(r[0] for r in p_rows) == ["211", "58"]
    assert [r[:-3] for r in m_rows] == p_rows
    # the port-0 CRS carries AMP^2 |g_0|^2 / 128 per sample (g_0 = 1), scaled by rel and (scale / 32768)^2
    tol_db = 10 * np.log10(1 + TOL["2port"][0]) + 0.1           # the restatement's spread and the channel filter's ripple
    for r in m_rows:
        planted = 10 * np.log10(rel[int(r[0])] * S.AMP ** 2 / 128 * (scale / 32768) ** 2)
        rsrp, rsrq, sinr = (float(v) for v in r[-3:])
        assert abs(rsrp - planted) < tol_db, (r, planted)
        assert np.isfinite(rsrq) and rsrq < 0 and sinr > 5, r
