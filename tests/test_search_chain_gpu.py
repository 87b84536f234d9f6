"""The FP64 cell-search stages between the correlator and the MIB decoder (csrc/chain_gpu.cu: psss_kernel, sss_getce_kernel,
sss_ml_kernel, tfg_kernel and their host geometry) against the CPU oracle, off the nominal clock.

Every capture is synthetic (track_oracle/lte_dl_synth.synth_cu8: one oscillator drives the LO and the sample clock) and both
sides get the same fc_programmed / fs_programmed, so every position that scales with 16/FS_LTE*fs_programmed*k_factor and
every FOC phase that scales with fs*k is exercised with a factor that is not 1:

  A   2-port normal CP at fs*(1+40e-6); the strongest peak sits at ind < 153 (the +9600*k shift of the PSS positions).
      The reference derives frame_start from the unshifted ind and loses the cell; so must the device (DESIGN section 2).
  B   4-port extended CP, 25 RB, fs*(1-60e-6), fc_programmed = fc - 3 kHz.
  C   1-port normal CP, 100 RB, at 614 400 samples (64 PSS positions per peak), at a length where the peaks of one buffer
      have 64 and 65 positions, and at 960 000 samples (100 positions).
  D   three cells in one buffer: both CP types, the three n_id_2, one at ind < 153; the peaks of one launch have
      different numbers of PSS positions.
  E   frame_start on each side of the -0.5 / 19199.5 wrap, and on each side of extract_tfg's one-frame step back.

Found cells and peaks are compared field by field (compare_cells, used by the other search tests too), the FP64 stages'
intermediates to 1e-8 of their largest magnitude or better."""
import contextlib
import ctypes as C
import os
import sys

import numpy as np
import pytest

import lcs_b200
import lcs_oracle
from conftest import synth_cu8 as noise_cu8

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "track_oracle"))
import lte_dl_synth as S  # noqa: E402

FC = 739e6
FS_LTE16 = 30720000.0 / 16
TH2 = 3.0                  # THRESH2_N_SIGMA of CellSearch.cpp:528

# Every field of lcs_cell is in exactly one of these classes: exact, within an absolute bound, or within a bound
# relative to the oracle's value.
EXACT = ("fc_requested", "fc_programmed", "freq", "ind", "n_id_1", "n_id_2", "cp_type", "n_ports", "n_rb_dl",
         "phich_duration", "phich_resource", "sfn")
ABS = {"frame_start": 1e-9, "freq_fine": 1e-6, "freq_superfine": 1e-6}
REL = {"pss_pow": 1e-6}


def bound(k, y):
    """How far field k may lie from the oracle's value y.  A field in no class fails, so that a new field of lcs_cell
    cannot go unchecked."""
    if k in ABS:
        return ABS[k]
    if k in REL:
        return REL[k] * abs(y)
    if k not in EXACT:
        pytest.fail(f"lcs_cell field {k} has no comparison class")
    return 0


def cell_fields(c):
    """The field names of c's structure, those of its ctypes base classes first."""
    return [k for t in reversed(type(c).__mro__) for k, _ in vars(t).get("_fields_", ())]


def compare_cells(got, ref):
    """Device cells or peaks against the oracle's: the same ones in the same order, then every field within its bound.
    A double is NaN on both sides or on neither (peaks carry NaN frame_start and freq_*)."""
    assert [(c.n_id_cell(), c.n_id_2, c.ind) for c in got] == [(c.n_id_cell(), c.n_id_2, c.ind) for c in ref]
    for a, b in zip(got, ref):
        for k in cell_fields(a):
            x, y = getattr(a, k), getattr(b, k)
            lim = bound(k, y)
            if isinstance(y, float) and (np.isnan(x) or np.isnan(y)):
                assert np.isnan(x) and np.isnan(y), k
            else:
                assert abs(x - y) <= lim, k


def same_cells(a, b):
    """Two device results bit for bit: every field, doubles by their bytes (NaNs included)."""
    def record(c):
        return tuple(np.float64(v).tobytes() if isinstance(v, float) else v for v in (getattr(c, k) for k in cell_fields(c)))
    assert [record(c) for c in a] == [record(c) for c in b]


A_CELL = dict(n_id_cell=137, n_ports=2, cp_type=1, n_rb_dl=50, phich_duration=1, phich_resource=2, t0=8900.0, sfn0=100)
B_CELL = dict(n_id_cell=301, n_ports=4, cp_type=2, n_rb_dl=25, phich_duration=2, phich_resource=4, t0=12345.0, sfn0=7)
C_CELL = dict(n_id_cell=55, n_ports=1, cp_type=1, n_rb_dl=100, phich_duration=1, phich_resource=1, t0=500.0, sfn0=1000)
D_CELLS = [A_CELL, B_CELL,
           dict(n_id_cell=192, n_ports=1, cp_type=1, n_rb_dl=15, phich_duration=1, phich_resource=1, t0=5000.0, sfn0=512,
                gains=[0.7])]
E_CELL = dict(n_id_cell=88, n_ports=2, cp_type=1, n_rb_dl=6, phich_duration=1, phich_resource=1, sfn0=300)

# name: (cells, f_true, fc_programmed, fs_programmed, n_cap, planted ids the oracle decodes)
SCEN = {
    "A": ([A_CELL], -22000.0, FC, 1.92e6 * (1 + 40e-6), 153600, []),
    "B": ([B_CELL], 41000.0, FC - 3000.0, 1.92e6 * (1 - 60e-6), 153600, [301]),
    "C614400": ([C_CELL], 12000.0, FC, 1.92e6 * (1 + 10e-6), 614400, [55]),
    "C_straddle": ([C_CELL], 12000.0, FC, 1.92e6 * (1 + 10e-6), None, [55]),
    "C960000": ([C_CELL], 12000.0, FC, 1.92e6 * (1 + 10e-6), 960000, [55]),
    "D": (D_CELLS, -7000.0, FC + 1500.0, 1.92e6 * (1 + 25e-6), 153600, [192, 301]),
    "E_wrapped": ([dict(E_CELL, t0=1.0)], 3000.0, FC, 1.92e6 * (1 - 20e-6), 153600, [88]),
    "E_unwrapped": ([dict(E_CELL, t0=2.5)], 3000.0, FC, 1.92e6 * (1 - 20e-6), 153600, [88]),
    "E_no_step_back": ([dict(E_CELL, t0=19190.5)], 3000.0, FC, 1.92e6 * (1 - 20e-6), 153600, [88]),
    "E_step_back": ([dict(E_CELL, t0=19192.5)], 3000.0, FC, 1.92e6 * (1 - 20e-6), 153600, [88]),
}


def n_pss(peak, n_cap, fc_req, fc_prog):
    """Number of PSS positions sss_detect combines for a peak (searcher.cpp:549-563, itpp_ext mrange)."""
    k = (fc_req - peak.freq) / fc_prog
    loc = peak.ind + (9600 * k if peak.ind + 9 < 162 else 0)
    return int(np.floor((n_cap - 125 - 9 - loc) / (9600 * k))) + 1


def tfg_step_back(cell, fc_req, fc_prog, fs_prog):
    """extract_tfg steps its first symbol back one frame when this is > -0.5 (searcher.cpp:887-889)."""
    k = (fc_req - cell.freq_fine) / fc_prog
    loc = cell.frame_start + (10 if cell.cp_type == 1 else 32) * (16 / 30720000.0 * fs_prog) * k
    return loc - .01 * fs_prog * k


def tfg_fits(cell, n_cap, fc_req, fc_prog, fs_prog):
    """Whether every DFT window of extract_tfg lies inside the buffer (the reference does not check, searcher.cpp:903-920)."""
    k = (fc_req - cell.freq_fine) / fc_prog
    r = 16 / 30720000.0 * fs_prog * k
    n_symb = 7 if cell.cp_type == 1 else 6
    loc = cell.frame_start + (10 if n_symb == 7 else 32) * r
    if loc - .01 * fs_prog * k > -0.5:
        loc -= .01 * fs_prog * k
    for t in range(6 * 10 * 2 * n_symb + 2 * n_symb):
        if np.rint(loc) < 0 or np.rint(loc) + 128 > n_cap:
            return False
        loc += ((138 if t % 7 == 6 else 137) if n_symb == 7 else 160) * r
    return True


class Scenarios:
    """Captures and the oracle's results, made on first use and kept for the module."""

    def __init__(self, oracle):
        self.oracle = oracle
        self._cu8 = {}
        self._chain = {}

    def params(self, name):
        cells, f_true, fcp, fs, _, ids = SCEN[name]
        return dict(f=f_true + 5000.0 * np.arange(-2, 3), fcr=FC, fcp=fcp, fs=fs, f_true=f_true, ids=ids, cells=cells)

    def cu8(self, name):
        if name not in self._cu8:
            cells, f_true, fcp, fs, n, _ = SCEN[name]
            if name.startswith("C"):
                full = self._cu8.get("C960000")
                if full is None:
                    full = self._cu8["C960000"] = S.synth_cu8(960000, cells, f_true=f_true, fc=FC, fc_programmed=fcp,
                                                              fs_programmed=fs, snr_db=5.0, seed=3)
                n = n or self.straddle_length(full[:614400])
                self._cu8[name] = full[:n]
            else:
                self._cu8[name] = S.synth_cu8(n, cells, f_true=f_true, fc=FC, fc_programmed=fcp, fs_programmed=fs,
                                              snr_db=5.0, seed=3)
        return self._cu8[name]

    def straddle_length(self, cu8):
        """A length at which the peaks of C have 64 and 65 PSS positions: halfway between the lengths at which the first and
        the last of the 614 400-sample capture's peaks reach 65."""
        p = self.params("C614400")
        _, peaks = self.oracle.cell_search_one(S.to_c128(cu8), p["f"], FC, p["fcp"], p["fs"])
        lo = 614400
        while max(n_pss(q, lo, FC, p["fcp"]) for q in peaks) < 65:
            lo += 1
        hi = lo
        while min(n_pss(q, hi, FC, p["fcp"]) for q in peaks) < 65:
            hi += 1
        return (lo + hi) // 2

    def cap(self, name):
        return S.to_c128(self.cu8(name))

    def chain(self, name):
        """The oracle's CellSearch chain (cells, peaks) on the scenario's samples."""
        if name not in self._chain:
            p = self.params(name)
            self._chain[name] = self.oracle.cell_search_one(self.cap(name), p["f"], p["fcr"], p["fcp"], p["fs"])
        return self._chain[name]


@pytest.fixture(scope="module")
def scen(oracle):
    return Scenarios(oracle)


def test_compare_cells_classes():
    """Every field of a cell and of a peak (NaN past n_id_2) moved just inside its bound passes compare_cells; moved just
    past it, or NaN on one side only, it fails.  A field in no class fails with its name."""
    assert lcs_b200.Cell._fields_ == lcs_oracle.Cell._fields_
    cell = lcs_b200.Cell(fc_requested=FC, fc_programmed=FC - 3e3, pss_pow=2.5e3, ind=1410, freq=35e3, n_id_2=1, n_id_1=92,
                         cp_type=1, frame_start=8898.62, freq_fine=35227.9, freq_superfine=35228.46, n_ports=2, n_rb_dl=50,
                         phich_duration=1, phich_resource=2, sfn=100)
    peak = lcs_b200.Cell(fc_requested=FC, fc_programmed=FC - 3e3, pss_pow=170.25, ind=6990, freq=-5e3, n_id_2=0, n_id_1=-1,
                         frame_start=np.nan, freq_fine=np.nan, freq_superfine=np.nan, n_ports=-1, n_rb_dl=-1, sfn=-1)
    ref = [cell, peak]
    for i, c in enumerate(ref):
        for k in cell_fields(c):
            y = getattr(c, k)
            if isinstance(y, int):
                moves = [(y, True), (y + 1, False), (y - 1, False)]
            elif np.isnan(y):
                moves = [(y, True), (0.0, False)]
            else:           # an exact double (bound 0) fails one ulp away
                lim = bound(k, y)
                moves = [(np.nan, False)] + [(y + s * 0.99 * lim, True) for s in (1, -1)]
                moves += [(np.nextafter(y + s * 1.01 * lim, s * np.inf), False) for s in (1, -1)]
            for v, ok in moves:
                got = [type(x).from_buffer_copy(x) for x in ref]
                setattr(got[i], k, v)
                with contextlib.nullcontext() if ok else pytest.raises(AssertionError):
                    compare_cells(got, ref)

    class Wider(lcs_b200.Cell):
        _fields_ = [("extra", C.c_int32)]
    with pytest.raises(pytest.fail.Exception, match="field extra "):
        compare_cells([Wider()], [Wider()])


def check_stages(ctx, lcs, oracle, peak, cap, p):
    """sss_detect -> pss_sss_foe -> extract_tfg of one peak, device against oracle, every intermediate.  Each stage gets
    the oracle's output of the stage before on both sides: a freq_fine 1e-9 Hz apart turns the FOC phase at the end of the
    grid by a few 1e-10 rad, more than extract_tfg's own tolerance."""
    fcr, fcp, fs = p["fcr"], p["fcp"], p["fs"]
    o, od = oracle.sss_detect(peak, cap, TH2, fcr, fcp, fs)
    d, dd = ctx.sss_detect(lcs.new_cell(**peak.as_dict()), cap, TH2, fcr, fcp, fs)
    for k in ("h1_np", "h2_np", "h1_nrm", "h2_nrm", "h1_ext", "h2_ext"):
        assert np.abs(dd[k] - od[k]).max() <= 1e-10 * np.abs(od[k]).max(), k
    for k in ("log_lik_nrm", "log_lik_ext"):
        assert np.abs(dd[k] - od[k]).max() <= 1e-8 * np.abs(od[k]).max(), k
    assert (d.n_id_1, d.cp_type) == (o.n_id_1, o.cp_type)
    if o.n_id_1 < 0:
        assert np.isnan(d.frame_start)
        return o
    assert abs(d.frame_start - o.frame_start) <= 1e-9
    o2 = oracle.pss_sss_foe(o, cap, fcr, fcp, fs)
    d2 = ctx.pss_sss_foe(lcs.new_cell(**o.as_dict()), cap, fcr, fcp, fs)
    assert abs(d2.freq_fine - o2.freq_fine) <= 1e-6
    assert abs(ctx.pss_sss_foe(d, cap, fcr, fcp, fs).freq_fine - o2.freq_fine) <= 1e-6     # from the device's own frame_start
    if not tfg_fits(o2, cap.size, fcr, fcp, fs):
        with pytest.raises(lcs.LcsError):
            ctx.extract_tfg(lcs.new_cell(**o2.as_dict()), cap, fcr, fcp, fs)
        return o2
    o_tfg, o_ts = oracle.extract_tfg(o2, cap, fcr, fcp, fs)
    d_tfg, d_ts = ctx.extract_tfg(lcs.new_cell(**o2.as_dict()), cap, fcr, fcp, fs)
    assert d_tfg.shape == o_tfg.shape == (854 if o2.cp_type == 1 else 732, 72)
    assert np.array_equal(d_ts, o_ts)
    assert np.abs(d_tfg - o_tfg).max() <= 1e-11 * np.abs(o_tfg).max()
    return o2


def check_scenario_shape(name, peaks, cells, p, n_cap):
    """What each scenario is there to reach, on the oracle's side."""
    npss = [n_pss(q, n_cap, p["fcr"], p["fcp"]) for q in peaks]
    assert sorted(c.n_id_cell() for c in cells) == p["ids"]
    if name == "A":
        assert peaks[0].ind < 153
    elif name == "C614400":
        assert set(npss) == {64}
    elif name == "C_straddle":
        assert set(npss) == {64, 65}
    elif name == "C960000":
        assert set(npss) == {100}
    elif name == "D":
        assert len(set(npss)) > 1 and min(q.ind for q in peaks) < 153 and len({q.n_id_2 for q in peaks}) == 3
    elif name.startswith("E"):
        c = cells[0]
        step = tfg_step_back(c, p["fcr"], p["fcp"], p["fs"])
        if name == "E_wrapped":       # raw frame_start < -0.5, wrapped to the end of the frame
            assert c.frame_start > 19190
        elif name == "E_unwrapped":
            assert -0.5 < c.frame_start < 1 and step < -0.5
        elif name == "E_no_step_back":
            assert 19180 < c.frame_start and step < -0.5
        else:
            assert step > -0.5
    return npss


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCEN))
def test_stages_per_peak(ctx, lcs, oracle, scen, name):
    """Every peak of the oracle's peak search through sss_detect, pss_sss_foe and extract_tfg on both sides."""
    p = scen.params(name)
    cap = scen.cap(name)
    cells, peaks = scen.chain(name)
    check_scenario_shape(name, peaks, cells, p, cap.size)
    for q in peaks:
        check_stages(ctx, lcs, oracle, q, cap, p)
    if name == "A":     # the strongest peak: SSS decided on the shifted positions, frame_start from the unshifted ind
        o, _ = oracle.sss_detect(peaks[0], cap, TH2, FC, p["fcp"], p["fs"])
        t0 = A_CELL["t0"]
        assert o.n_id_1 * 3 + o.n_id_2 == 137 and abs(o.frame_start - (t0 - 2) - 9600) < 2


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["cu8", "c128"])
@pytest.mark.parametrize("name", list(SCEN))
def test_cell_search(ctx, scen, name, fmt):
    """The whole chain (lcs_cell_search[_cu8]) against the oracle's: peaks, then every field of every cell."""
    p = scen.params(name)
    o_cells, o_peaks = scen.chain(name)
    buf = scen.cu8(name) if fmt == "cu8" else scen.cap(name)
    cells, peaks = ctx.cell_search(buf, p["f"], p["fcr"], p["fcp"], p["fs"])
    compare_cells(peaks, o_peaks)
    compare_cells(cells, o_cells)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["B", "C_straddle", "D"])
def test_cell_search_c128_not_8bit_exact(ctx, oracle, scen, name):
    """Samples scaled by 0.999 are no longer (u8-127)/128: the chain reads them as c128 and still equals the oracle."""
    p = scen.params(name)
    cap = scen.cap(name) * 0.999
    o_cells, o_peaks = oracle.cell_search_one(cap, p["f"], p["fcr"], p["fcp"], p["fs"])
    assert sorted(c.n_id_cell() for c in o_cells) == p["ids"]
    cells, peaks = ctx.cell_search(cap, p["f"], p["fcr"], p["fcp"], p["fs"])
    compare_cells(peaks, o_peaks)
    compare_cells(cells, o_cells)


@pytest.mark.gpu
def test_cell_search_batch_off_nominal_clock(ctx, lcs, oracle, scen):
    """lcs_cell_search_batch_cu8 with scenario B's clock: B between noise buffers, more buffers than one chunk."""
    p = scen.params("B")
    o_cells, _ = scen.chain("B")
    noise = noise_cu8(0xD00D)
    assert oracle.cell_search_one(S.to_c128(noise), p["f"], p["fcr"], p["fcp"], p["fs"])[0] == []
    order = [1, 0, 0, 1] + [0] * 31 + [1, 0]
    bufs = np.stack([scen.cu8("B") if k else noise for k in order])
    plan = ctx.plan(153600, p["f"], 2, p["fcr"], p["fcp"], p["fs"], max_batch=32)
    got = plan.cell_search_batch_cu8(bufs)
    plan.close()
    for k, cells in zip(order, got):
        if k:
            compare_cells(cells, o_cells)
        else:
            assert cells == []


@pytest.fixture(scope="module")
def sweep_channels(scen):
    """Scenario B's clock at two channels with their own fc_programmed (the second made at 1.8 GHz), and noise."""
    p = scen.params("B")
    fc2 = 1.8e9
    b2 = S.synth_cu8(153600, [dict(B_CELL, n_id_cell=46, t0=7000.0)], f_true=p["f_true"], fc=fc2, fc_programmed=fc2 + 2000.0,
                     fs_programmed=p["fs"], snr_db=5.0, seed=4)
    noise = noise_cu8(0xFACE)
    return dict(iq=np.stack([scen.cu8("B"), noise, b2, noise]), fcr=np.array([FC, FC + 5e6, fc2, fc2 + 1e6]),
                fcp=np.array([p["fcp"], FC + 5e6, fc2 + 2000.0, fc2 + 1e6]), fs=p["fs"], f=p["f"], f_true=p["f_true"])


@pytest.mark.gpu
def test_sweep_search_off_nominal_clock(ctx, lcs, oracle, sweep_channels):
    """lcs_sweep_search_cu8 with fs_programmed and per-channel fc_programmed against the oracle's chain per channel."""
    ch = sweep_channels
    sw = lcs.Sweep(ctx, 153600)
    got = sw.search_cu8(ch["iq"], ch["fcr"], ch["f"], fs_programmed=ch["fs"], fc_programmed=ch["fcp"])
    sw.close()
    for i in range(len(ch["fcr"])):
        o_cells, _ = oracle.cell_search_one(S.to_c128(ch["iq"][i]), ch["f"], ch["fcr"][i], ch["fcp"][i], ch["fs"])
        assert [c.n_id_cell() for c in o_cells] == ([301] if i == 0 else [46] if i == 2 else [])
        compare_cells(got[i], o_cells)
        for a in got[i]:
            assert a.fc_requested == ch["fcr"][i] and a.fc_programmed == ch["fcp"][i]


@pytest.mark.gpu
def test_tracker_search_off_nominal_clock(ctx, lcs, oracle, sweep_channels):
    """lcs_tracker_search_cu8 and lcs_sweep_track_cu8 at the cells' offset (n_f = 1) against the oracle's chain at n_f = 1;
    frame_timing = frame_start*(FS_LTE/16)/(fs*k) + late with k = (fc_requested - offset)/fc_programmed."""
    ch = sweep_channels
    off = [ch["f_true"]] * len(ch["fcr"])
    late = [0.25, 0.0, -0.5, 1.5]
    sw = lcs.Sweep(ctx, 153600)
    got = sw.track_cu8(ch["iq"], off, ch["fcr"], fs_programmed=ch["fs"], fc_programmed=ch["fcp"], late=late)
    sw.close()
    for i in range(len(ch["fcr"])):
        fcr, fcp, fs = ch["fcr"][i], ch["fcp"][i], ch["fs"]
        o_cells, _ = oracle.cell_search_one(S.to_c128(ch["iq"][i]), np.array([off[i]]), fcr, fcp, fs)
        assert [c.n_id_cell() for c in o_cells] == ([301] if i == 0 else [46] if i == 2 else [])
        new = ctx.tracker_search_cu8(ch["iq"][i], off[i], fcr, fcp, fs, late[i])
        compare_cells([c for c, _ in new], o_cells)
        k = (fcr - off[i]) / fcp
        for (c, ft), b in zip(new, o_cells):
            assert abs(ft - (b.frame_start * FS_LTE16 / (fs * k) + late[i])) < 1e-9
        same_cells([a for a, _ in got[i]], [b for b, _ in new])
        assert [fa for _, fa in got[i]] == [fb for _, fb in new]


@pytest.mark.gpu
def test_grid_outside_the_buffer(ctx, lcs, oracle):
    """A buffer too short for one cell's 732-symbol extended-CP grid: that cell is dropped (extract_tfg raises), the other
    cell is still decoded and equals the oracle's chain, which is run only where its DFT windows lie inside the buffer."""
    fs, f_true, n = 1.92e6 * (1 + 15e-6), -15000.0, 125000
    cells = [dict(n_id_cell=250, n_ports=2, cp_type=1, n_rb_dl=50, phich_duration=1, phich_resource=1, t0=500.0, sfn0=40),
             dict(n_id_cell=114, n_ports=1, cp_type=2, n_rb_dl=25, phich_duration=1, phich_resource=1, t0=12000.0, sfn0=900)]
    cu8 = S.synth_cu8(n, cells, f_true=f_true, fc=FC, fs_programmed=fs, snr_db=5.0, seed=3)
    cap = S.to_c128(cu8)
    p = dict(f=f_true + 5000.0 * np.arange(-2, 3), fcr=FC, fcp=FC, fs=fs)
    x = oracle.xcorr_pss(cap, p["f"], 2, FC, FC, fs)
    z = oracle.calc_Z_th1(x["sp_incoherent"], x["n_comb_xc"], 2)
    o_peaks = oracle.peak_search(x["pow"], x["frq"], z, p["f"], FC, FC, x["single"], 2)
    # the oracle's chain, cell by cell, on the peaks whose grid fits (CellSearch.cpp:510-558)
    o_cells, dropped = [], []
    for q in o_peaks:
        o = check_stages(ctx, lcs, oracle, q, cap, p)
        if o.n_id_1 < 0:
            continue
        if not tfg_fits(o, n, FC, FC, fs):
            dropped.append(o.n_id_cell())
            continue
        tfg, ts = oracle.extract_tfg(o, cap, FC, FC, fs)
        o3, tfg_c, _ = oracle.tfoec(o, tfg, ts, FC, FC)
        o4, _ = oracle.decode_mib(o3, tfg_c)
        if o4.n_rb_dl != -1:
            o_cells.append(o4)
    assert dropped == [114] and [c.n_id_cell() for c in o_cells] == [250]
    for buf in (cu8, cap):
        got, peaks = ctx.cell_search(buf, p["f"], FC, FC, fs)
        compare_cells(peaks, o_peaks)
        compare_cells(got, o_cells)
