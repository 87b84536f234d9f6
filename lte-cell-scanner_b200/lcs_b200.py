"""ctypes binding of liblcs_b200.so - the C ABI declared in include/lcs_b200.h.

This module is plumbing for tests/, bench.py and __graft_entry__.py: every call goes through the
same `extern "C"` entry points a C++/IT++ host would bind (INTEGRATION.md).  There is no CPU
fallback: importing works anywhere (the symbols are checked), but every compute call needs an
H100 and raises LcsError otherwise.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LCS_B200_LIB") or os.path.join(HERE, "liblcs_b200.so")
HEADER = os.path.join(HERE, "..", "include", "lcs_b200.h")

IQ_CF32, IQ_CU8, IQ_C128 = 0, 1, 2
KERNEL_AUTO, KERNEL_FP32, KERNEL_TC = 0, 1, 2
N_FOLD = 9600


class LcsError(RuntimeError):
    pass


class Cell(C.Structure):
    """lcs_cell: POD mirror of the reference's class Cell (include/common.h.in:101-129)."""
    _fields_ = [
        ("fc_requested", C.c_double), ("fc_programmed", C.c_double), ("pss_pow", C.c_double),
        ("ind", C.c_int32), ("freq", C.c_double), ("n_id_2", C.c_int32), ("n_id_1", C.c_int32),
        ("cp_type", C.c_int32), ("frame_start", C.c_double), ("freq_fine", C.c_double),
        ("freq_superfine", C.c_double), ("n_ports", C.c_int32), ("n_rb_dl", C.c_int32),
        ("phich_duration", C.c_int32), ("phich_resource", C.c_int32), ("sfn", C.c_int32),
    ]

    def n_id_cell(self):
        return self.n_id_2 + 3 * self.n_id_1 if (self.n_id_1 >= 0 and self.n_id_2 >= 0) else -1

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def build(force=False):
    """Compile the CUDA library in-tree (nvcc cross-compiles sm_90a without a GPU)."""
    if force or not os.path.exists(LIB_PATH):
        subprocess.check_call(["make", "-C", HERE, "-s", "-j8"])
    else:
        subprocess.check_call(["make", "-C", HERE, "-s", "-j8"])  # make is incremental
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LcsError("liblcs_b200.so is not built (run `make -C lte-cell-scanner_b200`); "
                           "there is no CPU fallback")
        _lib = C.CDLL(LIB_PATH)
        _lib.lcs_version.restype = C.c_char_p
        _lib.lcs_last_error.restype = C.c_char_p
        _lib.lcs_last_error.argtypes = [C.c_void_p]
        _lib.lcs_launch_count.restype = C.c_uint64
        _lib.lcs_launch_count.argtypes = [C.c_void_p]
        _lib.lcs_xcorr_plan_n_comb_xc.restype = C.c_uint16
        _lib.lcs_xcorr_plan_n_comb_sp.restype = C.c_uint16
        _lib.lcs_xcorr_plan_n_comb_xc.argtypes = [C.c_void_p]
        _lib.lcs_xcorr_plan_n_comb_sp.argtypes = [C.c_void_p]
        _lib.lcs_xcorr_plan_kernel.argtypes = [C.c_void_p, C.c_int]
        _lib.lcs_ctx_destroy.argtypes = [C.c_void_p]
        _lib.lcs_xcorr_plan_destroy.argtypes = [C.c_void_p]
        _lib.lcs_xcorr_plan_timing_enable.argtypes = [C.c_void_p, C.c_int]
        _lib.lcs_xcorr_plan_timing_read.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.lcs_framer_destroy.argtypes = [C.c_void_p]
        _lib.lcs_sweep_destroy.argtypes = [C.c_void_p]
        _lib.lcs_sweep_destroy.restype = None
        _lib.lcs_framer_destroy.restype = None
        _lib.lcs_framer_request.argtypes = [C.c_void_p]
        _lib.lcs_framer_request.restype = None
        _lib.lcs_framer_sample_time.argtypes = [C.c_void_p]
        _lib.lcs_framer_sample_time.restype = C.c_double
        _lib.lcs_track_destroy.argtypes = [C.c_void_p]
        _lib.lcs_track_destroy.restype = None
        _lib.lcs_track_add_cell.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_double]
        _lib.lcs_track_push_cu8.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        _lib.lcs_track_frequency_offset.argtypes = [C.c_void_p, C.c_void_p]
        _lib.lcs_track_read.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
        _lib.lcs_track_sample_time.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        _lib.lcs_track_timing_read.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _chk(rc, ctx=None):
    if rc != 0:
        msg = lib().lcs_last_error(ctx).decode() if ctx else lib().lcs_last_error(None).decode()
        raise LcsError("lcs_b200 error %d: %s" % (rc, msg))


def new_cell(**kw):
    c = Cell()
    lib().lcs_cell_init(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _copy(c):
    o = Cell()
    C.memmove(C.byref(o), C.byref(c), C.sizeof(Cell))
    return o


def f_search_set(freq_start, ppm):
    n = C.c_uint32(0)
    _chk(lib().lcs_f_search_set(C.c_double(freq_start), C.c_double(ppm), None, C.byref(n)))
    out = np.zeros(n.value)
    _chk(lib().lcs_f_search_set(C.c_double(freq_start), C.c_double(ppm), _p(out), C.byref(n)))
    return out


def calc_z_th1(sp_incoherent, n_comb_xc, ds_comb_arm):
    s = np.ascontiguousarray(sp_incoherent, np.float64)
    z = np.zeros_like(s)
    _chk(lib().lcs_calc_z_th1(_p(s), C.c_uint32(s.size), C.c_uint16(n_comb_xc), C.c_uint8(ds_comb_arm), _p(z)))
    return z


def peak_search(pw, frq, z_th1, f_set, fc_requested, fc_programmed, single_planar, ds_comb_arm, max_cells=256):
    """pw/frq: [3][9600]; single_planar: [3][n_f][9600] float32."""
    pw = np.ascontiguousarray(pw, np.float64); frq = np.ascontiguousarray(frq, np.int32)
    z = np.ascontiguousarray(z_th1, np.float64); f = np.ascontiguousarray(f_set, np.float64)
    sp = np.ascontiguousarray(single_planar, np.float32)
    cells = (Cell * max_cells)(); n = C.c_uint32(0)
    _chk(lib().lcs_peak_search(_p(pw), _p(frq), _p(z), _p(f), C.c_uint32(f.size), C.c_double(fc_requested),
                               C.c_double(fc_programmed), _p(sp), C.c_uint8(ds_comb_arm), cells,
                               C.c_uint32(max_cells), C.byref(n)))
    return [_copy(cells[i]) for i in range(min(n.value, max_cells))]


def dedup(cells):
    n = len(cells)
    arr = (Cell * max(n, 1))(*cells); out = (Cell * max(n, 1))(); m = C.c_uint32(0)
    _chk(lib().lcs_dedup(arr, C.c_uint32(n), out, C.byref(m)))
    return [_copy(out[i]) for i in range(m.value)]


def tfoec(cell, tfg, ts, fc_requested, fc_programmed):
    """searcher.h:101-112 - host stage (no GPU needed).  tfg: [n_ofdm][72] complex128."""
    n = ts.size
    g = np.asfortranarray(tfg, np.complex128)                        # column-major cmat for the ABI
    ts = np.ascontiguousarray(ts, np.float64)
    gc = np.zeros((n, 72), np.complex128, order="F"); tsc = np.zeros(n); out = Cell()
    _chk(lib().lcs_tfoec(None, C.byref(cell), C.c_void_p(g.ctypes.data), _p(ts), C.c_uint32(n),
                         C.c_double(fc_requested), C.c_double(fc_programmed), C.c_void_p(gc.ctypes.data), _p(tsc),
                         C.byref(out)))
    return out, np.ascontiguousarray(gc), tsc


def decode_mib(cell, tfg):
    """searcher.h:115-119 - host stage (no GPU needed)."""
    g = np.asfortranarray(tfg, np.complex128)
    out = Cell()
    _chk(lib().lcs_decode_mib(None, C.byref(cell), C.c_void_p(g.ctypes.data), C.c_uint32(g.shape[0]), C.byref(out)))
    return out


class Context:
    """lcs_ctx: one per process per GPU."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        _chk(lib().lcs_ctx_create(int(device), C.byref(self._h)))

    def close(self):
        if self._h:
            lib().lcs_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launches(self):
        return int(lib().lcs_launch_count(self._h))

    # ---- searcher.h:22-41 ----
    def xcorr_pss(self, capbuf, f_set, ds_comb_arm, fc_requested, fc_programmed, fs_programmed,
                  want_incoherent=True, want_xc=False, want_sp=False):
        capbuf = np.ascontiguousarray(capbuf, np.complex128)
        f = np.ascontiguousarray(f_set, np.float64)
        n_cap, n_f = capbuf.size, f.size
        pw = np.zeros((9600, 3)); frq = np.zeros((9600, 3), np.int32)      # column-major mat(3,9600)
        single = np.zeros((3, 9600, n_f), np.float32)
        inc = np.zeros((3, 9600, n_f), np.float32) if want_incoherent else None
        spi = np.zeros(9600)
        xc = np.zeros((3, n_cap - 136, n_f), np.complex64) if want_xc else None
        sp = np.zeros(((n_cap - 273) // 9600) * 9600) if want_sp else None
        ncx, ncs = C.c_uint16(0), C.c_uint16(0)
        _chk(lib().lcs_xcorr_pss(self._h, _p(capbuf), C.c_uint32(n_cap), _p(f), C.c_uint32(n_f), C.c_uint8(ds_comb_arm),
                                 C.c_double(fc_requested), C.c_double(fc_programmed), C.c_double(fs_programmed),
                                 _p(pw), _p(frq), _p(single), _p(inc), _p(spi), _p(xc), _p(sp), C.byref(ncx), C.byref(ncs)),
             self._h)
        return dict(pow=pw.T.copy(), frq=frq.T.copy(), single=single, incoherent=inc, sp_incoherent=spi, xc=xc, sp=sp,
                    n_comb_xc=ncx.value, n_comb_sp=ncs.value)

    def sss_detect(self, cell, capbuf, thresh2_n_sigma, fc_requested, fc_programmed, fs_programmed):
        capbuf = np.ascontiguousarray(capbuf, np.complex128)
        out = Cell()
        h1_np = np.zeros(62); h2_np = np.zeros(62)
        arrs = [np.zeros(62, np.complex128) for _ in range(4)]
        lln = np.zeros((2, 168)); lle = np.zeros((2, 168))
        _chk(lib().lcs_sss_detect(self._h, C.byref(cell), _p(capbuf), C.c_uint32(capbuf.size), C.c_double(thresh2_n_sigma),
                                  C.c_double(fc_requested), C.c_double(fc_programmed), C.c_double(fs_programmed),
                                  C.byref(out), _p(h1_np), _p(h2_np), _p(arrs[0]), _p(arrs[1]), _p(arrs[2]), _p(arrs[3]),
                                  _p(lln), _p(lle)), self._h)
        d = dict(h1_np=h1_np, h2_np=h2_np, h1_nrm=arrs[0], h2_nrm=arrs[1], h1_ext=arrs[2], h2_ext=arrs[3],
                 log_lik_nrm=lln.T.copy(), log_lik_ext=lle.T.copy())
        return out, d

    def pss_sss_foe(self, cell, capbuf, fc_requested, fc_programmed, fs_programmed):
        capbuf = np.ascontiguousarray(capbuf, np.complex128)
        out = Cell()
        _chk(lib().lcs_pss_sss_foe(self._h, C.byref(cell), _p(capbuf), C.c_uint32(capbuf.size), C.c_double(fc_requested),
                                   C.c_double(fc_programmed), C.c_double(fs_programmed), C.byref(out)), self._h)
        return out

    def extract_tfg(self, cell, capbuf, fc_requested, fc_programmed, fs_programmed):
        capbuf = np.ascontiguousarray(capbuf, np.complex128)
        tfg = np.zeros(72 * 854, np.complex128); ts = np.zeros(854); n = C.c_uint32(0)
        _chk(lib().lcs_extract_tfg(self._h, C.byref(cell), _p(capbuf), C.c_uint32(capbuf.size), C.c_double(fc_requested),
                                   C.c_double(fc_programmed), C.c_double(fs_programmed), _p(tfg), _p(ts), C.byref(n)),
             self._h)
        n = n.value
        return tfg[:72 * n].reshape(72, n).T.copy(), ts[:n].copy()      # cmat(n_ofdm,72) column-major

    def tfoec(self, cell, tfg, ts, fc_requested, fc_programmed):
        return tfoec(cell, tfg, ts, fc_requested, fc_programmed)

    def decode_mib(self, cell, tfg):
        return decode_mib(cell, tfg)

    def cell_search(self, capbuf, f_set, fc_requested, fc_programmed, fs_programmed, max_cells=64):
        """One centre frequency of CellSearch's main loop.  capbuf: complex128 [n_cap] or uint8 [n_cap,2]."""
        f = np.ascontiguousarray(f_set, np.float64)
        cells = (Cell * max_cells)(); peaks = (Cell * max_cells)()
        n = C.c_uint32(0); npk = C.c_uint32(0)
        if capbuf.dtype == np.uint8:
            cb = np.ascontiguousarray(capbuf)
            fn, n_cap = lib().lcs_cell_search_cu8, cb.size // 2
        else:
            cb = np.ascontiguousarray(capbuf, np.complex128)
            fn, n_cap = lib().lcs_cell_search, cb.size
        _chk(fn(self._h, _p(cb), C.c_uint32(n_cap), _p(f), C.c_uint32(f.size), C.c_double(fc_requested),
                C.c_double(fc_programmed), C.c_double(fs_programmed), cells, C.c_uint32(max_cells), C.byref(n), peaks,
                C.byref(npk)), self._h)
        return ([_copy(cells[i]) for i in range(min(n.value, max_cells))],
                [_copy(peaks[i]) for i in range(min(npk.value, max_cells))])

    def tracker_search_cu8(self, capbuf_cu8, frequency_offset, fc_requested, fc_programmed, fs_programmed, late,
                           tracked=(), max_cells=16):
        """One searcher-thread cycle (searcher_thread.cpp:95-232).  Returns [(Cell, frame_timing), ...] of NEW cells."""
        cb = np.ascontiguousarray(capbuf_cu8, np.uint8)
        tr = np.ascontiguousarray(list(tracked), np.int32)
        cells = (Cell * max_cells)(); ft = (C.c_double * max_cells)(); n = C.c_uint32(0)
        _chk(lib().lcs_tracker_search_cu8(self._h, _p(cb), C.c_uint32(cb.size // 2), C.c_double(frequency_offset),
                                          C.c_double(fc_requested), C.c_double(fc_programmed), C.c_double(fs_programmed),
                                          C.c_double(late), _p(tr) if tr.size else None, C.c_uint32(tr.size), cells, ft,
                                          C.c_uint32(max_cells), C.byref(n)), self._h)
        return [(_copy(cells[i]), ft[i]) for i in range(min(n.value, max_cells))]

    def kalibrate_cu8(self, capbuf_cu8, fc_requested, fc_programmed, fs_programmed, ppm, correction=1.0):
        """LTE-Tracker.cpp:565-741.  Returns (best Cell or None, correction_residual, number of cells found)."""
        cb = np.ascontiguousarray(capbuf_cu8, np.uint8)
        best = Cell(); res = C.c_double(0); n = C.c_uint32(0)
        _chk(lib().lcs_kalibrate_cu8(self._h, _p(cb), C.c_uint32(cb.size // 2), C.c_double(fc_requested), C.c_double(fc_programmed),
                                     C.c_double(fs_programmed), C.c_double(ppm), C.c_double(correction), C.byref(best), C.byref(res),
                                     C.byref(n)), self._h)
        return (best if n.value else None), res.value, n.value

    def plan(self, n_cap, f_set, ds_comb_arm, fc_requested, fc_programmed, fs_programmed, max_batch=1,
             kernel=KERNEL_AUTO):
        return XcorrPlan(self, n_cap, f_set, ds_comb_arm, fc_requested, fc_programmed, fs_programmed, max_batch, kernel)


class XcorrPlan:
    """lcs_xcorr_plan: templates + fold offsets + scratch for a fixed search configuration."""

    def __init__(self, ctx, n_cap, f_set, ds_comb_arm, fc_requested, fc_programmed, fs_programmed, max_batch, kernel):
        self.ctx = ctx
        self.n_cap = int(n_cap)
        self.f_set = np.ascontiguousarray(f_set, np.float64)
        self.n_f = self.f_set.size
        self.max_batch = int(max_batch)
        self._h = C.c_void_p()
        _chk(lib().lcs_xcorr_plan_create(ctx._h, C.c_uint32(n_cap), _p(self.f_set), C.c_uint32(self.n_f),
                                         C.c_uint8(ds_comb_arm), C.c_double(fc_requested), C.c_double(fc_programmed),
                                         C.c_double(fs_programmed), C.c_uint32(max_batch), int(kernel), C.byref(self._h)),
             ctx._h)
        self.n_comb_xc = lib().lcs_xcorr_plan_n_comb_xc(self._h)
        self.n_comb_sp = lib().lcs_xcorr_plan_n_comb_sp(self._h)

    def close(self):
        if self._h:
            lib().lcs_xcorr_plan_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def timing_enable(self, on=True):
        _chk(lib().lcs_xcorr_plan_timing_enable(self._h, int(bool(on))), self.ctx._h)

    def timing_read(self):
        ms = C.c_double(0); n = C.c_uint64(0)
        _chk(lib().lcs_xcorr_plan_timing_read(self._h, C.byref(ms), C.byref(n)), self.ctx._h)
        return ms.value, n.value

    def kernel_for(self, iq_format):
        return lib().lcs_xcorr_plan_kernel(self._h, int(iq_format))

    def run_device(self, d_iq_ptr, iq_format, batch, d_single_ptr, d_pow_ptr, d_frq_ptr, d_spi_ptr,
                   d_inc_ptr=None, stream=None):
        """Raw device pointers (ints, e.g. torch.Tensor.data_ptr()); asynchronous on `stream`."""
        _chk(lib().lcs_xcorr_pss_device(self._h, C.c_void_p(d_iq_ptr), int(iq_format), C.c_uint32(batch),
                                        C.c_void_p(d_single_ptr), C.c_void_p(d_pow_ptr), C.c_void_p(d_frq_ptr),
                                        C.c_void_p(d_spi_ptr), C.c_void_p(d_inc_ptr) if d_inc_ptr else None,
                                        C.c_void_p(stream) if stream else None), self.ctx._h)

    def run_host(self, h_iq_ptr, iq_format, batch, h_single_ptr, h_pow_ptr, h_frq_ptr, h_spi_ptr):
        """Host pointers (pinned for overlap): the e2e path."""
        _chk(lib().lcs_xcorr_pss_batch_host(self._h, C.c_void_p(h_iq_ptr), int(iq_format), C.c_uint32(batch),
                                            C.c_void_p(h_single_ptr) if h_single_ptr else None, C.c_void_p(h_pow_ptr),
                                            C.c_void_p(h_frq_ptr), C.c_void_p(h_spi_ptr)), self.ctx._h)

    def run_host_np(self, iq, iq_format, want_single=True):
        """numpy convenience over run_host: iq [batch][n_cap] in the given format."""
        iq = np.ascontiguousarray(iq)
        batch = iq.shape[0]
        single = np.zeros((batch, 3, self.n_f, N_FOLD), np.float32) if want_single else None
        pw = np.zeros((batch, 3, N_FOLD)); frq = np.zeros((batch, 3, N_FOLD), np.int32); spi = np.zeros((batch, N_FOLD))
        self.run_host(iq.ctypes.data, iq_format, batch, single.ctypes.data if want_single else None, pw.ctypes.data,
                      frq.ctypes.data, spi.ctypes.data)
        return dict(single=single, pow=pw, frq=frq, sp_incoherent=spi)

    def peaks_batch(self, iq, iq_format, max_peaks=32, host_ptr=None, batch=None):
        """xcorr_pss + threshold + peak_search on the device for a batch of host buffers (iq [batch][n_cap] in iq_format,
        or a raw host pointer + batch).  Returns a list (per buffer) of lists of PSS-peak Cells."""
        if host_ptr is None:
            iq = np.ascontiguousarray(iq)
            host_ptr, batch = iq.ctypes.data, iq.shape[0]
        peaks = (Cell * (batch * max_peaks))()
        n = (C.c_uint32 * batch)()
        _chk(lib().lcs_xcorr_peaks_batch_host(self._h, C.c_void_p(host_ptr), int(iq_format), C.c_uint32(batch), peaks,
                                              C.c_uint32(max_peaks), n), self.ctx._h)
        return [[_copy(peaks[b * max_peaks + k]) for k in range(min(n[b], max_peaks))] for b in range(batch)]

    def cell_search_batch_cu8(self, iq_cu8, max_cells=16, host_ptr=None, batch=None):
        """The whole CellSearch chain for every buffer of a batch of raw rtl-sdr byte buffers (uint8 [batch][n_cap][2])."""
        if host_ptr is None:
            iq_cu8 = np.ascontiguousarray(iq_cu8, np.uint8)
            host_ptr, batch = iq_cu8.ctypes.data, iq_cu8.shape[0]
        cells = (Cell * (batch * max_cells))()
        n = (C.c_uint32 * batch)()
        _chk(lib().lcs_cell_search_batch_cu8(self._h, C.c_void_p(host_ptr), C.c_uint32(batch), cells, C.c_uint32(max_cells), n),
             self.ctx._h)
        return [[_copy(cells[b * max_cells + k]) for k in range(min(n[b], max_cells))] for b in range(batch)]


class Sweep:
    """lcs_sweep: many channels (centre frequencies / tracked channels) through one correlator launch per chunk."""

    def __init__(self, ctx, n_cap=153600):
        self.ctx = ctx
        self.n_cap = int(n_cap)
        self._h = C.c_void_p()
        _chk(lib().lcs_sweep_create(ctx._h, C.c_uint32(n_cap), C.byref(self._h)), ctx._h)

    def close(self):
        if self._h:
            lib().lcs_sweep_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def search_cu8(self, iq_cu8, fc_requested, f_set, fs_programmed=1.92e6, fc_programmed=None, max_cells=8, host_ptr=None):
        """CellSearch.cpp:465-558 for all channels.  iq_cu8: uint8 [n_ch][n_cap][2] (or host_ptr).  Returns a list
        (per channel) of lists of Cells."""
        fc = np.ascontiguousarray(fc_requested, np.float64)
        n_ch = fc.size
        fcp = None if fc_programmed is None else np.ascontiguousarray(fc_programmed, np.float64)
        f = np.ascontiguousarray(f_set, np.float64)
        if host_ptr is None:
            iq_cu8 = np.ascontiguousarray(iq_cu8, np.uint8)
            host_ptr = iq_cu8.ctypes.data
        cells = (Cell * (n_ch * max_cells))()
        n = (C.c_uint32 * n_ch)()
        _chk(lib().lcs_sweep_search_cu8(self._h, C.c_void_p(host_ptr), C.c_uint32(n_ch), _p(fc), _p(fcp), C.c_double(fs_programmed),
                                        _p(f), C.c_uint32(f.size), cells, C.c_uint32(max_cells), n), self.ctx._h)
        return [[_copy(cells[b * max_cells + k]) for k in range(min(n[b], max_cells))] for b in range(n_ch)]

    def track_cu8(self, iq_cu8, frequency_offset, fc_requested, fs_programmed=1.92e6, fc_programmed=None, late=None, tracked=None,
                  max_cells=8, host_ptr=None):
        """searcher_thread.cpp:95-232 for all channels.  tracked: list (per channel) of lists of n_id_cell.  Returns a
        list (per channel) of [(Cell, frame_timing), ...]."""
        fo = np.ascontiguousarray(frequency_offset, np.float64)
        fc = np.ascontiguousarray(fc_requested, np.float64)
        n_ch = fc.size
        fcp = None if fc_programmed is None else np.ascontiguousarray(fc_programmed, np.float64)
        lt = None if late is None else np.ascontiguousarray(late, np.float64)
        tr = nt = None
        stride = 0
        if tracked is not None:
            stride = max(1, max(len(t) for t in tracked))
            tr = np.full((n_ch, stride), -1, np.int32)
            nt = np.zeros(n_ch, np.uint32)
            for c, t in enumerate(tracked):
                tr[c, :len(t)] = t
                nt[c] = len(t)
        if host_ptr is None:
            iq_cu8 = np.ascontiguousarray(iq_cu8, np.uint8)
            host_ptr = iq_cu8.ctypes.data
        cells = (Cell * (n_ch * max_cells))()
        ft = (C.c_double * (n_ch * max_cells))()
        n = (C.c_uint32 * n_ch)()
        _chk(lib().lcs_sweep_track_cu8(self._h, C.c_void_p(host_ptr), C.c_uint32(n_ch), _p(fo), _p(fc), _p(fcp), C.c_double(fs_programmed),
                                       _p(lt), _p(tr), _p(nt), C.c_uint32(stride), cells, ft, C.c_uint32(max_cells), n), self.ctx._h)
        return [[(_copy(cells[b * max_cells + k]), ft[b * max_cells + k]) for k in range(min(n[b], max_cells))] for b in range(n_ch)]


class Framer:
    """lcs_framer: producer-side framing of a raw IQ byte stream into searcher capture buffers (host only)."""

    def __init__(self, fc_requested, fc_programmed, fs_programmed, n_cap=153600):
        self._h = C.c_void_p()
        self.n_cap = n_cap
        _chk(lib().lcs_framer_create(C.c_double(fc_requested), C.c_double(fc_programmed), C.c_double(fs_programmed),
                                     C.c_uint32(n_cap), C.byref(self._h)))

    def request(self):
        lib().lcs_framer_request(self._h)

    def sample_time(self):
        return lib().lcs_framer_sample_time(self._h)

    def push(self, iq_u8, frequency_offset):
        """iq_u8: uint8 [n][2].  Returns None, or (capbuf uint8 [n_cap][2] copy, late) once a requested buffer is full."""
        iq = np.ascontiguousarray(iq_u8, np.uint8)
        ready = C.c_int(0); cap = C.POINTER(C.c_uint8)(); late = C.c_double(0)
        _chk(lib().lcs_framer_push(self._h, _p(iq), C.c_uint32(iq.size // 2), C.c_double(frequency_offset), C.byref(ready),
                                   C.byref(cap), C.byref(late)))
        if not ready.value:
            return None
        return np.ctypeslib.as_array(cap, shape=(self.n_cap, 2)).copy(), late.value

    def close(self):
        if self._h:
            lib().lcs_framer_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()


class TrackCell(C.Structure):
    """lcs_track_cell: one tracked cell as lcs_track_read reports it."""
    _fields_ = [
        ("n_id_cell", C.c_int32), ("n_ports", C.c_int32), ("cp_type", C.c_int32), ("dropped", C.c_int32),
        ("drop_sample", C.c_int64), ("n_symbols", C.c_int64), ("last_slice_start", C.c_int64),
        ("mib_attempts", C.c_int64), ("mib_successes", C.c_int64),
        ("frame_timing", C.c_double), ("mib_decode_failures", C.c_double),
        ("crs_tp", C.c_double * 4), ("crs_sp_raw", C.c_double * 4), ("crs_np", C.c_double * 4),
        ("crs_tp_av", C.c_double * 4), ("crs_sp_raw_av", C.c_double * 4), ("crs_np_av", C.c_double * 4),
        ("sync_tp", C.c_double), ("sync_sp", C.c_double), ("sync_np", C.c_double), ("sync_np_blank", C.c_double),
        ("sync_tp_av", C.c_double), ("sync_sp_av", C.c_double), ("sync_np_av", C.c_double),
        ("sync_np_blank_av", C.c_double),
        ("sync_ce", C.c_double * 144), ("ce", C.c_double * (4 * 144)),
    ]

    def as_dict(self):
        """Plain Python / numpy values; sync_ce is complex [72], ce complex [4][72]."""
        d = {}
        for k, _ in self._fields_:
            v = getattr(self, k)
            if k == "sync_ce":
                v = np.ctypeslib.as_array(v).copy().view(np.complex128)
            elif k == "ce":
                v = np.ctypeslib.as_array(v).copy().view(np.complex128).reshape(4, 72)
            elif not isinstance(v, (int, float)):
                v = np.ctypeslib.as_array(v).copy()
            d[k] = v
        return d


TRACK_BLOCK = 10000


class Tracker:
    """lcs_track: the per-cell tracker loop of LTE-Tracker for every cell of n_ch channels, one launch per push."""

    def __init__(self, ctx, fc_requested, frequency_offset, fs_programmed=1.92e6, fc_programmed=None, max_cells=8):
        self.ctx = ctx
        fc = np.ascontiguousarray(np.atleast_1d(fc_requested), np.float64)
        self.n_ch = fc.size
        fcp = None if fc_programmed is None else np.ascontiguousarray(np.atleast_1d(fc_programmed), np.float64)
        fo = np.ascontiguousarray(np.broadcast_to(np.asarray(frequency_offset, np.float64), (self.n_ch,)))
        self.max_cells = int(max_cells)
        self._h = C.c_void_p()
        _chk(lib().lcs_track_create(ctx._h, C.c_uint32(self.n_ch), _p(fc), _p(fcp), C.c_double(fs_programmed), _p(fo),
                                    C.c_uint32(self.max_cells), C.byref(self._h)), ctx._h)

    def add_cell(self, ch, cell, frame_timing):
        _chk(lib().lcs_track_add_cell(self._h, C.c_uint32(ch), C.byref(cell), C.c_double(frame_timing)), self.ctx._h)

    def push_cu8(self, iq_cu8):
        """iq_cu8: uint8 [n_ch][n][2] (or [n][2] for one channel)."""
        iq = np.ascontiguousarray(iq_cu8, np.uint8)
        n = iq.shape[-2]
        if iq.size != self.n_ch * n * 2:
            raise ValueError("push_cu8: expected [n_ch][n][2] samples")
        _chk(lib().lcs_track_push_cu8(self._h, _p(iq), C.c_uint32(n)), self.ctx._h)

    def frequency_offset(self):
        fo = np.zeros(self.n_ch)
        _chk(lib().lcs_track_frequency_offset(self._h, _p(fo)), self.ctx._h)
        return fo

    def sample_time(self, ch=0):
        v = C.c_double(0)
        _chk(lib().lcs_track_sample_time(self._h, C.c_uint32(ch), C.byref(v)), self.ctx._h)
        return v.value

    def timing_read(self):
        """(kernel ms, launches) since the last read, from CUDA events around each launch."""
        ms = C.c_double(0); n = C.c_uint64(0)
        _chk(lib().lcs_track_timing_read(self._h, C.byref(ms), C.byref(n)), self.ctx._h)
        return ms.value, n.value

    def read(self, ch=0):
        """The channel's cells in the order added, as dicts; a dropped cell is reported once."""
        out = (TrackCell * self.max_cells)()
        n = C.c_uint32(0)
        _chk(lib().lcs_track_read(self._h, C.c_uint32(ch), out, C.c_uint32(self.max_cells), C.byref(n)), self.ctx._h)
        return [out[i].as_dict() for i in range(n.value)]

    def close(self):
        if self._h:
            lib().lcs_track_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def declared_symbols():
    """Function names declared in include/lcs_b200.h (for the export test)."""
    import re
    txt = open(HEADER).read()
    return sorted(set(re.findall(r"\b(lcs_[a-z0-9_]+)\s*\(", txt)))
