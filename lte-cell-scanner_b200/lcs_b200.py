"""ctypes binding of liblcs_b200.so - the C ABI declared in include/lcs_b200.h - and of the three modules built on top of
it: liblcs_psd.so, the Welch spectrum of include/lcs_psd.h, liblcs_meas.so, the per-cell RSRP / RSRQ / SINR of
include/lcs_meas.h, liblcs_carrier.so, the same over each cell's whole carrier, of include/lcs_carrier.h,
liblcs_cir.so, the power delay profile of each cell over its whole carrier, of include/lcs_cir.h, liblcs_pcfich.so,
the control format indicator of each cell in every subframe, of include/lcs_pcfich.h, liblcs_pdcch.so, the
common-search-space DCIs of each cell in every subframe, of include/lcs_pdcch.h, and liblcs_sib1.so, the SIB1 of each
cell, of include/lcs_sib1.h.

This module is plumbing for tests/, bench.py and __graft_entry__.py: every call goes through the
same `extern "C"` entry points a C++/IT++ host would bind (INTEGRATION.md).  lib() gives every
function of the header its ctypes prototype, read from the header itself, so a call with a missing
or mistyped argument raises before it reaches the library.  There is no CPU fallback: importing
works anywhere, but every compute call needs an H100 and raises LcsError otherwise.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LCS_B200_LIB") or os.path.join(HERE, "liblcs_b200.so")
HEADER = os.path.join(HERE, "..", "include", "lcs_b200.h")
PSD_LIB_PATH = os.environ.get("LCS_PSD_LIB") or os.path.join(HERE, "liblcs_psd.so")
PSD_HEADER = os.path.join(HERE, "..", "include", "lcs_psd.h")
MEAS_LIB_PATH = os.environ.get("LCS_MEAS_LIB") or os.path.join(HERE, "liblcs_meas.so")
MEAS_HEADER = os.path.join(HERE, "..", "include", "lcs_meas.h")
CARRIER_LIB_PATH = os.environ.get("LCS_CARRIER_LIB") or os.path.join(HERE, "liblcs_carrier.so")
CARRIER_HEADER = os.path.join(HERE, "..", "include", "lcs_carrier.h")
CIR_LIB_PATH = os.environ.get("LCS_CIR_LIB") or os.path.join(HERE, "liblcs_cir.so")
CIR_HEADER = os.path.join(HERE, "..", "include", "lcs_cir.h")
PCFICH_LIB_PATH = os.environ.get("LCS_PCFICH_LIB") or os.path.join(HERE, "liblcs_pcfich.so")
PCFICH_HEADER = os.path.join(HERE, "..", "include", "lcs_pcfich.h")
PDCCH_LIB_PATH = os.environ.get("LCS_PDCCH_LIB") or os.path.join(HERE, "liblcs_pdcch.so")
PDCCH_HEADER = os.path.join(HERE, "..", "include", "lcs_pdcch.h")
SIB1_LIB_PATH = os.environ.get("LCS_SIB1_LIB") or os.path.join(HERE, "liblcs_sib1.so")
SIB1_HEADER = os.path.join(HERE, "..", "include", "lcs_sib1.h")

IQ_CF32, IQ_CU8, IQ_C128, IQ_CI16, IQ_CS8 = 0, 1, 2, 3, 4
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
    """Compile the CUDA library in-tree (nvcc cross-compiles sm_90a without a GPU).  make is incremental, so it rebuilds
    what changed whether or not `force` is set."""
    subprocess.check_call(["make", "-C", HERE, "-s", "-j8"])
    return LIB_PATH


# Scalar types of the header.  Every pointer (handles, arrays, structs, out-parameters) is a c_void_p: the callers pass
# array addresses, ctypes arrays, C.byref(...) and oracle Cells alike.
_SCALARS = {"double": C.c_double, "int": C.c_int, "lcs_status": C.c_int, "uint8_t": C.c_uint8, "uint16_t": C.c_uint16,
            "uint32_t": C.c_uint32, "uint64_t": C.c_uint64}


def _ctype(fn, decl, ret=False):
    words = re.sub(r"\bconst\b", " ", decl).replace("*", " * ").split()
    if "*" in words:
        return C.c_char_p if ret and words == ["char", "*"] else C.c_void_p
    if ret and words == ["void"]:
        return None
    if not words or words[0] not in _SCALARS:
        raise LcsError("%s: no ctypes type for %r in %s" % (fn, decl.strip(), HEADER))
    return _SCALARS[words[0]]


def prototypes(header=HEADER):
    """{name: (restype, argtypes)} for every function declared in `header` (default include/lcs_b200.h; included
    headers are not followed)."""
    txt = re.sub(r"/\*.*?\*/", " ", open(header).read(), flags=re.S)
    txt = re.sub(r"^\s*#.*$", "", txt, flags=re.M)
    table = {}
    for decl in re.split(r"[;{}]", txt):
        m = re.fullmatch(r"\s*(.+?)\b(lcs_\w+)\s*\((.*)\)\s*", decl, re.S)
        if m:
            ret, name, args = m.groups()
            args = [] if args.strip() == "void" else args.split(",")
            table[name] = (_ctype(name, ret, ret=True), [_ctype(name, a) for a in args])
    return table


def declared_symbols():
    """Function names declared in include/lcs_b200.h."""
    return sorted(prototypes())


_libs = {}


def _bind(path, header):
    """The library at `path` with every function of `header` given its prototype; raises naming any it lacks."""
    if path not in _libs:
        if not os.path.exists(path):
            raise LcsError("%s is not built (run `make -C lte-cell-scanner_b200`); there is no CPU fallback"
                           % os.path.basename(path))
        l = C.CDLL(path)
        table = prototypes(header)
        missing = sorted(name for name in table if not hasattr(l, name))
        if missing:
            raise LcsError("%s lacks functions declared in %s: %s" % (path, os.path.basename(header), ", ".join(missing)))
        for name, (restype, argtypes) in table.items():
            f = getattr(l, name)
            f.restype, f.argtypes = restype, argtypes
        _libs[path] = l
    return _libs[path]


def lib():
    return _bind(LIB_PATH, HEADER)


def psd_lib():
    """liblcs_psd.so (include/lcs_psd.h); it takes the contexts of lib()."""
    lib()
    return _bind(PSD_LIB_PATH, PSD_HEADER)


def meas_lib():
    """liblcs_meas.so (include/lcs_meas.h); it takes the contexts of lib()."""
    lib()
    return _bind(MEAS_LIB_PATH, MEAS_HEADER)


def _grid_lib(path, header):
    """A module on the whole-carrier grid (include/lcs_carrier.h, lcs_cir.h, lcs_pcfich.h, lcs_pdcch.h or lcs_sib1.h); it
    takes the contexts of lib()."""
    lib()
    return _bind(path, header)


def carrier_lib():
    return _grid_lib(CARRIER_LIB_PATH, CARRIER_HEADER)


def cir_lib():
    return _grid_lib(CIR_LIB_PATH, CIR_HEADER)


def pcfich_lib():
    return _grid_lib(PCFICH_LIB_PATH, PCFICH_HEADER)


def pdcch_lib():
    return _grid_lib(PDCCH_LIB_PATH, PDCCH_HEADER)


def sib1_lib():
    return _grid_lib(SIB1_LIB_PATH, SIB1_HEADER)


def _p(a):
    return None if a is None else a.ctypes.data


def _chk(rc, ctx=None):
    if rc != 0:
        raise LcsError("lcs_b200 error %d: %s" % (rc, lib().lcs_last_error(ctx).decode()))


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


def _cell_rows(cells, n, max_cells, values=None):
    """Row b of the [len(n)][max_cells] array `cells` holds n[b] Cells, truncated at max_cells: one list of copies per
    row, or of (Cell, values[i]) pairs when the parallel array `values` is given."""
    rows = []
    for b, nb in enumerate(n):
        idx = range(b * max_cells, b * max_cells + min(nb, max_cells))
        rows.append([_copy(cells[i]) if values is None else (_copy(cells[i]), values[i]) for i in idx])
    return rows


def _query_then_fill(fn, *args, dtype=np.float64):
    """fn(*args, out, &n) sets n when out is NULL, then fills an n-element out: the filled array."""
    n = C.c_uint32(0)
    _chk(fn(*args, None, C.byref(n)))
    out = np.zeros(n.value, dtype)
    _chk(fn(*args, _p(out), C.byref(n)))
    return out


class _Handle:
    """A library object: `_h` is its handle, freed by the function named `_destroy` on close() or garbage collection."""
    _h = None
    _destroy = None
    _timing_read = None               # the handle's lcs_*_timing_read, if it times its kernels

    _lib = staticmethod(lib)          # the library that owns `_destroy` and `_timing_read`

    def close(self):
        if self._h:
            getattr(self._lib(), self._destroy)(self._h)
            self._h = C.c_void_p()

    def timing_read(self):
        """(kernel ms, kernel launches) since the last read, from CUDA events around the launches."""
        ms = C.c_double(0); n = C.c_uint64(0)
        _chk(getattr(self._lib(), self._timing_read)(self._h, C.byref(ms), C.byref(n)), self.ctx._h)
        return ms.value, n.value

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def f_search_set(freq_start, ppm):
    return _query_then_fill(lib().lcs_f_search_set, freq_start, ppm)


def calc_z_th1(sp_incoherent, n_comb_xc, ds_comb_arm):
    s = np.ascontiguousarray(sp_incoherent, np.float64)
    z = np.zeros_like(s)
    _chk(lib().lcs_calc_z_th1(_p(s), s.size, n_comb_xc, ds_comb_arm, _p(z)))
    return z


def peak_search(pw, frq, z_th1, f_set, fc_requested, fc_programmed, single_planar, ds_comb_arm, max_cells=256):
    """pw/frq: [3][9600]; single_planar: [3][n_f][9600] float32."""
    pw = np.ascontiguousarray(pw, np.float64); frq = np.ascontiguousarray(frq, np.int32)
    z = np.ascontiguousarray(z_th1, np.float64); f = np.ascontiguousarray(f_set, np.float64)
    sp = np.ascontiguousarray(single_planar, np.float32)
    cells = (Cell * max_cells)(); n = C.c_uint32(0)
    _chk(lib().lcs_peak_search(_p(pw), _p(frq), _p(z), _p(f), f.size, fc_requested, fc_programmed, _p(sp), ds_comb_arm,
                               cells, max_cells, C.byref(n)))
    return [_copy(cells[i]) for i in range(min(n.value, max_cells))]


def dedup(cells):
    n = len(cells)
    arr = (Cell * max(n, 1))(*cells); out = (Cell * max(n, 1))(); m = C.c_uint32(0)
    _chk(lib().lcs_dedup(arr, n, out, C.byref(m)))
    return [_copy(out[i]) for i in range(m.value)]


def tfoec(cell, tfg, ts, fc_requested, fc_programmed):
    """searcher.h:101-112 - host stage (no GPU needed).  tfg: [n_ofdm][72] complex128."""
    n = ts.size
    g = np.asfortranarray(tfg, np.complex128)                        # column-major cmat for the ABI
    ts = np.ascontiguousarray(ts, np.float64)
    gc = np.zeros((n, 72), np.complex128, order="F"); tsc = np.zeros(n); out = Cell()
    _chk(lib().lcs_tfoec(None, C.byref(cell), _p(g), _p(ts), n, fc_requested, fc_programmed, _p(gc), _p(tsc),
                         C.byref(out)))
    return out, np.ascontiguousarray(gc), tsc


def decode_mib(cell, tfg):
    """searcher.h:115-119 - host stage (no GPU needed)."""
    g = np.asfortranarray(tfg, np.complex128)
    out = Cell()
    _chk(lib().lcs_decode_mib(None, C.byref(cell), _p(g), g.shape[0], C.byref(out)))
    return out


class Context(_Handle):
    """lcs_ctx: one per process per GPU."""
    _destroy = "lcs_ctx_destroy"

    def __init__(self, device=0):
        self._h = C.c_void_p()
        _chk(lib().lcs_ctx_create(int(device), C.byref(self._h)))

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
        _chk(lib().lcs_xcorr_pss(self._h, _p(capbuf), n_cap, _p(f), n_f, ds_comb_arm, fc_requested, fc_programmed,
                                 fs_programmed, _p(pw), _p(frq), _p(single), _p(inc), _p(spi), _p(xc), _p(sp),
                                 C.byref(ncx), C.byref(ncs)), self._h)
        return dict(pow=pw.T.copy(), frq=frq.T.copy(), single=single, incoherent=inc, sp_incoherent=spi, xc=xc, sp=sp,
                    n_comb_xc=ncx.value, n_comb_sp=ncs.value)

    def sss_detect(self, cell, capbuf, thresh2_n_sigma, fc_requested, fc_programmed, fs_programmed):
        capbuf = np.ascontiguousarray(capbuf, np.complex128)
        out = Cell()
        h1_np = np.zeros(62); h2_np = np.zeros(62)
        arrs = [np.zeros(62, np.complex128) for _ in range(4)]
        lln = np.zeros((2, 168)); lle = np.zeros((2, 168))
        _chk(lib().lcs_sss_detect(self._h, C.byref(cell), _p(capbuf), capbuf.size, thresh2_n_sigma, fc_requested,
                                  fc_programmed, fs_programmed, C.byref(out), _p(h1_np), _p(h2_np), _p(arrs[0]),
                                  _p(arrs[1]), _p(arrs[2]), _p(arrs[3]), _p(lln), _p(lle)), self._h)
        d = dict(h1_np=h1_np, h2_np=h2_np, h1_nrm=arrs[0], h2_nrm=arrs[1], h1_ext=arrs[2], h2_ext=arrs[3],
                 log_lik_nrm=lln.T.copy(), log_lik_ext=lle.T.copy())
        return out, d

    def pss_sss_foe(self, cell, capbuf, fc_requested, fc_programmed, fs_programmed):
        capbuf = np.ascontiguousarray(capbuf, np.complex128)
        out = Cell()
        _chk(lib().lcs_pss_sss_foe(self._h, C.byref(cell), _p(capbuf), capbuf.size, fc_requested, fc_programmed,
                                   fs_programmed, C.byref(out)), self._h)
        return out

    def extract_tfg(self, cell, capbuf, fc_requested, fc_programmed, fs_programmed):
        capbuf = np.ascontiguousarray(capbuf, np.complex128)
        tfg = np.zeros(72 * 854, np.complex128); ts = np.zeros(854); n = C.c_uint32(0)
        _chk(lib().lcs_extract_tfg(self._h, C.byref(cell), _p(capbuf), capbuf.size, fc_requested, fc_programmed,
                                   fs_programmed, _p(tfg), _p(ts), C.byref(n)), self._h)
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
        _chk(fn(self._h, _p(cb), n_cap, _p(f), f.size, fc_requested, fc_programmed, fs_programmed, cells, max_cells,
                C.byref(n), peaks, C.byref(npk)), self._h)
        return ([_copy(cells[i]) for i in range(min(n.value, max_cells))],
                [_copy(peaks[i]) for i in range(min(npk.value, max_cells))])

    def tracker_search_cu8(self, capbuf_cu8, frequency_offset, fc_requested, fc_programmed, fs_programmed, late,
                           tracked=(), max_cells=16):
        """One searcher-thread cycle (searcher_thread.cpp:95-232).  Returns [(Cell, frame_timing), ...] of NEW cells."""
        cb = np.ascontiguousarray(capbuf_cu8, np.uint8)
        tr = np.ascontiguousarray(list(tracked), np.int32)
        cells = (Cell * max_cells)(); ft = (C.c_double * max_cells)(); n = C.c_uint32(0)
        _chk(lib().lcs_tracker_search_cu8(self._h, _p(cb), cb.size // 2, frequency_offset, fc_requested, fc_programmed,
                                          fs_programmed, late, _p(tr) if tr.size else None, tr.size, cells, ft,
                                          max_cells, C.byref(n)), self._h)
        return [(_copy(cells[i]), ft[i]) for i in range(min(n.value, max_cells))]

    def kalibrate_cu8(self, capbuf_cu8, fc_requested, fc_programmed, fs_programmed, ppm, correction=1.0):
        """LTE-Tracker.cpp:565-741.  Returns (best Cell or None, correction_residual, number of cells found)."""
        cb = np.ascontiguousarray(capbuf_cu8, np.uint8)
        best = Cell(); res = C.c_double(0); n = C.c_uint32(0)
        _chk(lib().lcs_kalibrate_cu8(self._h, _p(cb), cb.size // 2, fc_requested, fc_programmed, fs_programmed, ppm,
                                     correction, C.byref(best), C.byref(res), C.byref(n)), self._h)
        return (best if n.value else None), res.value, n.value

    def plan(self, n_cap, f_set, ds_comb_arm, fc_requested, fc_programmed, fs_programmed, max_batch=1,
             kernel=KERNEL_AUTO):
        return XcorrPlan(self, n_cap, f_set, ds_comb_arm, fc_requested, fc_programmed, fs_programmed, max_batch, kernel)


class XcorrPlan(_Handle):
    """lcs_xcorr_plan: templates + fold offsets + scratch for a fixed search configuration."""
    _destroy = "lcs_xcorr_plan_destroy"
    _timing_read = "lcs_xcorr_plan_timing_read"

    def __init__(self, ctx, n_cap, f_set, ds_comb_arm, fc_requested, fc_programmed, fs_programmed, max_batch, kernel):
        self.ctx = ctx
        self.n_cap = int(n_cap)
        self.f_set = np.ascontiguousarray(f_set, np.float64)
        self.n_f = self.f_set.size
        self.max_batch = int(max_batch)
        self._h = C.c_void_p()
        _chk(lib().lcs_xcorr_plan_create(ctx._h, n_cap, _p(self.f_set), self.n_f, ds_comb_arm, fc_requested,
                                         fc_programmed, fs_programmed, max_batch, int(kernel), C.byref(self._h)), ctx._h)
        self.n_comb_xc = lib().lcs_xcorr_plan_n_comb_xc(self._h)
        self.n_comb_sp = lib().lcs_xcorr_plan_n_comb_sp(self._h)

    def timing_enable(self, on=True):
        _chk(lib().lcs_xcorr_plan_timing_enable(self._h, int(bool(on))), self.ctx._h)

    def kernel_for(self, iq_format):
        return lib().lcs_xcorr_plan_kernel(self._h, int(iq_format))

    def run_device(self, d_iq_ptr, iq_format, batch, d_single_ptr, d_pow_ptr, d_frq_ptr, d_spi_ptr,
                   d_inc_ptr=None, stream=None):
        """Raw device pointers (ints, e.g. torch.Tensor.data_ptr()); asynchronous on `stream`."""
        _chk(lib().lcs_xcorr_pss_device(self._h, d_iq_ptr, int(iq_format), batch, d_single_ptr, d_pow_ptr, d_frq_ptr,
                                        d_spi_ptr, d_inc_ptr, stream), self.ctx._h)

    def run_host(self, h_iq_ptr, iq_format, batch, h_single_ptr, h_pow_ptr, h_frq_ptr, h_spi_ptr):
        """Host pointers (pinned for overlap): the e2e path."""
        _chk(lib().lcs_xcorr_pss_batch_host(self._h, h_iq_ptr, int(iq_format), batch, h_single_ptr, h_pow_ptr, h_frq_ptr,
                                            h_spi_ptr), self.ctx._h)

    def run_host_np(self, iq, iq_format, want_single=True):
        """numpy convenience over run_host: iq [batch][n_cap] in the given format."""
        iq = np.ascontiguousarray(iq)
        batch = iq.shape[0]
        single = np.zeros((batch, 3, self.n_f, N_FOLD), np.float32) if want_single else None
        pw = np.zeros((batch, 3, N_FOLD)); frq = np.zeros((batch, 3, N_FOLD), np.int32); spi = np.zeros((batch, N_FOLD))
        self.run_host(_p(iq), iq_format, batch, _p(single), _p(pw), _p(frq), _p(spi))
        return dict(single=single, pow=pw, frq=frq, sp_incoherent=spi)

    def peaks_batch(self, iq, iq_format, max_peaks=32, host_ptr=None, batch=None):
        """xcorr_pss + threshold + peak_search on the device for a batch of host buffers (iq [batch][n_cap] in iq_format,
        or a raw host pointer + batch).  Returns a list (per buffer) of lists of PSS-peak Cells."""
        if host_ptr is None:
            iq = np.ascontiguousarray(iq)
            host_ptr, batch = iq.ctypes.data, iq.shape[0]
        peaks = (Cell * (batch * max_peaks))()
        n = (C.c_uint32 * batch)()
        _chk(lib().lcs_xcorr_peaks_batch_host(self._h, host_ptr, int(iq_format), batch, peaks, max_peaks, n), self.ctx._h)
        return _cell_rows(peaks, n, max_peaks)

    def cell_search_batch_cu8(self, iq_cu8, max_cells=16, host_ptr=None, batch=None):
        """The whole CellSearch chain for every buffer of a batch of raw rtl-sdr byte buffers (uint8 [batch][n_cap][2])."""
        if host_ptr is None:
            iq_cu8 = np.ascontiguousarray(iq_cu8, np.uint8)
            host_ptr, batch = iq_cu8.ctypes.data, iq_cu8.shape[0]
        cells = (Cell * (batch * max_cells))()
        n = (C.c_uint32 * batch)()
        _chk(lib().lcs_cell_search_batch_cu8(self._h, host_ptr, batch, cells, max_cells, n), self.ctx._h)
        return _cell_rows(cells, n, max_cells)


class Sweep(_Handle):
    """lcs_sweep: many channels (centre frequencies / tracked channels) through one correlator launch per chunk."""
    _destroy = "lcs_sweep_destroy"

    def __init__(self, ctx, n_cap=153600):
        self.ctx = ctx
        self.n_cap = int(n_cap)
        self._h = C.c_void_p()
        _chk(lib().lcs_sweep_create(ctx._h, n_cap, C.byref(self._h)), ctx._h)

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
        _chk(lib().lcs_sweep_search_cu8(self._h, host_ptr, n_ch, _p(fc), _p(fcp), fs_programmed, _p(f), f.size, cells,
                                        max_cells, n), self.ctx._h)
        return _cell_rows(cells, n, max_cells)

    def search_cu8_device(self, iq, fc_requested, f_set, fs_programmed=1.92e6, fc_programmed=None, max_cells=8, n_ch=None):
        """search_cu8 on capture buffers in device memory, read in place: iq is a uint8 CUDA tensor [n_ch][n_cap][2]
        (16-byte aligned, contiguous) or a raw device pointer (int) with n_ch given.  The caller's writes to it must be
        complete; for a tensor, its stream is synchronised first."""
        fc = np.ascontiguousarray(fc_requested, np.float64)
        n_ch = fc.size
        fcp = None if fc_programmed is None else np.ascontiguousarray(fc_programmed, np.float64)
        f = np.ascontiguousarray(f_set, np.float64)
        if isinstance(iq, int):
            ptr = iq
        else:
            if not (iq.is_cuda and iq.is_contiguous() and iq.numel() >= n_ch * self.n_cap * 2):
                raise ValueError("search_cu8_device: expected a contiguous uint8 CUDA tensor [n_ch][n_cap][2]")
            import torch
            torch.cuda.current_stream(iq.device).synchronize()
            ptr = iq.data_ptr()
        cells = (Cell * (n_ch * max_cells))()
        n = (C.c_uint32 * n_ch)()
        _chk(lib().lcs_sweep_search_cu8_device(self._h, ptr, n_ch, _p(fc), _p(fcp), fs_programmed, _p(f), f.size, cells,
                                               max_cells, n), self.ctx._h)
        return _cell_rows(cells, n, max_cells)

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
        _chk(lib().lcs_sweep_track_cu8(self._h, host_ptr, n_ch, _p(fo), _p(fc), _p(fcp), fs_programmed, _p(lt), _p(tr),
                                       _p(nt), stride, cells, ft, max_cells, n), self.ctx._h)
        return _cell_rows(cells, n, max_cells, ft)


class Framer(_Handle):
    """lcs_framer: producer-side framing of a raw IQ byte stream into searcher capture buffers (host only)."""
    _destroy = "lcs_framer_destroy"

    def __init__(self, fc_requested, fc_programmed, fs_programmed, n_cap=153600):
        self._h = C.c_void_p()
        self.n_cap = n_cap
        _chk(lib().lcs_framer_create(fc_requested, fc_programmed, fs_programmed, n_cap, C.byref(self._h)))

    def request(self):
        lib().lcs_framer_request(self._h)

    def sample_time(self):
        return lib().lcs_framer_sample_time(self._h)

    def push(self, iq_u8, frequency_offset):
        """iq_u8: uint8 [n][2].  Returns None, or (capbuf uint8 [n_cap][2] copy, late) once a requested buffer is full."""
        iq = np.ascontiguousarray(iq_u8, np.uint8)
        ready = C.c_int(0); cap = C.POINTER(C.c_uint8)(); late = C.c_double(0)
        _chk(lib().lcs_framer_push(self._h, _p(iq), iq.size // 2, frequency_offset, C.byref(ready), C.byref(cap),
                                   C.byref(late)))
        if not ready.value:
            return None
        return np.ctypeslib.as_array(cap, shape=(self.n_cap, 2)).copy(), late.value


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
        ("ac_fd", C.c_double * 24), ("ac_td", C.c_double * 144),
    ]

    def as_dict(self):
        """Plain Python / numpy values; sync_ce and ac_td are complex [72], ac_fd complex [12], ce complex [4][72]."""
        d = {}
        for k, _ in self._fields_:
            v = getattr(self, k)
            if k in ("sync_ce", "ac_fd", "ac_td"):
                v = np.ctypeslib.as_array(v).copy().view(np.complex128)
            elif k == "ce":
                v = np.ctypeslib.as_array(v).copy().view(np.complex128).reshape(4, 72)
            elif not isinstance(v, (int, float)):
                v = np.ctypeslib.as_array(v).copy()
            d[k] = v
        return d


TRACK_BLOCK = 10000


class Tracker(_Handle):
    """lcs_track: the per-cell tracker loop of LTE-Tracker for every cell of n_ch channels, one launch per push."""
    _destroy = "lcs_track_destroy"
    _timing_read = "lcs_track_timing_read"

    def __init__(self, ctx, fc_requested, frequency_offset, fs_programmed=1.92e6, fc_programmed=None, max_cells=8):
        self.ctx = ctx
        fc = np.ascontiguousarray(np.atleast_1d(fc_requested), np.float64)
        self.n_ch = fc.size
        fcp = None if fc_programmed is None else np.ascontiguousarray(np.atleast_1d(fc_programmed), np.float64)
        fo = np.ascontiguousarray(np.broadcast_to(np.asarray(frequency_offset, np.float64), (self.n_ch,)))
        self.max_cells = int(max_cells)
        self._h = C.c_void_p()
        _chk(lib().lcs_track_create(ctx._h, self.n_ch, _p(fc), _p(fcp), fs_programmed, _p(fo), self.max_cells,
                                    C.byref(self._h)), ctx._h)

    def add_cell(self, ch, cell, frame_timing):
        _chk(lib().lcs_track_add_cell(self._h, ch, C.byref(cell), frame_timing), self.ctx._h)

    def push_cu8(self, iq_cu8):
        """iq_cu8: uint8 [n_ch][n][2] (or [n][2] for one channel)."""
        iq = np.ascontiguousarray(iq_cu8, np.uint8)
        n = iq.shape[-2]
        if iq.size != self.n_ch * n * 2:
            raise ValueError("push_cu8: expected [n_ch][n][2] samples")
        _chk(lib().lcs_track_push_cu8(self._h, _p(iq), n), self.ctx._h)

    def frequency_offset(self):
        fo = np.zeros(self.n_ch)
        _chk(lib().lcs_track_frequency_offset(self._h, _p(fo)), self.ctx._h)
        return fo

    def sample_time(self, ch=0):
        v = C.c_double(0)
        _chk(lib().lcs_track_sample_time(self._h, ch, C.byref(v)), self.ctx._h)
        return v.value

    def read(self, ch=0):
        """The channel's cells in the order added, as dicts; a dropped cell is reported once."""
        out = (TrackCell * self.max_cells)()
        n = C.c_uint32(0)
        _chk(lib().lcs_track_read(self._h, ch, out, self.max_cells, C.byref(n)), self.ctx._h)
        return [out[i].as_dict() for i in range(n.value)]


def chan_design_taps(fs_in):
    """The channelizer's prototype low-pass for input rate fs_in (host only, no device needed): float32 [L]."""
    return _query_then_fill(lib().lcs_chan_design_taps, fs_in, dtype=np.float32)


def chan_design_rational(fs_in):
    """fs_in / 1.92 MHz = down / up in lowest terms and the prototype low-pass at up * fs_in, DC gain up (host only):
    (up, down, float32 [L])."""
    up, down = C.c_uint32(0), C.c_uint32(0)
    h = _query_then_fill(lib().lcs_chan_design_rational, fs_in, C.byref(up), C.byref(down), dtype=np.float32)
    return up.value, down.value, h


# sample format name -> (lcs format, numpy dtype of the [...][2] components)
IQ_FORMATS = {"cf32": (IQ_CF32, np.float32), "cu8": (IQ_CU8, np.uint8), "c128": (IQ_C128, np.float64),
              "ci16": (IQ_CI16, np.int16), "cs8": (IQ_CS8, np.int8)}
SEARCH_FORMATS = ("cf32", "cu8", "c128")             # what the correlator, the search and the cell measurement take
STREAM_FORMATS = ("ci16", "cs8", "cu8", "cf32")      # what the channelizer and the spectrum take


def _iq_format(fmt):
    """The lcs format of a sample format name of STREAM_FORMATS."""
    if fmt not in STREAM_FORMATS:
        raise ValueError("fmt must be one of %s" % ", ".join(STREAM_FORMATS))
    return IQ_FORMATS[fmt][0]


def _samples(iq, fmt, ndims=(2,)):
    """iq as contiguous [...][2] components of fmt's dtype with one of `ndims` dimensions; complex64 / complex128 arrays
    (one dimension fewer) are accepted for cf32 / c128."""
    dtype = IQ_FORMATS[fmt][1]
    iq = np.asarray(iq)
    if iq.dtype in (np.complex64, np.complex128):
        iq = iq.view(iq.real.dtype).reshape(iq.shape + (2,))
    if iq.dtype != dtype or iq.ndim not in ndims or iq.shape[-1] != 2:
        raise ValueError("expected %s samples: %s, %s dimensions, the last of 2" % (fmt, np.dtype(dtype).name,
                                                                                  " or ".join(map(str, ndims))))
    return np.ascontiguousarray(iq)


class RationalChannelizer(_Handle):
    """lcs_chan at any allowed SDR rate: a wideband ci16 / cs8 / cu8 / cf32 recording -> one 1.92 Msps cu8 stream per LTE
    raster channel, resampled by up / down (DESIGN.md sections 4.6 and 4.7)."""
    _destroy = "lcs_chan_destroy"
    _timing_read = "lcs_chan_timing_read"

    def __init__(self, ctx, fs_in, fc_in, fc_ch, fmt="ci16", gain=None):
        self._iq_format = _iq_format(fmt)
        self.ctx = ctx
        self.fmt = fmt
        fc = np.ascontiguousarray(np.atleast_1d(fc_ch), np.float64)
        self.n_ch = fc.size
        self.fc_ch = fc
        g = None if gain is None else np.ascontiguousarray(np.broadcast_to(np.asarray(gain, np.float32), (self.n_ch,)))
        self._h = C.c_void_p()
        _chk(self._create(fs_in, fc_in, fc, g), ctx._h)
        self.up, self.down, self.taps = chan_design_rational(fs_in)
        self.M = (self.taps.size - 1) // 2

    def _create(self, fs_in, fc_in, fc, g):
        return lib().lcs_chan_create_rational(self.ctx._h, fs_in, self._iq_format, fc_in, self.n_ch, _p(fc), _p(g),
                                              C.byref(self._h))

    def _samples(self, iq):
        return _samples(iq, self.fmt)

    def auto_gain(self, iq):
        """Set every channel's gain to 0.25 / RMS of its output over these samples (the stream is not touched)."""
        iq = self._samples(iq)
        _chk(lib().lcs_chan_auto_gain(self._h, _p(iq), iq.shape[0]), self.ctx._h)
        return self.gain

    @property
    def gain(self):
        g = np.zeros(self.n_ch, np.float32)
        _chk(lib().lcs_chan_gain(self._h, _p(g)), self.ctx._h)
        return g

    def n_out(self, n_in):
        k = C.c_uint32(0)
        _chk(lib().lcs_chan_n_out(self._h, n_in, C.byref(k)), self.ctx._h)
        return k.value

    def push(self, iq):
        """Push [n][2] samples.  Returns (cu8 [n_ch][n_out][2], n_clipped [n_ch])."""
        iq = self._samples(iq)
        k = self.n_out(iq.shape[0])
        out = np.zeros((self.n_ch, k, 2), np.uint8)
        clip = np.zeros(self.n_ch, np.uint64)
        got = C.c_uint32(0)
        _chk(lib().lcs_chan_push(self._h, _p(iq), iq.shape[0], _p(out), k, 0, C.byref(got), _p(clip)), self.ctx._h)
        return out, clip

    def push_device(self, iq, out):
        """Push [n][2] samples, writing the bytes into the uint8 CUDA tensor out [n_ch][capacity][2] from column 0 on.
        Returns (n_out, n_clipped [n_ch])."""
        iq = self._samples(iq)
        if not (out.is_cuda and out.is_contiguous() and str(out.dtype) == "torch.uint8" and out.dim() == 3 and
                out.shape[0] == self.n_ch and out.shape[2] == 2):
            raise ValueError("push_device: expected a contiguous uint8 CUDA tensor [n_ch][capacity][2]")
        clip = np.zeros(self.n_ch, np.uint64)
        got = C.c_uint32(0)
        _chk(lib().lcs_chan_push(self._h, _p(iq), iq.shape[0], out.data_ptr(), out.shape[1], 1, C.byref(got), _p(clip)),
             self.ctx._h)
        return got.value, clip


class Channelizer(RationalChannelizer):
    """The ci16 channelizer of DESIGN.md section 4.6, made by lcs_chan_create: fs_in must be D * 1.92 MHz."""

    def __init__(self, ctx, fs_in, fc_in, fc_ch, gain=None):
        super().__init__(ctx, fs_in, fc_in, fc_ch, "ci16", gain)
        self.D = self.down

    def _create(self, fs_in, fc_in, fc, g):
        return lib().lcs_chan_create(self.ctx._h, fs_in, fc_in, self.n_ch, _p(fc), _p(g), C.byref(self._h))

    def _samples(self, iq):
        """iq as contiguous int16 [n][2], cast from other integer types."""
        return _samples(np.asarray(iq, np.int16), "ci16")

    push_ci16 = RationalChannelizer.push
    push_ci16_device = RationalChannelizer.push_device


class Spectrum(_Handle):
    """lcs_psd: Welch's power spectral density of a wideband ci16 / cs8 / cu8 / cf32 recording pushed in pieces of any
    size, periodic Hann window of nfft points, hop nfft/2 (DESIGN.md section 4.8)."""
    _destroy = "lcs_psd_destroy"
    _timing_read = "lcs_psd_timing_read"
    _lib = staticmethod(psd_lib)

    def __init__(self, ctx, fs_in, fmt="ci16", nfft=4096, fc_in=0.0):
        iq_format = _iq_format(fmt)
        self.ctx = ctx
        self.fmt = fmt
        self.fs_in = float(fs_in)
        self.fc_in = float(fc_in)
        self.nfft = int(nfft)
        self._h = C.c_void_p()
        _chk(psd_lib().lcs_psd_create(ctx._h, fs_in, iq_format, nfft, C.byref(self._h)), ctx._h)

    def push(self, iq):
        """Push [n][2] samples in the handle's format (complex64 [n] is accepted for cf32)."""
        iq = _samples(iq, self.fmt)
        _chk(psd_lib().lcs_psd_push(self._h, _p(iq), iq.shape[0]), self.ctx._h)

    @property
    def freqs(self):
        """Centre frequency of every output bin, fc_in + (i - nfft/2) * fs_in / nfft."""
        return self.fc_in + (np.arange(self.nfft) - self.nfft // 2) * (self.fs_in / self.nfft)

    def read(self):
        """(freqs, psd, n_segments): the PSD in full-scale^2 per Hz, fftshift order, over the segments completed since the
        last read; the accumulator then restarts."""
        psd = np.zeros(self.nfft)
        n = C.c_uint64(0)
        _chk(psd_lib().lcs_psd_read(self._h, _p(psd), C.byref(n)), self.ctx._h)
        return self.freqs, psd, n.value


# lcs_cell_meas as a numpy record
CELL_MEAS = np.dtype([("rsrp", np.float64, 4), ("noise", np.float64, 4), ("sinr", np.float64, 4), ("rssi", np.float64),
                      ("rsrq", np.float64), ("n_pairs", np.uint32, 4)], align=True)


class CellMeasure(_Handle):
    """lcs_meas: RSRP, RSRQ and SINR of found cells from the CRS of their central six resource blocks (DESIGN.md section
    4.9), every cell of a call in one grid launch and one measurement launch."""
    _destroy = "lcs_meas_destroy"
    _timing_read = "lcs_meas_timing_read"
    _lib = staticmethod(meas_lib)

    def __init__(self, ctx):
        self.ctx = ctx
        self._h = C.c_void_p()
        _chk(meas_lib().lcs_meas_create(ctx._h, C.byref(self._h)), ctx._h)

    def measure(self, iq, cells, ch=None, fs_programmed=1.92e6, fmt="cu8"):
        """Measure `cells` (Cells, or lists of them) found in the capture buffers iq [n_ch][n_cap][2] (or [n_cap][2] for
        one channel) of format fmt: cu8 (uint8), cf32 (float32) or c128 (float64); complex64 / complex128 [n_ch][n_cap]
        are accepted for cf32 / c128.  iq may be a contiguous CUDA tensor (read in place; its stream is synchronised
        first).  ch[i] is the channel of cell i (default 0).  Returns a CELL_MEAS record array, one row per cell."""
        if fmt not in SEARCH_FORMATS:
            raise KeyError(fmt)
        iq_format = IQ_FORMATS[fmt][0]
        cells = list(cells)
        n = len(cells)
        arr = (Cell * max(n, 1))()
        for i, c in enumerate(cells):                   # any struct of lcs_cell's layout (the oracle's Cell too)
            C.memmove(C.addressof(arr) + i * C.sizeof(Cell), C.byref(c), C.sizeof(Cell))
        chv = np.ascontiguousarray(np.zeros(n) if ch is None else ch, np.uint32)
        if chv.shape != (n,):
            raise ValueError("ch must hold one channel per cell")
        if hasattr(iq, "is_cuda"):
            if not (iq.is_cuda and iq.is_contiguous()):
                raise ValueError("measure: expected a contiguous CUDA tensor")
            shape = tuple(iq.shape)
            if iq.is_complex():
                shape = shape + (2,)
            import torch
            torch.cuda.current_stream(iq.device).synchronize()
            ptr, on_device = iq.data_ptr(), 1
        else:
            iq = _samples(iq, fmt, (2, 3))
            shape, ptr, on_device = iq.shape, iq.ctypes.data, 0
        if len(shape) == 2:
            shape = (1,) + shape
        if len(shape) != 3 or shape[2] != 2:
            raise ValueError("expected capture buffers [n_ch][n_cap][2]")
        out = np.zeros(n, CELL_MEAS)
        self._iq = iq                                   # kept alive until the call has returned
        _chk(meas_lib().lcs_meas_cells(self._h, ptr, iq_format, on_device, shape[0], shape[1], arr, _p(chv), n,
                                       fs_programmed, _p(out)), self.ctx._h)
        self._iq = None
        return out


class _GridModule(_Handle):
    """A module on the whole-carrier grid: `_lib` is its library, `_prefix` the prefix of its C functions (lcs_carrier,
    lcs_cir, lcs_pcfich, lcs_pdcch or lcs_sib1) and `_dtype` its record."""
    _prefix = _dtype = None

    def __init__(self, ctx):
        self.ctx = ctx
        self._h = C.c_void_p()
        self._destroy = self._prefix + "_destroy"
        self._timing_read = self._prefix + "_timing_read"
        _chk(getattr(self._lib(), self._prefix + "_create")(ctx._h, C.byref(self._h)), ctx._h)

    def measure(self, iq, fmt, fs_in, fc_in, cells, fs_programmed):
        """Measure `cells` (Cells, or any struct of lcs_cell's layout) in the recording iq [n_in][2] of format fmt (ci16,
        cs8, cu8 or cf32; complex64 [n_in] is accepted for cf32) at fs_in, centred on fc_in.  iq may be a contiguous
        CUDA tensor (read in place; its stream is synchronised first).  Returns a record array of the module's dtype, one
        row per cell."""
        iq_format = _iq_format(fmt)
        cells = list(cells)
        n = len(cells)
        arr = (Cell * max(n, 1))()
        for i, c in enumerate(cells):
            C.memmove(C.addressof(arr) + i * C.sizeof(Cell), C.byref(c), C.sizeof(Cell))
        if hasattr(iq, "is_cuda"):
            if not (iq.is_cuda and iq.is_contiguous()):
                raise ValueError("measure: expected a contiguous CUDA tensor")
            shape = tuple(iq.shape) + ((2,) if iq.is_complex() else ())
            import torch
            torch.cuda.current_stream(iq.device).synchronize()
            ptr, on_device = iq.data_ptr(), 1
        else:
            iq = _samples(iq, fmt)
            shape, ptr, on_device = iq.shape, iq.ctypes.data, 0
        if len(shape) != 2 or shape[1] != 2:
            raise ValueError("expected a recording [n_in][2]")
        out = np.zeros(n, self._dtype)
        self._iq = iq                                   # kept alive until the call has returned
        _chk(getattr(self._lib(), self._prefix + "_cells")(self._h, ptr, iq_format, on_device, shape[0], fs_in, fc_in, arr,
                                                           n, fs_programmed, _p(out)), self.ctx._h)
        self._iq = None
        return out


# lcs_carrier_meas as a numpy record
CARRIER_MEAS = np.dtype([("rsrp", np.float64, 4), ("noise", np.float64, 4), ("sinr", np.float64, 4), ("rssi", np.float64),
                         ("rsrq", np.float64), ("rb_rsrp", np.float64, (4, 100)), ("rb_noise", np.float64, (4, 100)),
                         ("rb_rssi", np.float64, 100), ("n_pairs", np.uint32, 4), ("n_rb", np.uint32)], align=True)
CARRIER_CHUNK = 32                    # LCS_CARRIER_CHUNK: cells per chunk, two launches each


class CarrierMeasure(_GridModule):
    """lcs_carrier: RSRP, RSRQ and SINR of found cells over all their resource blocks, and per resource block, measured on
    the wideband recording they were found in (DESIGN.md section 4.10)."""
    _lib = staticmethod(carrier_lib)
    _prefix = "lcs_carrier"
    _dtype = CARRIER_MEAS


# lcs_cir_meas as a numpy record
CIR_TAPS = 320                        # LCS_CIR_TAPS: tap j is (j - 64) / 30.72 MHz
CIR_MEAS = np.dtype([("pdp", np.float64, (4, CIR_TAPS)), ("floor", np.float64, 4), ("peak_delay", np.float64, 4),
                     ("first_delay", np.float64, 4), ("mean_delay", np.float64, 4), ("rms_spread", np.float64, 4),
                     ("frame_arrival", np.float64), ("n_pairs", np.uint32, 4), ("n_taps", np.uint32, 4)], align=True)
CIR_CHUNK = 32                        # LCS_CIR_CHUNK: cells per chunk, two launches each


def cir_delays():
    """The delay of every tap of CIR_MEAS.pdp, seconds."""
    return (np.arange(CIR_TAPS) - 64) * (1 / 30.72e6)


class CellImpulse(_GridModule):
    """lcs_cir: the power delay profile of found cells over their whole carrier, with its first-path and peak delay, mean
    delay, RMS delay spread and the frame's arrival time, measured on the wideband recording they were found in (DESIGN.md
    section 4.11)."""
    _lib = staticmethod(cir_lib)
    _prefix = "lcs_cir"
    _dtype = CIR_MEAS


# lcs_pcfich_meas as a numpy record
PCFICH_SUBFRAMES = 61                 # LCS_PCFICH_SUBFRAMES
PCFICH_MEAS = np.dtype([("metric", np.float64, (PCFICH_SUBFRAMES, 3)), ("sinr", np.float64, PCFICH_SUBFRAMES),
                        ("cfi", np.uint32, PCFICH_SUBFRAMES), ("count", np.uint32, 4), ("cfi_mode", np.uint32),
                        ("n_ctrl_symbols", np.uint32), ("n_subframes", np.uint32)], align=True)
PCFICH_CHUNK = 32                     # LCS_PCFICH_CHUNK: cells per chunk, two launches each


class ControlFormat(_GridModule):
    """lcs_pcfich: the control format indicator of found cells in every subframe, decoded from their PCFICH over the
    whole carrier of the wideband recording they were found in (DESIGN.md section 4.12)."""
    _lib = staticmethod(pcfich_lib)
    _prefix = "lcs_pcfich"
    _dtype = PCFICH_MEAS


# lcs_pdcch_dci and lcs_pdcch_meas as numpy records
PDCCH_SUBFRAMES = 61                  # LCS_PDCCH_SUBFRAMES
PDCCH_MAX_DCI = 6                     # LCS_PDCCH_MAX_DCI
DCI_1A, DCI_1C = 1, 2                 # LCS_DCI_1A, LCS_DCI_1C
RNTI_SI, RNTI_P = 0xFFFF, 0xFFFE      # LCS_RNTI_SI, LCS_RNTI_P
PDCCH_DCI = np.dtype([("quality", np.float64), ("payload", np.uint64), ("format", np.uint32), ("agg", np.uint32),
                      ("cce", np.uint32), ("rnti", np.uint32), ("n_bits", np.uint32), ("riv", np.uint32),
                      ("rb_start", np.int32), ("n_rb", np.int32), ("localized", np.uint32), ("mcs", np.uint32),
                      ("harq", np.uint32), ("ndi", np.uint32), ("rv", np.uint32), ("tpc", np.uint32), ("gap", np.uint32),
                      ("tbs_index", np.uint32)], align=True)
PDCCH_MEAS = np.dtype([("dci", PDCCH_DCI, (PDCCH_SUBFRAMES, PDCCH_MAX_DCI)), ("cfi", np.uint32, PDCCH_SUBFRAMES),
                       ("n_ctrl", np.uint32, PDCCH_SUBFRAMES), ("n_reg", np.uint32, PDCCH_SUBFRAMES),
                       ("n_cce", np.uint32, PDCCH_SUBFRAMES), ("n_dci", np.uint32, PDCCH_SUBFRAMES), ("count", np.uint32, 3),
                       ("si_subframes", np.uint32), ("n_subframes", np.uint32)], align=True)
PDCCH_CHUNK = 32                      # LCS_PDCCH_CHUNK: cells per chunk, three launches each


class ControlChannel(_GridModule):
    """lcs_pdcch: the common-search-space DCIs (SI-, P- and RA-RNTI, formats 1A and 1C) of found cells in every
    subframe, decoded from their PDCCH over the whole carrier of the wideband recording they were found in (DESIGN.md
    section 4.13)."""
    _lib = staticmethod(pdcch_lib)
    _prefix = "lcs_pdcch"
    _dtype = PDCCH_MEAS


# lcs_sib1_occasion and lcs_sib1_meas as numpy records
SIB1_OCCASIONS = 3                    # LCS_SIB1_OCCASIONS
SIB1_TB_BYTES = 280                   # LCS_SIB1_TB_BYTES
SIB1_OCC = np.dtype([("sinr", np.float64), ("dci", PDCCH_DCI), ("subframe", np.uint32), ("sfn", np.uint32),
                     ("found", np.uint32), ("cfi", np.uint32), ("n_ctrl", np.uint32), ("format", np.uint32),
                     ("distributed", np.uint32), ("gap", np.uint32), ("vrb_start", np.int32), ("n_vrb", np.int32),
                     ("n_prb", np.uint32), ("prb", np.uint8, (2, 100)), ("tbs", np.uint32), ("K", np.uint32), ("F", np.uint32),
                     ("rv", np.uint32), ("n_re", np.uint32), ("crc_ok", np.uint32), ("iterations", np.uint32),
                     ("tb", np.uint8, SIB1_TB_BYTES)], align=True)
SIB1_PLMN = np.dtype([("mcc", np.uint32), ("mnc", np.uint32), ("mnc_digits", np.uint32), ("reserved", np.uint32)], align=True)
SIB1_MEAS = np.dtype([("occ", SIB1_OCC, SIB1_OCCASIONS), ("n_found", np.uint32), ("n_crc_ok", np.uint32),
                      ("consistent", np.uint32), ("parse_ok", np.uint32), ("n_plmn", np.uint32), ("plmn", SIB1_PLMN, 6),
                      ("tac", np.uint32), ("cell_identity", np.uint32), ("cell_barred", np.uint32),
                      ("intra_freq_reselection", np.uint32), ("csg_indication", np.uint32),
                      ("csg_identity_present", np.uint32), ("csg_identity", np.uint32), ("q_rx_lev_min", np.int32),
                      ("q_rx_lev_min_offset", np.uint32), ("p_max_present", np.uint32), ("p_max", np.int32),
                      ("freq_band_indicator", np.uint32), ("n_si", np.uint32), ("si_periodicity", np.uint32, 32),
                      ("si_sib_mask", np.uint32, 32), ("tdd_present", np.uint32), ("tdd_subframe_assignment", np.uint32),
                      ("tdd_special_subframe_patterns", np.uint32), ("si_window_ms", np.uint32),
                      ("system_info_value_tag", np.uint32), ("non_critical_extension", np.uint32)], align=True)
SIB1_CHUNK = 32                       # LCS_SIB1_CHUNK: cells per chunk, five launches each


class SystemInfo(_GridModule):
    """lcs_sib1: SystemInformationBlockType1 of found cells (their PLMNs, tracking area code and cell identity), decoded
    from the PDSCH their SI-RNTI DCIs schedule in the three SIB1 occasions of the wideband recording they were found in
    (DESIGN.md section 4.14).  Each cell's `sfn` must be that of its grid frame 0, as lcs_decode_mib reports it."""
    _lib = staticmethod(sib1_lib)
    _prefix = "lcs_sib1"
    _dtype = SIB1_MEAS
