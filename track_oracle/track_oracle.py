"""ctypes binding of the CPU oracle of the cell tracker (libtrack_oracle.so).  TEST INFRASTRUCTURE ONLY.

Same interface as lcs_b200.Tracker, without a device: the tests compare the two after every push."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "lte-cell-scanner_b200"))
from lcs_b200 import TrackCell, Cell  # noqa: E402  (the POD layouts of include/lcs_b200.h)

LIB_PATH = os.path.join(HERE, "libtrack_oracle.so")
_lib = None


def build():
    subprocess.check_call(["make", "-C", HERE, "-s"])
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()                                   # make is incremental: an edited track_oracle.cpp is rebuilt
        _lib = C.CDLL(LIB_PATH)
        _lib.to_create.restype = C.c_void_p
        _lib.to_create.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_uint32]
        _lib.to_destroy.argtypes = [C.c_void_p]
        _lib.to_add_cell.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_double]
        _lib.to_push_cu8.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        _lib.to_frequency_offset.argtypes = [C.c_void_p, C.c_void_p]
        _lib.to_sample_time.argtypes = [C.c_void_p, C.c_uint32]
        _lib.to_sample_time.restype = C.c_double
        _lib.to_read.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    return _lib


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


class Tracker:
    def __init__(self, fc_requested, frequency_offset, fs_programmed=1.92e6, fc_programmed=None, max_cells=8):
        fc = np.ascontiguousarray(np.atleast_1d(fc_requested), np.float64)
        self.n_ch = fc.size
        self._fc = fc
        self._fcp = None if fc_programmed is None else np.ascontiguousarray(np.atleast_1d(fc_programmed), np.float64)
        fo = np.ascontiguousarray(np.broadcast_to(np.asarray(frequency_offset, np.float64), (self.n_ch,)))
        self.max_cells = int(max_cells)
        self._h = lib().to_create(self.n_ch, _p(fc), _p(self._fcp), fs_programmed, _p(fo), self.max_cells)

    def add_cell(self, ch, cell, frame_timing):
        if lib().to_add_cell(self._h, ch, C.byref(cell), frame_timing) != 0:
            raise ValueError("add_cell: bad channel or channel full")

    def push_cu8(self, iq_cu8):
        iq = np.ascontiguousarray(iq_cu8, np.uint8)
        n = iq.shape[-2]
        assert iq.size == self.n_ch * n * 2
        lib().to_push_cu8(self._h, _p(iq), n)

    def frequency_offset(self):
        fo = np.zeros(self.n_ch)
        lib().to_frequency_offset(self._h, _p(fo))
        return fo

    def sample_time(self, ch=0):
        return lib().to_sample_time(self._h, ch)

    def read(self, ch=0):
        out = (TrackCell * self.max_cells)()
        n = C.c_uint32(0)
        lib().to_read(self._h, ch, out, self.max_cells, C.byref(n))
        return [out[i].as_dict() for i in range(n.value)]

    def close(self):
        if self._h:
            lib().to_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
