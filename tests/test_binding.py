"""The ctypes prototypes lcs_b200.lib() reads from include/lcs_b200.h: every declared function is bound, with the types
the header states, and a mistyped or missing argument is refused before the library runs (no GPU needed)."""
import ctypes as C
import re
import subprocess

import pytest


def test_prototype_table_covers_header_and_library(lcs):
    header = re.sub(r"/\*.*?\*/", " ", open(lcs.HEADER).read(), flags=re.S)
    names = set(re.findall(r"\b(lcs_\w+)\s*\(", header))
    assert set(lcs.prototypes()) == names
    assert len(names) == 61
    nm = subprocess.run(["nm", "-D", "--defined-only", lcs.LIB_PATH], check=True, capture_output=True, text=True).stdout
    exported = {line.split()[-1] for line in nm.splitlines() if line.split() and line.split()[-1].startswith("lcs_")}
    assert exported == names
    l = lcs.lib()
    for n in names:
        assert getattr(l, n).argtypes is not None, n


def test_prototypes_of_selected_functions(lcs):
    l = lcs.lib()
    assert l.lcs_xcorr_pss_device.argtypes == [C.c_void_p, C.c_void_p, C.c_int, C.c_uint32] + [C.c_void_p] * 6
    assert l.lcs_chan_n_out.argtypes[1] is C.c_uint64
    assert l.lcs_kalibrate_cu8.argtypes[3:8] == [C.c_double] * 5
    assert l.lcs_kalibrate_cu8.argtypes[2] is C.c_uint32 and l.lcs_kalibrate_cu8.argtypes[8] is C.c_void_p
    assert l.lcs_framer_sample_time.restype is C.c_double
    assert l.lcs_xcorr_plan_n_comb_xc.restype is C.c_uint16
    assert l.lcs_launch_count.restype is C.c_uint64
    assert l.lcs_version.restype is C.c_char_p and l.lcs_version.argtypes == []
    assert l.lcs_ctx_destroy.restype is None
    assert l.lcs_f_search_set.restype is C.c_int


def test_bad_calls_are_refused_before_the_library_runs(lcs):
    l = lcs.lib()
    n = C.c_uint32(0)
    with pytest.raises(C.ArgumentError):
        l.lcs_f_search_set("739e6", 120.0, None, C.byref(n))
    with pytest.raises(TypeError):
        l.lcs_f_search_set(739e6, 120.0, None)
    assert n.value == 0
    assert l.lcs_f_search_set(739e6, 120, None, C.byref(n)) == 0 and n.value == 37      # an int converts to double


def test_unknown_type_is_refused_by_name(lcs):
    with pytest.raises(lcs.LcsError, match="lcs_x.*unsigned"):
        lcs._ctype("lcs_x", "unsigned n")
