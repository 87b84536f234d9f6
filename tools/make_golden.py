#!/usr/bin/env python
"""Regenerate tests/golden/*.npz from the reference's own fixtures.

Needs a checkout of the reference project: `python tools/make_golden.py <reference dir>` (or
LCS_REFERENCE=<dir>).  The .it files are the reference's golden vectors (SURVEY.md section 4.1);
they are stored as compressed .npz so that no test needs the reference at run time.

  capbuf_0000.npz       real 8-bit capture (test/capbuf_0000.it) as raw cu8 + fc
  ref_xcorr_pss.npz     test/test_xcorr_pss.it  (Matlab-era semantics -> oracle legacy mode)
  ref_peak_search.npz   test/test_peak_search.it
  ref_sss_detect.npz    test/test_sss_detect.it
  ref_tfg.npz           test/test_tfg.it

The 19 MB `xc` and 1 MB `sp` debug arrays are thinned (a dense head + a strided
comb); everything else is stored in full, bit for bit (float64 / int32).
"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from itfile import read_it  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("LCS_REFERENCE", "")
OUT = os.path.join(HERE, "..", "tests", "golden")


def main():
    os.makedirs(OUT, exist_ok=True)
    t = os.path.join(REF, "test")

    v = read_it(os.path.join(t, "capbuf_0000.it"))
    q = v["capbuf"].view(np.float64) * 128 + 127
    assert np.all(q == np.round(q)) and q.min() >= 0 and q.max() <= 255
    np.savez_compressed(os.path.join(OUT, "capbuf_0000.npz"),
                        cu8=q.astype(np.uint8), fc=v["fc"])

    v = read_it(os.path.join(t, "test_xcorr_pss.it"))
    n_f = len(v["f_search_set"])
    n_lag = v["xc"].size // (3 * n_f)
    xc = v["xc"].reshape((n_f, n_lag, 3))            # flatten(): t fastest, then k, then f
    lag_idx = np.unique(np.concatenate([np.arange(4096), np.arange(0, n_lag, 97),
                                        np.arange(n_lag - 512, n_lag)]))
    sp_idx = np.unique(np.concatenate([np.arange(4096), np.arange(0, v["sp"].size, 16)]))
    np.savez_compressed(
        os.path.join(OUT, "ref_xcorr_pss.npz"),
        capbuf=v["capbuf"], f_search_set=v["f_search_set"], ds_comb_arm=v["ds_comb_arm"],
        fc=v["fc"], n_comb_xc=v["n_comb_xc"], n_comb_sp=v["n_comb_sp"],
        pow=v["xc_incoherent_collapsed_pow"], frq=v["xc_incoherent_collapsed_frq"],
        single=v["xc_incoherent_single"], incoherent=v["xc_incoherent"],
        sp_incoherent=v["sp_incoherent"],
        xc_lag_idx=lag_idx.astype(np.int32), xc_sub=xc[:, lag_idx, :],
        xc_n_lag=np.int32(n_lag),
        xc_abs2_sum=np.float64((np.abs(v["xc"]) ** 2).sum()),
        sp_idx=sp_idx.astype(np.int32), sp_sub=v["sp"][sp_idx], sp_sum=np.float64(v["sp"].sum()))

    v = read_it(os.path.join(t, "test_peak_search.it"))
    np.savez_compressed(os.path.join(OUT, "ref_peak_search.npz"), **v)

    v = read_it(os.path.join(t, "test_sss_detect.it"))
    np.savez_compressed(os.path.join(OUT, "ref_sss_detect.npz"), **v)

    w = read_it(os.path.join(t, "test_tfg.it"))
    same = np.array_equal(w["capbuf"], v["capbuf"])
    if same:
        w = dict(w)
        del w["capbuf"]          # identical to ref_sss_detect's capbuf
    w["capbuf_same_as_sss_detect"] = np.int32(same)
    np.savez_compressed(os.path.join(OUT, "ref_tfg.npz"), **w)
    for f in sorted(os.listdir(OUT)):
        print("%-24s %9d B" % (f, os.path.getsize(os.path.join(OUT, f))))


if __name__ == "__main__":
    main()
