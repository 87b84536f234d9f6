"""Parity of the CUDA path (through the C ABI) against the CPU oracle and the golden fixtures.

Tolerances: correlation magnitudes |a-b| <= 1e-6*max|ref| per array (BASELINE.md section 4); frequency indices at
detections bit-exact; found cells and peaks field by field under test_search_chain_gpu.compare_cells, two device
results bit for bit under same_cells."""
import numpy as np
import pytest

from conftest import cu8_to_c128, load, synth_cu8
from test_search_chain_gpu import compare_cells, same_cells

pytestmark = pytest.mark.gpu

REL = 1e-6


@pytest.fixture(scope="module")
def capbuf_chain(oracle, capbuf0000):
    """The oracle's chain on the recording at the +-120 ppm grid: (grid, cells, peaks)."""
    fc = capbuf0000["fc"]
    f = oracle.f_search_set(fc, 120.0)
    return (f, *oracle.cell_search_one(capbuf0000["capbuf"], f, fc, fc, 1.92e6))


def rel_err(a, ref):
    return np.abs(np.asarray(a, np.float64) - ref).max() / np.abs(ref).max()


def frq_mismatch_is_near_tie(frq_gpu, ref, tol=4e-6):
    """argmax over f may differ only where the two best hypotheses are within fp32 noise."""
    bad = np.argwhere(frq_gpu != ref["frq"])
    for t, k in bad:
        v = ref["incoherent"][t, k]
        if abs(v[frq_gpu[t, k]] - v[ref["frq"][t, k]]) > tol * ref["incoherent"].max():
            return False
    return len(bad) < 0.002 * frq_gpu.size


def check_xcorr(out, ref):
    assert out["n_comb_xc"] == ref["n_comb_xc"] and out["n_comb_sp"] == ref["n_comb_sp"]
    assert rel_err(out["single"], ref["single"]) < REL
    assert rel_err(out["incoherent"], ref["incoherent"]) < REL
    assert rel_err(out["pow"], ref["pow"]) < REL
    assert np.abs(out["sp_incoherent"] / ref["sp_incoherent"] - 1).max() < 1e-12
    assert frq_mismatch_is_near_tie(out["frq"], ref)


def test_xcorr_pss_dropin_capbuf_0000(ctx, oracle, capbuf0000):
    """searcher.h xcorr_pss drop-in, real capture, default ppm=120 grid (n_f=37)."""
    fc = capbuf0000["fc"]
    f = oracle.f_search_set(fc, 120.0)
    ref = oracle.xcorr_pss(capbuf0000["capbuf"], f, 2, fc, fc, 1.92e6)
    out = ctx.xcorr_pss(capbuf0000["capbuf"], f, 2, fc, fc, 1.92e6)
    check_xcorr(out, ref)
    # the detections are decided on exactly equal indices
    for (t, k) in [(1, 1410), (1, 6990), (2, 1314), (0, 1327)]:
        for d in range(-2, 3):
            assert out["frq"][t, k + d] == ref["frq"][t, k + d]


def test_xcorr_pss_dropin_debug_outputs(ctx, oracle):
    """xc and sp debug outputs on the reference's test_xcorr_pss capture (n_f=3)."""
    g = load("ref_xcorr_pss.npz")
    f = g["f_search_set"].astype(float); fc = float(g["fc"][0])
    ref = oracle.xcorr_pss(g["capbuf"], f, 2, fc, fc, 1.92e6, want_xc=True)
    out = ctx.xcorr_pss(g["capbuf"], f, 2, fc, fc, 1.92e6, want_xc=True, want_sp=True)
    check_xcorr(out, ref)
    assert np.abs(out["xc"].astype(np.complex128) - ref["xc"]).max() < REL * np.abs(ref["xc"]).max()
    assert np.abs(out["sp"] / ref["sp"] - 1).max() < 1e-11


@pytest.mark.parametrize("fmt", ["cu8", "cf32", "c128"])
def test_xcorr_batch_host_formats(ctx, lcs, oracle, fmt):
    """Batched host entry point with the three wire formats, synthetic 8-bit IQ, 2 buffers."""
    fc = 739e6
    f = oracle.f_search_set(fc, 20.0)          # n_f = 7 keeps the oracle fast
    cu8 = np.stack([synth_cu8(0xC0FFEE + i) for i in range(2)])
    plan = ctx.plan(153600, f, 2, fc, fc, 1.92e6, max_batch=2)
    if fmt == "cu8":
        out = plan.run_host_np(cu8, lcs.IQ_CU8)
    elif fmt == "cf32":
        x = ((cu8.astype(np.float32) - 127) / 128)
        out = plan.run_host_np(x, lcs.IQ_CF32)
    else:
        x = ((cu8.astype(np.float64) - 127) / 128)
        out = plan.run_host_np(x, lcs.IQ_C128)
    for b in range(2):
        ref = oracle.xcorr_pss(cu8_to_c128(cu8[b]), f, 2, fc, fc, 1.92e6)
        assert rel_err(out["single"][b].transpose(0, 2, 1), ref["single"]) < REL
        assert rel_err(out["pow"][b], ref["pow"]) < REL
        assert np.abs(out["sp_incoherent"][b] / ref["sp_incoherent"] - 1).max() < 1e-12
        assert frq_mismatch_is_near_tie(out["frq"][b], ref)
    plan.close()


def test_xcorr_edge_shapes(ctx, lcs, oracle):
    """Ragged grids and sizes: n_f=1 (tracker mode), n_f not a multiple of 8, asymmetric offsets,
    fc_programmed != fc_requested, short buffer (n_comb=2), arm=0."""
    rng = np.random.default_rng(3)
    cases = [
        (153600, np.array([35000.0]), 2, 739e6, 739e6, 1.92e6),
        (60000, np.arange(-4, 5) * 5000.0, 2, 739e6, 739.003e6, 1.92e6 * 1.00002),
        (29000, np.array([-20000.0, 0.0, 5000.0]), 0, 2.1e9, 2.1e9, 1.92e6),
        (153600, np.arange(-5, 6) * 7000.0 + 1234.5, 3, 451e6, 451e6, 1.92e6),
    ]
    for n_cap, f, arm, fcr, fcp, fs in cases:
        cap = (rng.standard_normal(n_cap) + 1j * rng.standard_normal(n_cap)) * 0.2
        ref = oracle.xcorr_pss(cap, f, arm, fcr, fcp, fs)
        out = ctx.xcorr_pss(cap, f, arm, fcr, fcp, fs)
        check_xcorr(out, ref)


def test_xcorr_argument_errors(ctx, lcs):
    with pytest.raises(lcs.LcsError):
        ctx.plan(5000, np.array([0.0]), 2, 739e6, 739e6, 1.92e6)           # shorter than a half frame
    with pytest.raises(lcs.LcsError):
        ctx.plan(153600, np.array([]), 2, 739e6, 739e6, 1.92e6)            # empty grid
    with pytest.raises(lcs.LcsError):
        ctx.plan(20000, np.array([0.0]), 2, 739e6, 600e6, 1.92e6)          # k_factor pushes the fold out of range


def test_xcorr_full_size_properties(ctx, lcs):
    """BASELINE config 2 size (n_f=31, batch 4): properties that need no oracle.
    - shift: delaying the buffer by d samples (d < 100) rotates the fold by d
    - scaling the 8-bit amplitude about 127 by 2 scales powers by 4 (exact in fp32)
    - batch entries are independent of their neighbours (same input -> bit-identical output)."""
    fc = 739e6
    f = lcs.f_search_set(fc, 100.0)
    assert f.size == 31
    base = synth_cu8(0xC0FFEE, sigma=10.0)
    d = 37
    shifted = np.roll(base, d, axis=0)
    doubled = np.clip((base.astype(np.int32) - 127) * 2 + 127, 0, 255).astype(np.uint8)
    assert np.array_equal((doubled.astype(np.int32) - 127), (base.astype(np.int32) - 127) * 2)
    plan = ctx.plan(153600, f, 2, fc, fc, 1.92e6, max_batch=4)
    out = plan.run_host_np(np.stack([base, shifted, doubled, base]), lcs.IQ_CU8)
    s = out["single"]
    assert np.array_equal(s[0], s[3]) and np.array_equal(out["frq"][0], out["frq"][3])
    if plan.kernel_for(lcs.IQ_CU8) == lcs.KERNEL_FP32:
        assert np.array_equal(s[2], s[0] * 4.0)          # every fp32 operation scales exactly
    else:
        # the integer path works on v-128 (not v-127), so doubling is exact only up to the final float roundings
        assert np.abs(s[2] - s[0] * 4.0).max() <= 3e-7 * (4 * s[0].max())
    fp = ctx.plan(153600, f, 2, fc, fc, 1.92e6, max_batch=2, kernel=lcs.KERNEL_FP32)
    o2 = fp.run_host_np(np.stack([base, doubled]), lcs.IQ_CU8)
    assert np.array_equal(o2["single"][1], o2["single"][0] * 4.0)
    fp.close()
    # the roll moves every lag by d except those touching the wrapped head/tail of the buffer
    a, b = s[0][:, :, : 9600 - d], s[1][:, :, d:]
    assert np.abs(a[:, :, 300:] - b[:, :, 300:]).max() <= 2e-6 * a.max()
    assert out["pow"].shape == (4, 3, 9600) and (out["frq"] >= 0).all() and (out["frq"] < 31).all()
    plan.close()


def test_sss_detect_foe_parity(ctx, oracle):
    """sss_detect + pss_sss_foe on the reference's synthetic capture: 24 peaks incl. 2 rejections."""
    g = load("ref_sss_detect.npz")
    cap = g["capbuf"]; fc = float(g["fc"][0]); th = float(g["thresh2_n_sigma"][0])
    for t in range(len(g["peaks_pow"])):
        kw = dict(pss_pow=g["peaks_pow"][t], ind=int(g["peaks_ind"][t]) - 1, freq=float(g["peaks_freq"][t]),
                  n_id_2=int(g["peaks_n_id_2"][t]))
        import lcs_b200
        o_out, o_d = oracle.sss_detect(oracle.new_cell(**kw), cap, th, fc, fc, 1.92e6)
        p_out, p_d = ctx.sss_detect(lcs_b200.new_cell(**kw), cap, th, fc, fc, 1.92e6)
        for k in ["h1_np", "h2_np", "h1_nrm", "h2_nrm", "h1_ext", "h2_ext"]:
            assert np.abs(p_d[k] - o_d[k]).max() < 1e-10 * max(1.0, np.abs(o_d[k]).max())
        assert np.abs(p_d["log_lik_nrm"] - o_d["log_lik_nrm"]).max() < 1e-8 * np.abs(o_d["log_lik_nrm"]).max()
        assert np.abs(p_d["log_lik_ext"] - o_d["log_lik_ext"]).max() < 1e-8 * np.abs(o_d["log_lik_ext"]).max()
        assert (p_out.n_id_1, p_out.cp_type) == (o_out.n_id_1, o_out.cp_type)
        if o_out.n_id_1 >= 0:
            assert abs(p_out.frame_start - o_out.frame_start) < 1e-9
            o2 = oracle.pss_sss_foe(o_out, cap, fc, fc, 1.92e6)
            p2 = ctx.pss_sss_foe(p_out, cap, fc, fc, 1.92e6)
            assert abs(p2.freq_fine - o2.freq_fine) < 1e-6
        else:
            assert np.isnan(p_out.frame_start)
    # golden decisions (mode independent): ids and CP types of test_sss_detect.it
    n1 = g["peaks_out_n_id_1"]
    assert np.isnan(n1).sum() == 2


def test_extract_tfg_parity(ctx, oracle, lcs):
    g = load("ref_tfg.npz")
    cap = g["capbuf"]; fc = float(g["fc"][0])
    kw = dict(n_id_1=92, n_id_2=1, cp_type=1, frame_start=float(g["peaks_in_frame_start"][0]) - 1,
              freq_fine=float(g["peaks_in_freq_fine"][0]))
    o_tfg, o_ts = oracle.extract_tfg(oracle.new_cell(**kw), cap, fc, fc, 1.92e6)
    p_tfg, p_ts = ctx.extract_tfg(lcs.new_cell(**kw), cap, fc, fc, 1.92e6)
    assert p_tfg.shape == (854, 72) and np.array_equal(p_ts, o_ts)
    assert np.abs(p_tfg - o_tfg).max() < 1e-11 * np.abs(o_tfg).max()
    kw["cp_type"] = 2                                   # extended CP: 732 symbols
    o_tfg, o_ts = oracle.extract_tfg(oracle.new_cell(**kw), cap, fc, fc, 1.92e6)
    p_tfg, p_ts = ctx.extract_tfg(lcs.new_cell(**kw), cap, fc, fc, 1.92e6)
    assert p_tfg.shape == (732, 72) and np.abs(p_tfg - o_tfg).max() < 1e-11 * np.abs(o_tfg).max()
    with pytest.raises(lcs.LcsError):
        ctx.extract_tfg(lcs.new_cell(n_id_1=92, n_id_2=1), cap, fc, fc, 1.92e6)     # cp_type unknown


@pytest.mark.parametrize("fmt", ["c128", "cu8"])
def test_full_chain_capbuf_0000(ctx, capbuf0000, capbuf_chain, fmt):
    """BASELINE config 3: xcorr_pss -> peak_search -> sss_detect -> pss_sss_foe -> extract_tfg -> tfoec ->
    decode_mib on the shipped real capture; peaks and cells 277 and 271 field by field against the oracle."""
    fc = capbuf0000["fc"]
    f, o_cells, o_peaks = capbuf_chain
    cap = capbuf0000["capbuf"] if fmt == "c128" else capbuf0000["cu8"]
    p_cells, p_peaks = ctx.cell_search(cap, f, fc, fc, 1.92e6)
    compare_cells(p_peaks, o_peaks)
    assert [c.n_id_cell() for c in o_cells] == [277, 271]
    compare_cells(p_cells, o_cells)


def test_cellsearch_cli_full_test(ctx, tmp_path, capbuf0000):
    """The reference's (commented-out) integration test, src/CMakeLists.txt:34-35:
    `CellSearch -s 739000000 -l -d test` must print `cell ID: 271`.  Run through the C++ drop-in
    (searcher.h mirror + CLI) on a capbuf_0000.it regenerated from the committed fixture."""
    import os
    import re
    import subprocess
    import sys
    root = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
    sys.path.insert(0, os.path.join(root, "tools"))
    from itfile import write_it
    host = os.path.join(root, "lte-cell-scanner_b200", "host")
    subprocess.check_call(["make", "-C", host, "-s"])
    write_it(str(tmp_path / "capbuf_0000.it"), {"capbuf": capbuf0000["capbuf"], "fc": np.array([739000000], np.int32)})
    out = subprocess.run([os.path.join(host, "CellSearch_b200"), "-s", "739000000", "-l", "-d", str(tmp_path)],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert re.search(r"cell.ID..271", out.stdout) and re.search(r"cell.ID..277", out.stdout)
    rows = [l for l in out.stdout.splitlines() if re.match(r"^\s*27[17]\s+2\s", l)]
    assert len(rows) == 2
    for r in rows:                      # CID A fc foff RXPWR C nRB P PR ...  (doc/CellSearch.html example)
        assert " N  50 N one " in r and "739M" in r
    # raw rtl_sdr byte dump path
    capbuf0000["cu8"].tofile(str(tmp_path / "capbuf_0000.bin"))
    out2 = subprocess.run([os.path.join(host, "CellSearch_b200"), "-s", "739000000", "-l", "--raw", "-b", "-d", str(tmp_path)],
                          capture_output=True, text=True, timeout=300)
    assert out2.returncode == 0 and len([l for l in out2.stdout.splitlines() if re.match(r"^\s*27[17]\s+2\s", l)]) == 2


# ---------------------------------------------------------------------------------------------
# Tensor-core correlator (wgmma s8 x s8 -> s32, exact integer arithmetic for 8-bit IQ)
# ---------------------------------------------------------------------------------------------
def _tc_vs_oracle(ctx, lcs, oracle, cu8_batch, f, fcr, fcp, fs, arm=2):
    plan = ctx.plan(cu8_batch.shape[1], f, arm, fcr, fcp, fs, max_batch=cu8_batch.shape[0], kernel=lcs.KERNEL_TC)
    assert plan.kernel_for(lcs.IQ_CU8) == lcs.KERNEL_TC
    out = plan.run_host_np(cu8_batch, lcs.IQ_CU8)
    for b in range(cu8_batch.shape[0]):
        ref = oracle.xcorr_pss(cu8_to_c128(cu8_batch[b]), f, arm, fcr, fcp, fs)
        assert rel_err(out["single"][b].transpose(0, 2, 1), ref["single"]) < 5e-7      # exact integers + 2 float roundings
        assert rel_err(out["pow"][b], ref["pow"]) < 5e-7
        assert np.abs(out["sp_incoherent"][b] / ref["sp_incoherent"] - 1).max() < 1e-12
        assert frq_mismatch_is_near_tie(out["frq"][b], ref)
    plan.close()
    return out


def test_tc_capbuf_0000(ctx, lcs, oracle, capbuf0000):
    f = oracle.f_search_set(capbuf0000["fc"], 120.0)
    _tc_vs_oracle(ctx, lcs, oracle, capbuf0000["cu8"][None], f, 739e6, 739e6, 1.92e6)


def test_tc_synthetic_batch_and_extremes(ctx, lcs, oracle):
    """Batch of 3 incl. a full-scale buffer (bytes 0 and 255 everywhere: the int8 edge cases of the
    v-128 / ~I representation) and an all-127 (zero signal) buffer."""
    rng = np.random.default_rng(11)
    full = rng.choice(np.array([0, 255], np.uint8), size=(153600, 2))
    zero = np.full((153600, 2), 127, np.uint8)
    cu8 = np.stack([synth_cu8(0xC0FFEE), full, zero])
    f = oracle.f_search_set(739e6, 20.0)
    plan = ctx.plan(153600, f, 2, 739e6, 739e6, 1.92e6, max_batch=3, kernel=lcs.KERNEL_TC)
    out = plan.run_host_np(cu8, lcs.IQ_CU8)
    for b in range(2):
        ref = oracle.xcorr_pss(cu8_to_c128(cu8[b]), f, 2, 739e6, 739e6, 1.92e6)
        assert rel_err(out["single"][b].transpose(0, 2, 1), ref["single"]) < 5e-7
        assert frq_mismatch_is_near_tie(out["frq"][b], ref)
    assert np.all(out["single"][2] == 0) and np.all(out["pow"][2] == 0) and np.all(out["sp_incoherent"][2] == 0)
    plan.close()


def test_tc_edge_shapes(ctx, lcs, oracle):
    """Chunking of the template columns (<= 32 hypotheses = 96 columns per pass): n_f=1 (one job of C=16), 42 (2 passes of
    21 -> two jobs of C=32), 51 (26+25 -> two jobs of C=48), 64 (2 full passes), 70 (3 passes), 9 (two jobs of C=24);
    short buffers, fc_programmed != fc_requested, arm=0/1."""
    cases = [
        (153600, np.array([35000.0]), 2, 739e6, 739e6, 1.92e6),
        (40000, np.arange(-20, 22) * 2500.0, 2, 739e6, 739.002e6, 1.92e6 * 1.00001),
        (29000, np.array([-20000.0, 0.0, 5000.0]), 0, 2.1e9, 2.1e9, 1.92e6),
        (30000, np.arange(-25, 26) * 3000.0, 1, 739e6, 739e6, 1.92e6),          # 51 hypotheses -> 2 chunks
        (30000, np.arange(-32, 32) * 2000.0 + 500.0, 2, 739e6, 739e6, 1.92e6),  # 64 hypotheses -> 2 x 32 (all 96 columns live)
        (30000, np.arange(-35, 35) * 1500.0, 2, 1.8e9, 1.8e9, 1.92e6),          # 70 hypotheses -> 3 chunks
        (60000, np.arange(-4, 5) * 5000.0, 2, 739e6, 739e6, 1.92e6),            # n_comb = 6: the write-out divides with the division sequence (not in the exact-reciprocal set)
        (106000, np.arange(-2, 3) * 5000.0, 1, 739e6, 739e6, 1.92e6),           # n_comb = 11, N = 48 single-job layout
    ]
    for i, (n_cap, f, arm, fcr, fcp, fs) in enumerate(cases):
        _tc_vs_oracle(ctx, lcs, oracle, synth_cu8(77 + i, n_cap)[None], f, fcr, fcp, fs, arm)


def test_tc_matches_fp32_kernel_and_auto_selection(ctx, lcs):
    """Same plan parameters, both kernels: powers agree to fp32 noise; AUTO picks TC for cu8 only."""
    f = lcs.f_search_set(739e6, 100.0)
    cu8 = np.stack([synth_cu8(5), synth_cu8(6)])
    res = {}
    for k in (lcs.KERNEL_TC, lcs.KERNEL_FP32, lcs.KERNEL_AUTO):
        plan = ctx.plan(153600, f, 2, 739e6, 739e6, 1.92e6, max_batch=2, kernel=k)
        if k == lcs.KERNEL_AUTO:
            assert plan.kernel_for(lcs.IQ_CU8) == lcs.KERNEL_TC and plan.kernel_for(lcs.IQ_CF32) == lcs.KERNEL_FP32
        res[k] = plan.run_host_np(cu8, lcs.IQ_CU8)
        plan.close()
    a, b = res[lcs.KERNEL_TC]["single"], res[lcs.KERNEL_FP32]["single"]
    assert np.abs(a - b).max() < 1e-6 * b.max()
    assert np.array_equal(res[lcs.KERNEL_AUTO]["single"], a)
    # wide grids (3*n_f > 128 template rows) run as several <=42-hypothesis chunks
    wide = np.arange(-30, 31) * 2000.0
    outs = {}
    for k in (lcs.KERNEL_TC, lcs.KERNEL_FP32):
        plan = ctx.plan(153600, wide, 2, 739e6, 739e6, 1.92e6, max_batch=1, kernel=k)
        outs[k] = plan.run_host_np(cu8[:1], lcs.IQ_CU8)
        plan.close()
    assert np.abs(outs[lcs.KERNEL_TC]["single"] - outs[lcs.KERNEL_FP32]["single"]).max() < 1e-6 * outs[lcs.KERNEL_FP32]["single"].max()
    assert (outs[lcs.KERNEL_TC]["frq"] != outs[lcs.KERNEL_FP32]["frq"]).mean() < 0.002


# ---------------------------------------------------------------------------------------------
# device-side threshold + peak_search, batched search (SURVEY 8f rank 2)
# ---------------------------------------------------------------------------------------------
def _host_peaks(ctx, lcs, plan, cu8, f, fc):
    """xcorr_pss through the plan, then threshold + peak_search with the HOST implementation (lcs_peak_search)."""
    out = plan.run_host_np(cu8[None], lcs.IQ_CU8)
    z = lcs.calc_z_th1(out["sp_incoherent"][0], plan.n_comb_xc, 2)
    return lcs.peak_search(out["pow"][0], out["frq"][0], z, f, fc, fc, out["single"][0], 2)


def test_device_peak_search_matches_host(ctx, lcs, capbuf0000):
    """Device peak_search kernel == host peak_search (searcher.cpp:422-510) on the same device-computed pow/frq:
    real capture (several peaks incl. ghost cancellation), noise (none), the same capture rolled so that a peak sits
    at column < arm (the reference's uint16 wrap), and an all-equal buffer (zero power everywhere: the reference's loop
    would not terminate there, both implementations stop)."""
    fc = capbuf0000["fc"]
    f = lcs.f_search_set(fc, 120.0)
    real = capbuf0000["cu8"]
    plan = ctx.plan(real.shape[0], f, 2, fc, fc, 1.92e6, max_batch=8)
    ref0 = _host_peaks(ctx, lcs, plan, real, f, fc)
    assert len(ref0) >= 2
    rolled = np.roll(real, -(ref0[0].ind - 1), axis=0)          # strongest peak to fold position 1
    bufs = [real, synth_cu8(0xC0FFEE), rolled, np.full_like(real, 127), synth_cu8(3, sigma=3.0)]
    got = plan.peaks_batch(np.stack(bufs), lcs.IQ_CU8)
    n_wrapped = 0
    for b, cu8 in enumerate(bufs):
        ref = _host_peaks(ctx, lcs, plan, cu8, f, fc)
        same_cells(got[b], ref)
        n_wrapped += sum(p.ind == -1 for p in ref)
        for p in got[b]:
            assert p.fc_requested == fc and p.fc_programmed == fc and p.n_id_1 == -1
    assert len(got[1]) == 0 and len(got[3]) == 0
    plan.close()


def test_cell_search_batch_matches_single(ctx, lcs, capbuf0000):
    """lcs_cell_search_batch_cu8 == lcs_cell_search_cu8 (a batch of one) per buffer (cells 277/271 on the real capture,
    none on noise); more buffers than one chunk so that the stream rotation and the chunk hand-over are exercised."""
    fc = capbuf0000["fc"]
    f = lcs.f_search_set(fc, 120.0)
    real = capbuf0000["cu8"]
    order = [0, 1, 1, 0] + [1] * 31 + [0, 1]
    noise = synth_cu8(0xBEEF)
    bufs = np.stack([real if k == 0 else noise for k in order])
    plan = ctx.plan(real.shape[0], f, 2, fc, fc, 1.92e6, max_batch=32)
    got = plan.cell_search_batch_cu8(bufs)
    ref_cells, _ = ctx.cell_search(real, f, fc, fc, 1.92e6)
    assert [c.n_id_cell() for c in ref_cells] == [277, 271]
    for k, cells in zip(order, got):
        if k == 1:
            assert cells == []
        else:
            same_cells(cells, ref_cells)
    plan.close()


def test_tracker_search_cycle(ctx, lcs, capbuf0000):
    """Streaming mode (SURVEY 8f rank 3): raw bytes -> lcs_framer -> lcs_tracker_search_cu8 == the n_f=1 chain of
    searcher_thread.cpp:95-232 on the framed buffer; frame_timing = frame_start*(FS_LTE/16)/(fs*k)+late; tracked cells
    are skipped."""
    fc = capbuf0000["fc"]
    real = capbuf0000["cu8"]
    full, _ = ctx.cell_search(real, lcs.f_search_set(fc, 120.0), fc, fc, 1.92e6)
    f_off = float(np.round(full[0].freq_superfine))          # the tracker searches at its current offset estimate
    fs = 1.92e6
    rng = np.random.default_rng(5)
    lead = rng.integers(100, 156, size=(19200 + 777, 2), dtype=np.uint8)
    stream = np.concatenate([lead, real, lead])
    fr = lcs.Framer(fc, fc, fs, real.shape[0])
    fr.push(stream[:500], f_off)
    fr.request()
    got = None
    for lo in range(500, stream.shape[0], 10000):            # BLOCK_SIZE of producer_thread.cpp:95
        got = got or fr.push(stream[lo:lo + 10000], f_off)
    assert got is not None
    cap, late = got
    assert abs(late) < 0.5
    k = (fc - f_off) / fc
    ref_cells, _ = ctx.cell_search(cap, np.array([f_off]), fc, fc, fs)
    new = ctx.tracker_search_cu8(cap, f_off, fc, fc, fs, late)
    assert len(ref_cells) >= 1
    same_cells([c for c, _ in new], ref_cells)
    for (c, ft), r in zip(new, ref_cells):
        assert ft == r.frame_start * (30720000.0 / 16) / (fs * k) + late
    first = new[0][0].n_id_cell()
    rest = ctx.tracker_search_cu8(cap, f_off, fc, fc, fs, late, tracked=[first])
    assert [c.n_id_cell() for c, _ in rest] == [c.n_id_cell() for c, _ in new if c.n_id_cell() != first]
    fr.close()


# ---------------------------------------------------------------------------------------------
# bench configuration, unaligned buffer strides, device peak search and tracker search against the oracle
# ---------------------------------------------------------------------------------------------
def test_tc_bench_config_vs_oracle(ctx, lcs, oracle):
    """The configuration bench.py times (BASELINE configs[1]: n_f=31, n_cap=153600) with enough buffers that every
    persistent CTA walks more than one work item (8 buffers): EVERY buffer against the oracle, <= 5e-7."""
    f = lcs.f_search_set(739e6, 100.0)
    assert f.size == 31
    cu8 = np.stack([synth_cu8(0xC0FFEE + i) for i in range(8)])
    _tc_vs_oracle(ctx, lcs, oracle, cu8, f, 739e6, 739e6, 1.92e6)


def test_tc_unaligned_buffer_stride(ctx, lcs, oracle):
    """batch > 1 with n_cap*2 % 16 != 0 (n_cap = 29004): buffers 1.. start at byte offsets that are not 16-byte aligned."""
    f = np.arange(-3, 4) * 5000.0
    cu8 = np.stack([synth_cu8(500 + i, 29004) for i in range(3)])
    _tc_vs_oracle(ctx, lcs, oracle, cu8, f, 739e6, 739e6, 1.92e6)
    cu8 = np.stack([synth_cu8(600 + i, 29001) for i in range(2)])       # odd sample count
    _tc_vs_oracle(ctx, lcs, oracle, cu8, f, 739e6, 739e6, 1.92e6)


def test_device_peak_search_vs_oracle(ctx, lcs, capbuf0000, capbuf_chain):
    """Device threshold + peak_search against the ORACLE's xcorr_pss + Z_th1 + peak_search (searcher.cpp:422-510,
    CellSearch.cpp:500-503) on the same capture."""
    fc = capbuf0000["fc"]
    f, _, o_peaks = capbuf_chain
    real = capbuf0000["cu8"]
    plan = ctx.plan(real.shape[0], f, 2, fc, fc, 1.92e6, max_batch=2)
    got = plan.peaks_batch(np.stack([real, synth_cu8(0xC0FFEE)]), lcs.IQ_CU8)
    compare_cells(got[0], o_peaks)
    assert got[1] == []
    plan.close()


def test_peak_list_holds_more_than_32_peaks(ctx, lcs, oracle):
    """A buffer with 48 PSS peaks: 16 copies of every root's pss_td, 600 samples apart within a root and 200 samples
    between roots so that no two overlap, repeated in every half frame so that they fold coherently, over weak noise.
    The device peak list holds 102 entries, the most a buffer can have, so the batched peak search (the buffer second in
    its chunk) and the single-buffer cell search report exactly the host peak_search list, which matches the oracle's."""
    fc = 739e6
    f = lcs.f_search_set(fc, 120.0)
    half = np.zeros(9600, np.complex128)
    for r in range(3):
        for k in range(16):
            s = 200 * r + 600 * k
            half[s:s + 137] += oracle.pss_td(r)
    sig = np.tile(half, 16) * (40.0 / np.abs(half).max())
    cu8 = np.clip(np.round(synth_cu8(0x5EED, sigma=3.0) + np.stack([sig.real, sig.imag], axis=1)), 0, 255).astype(np.uint8)
    plan = ctx.plan(cu8.shape[0], f, 2, fc, fc, 1.92e6, max_batch=2)
    ref = _host_peaks(ctx, lcs, plan, cu8, f, fc)
    assert len(ref) > 32
    got = plan.peaks_batch(np.stack([synth_cu8(0xC0FFEE), cu8]), lcs.IQ_CU8, max_peaks=128)
    assert got[0] == []
    same_cells(got[1], ref)
    o = oracle.xcorr_pss(cu8_to_c128(cu8), f, 2, fc, fc, 1.92e6)
    z = oracle.calc_Z_th1(o["sp_incoherent"], o["n_comb_xc"], 2)
    compare_cells(got[1], oracle.peak_search(o["pow"], o["frq"], z, f, fc, fc, o["single"], 2))
    _, peaks = ctx.cell_search(cu8, f, fc, fc, 1.92e6, max_cells=128)
    same_cells(peaks, ref)
    plan.close()


def test_tracker_search_vs_oracle(ctx, lcs, oracle, capbuf0000):
    """One searcher cycle (n_f = 1 at the tracked offset, searcher_thread.cpp:95-232) against the oracle's chain on the
    same framed buffer: every field as in the full-chain test, and the frame timing."""
    fc = capbuf0000["fc"]; fs = 1.92e6
    f_off = 35228.0
    cap_u8 = capbuf0000["cu8"]
    o_cells, _ = oracle.cell_search_one(capbuf0000["capbuf"], np.array([f_off]), fc, fc, fs)
    new = ctx.tracker_search_cu8(cap_u8, f_off, fc, fc, fs, 0.25)
    assert len(o_cells) >= 1
    compare_cells([a for a, _ in new], o_cells)
    k = (fc - f_off) / fc
    for (a, ft), b in zip(new, o_cells):
        assert abs(ft - (b.frame_start * (30720000.0 / 16) / (fs * k) + 0.25)) < 1e-9


# ---------------------------------------------------------------------------------------------
# many channels at once (BASELINE configs 4 and 5): one plan per channel, one correlator launch per chunk
# ---------------------------------------------------------------------------------------------
def test_sweep_search_vs_oracle(ctx, lcs, oracle, capbuf0000, capbuf_chain):
    """lcs_sweep_search_cu8 = the per-centre-frequency loop of CellSearch.cpp:465-558.  The real capture is presented at
    three different centre frequencies (different k_factor => different templates and fold offsets per channel) between
    noise channels, more channels than one chunk; every channel is compared with the oracle's chain for that channel."""
    f = lcs.f_search_set(739e6, 120.0)                       # one f_search_set for the sweep (CellSearch.cpp:463-464)
    f0, o_cells0, _ = capbuf_chain
    assert f.tobytes() == f0.tobytes() and capbuf0000["fc"] == 739e6
    real, noise = capbuf0000["cu8"], synth_cu8(0xBEEF)
    fcs = 739e6 + 100e3 * np.arange(70)
    is_real = {0: 0, 33: 1, 69: 2}
    iq = np.stack([real if i in is_real else noise for i in range(fcs.size)])
    sw = lcs.Sweep(ctx, real.shape[0])
    got = sw.search_cu8(iq, fcs, f)
    o_noise, _ = oracle.cell_search_one(cu8_to_c128(noise), f, 739e6, 739e6, 1.92e6)
    assert o_noise == []
    for i, fc in enumerate(fcs):
        if i not in is_real:
            assert got[i] == [], i
            continue
        o_cells = o_cells0 if i == 0 else oracle.cell_search_one(capbuf0000["capbuf"], f, fc, fc, 1.92e6)[0]
        assert len(o_cells) >= 1
        compare_cells(got[i], o_cells)
    # a second sweep through the same handle with other channels (plans are rebuilt)
    got2 = sw.search_cu8(iq[:3], fcs[:3] + 5e6, f)
    assert len(got2[0]) >= 1 and got2[1] == [] and got2[2] == []
    sw.close()


def test_sweep_track_matches_tracker_search(ctx, lcs, capbuf0000):
    """lcs_sweep_track_cu8 (all channels in one launch, per-channel offset) == lcs_tracker_search_cu8 per channel."""
    fc = capbuf0000["fc"]
    real, noise = capbuf0000["cu8"], synth_cu8(0xFEED)
    offs = [35228.0, 35000.0, -1200.0, 35228.0, 36000.0]
    fcs = [fc, fc, fc + 1e6, fc + 2e6, fc]
    bufs = [real, real, noise, real, real]
    late = [0.25, -0.5, 0.0, 1.5, 0.0]
    tracked = [[], [], [], [277], [271, 5]]
    sw = lcs.Sweep(ctx, real.shape[0])
    got = sw.track_cu8(np.stack(bufs), offs, fcs, late=late, tracked=tracked)
    for c in range(len(bufs)):
        ref = ctx.tracker_search_cu8(bufs[c], offs[c], fcs[c], fcs[c], 1.92e6, late[c], tracked=tracked[c])
        same_cells([a for a, _ in got[c]], [b for b, _ in ref])
        assert [fa for _, fa in got[c]] == [fb for _, fb in ref], c
    assert [c.n_id_cell() for c, _ in got[0]] == [277, 271] and got[2] == []
    assert 277 not in [c.n_id_cell() for c, _ in got[3]]
    sw.close()


def test_kalibrate_vs_oracle(ctx, lcs, oracle, capbuf0000, capbuf_chain):
    """kalibrate (LTE-Tracker.cpp:565-741): offset-centred grid, chain, dedup, strongest cell, residual correction factor -
    against the same steps done with the oracle.  capbuf_0000: cell 277, freq_superfine 35 228.46 Hz."""
    fc = capbuf0000["fc"]; fs = 1.92e6
    f0, o_cells0, _ = capbuf_chain
    for correction in (1.0, 1.00004):
        f = (fc * correction - fc) + oracle.f_search_set(fc, 120.0)                       # :586-587
        if correction == 1.0:
            assert f.tobytes() == f0.tobytes()
        o_cells = o_cells0 if correction == 1.0 else oracle.cell_search_one(capbuf0000["capbuf"], f, fc, fc, fs)[0]
        o_fin = oracle.dedup(o_cells)
        o_best = max(o_fin, key=lambda c: c.pss_pow)
        best, resid, n = ctx.kalibrate_cu8(capbuf0000["cu8"], fc, fc, fs, 120.0, correction)
        assert n == len(o_fin) and best is not None and o_best.n_id_cell() == 277
        compare_cells([best], [o_best])
        assert abs(resid - fc / (fc - o_best.freq_superfine)) < 1e-15
    assert abs(best.freq_superfine - 35228.46) < 0.5
    none, _, n0 = ctx.kalibrate_cu8(synth_cu8(1), fc, fc, fs, 120.0)
    assert none is None and n0 == 0


def test_stream_search_cli_kalibrate(ctx, tmp_path, capbuf0000):
    """StreamSearch_b200 = LTE-Tracker's start-up on a recorded stream: kalibrate on the first buffer (LTE-Tracker.cpp:795-798),
    then producer framing + searcher cycles at the calibrated offset."""
    import os
    import re
    import subprocess
    root = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
    host = os.path.join(root, "lte-cell-scanner_b200", "host")
    subprocess.check_call(["make", "-C", host, "-s"])
    real = capbuf0000["cu8"]
    stream = np.concatenate([real, real, real[:40000]])
    stream.tofile(str(tmp_path / "stream.bin"))
    out = subprocess.run([os.path.join(host, "StreamSearch_b200"), "-f", "739000000", "-n", "1", str(tmp_path / "stream.bin")],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    m = re.search(r"Residual frequency offset: ([0-9.]+) Hz", out.stdout)
    assert m and abs(float(m.group(1)) - 35228.46) < 0.5
    assert re.search(r"new cell 277 ", out.stdout)


def test_cellsearch_cli_batched_sweep(ctx, tmp_path, capbuf0000):
    """`CellSearch_b200 -s 738.9M -e 739.1M -l --raw --sweep`: three centre frequencies through lcs_sweep_search_cu8 print
    the same table rows as the one-frequency-at-a-time loop (cells 277 and 271 at 739.0 MHz)."""
    import os
    import re
    import subprocess
    root = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
    host = os.path.join(root, "lte-cell-scanner_b200", "host")
    subprocess.check_call(["make", "-C", host, "-s"])
    synth_cu8(11).tofile(str(tmp_path / "capbuf_0000.bin"))
    capbuf0000["cu8"].tofile(str(tmp_path / "capbuf_0001.bin"))
    synth_cu8(12).tofile(str(tmp_path / "capbuf_0002.bin"))
    outs = []
    for extra in ([], ["--sweep"]):
        out = subprocess.run([os.path.join(host, "CellSearch_b200"), "-s", "738900000", "-e", "739100000", "-l", "--raw", "-b",
                              "-d", str(tmp_path)] + extra, capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr + out.stdout
        rows = [l for l in out.stdout.splitlines() if re.match(r"^\s*27[17]\s+2\s", l)]
        assert len(rows) == 2
        outs.append(rows)
    assert outs[0] == outs[1]


def test_dropin_routes_8bit_exact_input_to_the_tensor_core_kernel(ctx, lcs, capbuf0000):
    """lcs_xcorr_pss takes the IT++ c128 vector; a capture that holds exactly (u8-127)/128 (capbuf.cpp:172-175) must be
    served by the tensor-core correlator: its `single` is bit-identical to an explicit tensor-core plan on the raw bytes,
    while the same samples scaled by 0.999 (no longer 8-bit exact) take the FP32 correlator and differ in the last bits."""
    fc = capbuf0000["fc"]
    f = lcs.f_search_set(fc, 120.0)
    out = ctx.xcorr_pss(capbuf0000["capbuf"], f, 2, fc, fc, 1.92e6, want_incoherent=False)
    plan = ctx.plan(capbuf0000["cu8"].shape[0], f, 2, fc, fc, 1.92e6, max_batch=1, kernel=lcs.KERNEL_TC)
    tc = plan.run_host_np(capbuf0000["cu8"][None], lcs.IQ_CU8)
    plan.close()
    assert np.array_equal(out["single"], tc["single"][0].transpose(0, 2, 1))
    assert np.array_equal(out["pow"], tc["pow"][0]) and np.array_equal(out["frq"], tc["frq"][0])
    scaled = ctx.xcorr_pss(capbuf0000["capbuf"] * 0.999, f, 2, fc, fc, 1.92e6, want_incoherent=False)
    ratio = scaled["single"] / (out["single"] * 0.999 ** 2)
    assert not np.array_equal(scaled["single"], out["single"]) and np.abs(ratio - 1).max() < 1e-4


def test_sweep_on_a_grid_the_tensor_core_tiling_cannot_hold(ctx, lcs, oracle, capbuf0000):
    """A sweep whose frequency grid is too sparse for the tensor-core tiling (fold-offset spread > 32 samples) falls back
    to the FP32 correlator with per-channel templates; cells still equal the oracle's per channel."""
    f = np.arange(-8, 9) * 35000.0
    real, noise = capbuf0000["cu8"], synth_cu8(0xABCD)
    fcs = np.array([739e6, 739.1e6, 745e6])
    iq = np.stack([real, noise, real])
    sw = lcs.Sweep(ctx, real.shape[0])
    got = sw.search_cu8(iq, fcs, f)
    for i, fc in enumerate(fcs):
        cap = capbuf0000["capbuf"] if i != 1 else cu8_to_c128(noise)
        o_cells, _ = oracle.cell_search_one(cap, f, fc, fc, 1.92e6)
        compare_cells(got[i], o_cells)
    assert len(got[0]) >= 1 and got[1] == []
    sw.close()


def test_long_capture_falls_back_to_the_fp32_correlator(ctx, lcs, oracle):
    """More than 24 half frames (n_cap = 250000 -> n_comb = 26) exceed the tensor-core kernel's offset table: AUTO serves
    the 8-bit buffer with the FP32 correlator, an explicit tensor-core plan fails cleanly."""
    f = np.array([-5000.0, 0.0, 5000.0])
    cu8 = synth_cu8(321, 250000)
    plan = ctx.plan(250000, f, 2, 739e6, 739e6, 1.92e6, max_batch=1)
    assert plan.kernel_for(lcs.IQ_CU8) == lcs.KERNEL_FP32
    out = plan.run_host_np(cu8[None], lcs.IQ_CU8)
    ref = oracle.xcorr_pss(cu8_to_c128(cu8), f, 2, 739e6, 739e6, 1.92e6)
    assert ref["n_comb_xc"] == 26
    assert rel_err(out["single"][0].transpose(0, 2, 1), ref["single"]) < REL and rel_err(out["pow"][0], ref["pow"]) < REL
    plan.close()
    tcp = ctx.plan(250000, f, 2, 739e6, 739e6, 1.92e6, max_batch=1, kernel=lcs.KERNEL_TC)
    with pytest.raises(lcs.LcsError):
        tcp.run_host_np(cu8[None], lcs.IQ_CU8)
    tcp.close()


def test_tc_last_samples_of_the_last_buffer(ctx, lcs, oracle):
    """An extreme k_factor (fc_programmed = fc_requested / 2.00677) pushes the last fold offset to the limit the plan accepts:
    the very last sample of the capture buffer enters the correlation, and with n_cap = 29001 it sits in a partial 16-byte
    chunk at the end of the allocation (the TMA staging copies whole chunks; the tail is copied by lanes)."""
    n_cap = 29001
    fcr = 739e6
    fcp = fcr / 2.00677
    f = np.array([0.0])
    assert int(np.rint(9600 * (fcr / fcp))) + 9599 == n_cap - 136 - 1
    cu8 = synth_cu8(77, n_cap)
    cu8[-40:] = 255                                  # make the tail samples matter
    for batch in (1, 2):
        _tc_vs_oracle(ctx, lcs, oracle, np.stack([cu8] * batch), f, fcr, fcp, 1.92e6)
