"""CPU-side checks of the product: the C-ABI library loads and exports every symbol that
include/lcs_b200.h declares, fails loudly without a GPU, and its host stages (threshold,
peak_search, tfoec, decode_mib, dedup) agree with the oracle and with the reference's goldens."""
import ctypes as C

import numpy as np
import pytest

from conftest import has_gpu, load


def test_library_exports_every_declared_symbol(lcs):
    l = lcs.lib()
    names = lcs.declared_symbols()
    assert len(names) >= 25
    missing = [n for n in names if not hasattr(l, n)]
    assert not missing, missing
    assert b"sm_90a" in l.lcs_version()
    assert C.sizeof(lcs.Cell) == 104


@pytest.mark.skipif(has_gpu(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback(lcs):
    with pytest.raises(lcs.LcsError, match="no CUDA device"):
        lcs.Context(0)


def test_f_search_set_matches_reference_formula(lcs, oracle):
    for fc, ppm in [(739e6, 120.0), (739e6, 100.0), (715e6, 120.0), (768e6, 120.0), (2.6e9, 20.0)]:
        a, b = lcs.f_search_set(fc, ppm), oracle.f_search_set(fc, ppm)
        assert np.array_equal(a, b)
    assert lcs.f_search_set(739e6, 100.0).size == 31 and lcs.f_search_set(739e6, 120.0).size == 37


def test_z_th1_matches_oracle(lcs, oracle):
    rng = np.random.default_rng(0)
    spi = 0.05 + 0.01 * rng.random(9600)
    for n_comb, arm in [(15, 2), (14, 2), (15, 0)]:
        a, b = lcs.calc_z_th1(spi, n_comb, arm), oracle.calc_Z_th1(spi, n_comb, arm) if arm == 2 or True else None
        assert np.abs(a / b - 1).max() < 1e-12


def test_peak_search_golden(lcs):
    g = load("ref_peak_search.npz")
    pw = g["xc_incoherent_collapsed_pow"]; frq = g["xc_incoherent_collapsed_frq"] - 1
    f = g["f_search_set"].astype(float)
    single = np.repeat(pw[:, None, :], f.size, axis=1).astype(np.float32)     # planar [3][n_f][9600]
    cells = lcs.peak_search(pw, frq, g["Z_th1"], f, 739e6, 739e6, single, 0)
    assert len(cells) == 20
    for c, p, i, fr, n in zip(cells, g["peaks_pow"], g["peaks_ind"], g["peaks_freq"], g["peaks_n_id_2"]):
        assert abs(c.pss_pow - p) < 1e-6 and c.ind == i - 1 and c.freq == fr and c.n_id_2 == n


def test_peak_search_matches_oracle_random(lcs, oracle):
    rng = np.random.default_rng(5)
    n_f = 5
    f = np.arange(-2, 3) * 5000.0
    for trial in range(4):
        single = rng.random((3, n_f, 9600)).astype(np.float32) * 0.01
        for _ in range(6):                                    # plant peaks, some at the wrap-around edges
            t, fi = rng.integers(0, 3), rng.integers(0, n_f)
            idx = [0, 1, 9599, 4000, 7000, 9598][_] if trial == 0 else rng.integers(0, 9600)
            single[t, fi, idx] += rng.random() * 2 + 0.5
        inc = single.astype(np.float64)
        pw = inc.max(axis=1); frq = inc.argmax(axis=1).astype(np.int32)
        z = np.full(9600, 0.3)
        a = lcs.peak_search(pw, frq, z, f, 739e6, 739.01e6, single, 2)
        b = oracle.peak_search(pw, frq, z, f, 739e6, 739.01e6, single.transpose(0, 2, 1).astype(np.float64), 2)
        assert len(a) == len(b) and len(a) > 0
        for x, y in zip(a, b):
            assert (x.ind, x.freq, x.n_id_2, x.pss_pow, x.fc_programmed) == (y.ind, y.freq, y.n_id_2, y.pss_pow, y.fc_programmed)


def _golden_tfg_cell(m):
    return m.new_cell(n_id_1=92, n_id_2=1, cp_type=1, frame_start=17448.5250338295, freq_fine=39684.07746316391)


def test_tfoec_and_decode_mib_match_oracle(lcs, oracle):
    """Product host stages vs the oracle (HEAD semantics) on the golden TFG of cell 277."""
    g = load("ref_tfg.npz")
    fc = float(g["fc"][0])
    o_cell, o_tc, o_ts = oracle.tfoec(_golden_tfg_cell(oracle), g["tfg"], g["tfg_timestamp"] - 1, fc, fc)
    p_cell, p_tc, p_ts = lcs.tfoec(_golden_tfg_cell(lcs), g["tfg"], g["tfg_timestamp"] - 1, fc, fc)
    assert np.abs(p_tc - o_tc).max() < 1e-11 and np.abs(p_ts - o_ts).max() < 1e-9
    assert abs(p_cell.freq_superfine - o_cell.freq_superfine) < 1e-7
    o_m, dbg = oracle.decode_mib(o_cell, o_tc)
    p_m = lcs.decode_mib(p_cell, p_tc)
    for k in ("n_ports", "n_rb_dl", "phich_duration", "phich_resource", "sfn"):
        assert getattr(p_m, k) == getattr(o_m, k)
    assert (p_m.n_ports, p_m.n_rb_dl, p_m.sfn) == (2, 50, 649)


def test_decode_mib_kat(lcs):
    """Bit-exact KAT on the reference's stored tfg_comp (test/test_tfg.it; SURVEY 4.4)."""
    g = load("ref_tfg.npz")
    m = lcs.decode_mib(lcs.new_cell(n_id_1=92, n_id_2=1, cp_type=1), g["tfg_comp"])
    assert (m.n_ports, m.n_rb_dl, m.phich_duration, m.phich_resource, m.sfn) == (2, 50, 1, 3, 649)
    # a wrong cell id must not decode (CRC + scrambling)
    m2 = lcs.decode_mib(lcs.new_cell(n_id_1=91, n_id_2=1, cp_type=1), g["tfg_comp"])
    assert m2.n_rb_dl == -1 and m2.n_ports == -1


def test_chan_est_noise_and_errors(lcs):
    g = load("ref_tfg.npz")
    with pytest.raises(lcs.LcsError):
        lcs.decode_mib(lcs.new_cell(n_id_1=92, n_id_2=1, cp_type=0), g["tfg_comp"])        # cp_type unknown
    with pytest.raises(lcs.LcsError):
        lcs.decode_mib(lcs.new_cell(n_id_1=92, n_id_2=1, cp_type=1), g["tfg_comp"][:100])  # grid too short


def test_dedup_matches_oracle(lcs, oracle):
    def mk(m, cid, fc, sf, pw):
        return m.new_cell(n_id_1=cid // 3, n_id_2=cid % 3, fc_requested=fc, freq_superfine=sf, pss_pow=pw)
    spec = [(277, 739e6, 35e3, 0.06), (271, 739e6, 35e3, 0.016), (277, 739.1e6, -65e3, 0.08),
            (277, 741e6, 0.0, 0.01), (271, 739.1e6, -65e3, 0.001)]
    a = lcs.dedup([mk(lcs, *s) for s in spec])
    b = oracle.dedup([mk(oracle, *s) for s in spec])
    assert [(c.n_id_cell(), c.fc_requested, c.pss_pow) for c in a] == [(c.n_id_cell(), c.fc_requested, c.pss_pow) for c in b]
    assert [(c.n_id_cell(), c.fc_requested) for c in a] == [(277, 739.1e6), (271, 739e6), (277, 741e6)]
    assert lcs.dedup([]) == []


def _producer_restatement(stream, fc_req, fc_prog, fs_prog, f_off, n_cap, request_at):
    """src/producer_thread.cpp:96-161 written out directly (searcher capture buffer only): returns (start index, late)."""
    import math
    k = (fc_req - f_off) / fc_prog
    st = -1.0
    request = False
    for t in range(stream.shape[0]):
        if t == request_at:
            request = True
        st += (30720000.0 / 16) / (fs_prog * k)
        if st > 19200.0:
            st -= 19200.0
        w = (st + 9600.0) - 19200.0 * math.floor((st + 9600.0) / 19200.0) - 9600.0
        if request and abs(w) < 0.5:
            return t, w
    return None, None


def test_framer_matches_producer_thread(lcs):
    """lcs_framer (host framing of a raw IQ stream) against a direct restatement of producer_thread.cpp:96-161: capture
    starts at the first sample whose time stamp is within +-0.5 of a frame-pair boundary after the request, `late` is that
    stamp, the buffer holds the next n_cap samples verbatim; pushes of ragged block sizes give the same answer."""
    L = lcs
    rng = np.random.default_rng(11)
    n_cap = 5000
    stream = rng.integers(0, 256, size=(60000, 2), dtype=np.uint8)
    for fc_req, fc_prog, fs_prog, f_off, req_at in [(739e6, 739e6, 1.92e6, 0.0, 0), (739e6, 739.002e6, 1.92e6 * 1.00003, 1234.5, 7000),
                                                   (2.1e9, 2.1e9, 1.92e6 * 0.99995, -30000.0, 19190)]:
        t0, late = _producer_restatement(stream, fc_req, fc_prog, fs_prog, f_off, n_cap, req_at)
        assert t0 is not None
        for blocks in ([10000] * 6, [1, 6999, 3, 12187, 810, 40000]):
            fr = L.Framer(fc_req, fc_prog, fs_prog, n_cap)
            pos, got = 0, None
            requested = False
            for b in blocks:
                # the request arrives between two samples: split the block there
                parts = [(pos, pos + b)]
                if not requested and pos <= req_at < pos + b:
                    parts = [(pos, req_at), (req_at, pos + b)]
                for lo, hi in parts:
                    if lo == req_at and not requested:
                        fr.request(); requested = True
                    if hi > lo:
                        r = fr.push(stream[lo:hi], f_off)
                        if r is not None and got is None:
                            got = r
                pos += b
            assert got is not None
            cap, glate = got
            assert glate == late
            assert np.array_equal(cap, stream[t0:t0 + n_cap])
            fr.close()


def test_tc_integer_formulation_numpy(oracle):
    """The arithmetic of the tensor-core correlator (DESIGN.md 4.2) restated in numpy integers and checked against the oracle's
    `xc`: 24-bit fixed-point templates in three balanced base-256 digits, x' = byte-128, second byte stream (Q', ~I') for the
    imaginary part, additive corrections sum(a) / sum(a[even]), int32-safe partial sums, exact reconstruction."""
    from conftest import synth_cu8, cu8_to_c128
    n_cap, fc, fs = 12000, 739e6, 1.92e6
    f = np.array([-40000.0, 5000.0, 70000.0])
    cu8 = synth_cu8(99, n_cap, sigma=40.0)
    cu8[100:130] = 255; cu8[500:520] = 0                       # saturated samples: the "+1" correction must hold there too
    ref = oracle.xcorr_pss(cu8_to_c128(cu8), f, 2, fc, fc, fs, want_xc=True, want_sp=False)["xc"]     # [3][n_cap-136][n_f]
    z = cu8.reshape(-1).astype(np.int64)                       # interleaved I,Q bytes
    xs = z - 128                                               # (I', Q')
    ys = np.empty_like(xs); ys[0::2] = xs[1::2]; ys[1::2] = -xs[0::2] - 1      # (Q', ~I')
    w = np.empty((f.size, 3, 137), np.complex128)
    for fi, fo in enumerate(f):
        k_factor = (fc - fo) / fc
        k = np.pi * fo / ((fs * k_factor) / 2)
        for t in range(3):
            w[fi, t] = np.conj(oracle.pss_td(t) * np.exp(1j * k * np.arange(137))) / 137
    maxabs = max(np.abs(w.real).max(), np.abs(w.imag).max())
    limit = 127 * 65536 + 127 * 256 + 127
    e = int(np.floor(np.log2(limit / maxabs)))
    S = 2.0 ** e
    assert maxabs * S <= limit
    lags = np.random.default_rng(1).integers(0, n_cap - 136, 150)
    # the bit-exact model of the kernel (xcorr_tc_model) builds the same integer templates with the library's pss_td
    from xcorr_tc_model import TcModel
    model = TcModel(n_cap, f, fc, fc, fs)
    assert model.S == S
    worst = 0.0
    for fi in range(f.size):
        for t in range(3):
            wr, wi = np.rint(w[fi, t].real * S).astype(np.int64), np.rint(w[fi, t].imag * S).astype(np.int64)
            a = np.empty(274, np.int64); a[0::2] = wr; a[1::2] = -wi
            assert np.array_equal(model.a[fi, t], a)
            d2 = ((a + 128) % 256) - 128; r1 = (a - d2) // 256
            d1 = ((r1 + 128) % 256) - 128; d0 = (r1 - d1) // 256
            assert np.array_equal((d0 * 256 + d1) * 256 + d2, a)
            assert d0.min() >= -128 and d0.max() <= 127 and d1.min() >= -128 and d2.max() <= 127
            c_re, c_im = a.sum(), a[0::2].sum()
            for L in lags:
                seg_x, seg_y = xs[2 * L:2 * L + 274], ys[2 * L:2 * L + 274]
                acc = [[int((d * s).sum()) for d in (d0, d1, d2)] for s in (seg_x, seg_y)]
                assert max(abs(v) for part in acc for v in part) < 2 ** 23          # fits the int32 accumulators with room
                v_re = (acc[0][0] * 256 + acc[0][1]) * 256 + acc[0][2] + c_re
                v_im = (acc[1][0] * 256 + acc[1][1]) * 256 + acc[1][2] + c_im
                got = complex(v_re, v_im) / (S * 128)
                worst = max(worst, abs(got - ref[t, L, fi]) / np.abs(ref[t, :, fi]).max())
    assert worst < 3e-7, worst            # float32 rounding of the reference's stored xc + 2^-24 template quantisation


def test_tc_run_decomposition_covers_every_position_once():
    """The tensor-core correlator distributes work in tile space (xcorr_tc.cu: launch_xcorr_fold_tc / TcRunIter): CTA i takes
    tiles [i*t_cta, (i+1)*t_cta) of the sequence [unit][tu]; a run of T tiles yields 256*T - 32 fold positions.  Restated
    in xcorr_tc_model (which the bit-exact model's fold order uses too): for many (units, SMs) every position 0..9599 of
    every unit is produced by exactly one run, and no run needs more tiles than it was given."""
    from xcorr_tc_model import HALO, N_FOLD, NT, tc_plan, tc_runs

    for n_units, n_sm in [(1, 132), (2, 132), (3, 7), (8, 132), (32, 132), (64, 132), (128, 132), (384, 132), (768, 132), (5, 1), (37, 13),
                          (3, 114), (128, 114), (6, 78)]:
        tu, t_cta = tc_plan(n_units, n_sm)
        cover = np.zeros((n_units, N_FOLD), np.int32)
        grid = (n_units * tu + t_cta - 1) // t_cta
        assert grid <= max(n_sm, 1) or t_cta == 1
        for cta, u, p0, p1, n_tiles, given in tc_runs(n_units, n_sm):
            assert cta < grid and p1 > p0
            assert n_tiles <= given and NT * n_tiles - HALO >= p1 - p0          # the run's tiles suffice for its positions
            cover[u, p0:p1] += 1
        assert (cover == 1).all(), (n_units, n_sm, tu, t_cta)


def test_three_instruction_division_matches_ieee_on_samples():
    """q = RN(x*r); q += RN(x - n*q) * r with r = RN(1/n) is used instead of x / n for n = n_comb (15) and 2*arm+1 (3, 5, 7, 9).
    tools/divchk.c proves equality for EVERY non-negative float; here a sampled re-check in float32 arithmetic."""
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.random(200000, np.float32) * np.float32(10.0) ** rng.integers(-30, 30, 200000).astype(np.float32),
                        np.array([0.0, 1e-45, 1.1754944e-38, 3.4028235e38], np.float32)]).astype(np.float32)
    for n in (3, 5, 7, 9, 15):
        d = np.float32(n)
        r = np.float32(1.0) / d
        q = (x * r).astype(np.float32)
        e = (x.astype(np.float64) - d.astype(np.float64) * q.astype(np.float64)).astype(np.float32)   # fma(-n, q, x): exact product, one rounding
        q2 = (e.astype(np.float64) * r.astype(np.float64) + q.astype(np.float64)).astype(np.float32)
        assert np.array_equal(q2, (x / d).astype(np.float32)), n


def test_library_contains_hopper_native_instructions(lcs):
    """The shipped liblcs_b200.so must carry the warpgroup-MMA / TMA / mbarrier code paths of the tensor-core correlator
    (SASS mnemonics): IGMMA = wgmma.mma_async on s8 operands, WARPGROUP.ARRIVE = wgmma.fence, UBLKCP = cp.async.bulk
    (1-D TMA), SYNCS.ARRIVE.TRANS64 = mbarrier arrive / expect_tx."""
    import os
    import shutil
    import subprocess
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([exe, "-sass", lcs.LIB_PATH], capture_output=True, text=True, timeout=600).stdout
    for mnemonic in ("IGMMA.64x144x32.S8.S8", "WARPGROUP.ARRIVE", "UBLKCP", "SYNCS.ARRIVE.TRANS64"):
        assert sass.count(mnemonic) > 0, mnemonic
    assert "sm_90a" in subprocess.run([exe, "-lelf", lcs.LIB_PATH], capture_output=True, text=True, timeout=600).stdout
