"""The tensor-core correlator's `single` (xc_incoherent_single) bit for bit against a numpy model of its arithmetic.

For 8-bit IQ the kernel is exact integer arithmetic followed by a fixed, short sequence of correctly rounded float32
operations (xcorr_tc_model.py), so its output is determined to the last bit.  The model is checked against the oracle on
the CPU at the bound the parity tests use, and then the device is compared with it without a tolerance: at every layout
pick_layout chooses (C = 16, 24, 32, 48; one, two and three passes), at n_comb inside and outside the set the write-out
divides by reciprocal, with fc_programmed != fc_requested, the last sample of the last buffer, full-scale and zero-signal
buffers and an odd buffer stride, and at batch sizes that start the work runs at different tile phases.

The half frames of a fold position are added in ascending m at every batch size: planset_build chooses each pass' staging
start so that every column's fold offset relative to it is non-decreasing in m, and the kernel adds the half frames of a
tile in order.  The grids include columns whose offsets relative to the per-half-frame minimum are not monotone."""
import numpy as np
import pytest

import xcorr_tc_model as M
from conftest import cu8_to_c128, synth_cu8
from test_gpu_parity import rel_err
from test_xcorr_writeout_gpu import assert_bitwise

FC, FS = 739e6, 1.92e6


def f_search_set(fc, ppm):
    """f_search_set of the library and the oracle (test_f_search_set_matches_reference_formula)."""
    n = int(np.floor((fc * ppm / 1e6 + 2.5e3) / 5e3))
    return 5000.0 * np.arange(-n, n + 1)


def full_scale(seed, n_cap):
    return np.random.default_rng(seed).choice(np.array([0, 255], np.uint8), size=(n_cap, 2))


def tail_255(n_cap):
    x = synth_cu8(77, n_cap)
    x[-40:] = 255
    return x


# name: (n_cap, f, fc_requested, fc_programmed, fs_programmed, buffers, batch sizes); the buffers repeat over a batch
CASES = {
    "ppm120_two_passes_C32": (153600, f_search_set(FC, 120.0), FC, FC, FS, "synth real full zero", (1, 2, 3, 8, 64)),
    "bench_C48": (153600, f_search_set(FC, 100.0), FC, FC, FS, "synth", (1, 8)),
    "C16_ncomb11": (106000, np.arange(-2, 3) * 5000.0, FC, FC, FS, "synth full", (1, 3)),
    "C24_ncomb6": (60000, np.arange(-4, 5) * 5000.0, FC, FC, FS, "synth zero", (1, 2, 8)),
    "C24_ncomb10_n_f16": (100000, np.arange(-8, 8) * 4000.0 + 700.0, FC, FC, FS, "synth", (1, 3)),
    "C32_fc_programmed": (40000, np.arange(-10, 11) * 2500.0, FC, 739.002e6, FS * 1.00001, "synth", (1, 3)),
    "two_passes_42": (40000, np.arange(-20, 22) * 2500.0, FC, 739.002e6, FS * 1.00001, "synth full", (1, 2, 8)),
    "three_passes_70": (30000, np.arange(-35, 35) * 1500.0, 1.8e9, 1.8e9, FS, "synth", (1, 2)),
    "last_sample_odd_stride": (29001, np.array([0.0]), FC, FC / 2.00677, FS, "tail", (1, 2)),
    "odd_stride_C24": (29001, np.arange(-3, 4) * 5000.0, FC, FC, FS, "synth full synth", (3,)),
}
# grids whose fold offsets relative to the per-half-frame minimum of their pass are not monotone in m in some column
NON_MONOTONE = ("ppm120_two_passes_C32", "C16_ncomb11", "C24_ncomb6", "C24_ncomb10_n_f16", "C32_fc_programmed", "two_passes_42")


def buffers(kind, n_cap, real=None):
    out = []
    for i, k in enumerate(kind.split()):
        if k == "synth":
            out.append(synth_cu8(0xC0FFEE + 17 * i + n_cap, n_cap))
        elif k == "real":
            out.append(real[:n_cap])
        elif k == "full":
            out.append(full_scale(n_cap + i, n_cap))
        elif k == "zero":
            out.append(np.full((n_cap, 2), 127, np.uint8))
        elif k == "tail":
            out.append(tail_255(n_cap))
    return out


def model(name):
    n_cap, f, fcr, fcp, fs, _, _ = CASES[name]
    return M.TcModel(n_cap, f, fcr, fcp, fs)


# ---------------------------------------------------------------------------------------------------------------------
# the model on the CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_every_layout_is_covered():
    layouts = {M.pick_layout(len(c[1])) for c in CASES.values()}
    assert layouts >= {(16, 1, 1), (24, 2, 1), (32, 2, 1), (48, 2, 1), (32, 2, 2), (48, 2, 3)}
    n_comb = {M.n_comb_xc(c[0]) for c in CASES.values()}
    assert n_comb & set(M.EXACT_RCP) and n_comb - set(M.EXACT_RCP)


@pytest.mark.parametrize("name", list(CASES))
def test_fold_offsets_fit_and_are_monotone(name):
    """Every case runs on tensor cores (0 <= dsh <= 32), dsh is non-decreasing in m in every column, so that the kernel's
    (tile, m) order is ascending m for every run start, and the listed grids would not be monotone relative to the
    per-half-frame minimum."""
    mod = model(name)
    assert mod.fits
    assert (np.diff(mod.dsh, axis=0) >= 0).all()
    old = np.zeros_like(mod.off)
    for f0, f1 in M.passes(len(mod.f)):
        old[:, f0:f1] = mod.off[:, f0:f1] - mod.off[:, f0:f1].min(axis=1)[:, None]
    assert (np.diff(old, axis=0) < 0).any() == (name in NON_MONOTONE)
    rr = np.random.default_rng(1).random((mod.n_comb, len(mod.f), 3, M.N_FOLD)).astype(np.float32)
    base = mod.fold(rr)
    for batch in (1, 3, 64):
        for b in (0, batch - 1):
            assert np.array_equal(mod.fold(rr, mod.run_starts(batch, 132, b)), base)


def test_default_and_bench_grids_keep_the_tensor_cores():
    """The +-120 ppm grid at 739 MHz and the benchmark's +-100 ppm grid fit the halo with monotone offsets; the bench grid's
    offsets are the ones the per-half-frame minimum gives (its output is unchanged)."""
    for ppm in (120.0, 100.0):
        mod = M.TcModel(153600, f_search_set(FC, ppm), FC, FC, FS)
        assert mod.fits
    assert np.array_equal(mod.dsh, mod.off - mod.off.min(axis=1)[:, None])


def test_fma32_rounds_once():
    """fma32 against exact rational arithmetic, on random operands and on sums that fall exactly between two float32
    values in float64 (where rounding the float64 sum again would be wrong), with normal and subnormal results."""
    from fractions import Fraction
    rng = np.random.default_rng(3)
    a = (rng.standard_normal(4000) * 2.0 ** rng.integers(-20, 20, 4000)).astype(np.float32)
    b = (rng.standard_normal(4000) * 2.0 ** rng.integers(-20, 20, 4000)).astype(np.float32)
    c = (rng.standard_normal(4000) * 2.0 ** rng.integers(-40, 40, 4000)).astype(np.float32)
    # c = 1 + 2^-24 (a float32 midpoint in float64 once the tiny product is added and rounded away)
    a[:4] = np.float32(2.0 ** -30); b[:4] = np.float32([1.0, -1.0, 2.0 ** -25, -(2.0 ** -25)]); c[:4] = np.float32(1.0) + np.float32(2.0 ** -23)
    a[4:8] = np.float32(1.0 + 2.0 ** -23); b[4:8] = np.float32([2.0 ** -24, -(2.0 ** -24), 2.0 ** -25, 3.0]); c[4:8] = np.float32(1.0)
    # subnormal results: a quarter of random operands below 2^-126, and a product 2^-150 (1 -+ 2^-46) that takes the
    # float64 sum with an odd c = (2^9 + 1) 2^-149 exactly halfway between two subnormals
    sub = slice(1000, 2000)
    a[sub] = (rng.standard_normal(1000) * 2.0 ** rng.integers(-80, -60, 1000)).astype(np.float32)
    b[sub] = (rng.standard_normal(1000) * 2.0 ** rng.integers(-80, -60, 1000)).astype(np.float32)
    c[sub] = (rng.standard_normal(1000) * 2.0 ** rng.integers(-150, -127, 1000)).astype(np.float32)
    a[8:12] = np.float32((1 + 2.0 ** -23) * 2.0 ** -75)
    b[8:12] = np.float32([(1 - 2.0 ** -23) * 2.0 ** -75, -(1 - 2.0 ** -23) * 2.0 ** -75, (1 + 2.0 ** -23) * 2.0 ** -75,
                          -(1 + 2.0 ** -23) * 2.0 ** -75])
    c[8:12] = np.float32(2.0 ** -140 + 2.0 ** -149)
    assert (np.abs(c[8:12]) < 2.0 ** -126).all() and (np.abs(c[sub]) < 2.0 ** -126).mean() > 0.9
    got = M.fma32(a, b, c)
    for x, y, z, g in zip(a, b, c, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        lo = np.float32(float(exact))
        cand = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        err = [abs(Fraction(float(v)) - exact) for v in cand]
        best = min(err)
        ties = [v for v, e in zip(cand, err) if e == best]
        want = ties[0] if len(ties) == 1 else [v for v in ties if (np.float32(v).view(np.int32) & 1) == 0][0]
        assert g == want, (x, y, z, g, want)


def test_division_rule_is_the_ieee_quotient():
    rng = np.random.default_rng(2)
    x = (rng.random(200000) * 2.0 ** rng.integers(-60, 60, 200000)).astype(np.float32)
    for n in range(1, 25):
        assert np.array_equal(M.divide(x, n), x / np.float32(n)), n


@pytest.mark.parametrize("name", ["C16_ncomb11", "C24_ncomb6", "C32_fc_programmed", "two_passes_42", "three_passes_70",
                                  "last_sample_odd_stride"])
def test_model_matches_oracle(oracle, name):
    """The model against the oracle's float64 `single` at the tensor-core parity bound (5e-7 of the largest value)."""
    n_cap, f, fcr, fcp, fs, kind, _ = CASES[name]
    mod = model(name)
    for cu8 in buffers(kind, n_cap)[:2]:
        ref = oracle.xcorr_pss(cu8_to_c128(cu8), f, 2, fcr, fcp, fs)["single"]
        got = mod.single(cu8).transpose(0, 2, 1)
        if np.abs(ref).max() == 0:
            assert np.all(got == 0)
        else:
            assert rel_err(got, ref) < 5e-7


def test_model_accumulators_are_the_integer_formulation():
    """The model's recombined x equals (a0*256 + a1)*256 + a2 + sum(a) (re) / sum(a[even]) (im) computed in Python integers
    from the model's own templates and bytes, wherever float32 holds that integer exactly."""
    n_cap = 12000
    f = np.array([-40000.0, 5000.0, 70000.0])
    mod = M.TcModel(n_cap, f, FC, FC, FS)
    cu8 = synth_cu8(99, n_cap, sigma=40.0)
    cu8[100:130] = 255; cu8[500:520] = 0
    x_re, x_im = M.lag_values(cu8, mod.a, mod.c_re, mod.c_im, 1000)
    z = cu8.reshape(-1).astype(np.int64) - 128
    y = np.empty_like(z); y[0::2] = z[1::2]; y[1::2] = -z[0::2] - 1
    for j in range(3):
        for t in range(3):
            a = mod.a[j, t]
            for L in range(0, 1000, 7):
                v_re = int((a * z[2 * L:2 * L + 274]).sum()) + int(a.sum())
                v_im = int((a * y[2 * L:2 * L + 274]).sum()) + int(a[0::2].sum())
                for got, want, c in ((x_re[j, t, L], v_re, mod.c_re[j, t]), (x_im[j, t, L], v_im, mod.c_im[j, t])):
                    # three float32 roundings: float(a0*256 + a1), the recombination (want - c) and the sum; exact below 2^24
                    assert abs(int(got) - want) <= (2 * abs(want - int(c)) + abs(want)) * 2.0 ** -24


# ---------------------------------------------------------------------------------------------------------------------
# the device against the model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_tc_single_bitwise(ctx, lcs, capbuf0000, name):
    """Device `single` == the model at each batch size: in the kernel's (tile, m) order for the run decomposition of that
    launch (n_sm from the device), which is ascending m, so the same buffer gives the same bits at every batch size."""
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    n_cap, f, fcr, fcp, fs, kind, batches = CASES[name]
    mod = model(name)
    bufs = buffers(kind, n_cap, capbuf0000["cu8"])
    rr = [mod.powers(b) for b in bufs]
    ascending = [mod.fold(r) for r in rr]
    first = {}
    for batch in batches:
        plan = ctx.plan(n_cap, f, 2, fcr, fcp, fs, max_batch=batch, kernel=lcs.KERNEL_TC)
        assert plan.kernel_for(lcs.IQ_CU8) == lcs.KERNEL_TC
        out = plan.run_host_np(np.stack([bufs[b % len(bufs)] for b in range(batch)]), lcs.IQ_CU8)["single"]
        plan.close()
        for b in range(batch):
            k = b % len(bufs)
            want = mod.fold(rr[k], mod.run_starts(batch, n_sm, b))
            assert_bitwise(want, ascending[k], f"{name}: model order at batch {batch}, buffer {b}")
            assert_bitwise(out[b], want, f"{name}: batch {batch}, buffer {b} ({kind.split()[k]})")
            first.setdefault(k, out[b])
            assert np.array_equal(out[b], first[k])
