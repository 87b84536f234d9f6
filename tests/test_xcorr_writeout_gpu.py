"""The correlator's write-out bit for bit, through the device entry point bench.py times (lcs_xcorr_pss_device).

Downstream of `single` (xc_incoherent_single) every stage is exact by construction, so it is checked without a tolerance:
- the delay-spread box filter and the frequency arg-max (epilogue4_kernel for ds_comb_arm <= 4, epilogue_kernel above):
  given the device's own `single`, incoherent = (s[idx] + (s[idx-1] + s[idx+1]) + ... + (s[idx-arm] + s[idx+arm])) / (2 arm + 1)
  in float32 with a circular index (searcher.cpp:330-343), then a strict-'>' first maximum over f (:369-382);
- sp_fold_kernel on 8-bit input: integer sample powers, one rounded division per sp[t], the fold in half-frame order,
  / n_comb_sp and the shift by 137 (searcher.cpp:185-221).
Both are restated in numpy (epilogue_model, sp_model_cu8), checked against the oracle on the CPU, and then against the
device bit for bit at every ds_comb_arm width the two epilogue kernels take, on both correlators and all three input formats.
`single` itself is compared with the oracle at the usual bounds (DESIGN section 5).

The device peak search (threshold + peak_search_kernel) is compared with the oracle at arms other than 2, with the
strongest peak rolled onto the edges of its +-arm refinement window."""
import numpy as np
import pytest

from conftest import cu8_to_c128, synth_cu8
from test_gpu_parity import REL, frq_mismatch_is_near_tie, rel_err
from test_search_chain_gpu import compare_cells, same_cells

N_FOLD = 9600
FC = 739e6
FS = 1.92e6
ARMS = (0, 1, 2, 3, 4, 5, 7, 16, 64)
GAP = (3000, 3700)      # samples of every half frame that are exactly zero: `single` ties at 0 over all f there


# ---------------------------------------------------------------------------------------------------------------------
# numpy models of the write-out (plain float32 / float64 operations; numpy neither fuses nor reorders them)
# ---------------------------------------------------------------------------------------------------------------------
def epilogue_model(single, arm):
    """xc_delay_spread + xc_peak_freq on single [3][n_f][9600] float32: incoherent [3][n_f][9600] float32,
    pow [3][9600] float64 and frq [3][9600] int32, in the reference's operation order."""
    s = np.ascontiguousarray(single, np.float32)
    idx = np.arange(N_FOLD)
    v = s.copy()
    for a in range(1, arm + 1):
        v = v + (s[..., (idx - a) % N_FOLD] + s[..., (idx + a) % N_FOLD])     # :336 += single[idx-t] + single[idx+t]
    inc = v / np.float32(2 * arm + 1)                                         # :343, IEEE float32 quotient
    best = inc[:, 0, :].copy()
    frq = np.zeros((3, N_FOLD), np.int32)
    for f in range(1, s.shape[1]):
        better = inc[:, f, :] > best                                          # :371-377 strict '>': first maximum wins
        best = np.where(better, inc[:, f, :], best)
        frq[better] = f
    return dict(incoherent=inc, pow=best.astype(np.float64), frq=frq)


def sp_model_cu8(cu8, n_cap):
    """sp_incoherent [9600] of an 8-bit buffer (uint8 [n_cap][2]) as sp_fold_kernel computes it: the power of a 274-sample
    window is an exact integer multiple of 2^-14, sp[t] its one rounded quotient by 274, the fold summed in half-frame
    order, divided by n_comb_sp and shifted right by 137."""
    x = cu8[:n_cap].astype(np.int64) - 127
    p = x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]
    csum = np.concatenate([[0], np.cumsum(p)])
    n_comb_sp = (n_cap - 136 - 137) // N_FOLD
    acc = None
    for m in range(n_comb_sp):
        t = m * N_FOLD + np.arange(N_FOLD)
        sp = ((csum[t + 274] - csum[t]).astype(np.float64) * (1.0 / 16384)) / 274
        acc = sp if m == 0 else acc + sp
    return np.roll(acc / n_comb_sp, 137)


def with_gap(x):
    """x [n][2] with the samples of GAP in every half frame set to zero signal (127 for bytes)."""
    x = x.copy()
    pos = np.arange(x.shape[0]) % N_FOLD
    x[(pos >= GAP[0]) & (pos < GAP[1])] = 127 if x.dtype == np.uint8 else 0
    return x


def real_cf32(seed, n_cap):
    """Float32 samples that are not 8-bit exact, with the zero gap: [n_cap][2]."""
    rng = np.random.default_rng(seed)
    return with_gap((rng.standard_normal((n_cap, 2)) * 0.15).astype(np.float32))


def grid(n_f):
    return (np.arange(n_f) - n_f // 2) * 5000.0 + 1234.5


def assert_bitwise(got, ref, what):
    got, ref = np.ascontiguousarray(got), np.ascontiguousarray(ref)
    assert got.dtype == ref.dtype and got.shape == ref.shape, what
    g = got.view(np.uint8).reshape(got.shape + (-1,))
    r = ref.view(np.uint8).reshape(ref.shape + (-1,))
    bad = np.argwhere((g != r).any(axis=-1))
    assert bad.size == 0, f"{what}: {len(bad)} elements differ, first at {tuple(bad[0])}: {got[tuple(bad[0])]!r} vs {ref[tuple(bad[0])]!r}"


def sp_close(got, ref):
    """|got - ref| <= 1e-12 max|ref|.  The oracle's sp_est is a running sum (searcher.cpp:206-208) whose absolute error
    scales with the largest window power, so next to the zero gap, where sp falls to 0, an elementwise relative bound
    measures the oracle's cancellation error rather than the device's."""
    return np.all(np.abs(got - ref) <= 1e-12 * np.abs(ref).max())


# ---------------------------------------------------------------------------------------------------------------------
# the models against the oracle (CPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arm", [0, 1, 4, 5, 64])
def test_epilogue_model_matches_oracle(oracle, arm):
    """On the oracle's own `single`, the model reproduces the oracle's incoherent, pow and frq exactly."""
    cap = cu8_to_c128(with_gap(synth_cu8(40 + arm, 29000)))
    f = grid(6)
    ref = oracle.xcorr_pss(cap, f, arm, FC, FC, FS)
    single = ref["single"].astype(np.float32)
    assert np.array_equal(single, ref["single"])                          # the oracle's vf3d holds float32 values
    m = epilogue_model(single.transpose(0, 2, 1), arm)
    assert np.array_equal(m["incoherent"].transpose(0, 2, 1).astype(np.float64), ref["incoherent"])
    assert np.array_equal(m["pow"], ref["pow"]) and np.array_equal(m["frq"], ref["frq"])
    lo, hi = GAP[0] + 10 + arm, GAP[1] - 150 - arm                         # ties at zero: frq 0 there
    assert np.all(ref["pow"][:, lo:hi] == 0) and np.all(m["frq"][:, lo:hi] == 0)


@pytest.mark.parametrize("n_cap", [29000, 60001])
def test_sp_model_cu8_matches_oracle(oracle, n_cap):
    cu8 = with_gap(synth_cu8(7, n_cap))
    ref = oracle.xcorr_pss(cu8_to_c128(cu8), grid(1), 0, FC, FC, FS)
    assert sp_close(sp_model_cu8(cu8, n_cap), ref["sp_incoherent"])


# ---------------------------------------------------------------------------------------------------------------------
# the device entry point: torch tensors, raw pointers
# ---------------------------------------------------------------------------------------------------------------------
def dev_outputs(batch, n_f, inc=True):
    """Output tensors filled with values the write-out never produces, so that a position it skips fails."""
    import torch
    nan = float("nan")
    o = dict(single=torch.full((batch, 3, n_f, N_FOLD), nan, dtype=torch.float32, device="cuda"),
             pow=torch.full((batch, 3, N_FOLD), nan, dtype=torch.float64, device="cuda"),
             frq=torch.full((batch, 3, N_FOLD), -7, dtype=torch.int32, device="cuda"),
             sp_incoherent=torch.full((batch, N_FOLD), nan, dtype=torch.float64, device="cuda"))
    if inc:
        o["incoherent"] = torch.full((batch, 3, n_f, N_FOLD), nan, dtype=torch.float32, device="cuda")
    return o


def run_device(plan, iq, fmt, batch, inc=True, stream=None, iq_ptr=None):
    """plan.run_device on a device tensor iq [>= batch][n_cap][2]; returns the outputs as numpy arrays."""
    import torch
    o = dev_outputs(batch, plan.n_f, inc)
    if stream is not None:
        stream.wait_stream(torch.cuda.current_stream())
    plan.run_device(iq.data_ptr() if iq_ptr is None else iq_ptr, fmt, batch, o["single"].data_ptr(), o["pow"].data_ptr(),
                    o["frq"].data_ptr(), o["sp_incoherent"].data_ptr(), o["incoherent"].data_ptr() if inc else None,
                    stream=stream.cuda_stream if stream is not None else None)
    if stream is not None:
        stream.synchronize()
    else:
        torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def to_dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def check_writeout(out, arm, cu8=None):
    """Every buffer's incoherent / pow / frq bit for bit against the model on the device's own single."""
    for b in range(out["single"].shape[0]):
        m = epilogue_model(out["single"][b], arm)
        assert_bitwise(out["incoherent"][b], m["incoherent"], f"incoherent[{b}]")
        assert_bitwise(out["pow"][b], m["pow"], f"pow[{b}]")
        assert_bitwise(out["frq"][b], m["frq"], f"frq[{b}]")
        if cu8 is not None:
            assert_bitwise(out["sp_incoherent"][b], sp_model_cu8(cu8[b], cu8.shape[1]), f"sp_incoherent[{b}]")


def check_vs_oracle(out, refs, tol):
    for b, ref in enumerate(refs):
        assert rel_err(out["single"][b].transpose(0, 2, 1), ref["single"]) < tol
        assert rel_err(out["incoherent"][b].transpose(0, 2, 1), ref["incoherent"]) < tol
        assert rel_err(out["pow"][b], ref["pow"]) < tol
        assert sp_close(out["sp_incoherent"][b], ref["sp_incoherent"])
        assert frq_mismatch_is_near_tie(out["frq"][b], ref)


# (arm, n_cap, n_f, batch, max_batch, fc_programmed, fs_programmed)
#   n_f = 1: the FP32 correlator's FW = 1 path on cf32 / c128; n_f = 7 and 9 leave the last 8-hypothesis chunk partial
CASES = [
    (0, 29000, 1, 1, 1, FC, FS),
    (1, 30001, 9, 3, 5, FC, FS),
    (2, 60000, 5, 1, 1, FC + 2000.0, FS * 1.00002),
    (3, 40000, 7, 1, 1, FC, FS),
    (4, 35000, 1, 1, 2, FC, FS),
    (5, 29000, 9, 1, 1, FC, FS),
    (7, 50000, 3, 1, 1, FC - 3000.0, FS * (1 - 1e-5)),
    (16, 45000, 1, 1, 1, FC, FS),
    (64, 33333, 9, 3, 5, FC, FS),
]
assert sorted(c[0] for c in CASES) == list(ARMS)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=["arm%d" % c[0] for c in CASES])
def test_writeout_bitwise_every_arm(ctx, lcs, oracle, case):
    """run_device at one ds_comb_arm: cu8 through the tensor-core and the FP32 correlator, cf32 and c128 (the same float32
    samples, not 8-bit exact) through the FP32 correlator.  The write-out bit for bit against the models, everything
    against the oracle at the usual bounds."""
    arm, n_cap, n_f, batch, max_batch, fcp, fs = case
    f = grid(n_f)
    cu8 = np.stack([with_gap(synth_cu8(1000 * arm + b, n_cap)) for b in range(batch)])
    x32 = np.stack([real_cf32(2000 * arm + b, n_cap) for b in range(batch)])
    ref_u8 = [oracle.xcorr_pss(cu8_to_c128(c), f, arm, FC, fcp, fs) for c in cu8]
    ref_f = [oracle.xcorr_pss(x.astype(np.float64).view(np.complex128).reshape(-1), f, arm, FC, fcp, fs) for x in x32]
    d_u8, d_f32, d_c128 = to_dev(cu8), to_dev(x32), to_dev(x32.astype(np.float64))

    tc = ctx.plan(n_cap, f, arm, FC, fcp, fs, max_batch=max_batch, kernel=lcs.KERNEL_TC)
    fp = ctx.plan(n_cap, f, arm, FC, fcp, fs, max_batch=max_batch, kernel=lcs.KERNEL_FP32)
    assert tc.kernel_for(lcs.IQ_CU8) == lcs.KERNEL_TC and fp.kernel_for(lcs.IQ_CU8) == lcs.KERNEL_FP32
    out = run_device(tc, d_u8, lcs.IQ_CU8, batch)
    check_writeout(out, arm, cu8)
    check_vs_oracle(out, ref_u8, 5e-7)
    out = run_device(fp, d_u8, lcs.IQ_CU8, batch)
    check_writeout(out, arm, cu8)
    check_vs_oracle(out, ref_u8, REL)
    o32 = run_device(fp, d_f32, lcs.IQ_CF32, batch)
    check_writeout(o32, arm)
    check_vs_oracle(o32, ref_f, REL)
    o128 = run_device(fp, d_c128, lcs.IQ_C128, batch)
    check_writeout(o128, arm)
    check_vs_oracle(o128, ref_f, REL)
    # the c128 samples are the cf32 ones widened: the correlator rounds them back to the same floats
    assert_bitwise(o128["single"], o32["single"], "single c128 vs cf32")
    tc.close()
    fp.close()


# ---------------------------------------------------------------------------------------------------------------------
# entry-point behaviour
# ---------------------------------------------------------------------------------------------------------------------
def assert_bitwise_outputs(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert_bitwise(a[k], b[k], k)


@pytest.mark.gpu
def test_side_stream_and_timing_give_the_default_stream_result(ctx, lcs):
    """A caller's stream (only that stream synchronised) and the timing hook leave every output bit for bit unchanged;
    timing_read counts one bracketed launch per call."""
    import torch
    f = grid(9)
    cu8 = np.stack([with_gap(synth_cu8(60 + b, 40000)) for b in range(2)])
    d = to_dev(cu8)
    for kernel in (lcs.KERNEL_TC, lcs.KERNEL_FP32):
        plan = ctx.plan(40000, f, 5, FC, FC, FS, max_batch=2, kernel=kernel)
        base = run_device(plan, d, lcs.IQ_CU8, 2)
        side = torch.cuda.Stream()
        assert_bitwise_outputs(run_device(plan, d, lcs.IQ_CU8, 2, stream=side), base)
        assert plan.timing_read()[1] == 0
        plan.timing_enable(True)
        timed = [run_device(plan, d, lcs.IQ_CU8, 2), run_device(plan, d, lcs.IQ_CU8, 2, stream=side)]
        ms, n = plan.timing_read()
        assert n == 2 and ms > 0
        for t in timed:
            assert_bitwise_outputs(t, base)
        plan.timing_enable(False)
        run_device(plan, d, lcs.IQ_CU8, 2)
        assert plan.timing_read()[1] == 0
        plan.close()


@pytest.mark.gpu
def test_arm_limit(ctx, lcs):
    f = grid(3)
    with pytest.raises(lcs.LcsError):
        ctx.plan(29000, f, 65, FC, FC, FS)
    ctx.plan(29000, f, 64, FC, FC, FS).close()


@pytest.mark.gpu
@pytest.mark.parametrize("arm", [3, 5])
def test_dropin_incoherent_is_the_planar_write_out(ctx, lcs, capbuf0000, arm):
    """lcs_xcorr_pss's incoherent ([t][idx][f]) is the transposed d_incoherent_planar of a plan with the same parameters:
    an 8-bit exact capture (the drop-in routes it to the tensor-core correlator, the plan gets its bytes) and samples that
    are not 8-bit exact (FP32 correlator on both sides)."""
    f = 35000.0 + grid(5)
    cu8 = capbuf0000["cu8"][:60000]
    x = real_cf32(arm, 60000).astype(np.float64)
    for cap, iq, fmt in ((cu8_to_c128(cu8), cu8, lcs.IQ_CU8), (x.view(np.complex128).reshape(-1), x, lcs.IQ_C128)):
        ref = ctx.xcorr_pss(cap, f, arm, FC, FC, FS)
        plan = ctx.plan(60000, f, arm, FC, FC, FS, max_batch=1)
        out = run_device(plan, to_dev(iq[None]), fmt, 1)
        assert_bitwise(out["incoherent"][0].transpose(0, 2, 1), ref["incoherent"], "incoherent")
        assert_bitwise(out["single"][0].transpose(0, 2, 1), ref["single"], "single")
        assert_bitwise(out["pow"][0], ref["pow"], "pow")
        assert_bitwise(out["frq"][0], ref["frq"], "frq")
        plan.close()


@pytest.mark.gpu
def test_auto_serves_an_unaligned_cu8_pointer_with_the_fp32_correlator(ctx, lcs):
    """A cu8 pointer one sample (2 bytes) past a 16-byte boundary: AUTO runs the FP32 correlator and returns bitwise what
    an explicit FP32 plan returns on an aligned copy; an explicit tensor-core plan refuses it without a launch."""
    import torch
    n_cap, f = 30000, grid(5)
    cu8 = with_gap(synth_cu8(90, n_cap))
    raw = torch.zeros((n_cap + 8) * 2, dtype=torch.uint8, device="cuda")
    raw[2:2 + 2 * n_cap] = torch.from_numpy(cu8.reshape(-1)).cuda()
    ptr = raw.data_ptr() + 2
    assert ptr % 16 != 0
    auto = ctx.plan(n_cap, f, 2, FC, FC, FS)
    assert auto.kernel_for(lcs.IQ_CU8) == lcs.KERNEL_TC
    fp = ctx.plan(n_cap, f, 2, FC, FC, FS, kernel=lcs.KERNEL_FP32)
    got = run_device(auto, raw, lcs.IQ_CU8, 1, iq_ptr=ptr)
    assert_bitwise_outputs(got, run_device(fp, to_dev(cu8[None]), lcs.IQ_CU8, 1))
    check_writeout(got, 2, cu8[None])
    tc = ctx.plan(n_cap, f, 2, FC, FC, FS, kernel=lcs.KERNEL_TC)
    n0 = ctx.launches
    with pytest.raises(lcs.LcsError):
        run_device(tc, raw, lcs.IQ_CU8, 1, iq_ptr=ptr)
    assert ctx.launches == n0
    for p in (auto, fp, tc):
        p.close()


@pytest.mark.gpu
def test_rejected_calls_launch_nothing(ctx, lcs):
    """Bad batch sizes, an unknown format, cf32 on an explicit tensor-core plan, and pointers that the kernels would read
    or write with misaligned vector accesses: LcsError before any launch."""
    import torch
    n_cap, f = 30000, grid(3)
    fp = ctx.plan(n_cap, f, 2, FC, FC, FS, max_batch=2, kernel=lcs.KERNEL_FP32)
    tc = ctx.plan(n_cap, f, 2, FC, FC, FS, max_batch=2, kernel=lcs.KERNEL_TC)
    auto = ctx.plan(n_cap, f, 2, FC, FC, FS, max_batch=2)
    raw = {k: torch.zeros(2 * n_cap * 16 + 64, dtype=torch.uint8, device="cuda") for k in ("iq", "iq32")}
    o = dev_outputs(2, 3)
    ptrs = dict(single=o["single"].data_ptr(), pow=o["pow"].data_ptr(), frq=o["frq"].data_ptr(),
                sp_incoherent=o["sp_incoherent"].data_ptr(), incoherent=o["incoherent"].data_ptr())

    def call(plan, fmt=lcs.IQ_CU8, batch=1, iq=None, **shift):
        p = {k: v + shift.get(k, 0) for k, v in ptrs.items()}
        plan.run_device(raw["iq"].data_ptr() if iq is None else iq, fmt, batch, p["single"], p["pow"], p["frq"],
                        p["sp_incoherent"], p["incoherent"])

    call(fp)                                   # the well-formed call goes through
    call(auto, batch=2)
    torch.cuda.synchronize()
    bad = [(fp, dict(batch=0)), (fp, dict(batch=3)), (auto, dict(batch=3)), (fp, dict(fmt=7)), (auto, dict(fmt=-1)),
           (tc, dict(fmt=lcs.IQ_CF32)), (tc, dict(fmt=lcs.IQ_C128))]
    # one byte off: the IQ pointer for every format and plan, then each output in turn
    base = raw["iq32"].data_ptr()
    for plan in (fp, tc, auto):
        bad.append((plan, dict(iq=base + 1)))
    for fmt in (lcs.IQ_CF32, lcs.IQ_C128):
        bad += [(fp, dict(fmt=fmt, iq=base + 1)), (fp, dict(fmt=fmt, iq=base + 4)), (auto, dict(fmt=fmt, iq=base + 1))]
    bad.append((fp, dict(fmt=lcs.IQ_C128, iq=base + 8)))
    for k in ptrs:
        for plan in (fp, tc):
            bad.append((plan, {k: 1}))
    for k in ("single", "incoherent"):                     # a float slice: 4-byte aligned, not 16
        bad.append((fp, {k: 4}))
    bad += [(fp, dict(pow=8)), (fp, dict(frq=4)), (fp, dict(frq=8))]
    for plan, kw in bad:
        n0 = ctx.launches
        with pytest.raises(lcs.LcsError):
            call(plan, **kw)
        assert ctx.launches == n0, kw
    # sp_incoherent needs only 8 bytes (scalar doubles)
    call(fp, sp_incoherent=8)
    torch.cuda.synchronize()
    for p in (fp, tc, auto):
        p.close()


# ---------------------------------------------------------------------------------------------------------------------
# device peak search at arms other than 2
# ---------------------------------------------------------------------------------------------------------------------
def oracle_peaks(oracle, cu8, f, arm):
    o = oracle.xcorr_pss(cu8_to_c128(cu8), f, arm, FC, FC, FS)
    z = oracle.calc_Z_th1(o["sp_incoherent"], o["n_comb_xc"], arm)
    return o, oracle.peak_search(o["pow"], o["frq"], z, f, FC, FC, o["single"], arm)


def strongest_col(o):
    return int(np.argmax(o["pow"]) % N_FOLD)


def rolled_copies(oracle, cu8, f, arm, lo, hi):
    """{column: (buffer, oracle peaks)} for the rolls of cu8 that put the oracle's strongest pow column between lo and hi
    (inclusive, lo > hi wraps past 9599).  Near the ends of the fold the box filter sums neighbours from the other end,
    which moves the arg-max of a broad peak by a sample or two: some columns are skipped, so every roll in the range is
    tried."""
    o, _ = oracle_peaks(oracle, cu8, f, arm)
    c0 = strongest_col(o)
    out = {}
    for d in range(lo - c0 - 2, lo - c0 + (hi - lo) % N_FOLD + 3):
        r = np.roll(cu8, d, axis=0)
        o, peaks = oracle_peaks(oracle, r, f, arm)
        out.setdefault(strongest_col(o), (r, peaks))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("arm", [0, 1, 4, 7])
def test_device_peak_search_at_arm(ctx, lcs, oracle, capbuf0000, arm):
    """peaks_batch at ds_comb_arm = arm against the oracle's xcorr_pss -> calc_Z_th1 -> peak_search at the same arm, and
    against the host peak_search on the device's own pow / frq / single.  Besides the capture itself, rolled copies put
    the strongest peak at the last column below arm the peak can take (the reference's uint16 wrap: ind = -1), at the
    first column from arm on (column arm itself at arm 0 and 1: the first column that refines) and, for arm > 0, at a
    column above 9599 - arm (the refinement window wraps forward past 9599)."""
    f = 35000.0 + grid(5)
    real = capbuf0000["cu8"]
    bufs, refs = [real], [oracle_peaks(oracle, real, f, arm)[1]]
    near0 = rolled_copies(oracle, real, f, arm, 0, arm + 2)
    picks = []
    if arm:
        picks.append(max(c for c in near0 if c < arm))
        assert near0[picks[-1]][1][0].ind == -1
    picks.append(min(c for c in near0 if arm <= c < N_FOLD // 2))
    assert picks[-1] == arm or (arm > 1 and picks[-1] <= arm + 2)
    assert near0[picks[-1]][1][0].ind >= 0
    copies = [near0[c] for c in picks]
    if arm:
        near_end = rolled_copies(oracle, real, f, arm, N_FOLD - arm, N_FOLD - 1)
        copies.append(near_end[min(c for c in near_end if c >= N_FOLD - arm)])
    for b, p in copies:
        bufs.append(b)
        refs.append(p)
    plan = ctx.plan(real.shape[0], f, arm, FC, FC, FS, max_batch=len(bufs))
    got = plan.peaks_batch(np.stack(bufs), lcs.IQ_CU8)
    out = plan.run_host_np(np.stack(bufs), lcs.IQ_CU8)
    for b in range(len(bufs)):
        assert len(refs[b]) >= 2
        compare_cells(got[b], refs[b])
        z = lcs.calc_z_th1(out["sp_incoherent"][b], plan.n_comb_xc, arm)
        same_cells(got[b], lcs.peak_search(out["pow"][b], out["frq"][b], z, f, FC, FC, out["single"][b], arm))
    plan.close()
