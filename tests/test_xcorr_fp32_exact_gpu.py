"""The FP32 correlator's `single` (xcorr_fold_fp32_kernel), its templates, and sp_incoherent of float input, bit for bit.

The kernel is a fixed sequence of correctly rounded float32 operations (explicit fmaf, __fadd_rn / __fmul_rn, __fdiv_rn)
and sp_fold_kernel a fixed sequence of float64 ones, so both outputs are determined to the last bit and
xcorr_fp32_model.py restates them.  On the CPU the models are checked against the oracle, the comparison is shown to
resolve plausible slips (one tap chain, a fused power, descending half frames, templates divided in float32, a sequential
prefix sum), and the SASS is checked for the facts the model rests on.  On the device:
- the plan's FP32 templates (d_w01 / d_w2) equal the model's, read back through the drop-in's debug `xc` of a unit impulse;
- `single` equals the model at every hypothesis-chunk shape (FW = 1; FW = 8 with partial, exact and one-hypothesis chunks;
  37 and 300 hypotheses), fold offsets spread by fc_programmed != fc_requested and an off-nominal fs, the widest tile the
  plan accepts, n_comb 1, 2, 4, 6, 15 and 26, an odd n_cap whose last tile reads past it, every route to the kernel (explicit,
  AUTO for cf32 / c128 / long cu8 / > 256 hypotheses / sparse grids / an unaligned cu8 pointer, the c128 drop-in), noise,
  the recording with a dither, a cell 40 dB over noise, zero and subnormal-scale buffers, at batch sizes 1, 2 and 8;
- sp_incoherent equals the block-scan model for cf32 and c128 (and the integer model for cu8) in the same runs."""
import functools
import os
import re
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import xcorr_fp32_model as F
from conftest import ROOT, synth_cu8
from test_xcorr_writeout_gpu import run_device, sp_model_cu8

FC, FS = 739e6, 1.92e6
PSS_TD = functools.lru_cache(maxsize=None)(F.pss_td)
WIDE_STEP = 392400.0       # 9 hypotheses at 100 MHz: fold-offset spread 3692, the widest tile planset_build accepts


def f_search_set(fc, ppm):
    n = int(np.floor((fc * ppm / 1e6 + 2.5e3) / 5e3))
    return 5000.0 * np.arange(-n, n + 1)


# name: (n_cap, f, fc_requested, fc_programmed, fs_programmed, formats, route, buffers, batch sizes)
#   route: "fp32" an explicit FP32 plan, "auto" an AUTO plan that resolves the format to the FP32 kernel,
#   "auto_unaligned" an AUTO plan on a cu8 pointer 2 bytes past a 16-byte boundary, "dropin" lcs_xcorr_pss (c128)
CASES = {
    "fw1_auto": (29000, np.array([35000.0]), FC, FC, FS, ("cf32", "c128"), "auto", "noise cell zero", (1, 2, 8)),
    "fw1_ncomb15": (153600, np.array([-1234.5]), FC, FC, FS, ("c128", "cf32"), "fp32", "cell", (1,)),
    "nf7_fc_programmed": (60000, np.arange(-3, 4) * 5000.0, FC, FC + 2000.0, FS * 1.00002, ("c128",), "auto",
                          "noise cell", (1, 2)),
    "nf8_ncomb15_cu8": (153600, np.arange(-4, 4) * 5000.0 + 700.0, FC, FC, FS, ("cu8",), "fp32", "noise capbuf", (1, 2)),
    "nf9_subnormal": (40000, np.arange(-4, 5) * 5000.0, FC, FC, FS, ("cf32",), "fp32", "subnormal noise zero", (1, 8)),
    "nf9_ncomb1": (9873, np.arange(-4, 5) * 5000.0, FC, 739.004e6, FS * 0.99998, ("cf32", "c128"), "auto", "noise",
                   (1, 2)),
    "nf9_odd_tail": (29001, np.arange(0, 9) * 2500.0, FC, FC / 2.00677, FS, ("c128",), "fp32", "noise", (1, 2)),
    "ppm120": (153600, f_search_set(FC, 120.0), FC, FC, FS, ("c128", "cf32"), "auto", "capbuf cell", (1, 2)),
    "ppm120_dropin": (153600, f_search_set(FC, 120.0), FC, FC, FS, ("c128",), "dropin", "capbuf", (1,)),
    "nf300_cu8": (29000, np.arange(-150, 150) * 2000.0 + 500.0, FC, FC, FS, ("cu8",), "auto", "noise", (1,)),
    "ncomb26_cu8": (250000, np.arange(-1, 2) * 5000.0, FC, FC, FS, ("cu8",), "auto", "noise", (1,)),
    "wide_tile_cu8": (153600, np.arange(9) * WIDE_STEP, 100e6, 100e6, FS, ("cu8",), "auto", "noise", (1,)),
    "unaligned_cu8": (30001, np.arange(-4, 5) * 5000.0, FC, FC, FS, ("cu8",), "auto_unaligned", "noise capbuf", (1, 2)),
}
PARAMS = [(name, fmt) for name, c in CASES.items() for fmt in c[5]]

# fold positions every hypothesis is compared at: every lane x register slot (idx mod 224), both sides of every CTA
# edge (the FW = 1 sub-tiles are 224 wide too) and the last, partial CTA
POSITIONS = np.array(sorted(set(range(224)) | {224 * k + d for k in range(1, 43) for d in (-1, 0)}
                            | set(range(9408, 9600))))


def model(name):
    n_cap, f, fcr, fcp, fs = CASES[name][:5]
    return F.Fp32Model(n_cap, f, fcr, fcp, fs)


def edge_hypotheses(mod):
    """The hypotheses compared at every position: chunk edges, the last one, and the smallest and largest offsets."""
    last = mod.off[-1]
    fs = {0, 7, 8, 15, mod.n_f - 1, int(np.argmin(last)), int(np.argmax(last))}
    return np.array(sorted(f for f in fs if f < mod.n_f))


def full(mod):
    return mod.n_f <= 9


# ---------------------------------------------------------------------------------------------------------------------
# buffers: float kinds are float64 [n][2] (cast to float32 for cf32), cu8 kinds uint8 [n][2]
# ---------------------------------------------------------------------------------------------------------------------
def noise(seed, n, scale=0.2):
    return np.random.default_rng(seed).standard_normal((n, 2)) * scale


def cell(seed, n):
    """Root 1 of the PSS in every half frame at 40 dB over the noise per sample (most positions far below the peak)."""
    td = PSS_TD()[1]
    x = noise(seed, n, 0.002)
    amp = 100 * 0.002 * np.sqrt(2) / np.sqrt(np.mean(np.abs(td) ** 2))
    for s in range(2000, n - 137, 9600):
        x[s:s + 137, 0] += amp * td.real
        x[s:s + 137, 1] += amp * td.imag
    return x


def buffers(name, fmt, capbuf=None):
    n_cap, kinds = CASES[name][0], CASES[name][7]
    out = []
    for i, k in enumerate(kinds.split()):
        seed = 0xF32 + 31 * i + n_cap
        if fmt == "cu8":
            x = {"noise": lambda: synth_cu8(seed, n_cap), "capbuf": lambda: capbuf[:n_cap],
                 "zero": lambda: np.full((n_cap, 2), 127, np.uint8)}[k]()
        else:
            x = {"noise": lambda: noise(seed, n_cap), "cell": lambda: cell(seed, n_cap),
                 "zero": lambda: np.zeros((n_cap, 2)),
                 "capbuf": lambda: (capbuf[:n_cap].astype(np.float64) - 127) / 128 + noise(seed, n_cap, 1e-4),
                 "subnormal": lambda: noise(seed, n_cap, 2.0 ** -64)}[k]()
            x = x.astype(np.float32) if fmt == "cf32" else x
        out.append(np.ascontiguousarray(x))
    return out


def capbuf_cu8():
    from conftest import load
    return load("capbuf_0000.npz")["cu8"].reshape(-1, 2)


def sp_ref(buf, fmt, n_cap):
    if fmt == "cu8":
        return sp_model_cu8(buf, n_cap)
    return F.sp_model(F.sample_power(buf, fmt), n_cap)


def mismatches(got, want, fs, idx, what):
    """'' if got == want bit for bit, else the first few (buffer, t, f, idx, device, model)."""
    assert got.shape == want.shape and got.dtype == want.dtype, what
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    if not bad.size:
        return ""
    rows = [(what, int(t), int(fs[j]), int(idx[i]), float(got[t, j, i]), float(want[t, j, i])) for t, j, i in bad[:6]]
    return "%d of %d values differ; first (buffer, t, f, idx, device, model): %s" % (len(bad), got.size, rows)


# ---------------------------------------------------------------------------------------------------------------------
# the cases and the model on the CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_every_case_is_covered():
    mods = {name: model(name) for name in CASES}
    assert all(m.accepted for m in mods.values())
    n_f = {m.n_f for m in mods.values()}
    assert {m.fw for m in mods.values()} == {1, 8}
    assert {7, 9} <= {k for k in n_f if k % 8}, "partial chunks"                  # 9 leaves a one-hypothesis chunk
    assert 8 in n_f and 37 in n_f and max(n_f) > 256
    n_comb = {m.n_comb for m in mods.values()}
    assert {1, 15} <= n_comb and max(n_comb) > 24
    routes = {(fmt, c[6]) for c in CASES.values() for fmt in c[5]}
    assert {("cf32", "auto"), ("c128", "auto"), ("cu8", "fp32"), ("cu8", "auto_unaligned"), ("c128", "dropin")} <= routes
    assert {"noise", "capbuf", "cell", "zero", "subnormal"} <= {k for c in CASES.values() for k in c[7].split()}
    assert {1, 2, 8} <= {b for c in CASES.values() for b in c[8]}
    # offsets spread within a chunk by the clocks; the widest tile; a last tile that reads past an odd n_cap
    m = mods["nf7_fc_programmed"]
    assert CASES["nf7_fc_programmed"][3] != FC and CASES["nf7_fc_programmed"][4] != FS and m.spread >= 1
    assert mods["wide_tile_cu8"].smem == F.SMEM_CAP
    tail = mods["nf9_odd_tail"]
    assert tail.n_cap % 2 == 1 and tail.last_tile_end() > tail.n_cap
    assert tail.off.max() + F.N_FOLD - 1 == tail.n_cap - 137            # the last real tap reads the last sample
    # AUTO routes that land on the FP32 kernel for cu8: > 256 hypotheses, > 24 half frames, a grid too sparse for the
    # tensor-core tiling (offsets more than 32 samples above the staging start)
    assert mods["nf300_cu8"].n_f > 256 and mods["ncomb26_cu8"].n_comb > 24 and mods["wide_tile_cu8"].spread > 32
    # the position set: every lane x slot, both sides of every CTA edge, the last partial CTA
    assert set(POSITIONS % 224) == set(range(224))
    for k in range(1, 43):
        assert {224 * k - 1, 224 * k} <= set(POSITIONS)
    assert set(range(9408, 9600)) <= set(POSITIONS)


def test_wide_grid_sits_at_the_tile_limit():
    """The widest grid fills the FP32 correlator's 100 KiB of shared memory exactly; one sample more of spread is rejected
    by planset_build (test_wider_grid_is_rejected checks the device)."""
    m = model("wide_tile_cu8")
    assert m.spread == 3692 and m.smem == F.SMEM_CAP and m.accepted
    wider = F.Fp32Model(153600, np.arange(9) * (WIDE_STEP + 100.0), 100e6, 100e6, FS)
    assert wider.in_range and wider.spread == 3693 and not wider.accepted


def test_compiled_fmaf_is_one_rounding():
    """The model's std::fmaf equals fma32 (one rounding, checked against exact arithmetic in test_fma32_rounds_once) on
    random operands, normal and subnormal results, and sums halfway between two float32 values in float64."""
    rng = np.random.default_rng(11)
    n = 200000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-80, 20, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-80, 20, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-149, 40, n)).astype(np.float32)
    a[:4] = np.float32((1 + 2.0 ** -23) * 2.0 ** -75)
    b[:4] = np.float32([(1 - 2.0 ** -23) * 2.0 ** -75, -(1 - 2.0 ** -23) * 2.0 ** -75, 2.0 ** -75, -(2.0 ** -75)])
    c[:4] = np.float32(2.0 ** -140 + 2.0 ** -149)
    got, want = F.fmaf(a, b, c), F.fma32(a, b, c)
    assert ((want != 0) & (np.abs(want) < 2.0 ** -126)).sum() > 1000
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_fma64_rounds_once():
    """fma64 (the c128 sample power) against exact rational arithmetic."""
    rng = np.random.default_rng(12)
    x = rng.standard_normal(3000) * 2.0 ** rng.integers(-30, 30, 3000)
    y = rng.standard_normal(3000) * 2.0 ** rng.integers(-30, 30, 3000)
    c = y * y
    got = F.fma64(x, x, c)
    for xi, ci, g in zip(x, c, got):
        exact = Fraction(xi) * Fraction(xi) + Fraction(ci)
        lo = float(exact)                                           # Fraction -> float rounds to nearest, ties to even
        assert g == lo, (xi, ci, g, lo)


@pytest.mark.parametrize("name,fmt", [("nf9_subnormal", "cf32"), ("fw1_auto", "c128"), ("nf7_fc_programmed", "c128"),
                                      ("ppm120", "c128"), ("nf9_odd_tail", "c128"), ("nf8_ncomb15_cu8", "cu8")])
def test_model_matches_oracle(oracle, name, fmt):
    """The model against the oracle's float64 `single` at the parity bound (1e-6 of the largest value) and, where the
    oracle's value exceeds 1e-3 of the largest, at 5e-7 of the largest."""
    n_cap, f, fcr, fcp, fs = CASES[name][:5]
    mod = model(name)
    for buf in buffers(name, fmt, capbuf_cu8())[-2:]:
        x32 = F.samples(buf, fmt)
        ref = oracle.xcorr_pss(x32.astype(np.float64).view(np.complex128).reshape(-1), f, 2, fcr, fcp, fs)["single"]
        got = mod.single(x32).transpose(0, 2, 1)
        top = np.abs(ref).max()
        if top == 0:
            assert np.all(got == 0)
            continue
        err = np.abs(got - ref)
        assert err.max() < 1e-6 * top
        assert err[ref > 1e-3 * top].max() < 5e-7 * top


@pytest.mark.parametrize("fmt", ["cf32", "c128"])
@pytest.mark.parametrize("n_cap", [9873, 29000, 153600])
def test_sp_model_matches_oracle(oracle, fmt, n_cap):
    """The block-scan model of sp_incoherent against the oracle at the parity bound (1e-12 relative), n_comb_sp 1, 2, 15."""
    x = noise(n_cap, n_cap)
    x = x.astype(np.float32) if fmt == "cf32" else x
    ref = oracle.xcorr_pss(x.astype(np.float64).view(np.complex128).reshape(-1), np.array([0.0]), 2, FC, FC, FS)
    assert np.abs(sp_ref(x, fmt, n_cap) / ref["sp_incoherent"] - 1).max() < 1e-12


# fraction of the n_f = 9 noise case's positions at which a variant of the model differs from the model, as measured
# (0.877, 0.136, 0.333, 0.623 of `single`; 0.949 of sp_incoherent) and rounded down
SENSITIVITY = {"one 140-tap chain": 0.87, "fused power": 0.13, "descending m": 0.33, "templates float(re) / 137": 0.62,
               "sequential prefix sum": 0.94}


def test_the_comparison_resolves_plausible_slips():
    name = "nf9_subnormal"
    mod = model(name)
    buf = buffers(name, "cf32")[1]                                  # the noise buffer
    assert CASES[name][7].split()[1] == "noise" and mod.n_f == 9 and mod.n_comb == 4
    x32 = F.samples(buf, "cf32")
    base = mod.single(x32)
    frac = {"one 140-tap chain": mod.single(x32, flags=F.ONE_CHAIN),
            "fused power": mod.single(x32, flags=F.FUSED_POWER),
            "descending m": mod.single(x32, flags=F.DESCENDING_M),
            "templates float(re) / 137": mod.single(x32, exact_w=False)}
    frac = {k: float((v != base).mean()) for k, v in frac.items()}
    sp = sp_ref(buf, "cf32", mod.n_cap)
    frac["sequential prefix sum"] = float((F.sp_model(F.sample_power(buf, "cf32"), mod.n_cap, block_scan=False) != sp).mean())
    for k, th in SENSITIVITY.items():
        assert frac[k] >= th, (k, frac)


def test_subnormal_buffer_reaches_subnormal_powers():
    """The subnormal-scale buffer puts most squares re^2, im^2 below 2^-126: a flush to zero would change `single`."""
    mod = model("nf9_subnormal")
    s = mod.single(F.samples(buffers("nf9_subnormal", "cf32")[0], "cf32"))
    tiny = np.float32(2.0 ** -126)
    assert (s > 0).mean() > 0.95 and ((s > 0) & (s < tiny)).mean() > 0.5


# ---------------------------------------------------------------------------------------------------------------------
# the SASS facts the model rests on
# ---------------------------------------------------------------------------------------------------------------------
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\s*([^;]*);")


def functions(sass):
    """{mangled name: [(address, opcode, [operands])]} of a cuobjdump -sass listing."""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        m = INSN.search(line)
        if m and cur is not None:
            ops = [o.strip() for o in m.group(4).split(",")] if m.group(4).strip() else []
            cur.append((int(m.group(1), 16), m.group(3), ops))
    return out


def reads(ops, reg):
    return any(re.fullmatch(r"-?\|?%s\|?(\.reuse)?" % reg, o) for o in ops[1:])


def test_fp32_kernel_sass_keeps_the_power_unfused_and_no_ftz(tmp_path):
    """xcorr_fp32.cu compiled with the Makefile's flags: in every xcorr_fold_fp32_kernel instance each square re^2 / im^2
    is an FMUL whose result an FADD consumes, no FFMA squares a register (a fused power), and every .FTZ instruction lies
    inside the division's called slow path.  In sp_fold_kernel<C128> the sample power squares one component with a DMUL
    and fuses the other into a DFMA (the model's fma(x, x, RN(y^2)))."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    obj = str(tmp_path / "xcorr_fp32.o")
    subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                    "-lineinfo", "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function", "-c",
                    os.path.join(ROOT, "lte-cell-scanner_b200", "csrc", "xcorr_fp32.cu"), "-o", obj], check=True)
    fns = functions(subprocess.run([exe, "-sass", obj], capture_output=True, text=True, check=True).stdout)
    kernels = [k for k in fns if "xcorr_fold_fp32_kernel" in k]
    assert len(kernels) == 6                                        # cf32 / cu8 / c128 x FW 8 / 1
    for k in kernels:
        code = fns[k]
        squares = 0
        for i, (addr, op, ops) in enumerate(code):
            if op.startswith("FFMA"):
                assert ops[1].replace(".reuse", "") != ops[2].replace(".reuse", ""), (k, hex(addr), op, ops)
            if op == "FMUL" and ops[1].replace(".reuse", "") == ops[2].replace(".reuse", ""):
                squares += 1
                user = next(c for c in code[i + 1:] if reads(c[2], ops[0]))
                assert user[1] == "FADD", (k, hex(addr), user)
        assert squares == 42, k                                     # 3 roots x 7 positions x (re^2, im^2)
        calls = [int(ops[0], 16) for _, op, ops in code if op.startswith("CALL.REL")]
        rets = [addr for addr, op, _ in code if op.startswith("RET")]
        assert calls and rets
        lo, hi = min(calls), max(rets)
        ftz = [(hex(a), op) for a, op, _ in code if ".FTZ" in op]
        assert ftz and all(lo <= int(a, 16) <= hi for a, _ in ftz), (k, ftz, hex(lo), hex(hi))
    sp = fns[next(k for k in fns if "sp_fold_kernelILi2E" in k)]

    def square(i, reg):                                             # the last writer of reg before instruction i squares
        op, ops = next(((op, ops) for _, op, ops in reversed(sp[:i]) if ops and ops[0] == reg), (None, None))
        return op == "DMUL" and ops[1] == ops[2]

    fused = [(i, ops) for i, (_, op, ops) in enumerate(sp) if op == "DFMA" and ops[1] == ops[2] != ops[3]]
    assert fused and all(square(i, ops[3]) for i, ops in fused)
    assert not [ops for i, (_, op, ops) in enumerate(sp) if op == "DADD" and square(i, ops[1]) and square(i, ops[2])]


# ---------------------------------------------------------------------------------------------------------------------
# the device against the model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_fp32_templates_bitwise(ctx, name):
    """The plan's FP32 templates equal the model's bit for bit: on a c128 capture that is zero except 1.0 at sample P,
    the drop-in's debug xc (xc_debug_kernel on d_w01 / d_w2) holds xc[t][P - k][f] = (Re W, Im W) of tap k exactly."""
    _, f, fcr, fcp, fs = CASES[name][:5]
    n_cap, P = 10000, 5000
    cap = np.zeros(n_cap, np.complex128)
    cap[P] = 1.0
    xc = ctx.xcorr_pss(cap, f, 2, fcr, fcp, fs, want_incoherent=False, want_xc=True)["xc"]
    k = np.arange(F.N_TAPS)
    dev = xc[:, P - k, :].transpose(2, 0, 1)                        # [n_f][3][137]
    w = F.templates(f, fcr, fcp, fs)[:, :, :F.N_TAPS]
    want = (w[..., 0] + 1j * w[..., 1]).astype(np.complex64)
    bad = np.argwhere(dev.view(np.uint64) != want.view(np.uint64))
    assert not bad.size, "%d template taps differ; first (f, t, tap, device, model): %s" % (
        len(bad), [(int(a), int(b), int(c), complex(dev[a, b, c]), complex(want[a, b, c])) for a, b, c in bad[:6]])


def run_route(ctx, lcs, name, fmt, stack):
    """single [batch][3][n_f][9600] and sp_incoherent [batch][9600] of one call along the case's route."""
    n_cap, f, fcr, fcp, fs, _, route = CASES[name][:7]
    code = {"cu8": lcs.IQ_CU8, "cf32": lcs.IQ_CF32, "c128": lcs.IQ_C128}[fmt]
    batch = stack.shape[0]
    if route == "dropin":
        assert batch == 1
        out = ctx.xcorr_pss(stack[0].view(np.complex128).reshape(-1), f, 2, fcr, fcp, fs, want_incoherent=False)
        return out["single"].transpose(0, 2, 1)[None], out["sp_incoherent"][None]
    plan = ctx.plan(n_cap, f, 2, fcr, fcp, fs, max_batch=batch, kernel=lcs.KERNEL_FP32 if route == "fp32" else lcs.KERNEL_AUTO)
    try:
        if route == "auto_unaligned":
            import torch
            assert plan.kernel_for(code) == lcs.KERNEL_TC                   # an aligned pointer would take the tensor cores
            raw = torch.zeros(stack.nbytes + 16, dtype=torch.uint8, device="cuda")
            raw[2:2 + stack.nbytes] = torch.from_numpy(stack.reshape(-1)).cuda()
            out = run_device(plan, raw, code, batch, inc=False, iq_ptr=raw.data_ptr() + 2)
        else:
            assert plan.kernel_for(code) == lcs.KERNEL_FP32
            out = plan.run_host_np(stack, code)
    finally:
        plan.close()
    return out["single"], out["sp_incoherent"]


@pytest.mark.gpu
@pytest.mark.parametrize("name,fmt", PARAMS, ids=["%s-%s" % p for p in PARAMS])
def test_fp32_single_bitwise(ctx, lcs, name, fmt):
    """Device `single` == the model bit for bit (every position of every hypothesis for n_f <= 9; for more hypotheses every
    position of the edge hypotheses and every hypothesis at POSITIONS), and sp_incoherent == its model, at each batch
    size; the same buffer gives the same bits at every batch position."""
    mod = model(name)
    bufs = buffers(name, fmt, capbuf_cu8() if "capbuf" in CASES[name][7] else None)
    want, first = [], {}
    for buf in bufs:
        x32 = F.samples(buf, fmt)
        if full(mod):
            want.append([(np.arange(mod.n_f), np.arange(F.N_FOLD), mod.single(x32))])
        else:
            fe = edge_hypotheses(mod)
            want.append([(fe, np.arange(F.N_FOLD), mod.single(x32, fs=fe)),
                         (np.arange(mod.n_f), POSITIONS, mod.single(x32, idx=POSITIONS))])
    sp_want = [sp_ref(b, fmt, mod.n_cap) for b in bufs]
    kinds = CASES[name][7].split()
    for batch in CASES[name][8]:
        single, spi = run_route(ctx, lcs, name, fmt, np.stack([bufs[b % len(bufs)] for b in range(batch)]))
        for b in range(batch):
            k = b % len(bufs)
            what = "%s batch %d buffer %d (%s)" % (name, batch, b, kinds[k])
            for fs, idx, w in want[k]:
                msg = mismatches(np.ascontiguousarray(single[b][:, fs][:, :, idx]), w, fs, idx, what)
                assert not msg, msg
            assert np.array_equal(spi[b].view(np.uint64), sp_want[k].view(np.uint64)), \
                "%s sp_incoherent: %d positions differ" % (what, int((spi[b] != sp_want[k]).sum()))
            first.setdefault(k, single[b])
            assert np.array_equal(single[b].view(np.uint32), first[k].view(np.uint32)), what


@pytest.mark.gpu
def test_wider_grid_is_rejected(ctx, lcs):
    """One sample more fold-offset spread than the widest case: the plan is refused with LCS_ERR_RANGE."""
    with pytest.raises(lcs.LcsError, match="error 3: .*too sparse for one shared-memory tile"):
        ctx.plan(153600, np.arange(9) * (WIDE_STEP + 100.0), 2, 100e6, 100e6, FS, kernel=lcs.KERNEL_FP32)
    ctx.plan(153600, np.arange(9) * WIDE_STEP, 2, 100e6, 100e6, FS, kernel=lcs.KERNEL_FP32).close()
