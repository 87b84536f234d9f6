"""A bit-exact numpy model of the tensor-core correlator's xc_incoherent_single for 8-bit IQ (xcorr_tc.cu, planset.cu).

Everything the kernel does before its float steps is integer arithmetic, and the float steps are a fixed sequence of
correctly rounded float32 operations, so `single` is determined to the last bit:
- templates: W = conj(fshift(pss_td))/137 in double, llrint(W * S) with S the context's power of two, three balanced
  base-256 digits per component, constants corr = float(sum(a) - MAGIC_VAL) (plan_build_kernel, lcs_ctx_create);
- per lag and part: integer accumulators a0, a1, a2 of the digit planes against v - 128 (re) and (Q', ~I') (im);
- x = RN(RN(fma(float(a0*256 + a1), 256, MAGIC_VAL + a2)) + corr), rr = fma(x_im, x_im, RN(x_re^2));
- the fold: rr of the n_comb half frames added into a float32 window in the kernel's order, then * inv2s (exact) and / n_comb
  (launch_xcorr_fold_tc's reciprocal sequence for the divisors it proves exact, the IEEE quotient otherwise).

The work decomposition (TcRunIter) is restated once here and used both by the model's fold order and by the CPU check that
every fold position is produced exactly once."""
import math

import numpy as np

NT, HALO, N_FOLD, M_MAX = 256, 32, 9600, 24
MAGIC_VAL = 12582912.0
N_TAPS = 137
EXACT_RCP = (1, 2, 3, 4, 5, 7, 8, 9, 11, 13, 15, 16, 17, 19, 21, 23)     # kExactRcp of launch_xcorr_fold_tc


# ---------------------------------------------------------------------------------------------------------------------
# plan geometry (planset.cu)
# ---------------------------------------------------------------------------------------------------------------------
def pick_layout(n_f):
    """(C, J, n_pass) of pick_layout."""
    if n_f <= 5:
        return 16, 1, 1
    if n_f <= 16:
        return 24, 2, 1
    if n_f <= 21:
        return 32, 2, 1
    if n_f <= 32:
        return 48, 2, 1
    if n_f <= 42:
        return 32, 2, 2
    return 48, 2, (n_f + 31) // 32


def n_comb_xc(n_cap):
    return (n_cap - 136 - 100) // N_FOLD


def fold_offsets(f, fc_req, fc_prog, fs_prog, n_comb):
    """off[m][f] = round_i(m * .005 * k_factor * fs) as int64 (planset_build)."""
    off = np.empty((n_comb, len(f)), np.int64)
    for j, fo in enumerate(f):
        k_factor = (fc_req - fo) / fc_prog
        for m in range(n_comb):
            off[m, j] = int(np.rint(m * .005 * k_factor * fs_prog))
    return off


def passes(n_f):
    """[(f0, f1)] hypotheses of each pass."""
    _, _, n_pass = pick_layout(n_f)
    hpp = -(-n_f // n_pass)
    return [(p * hpp, min(n_f, (p + 1) * hpp)) for p in range(n_pass)]


def pass_start(off):
    """smin[m] of one pass (off [n_comb][hypotheses of the pass]): the staging start of half frame m.  It follows the
    smallest step of the fold offsets from one half frame to the next, so dsh = off - smin is non-negative and
    non-decreasing in m for every column."""
    step = np.diff(off, axis=0).min(axis=1)
    return np.concatenate([off[:1].min(axis=1), off[0].min() + np.cumsum(step)])


def dsh_table(off, n_f):
    """dsh [n_comb][n_f] (per column = per hypothesis; the three roots share it), and whether every pass fits the halo."""
    dsh = np.zeros_like(off)
    for f0, f1 in passes(n_f):
        dsh[:, f0:f1] = off[:, f0:f1] - pass_start(off[:, f0:f1])[:, None]
    return dsh, bool((dsh >= 0).all() and dsh.max() <= HALO)


# ---------------------------------------------------------------------------------------------------------------------
# work decomposition (launch_xcorr_fold_tc + TcRunIter)
# ---------------------------------------------------------------------------------------------------------------------
def tc_plan(n_units, n_sm):
    """(tu, t_cta): tiles per unit and per CTA."""
    tu = (N_FOLD + HALO + NT - 1) // NT
    while True:
        t_cta = (n_units * tu + n_sm - 1) // n_sm
        runs = (tu + t_cta - 1) // t_cta + 1
        if NT * tu - HALO * runs >= N_FOLD:
            return tu, t_cta
        tu += 1


def tc_runs(n_units, n_sm):
    """Every run of the launch as (cta, unit, p0, p1, n_tiles, tiles given): CTA i walks tiles [i t_cta, (i+1) t_cta) of the
    sequence [unit][tu]; a run of T tiles yields 256 T - 32 fold positions."""
    tu, t_cta = tc_plan(n_units, n_sm)
    total = n_units * tu
    out = []
    for cta in range((total + t_cta - 1) // t_cta):
        t, t_end = cta * t_cta, min((cta + 1) * t_cta, total)
        while t < t_end:
            u = t // tu
            base = u * tu
            a = t - base
            e = min(t_end, base + tu)
            bb = e - base
            nb = (base + a) // t_cta - base // t_cta
            t = e
            p0 = NT * a - HALO * nb
            if p0 >= N_FOLD:
                continue
            p1 = min(NT * bb - HALO * (nb + 1), N_FOLD)
            out.append((cta, u, p0, p1, min(bb - a, (p1 - p0 + HALO + NT - 1) // NT), bb - a))
    return out


def run_starts(n_units, n_sm):
    """p0 of the run that produces each fold position: int64 [n_units][9600]."""
    p0 = np.full((n_units, N_FOLD), -1, np.int64)
    for _, u, a, b, _, _ in tc_runs(n_units, n_sm):
        p0[u, a:b] = a
    assert (p0 >= 0).all()
    return p0


# ---------------------------------------------------------------------------------------------------------------------
# templates (lte_tables.cpp pss_td, lcs_ctx_create's scale, plan_build_kernel)
# ---------------------------------------------------------------------------------------------------------------------
def pss_td():
    """The library's time-domain PSS [3][137]: direct inverse DFT in double with exact argument reduction."""
    out = np.empty((3, N_TAPS), np.complex128)
    for t, root in enumerate((25, 29, 34)):
        fd = []
        for n in range(63):
            if n != 31:
                ph = -math.pi * root * float(n * (n + 1)) / 63.0
                fd.append(complex(math.cos(ph), math.sin(ph)))
        X = [0j] * 128
        for i in range(31):
            X[1 + i] = fd[31 + i]
            X[97 + i] = fd[i]
        sc = math.sqrt(128.0) * math.sqrt(128.0 / 62.0) / 128.0
        td = []
        for n in range(128):
            s = 0j
            for k in range(128):
                if X[k] != 0:
                    ph = 2 * math.pi * ((n * k) & 127) / 128.0
                    s += X[k] * complex(math.cos(ph), math.sin(ph))
            td.append(complex(s.real * sc, s.imag * sc))
        out[t] = td[119:] + td
    return out


def tc_scale(td):
    """S: the largest power of two with |template component| * S <= 127*65536 + 127*256 + 127."""
    maxmag = max(abs(complex(v)) / 137.0 for v in td.reshape(-1))
    limit = 127.0 * 65536 + 127 * 256 + 127
    ex = math.floor(math.log2(limit / maxmag))
    while math.ldexp(maxmag, ex) > limit:
        ex -= 1
    return math.ldexp(1.0, ex)


def balanced_digits(v):
    d2 = ((v + 128) % 256) - 128
    r1 = (v - d2) // 256
    d1 = ((r1 + 128) % 256) - 128
    return (r1 - d1) // 256, d1, d2


def templates(td, S, f, fc_req, fc_prog, fs_prog):
    """Integer template rows a [n_f][3][274] (a[2 tap] = round(Re W * S), a[2 tap + 1] = -round(Im W * S)) and the
    constants corr_re, corr_im [n_f][3] float32 with -MAGIC_VAL folded in."""
    tap = np.arange(N_TAPS, dtype=np.float64)
    a = np.empty((len(f), 3, 2 * N_TAPS), np.int64)
    for j, fo in enumerate(f):
        k_factor = (fc_req - fo) / fc_prog
        k = (math.pi * fo) / ((fs_prog * k_factor) / 2.0)
        ph = k * tap
        cs, sn = np.cos(ph), np.sin(ph)
        re = td.real * cs - td.imag * sn
        im = td.real * sn + td.imag * cs
        a[j, :, 0::2] = np.rint((re / 137.0) * S).astype(np.int64)
        a[j, :, 1::2] = -np.rint((-im / 137.0) * S).astype(np.int64)
    c_re = (a.sum(axis=2).astype(np.float64) - MAGIC_VAL).astype(np.float32)
    c_im = (a[:, :, 0::2].sum(axis=2).astype(np.float64) - MAGIC_VAL).astype(np.float32)
    d0, _, d2 = balanced_digits(a)
    assert d0.min() >= -128 and d0.max() <= 127, "template digits outside int8"
    assert (np.abs(d2).sum(axis=2) * 128 < 2 ** 22).all(), "low digit plane outside the exact magic-number range"
    return a, c_re, c_im


# ---------------------------------------------------------------------------------------------------------------------
# float32 steps
# ---------------------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """RN_float32(a * b + c) for float32 arrays with one rounding: the product is exact in float64, the sum is
    float64 + TwoSum error, and a float64 sum that lies exactly between two float32 values (normal or subnormal) is
    resolved by the error's sign."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c = c.astype(np.float64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    d = s - r.astype(np.float64)                                   # exact: s and r are within one float32 step
    other = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)))
    tie = (d != 0) & (e != 0) & (2 * d == other.astype(np.float64) - r.astype(np.float64))
    if tie.any():
        r[tie] = np.where((e[tie] > 0) == (d[tie] > 0), other[tie], r[tie])
    return r


def lag_values(cu8, a, c_re, c_im, n_lag):
    """x_re, x_im [n_f][3][n_lag] float32: recombined correlation at every lag, as the epilogue computes it."""
    z = cu8.reshape(-1).astype(np.int64)
    xs = (z - 128).astype(np.float32)
    ys = np.empty_like(xs)
    ys[0::2] = xs[1::2]
    ys[1::2] = -xs[0::2] - 1
    L = 2 * N_TAPS
    d = np.stack(balanced_digits(a.reshape(-1, L)), axis=0)                # [3 digits][cols][274]
    assert np.abs(d).max() <= 128
    out = []
    for s in (xs, ys):
        H = np.lib.stride_tricks.as_strided(s, shape=(n_lag, L), strides=(2 * s.itemsize, s.itemsize))
        # every partial sum is an integer of magnitude <= 274 * 128 * 128 < 2^24: float32 GEMM is exact in any order
        acc = [np.rint(H @ d[j].T.astype(np.float32)).astype(np.int64).T for j in range(3)]   # [cols][n_lag]
        out.append(acc)
    x = []
    for (a0, a1, a2), kk in zip(out, (c_re.reshape(-1), c_im.reshape(-1))):
        t = a0 * 256 + a1
        assert np.abs(t).max() < 2 ** 31 and np.abs(a2).max() < 2 ** 22
        f2 = (a2 + 12582912).astype(np.float32)                             # MAGIC_BITS + a2 reinterpreted: exact
        v = t.astype(np.float32) * np.float32(256) + f2                      # fma(float(t), 256, f2): the product is exact
        x.append((v + kk[:, None]).reshape(a.shape[0], 3, n_lag))
    return x[0], x[1]


def power(x_re, x_im):
    return fma32(x_im, x_im, x_re * x_re)


def divide(x, n):
    """x / n in launch_xcorr_fold_tc's write-out rule."""
    n32 = np.float32(n)
    if n in EXACT_RCP:
        r = np.float32(1.0) / n32
        q = x * r
        return fma32(fma32(np.full_like(q, -n32), q, x), np.full_like(q, r), q)
    return x / n32


# ---------------------------------------------------------------------------------------------------------------------
# the whole correlator
# ---------------------------------------------------------------------------------------------------------------------
class TcModel:
    """Templates, fold offsets and scale of one plan (f, fc_requested, fc_programmed, fs_programmed, n_cap)."""

    _td = None

    def __init__(self, n_cap, f, fc_req, fc_prog, fs_prog):
        if TcModel._td is None:
            TcModel._td = pss_td()
        self.n_cap, self.f = n_cap, np.asarray(f, np.float64)
        self.n_comb = n_comb_xc(n_cap)
        assert 1 <= self.n_comb <= M_MAX
        self.S = tc_scale(TcModel._td)
        self.a, self.c_re, self.c_im = templates(TcModel._td, self.S, self.f, fc_req, fc_prog, fs_prog)
        self.off = fold_offsets(self.f, fc_req, fc_prog, fs_prog, self.n_comb)
        self.dsh, self.fits = dsh_table(self.off, len(self.f))
        self.n_pass = pick_layout(len(self.f))[2]
        inv = np.float32(1.0 / (self.S * 128.0))
        self.inv2s = inv * inv

    def powers(self, cu8):
        """rr [n_comb][n_f][3][9600]: |xc|^2 of half frame m at fold position p (lag p + off[m][f])."""
        n_lag = int(self.off.max()) + N_FOLD
        p = np.arange(N_FOLD)
        out = np.empty((self.n_comb, len(self.f), 3, N_FOLD), np.float32)
        for j0 in range(0, len(self.f), 8):
            j1 = min(len(self.f), j0 + 8)
            x_re, x_im = lag_values(cu8, self.a[j0:j1], self.c_re[j0:j1], self.c_im[j0:j1], n_lag)
            rr = power(x_re, x_im)
            for m in range(self.n_comb):
                for j in range(j0, j1):
                    out[m, j] = rr[j - j0][:, p + self.off[m, j]]
        return out

    def fold(self, rr, p0=None):
        """single [3][n_f][9600] from rr.  p0 [n_f][9600] are the starts of the runs that produce each position of each
        hypothesis (its pass' unit): the kernel adds the half frames of a position in (tile, m) order, where half frame m
        of position p lands in tile (p - p0 + dsh[m]) // 256 of its run.  p0 = None adds them in ascending m, the
        reference's order."""
        acc = np.zeros(rr.shape[1:], np.float32)
        if p0 is None:
            for m in range(self.n_comb):
                acc = acc + rr[m]
        else:
            late = ((np.arange(N_FOLD) - p0) % NT)[None] + self.dsh[:, :, None] >= NT    # [n_comb][n_f][9600]
            for second in (False, True):
                for m in range(self.n_comb):
                    sel = (late[m] == second)[:, None, :]
                    acc = np.where(sel, acc + rr[m], acc)
        return divide(acc * self.inv2s, self.n_comb).transpose(1, 0, 2)

    def run_starts(self, batch, n_sm, b):
        """p0 [n_f][9600] of buffer b in a single-plan launch of `batch` buffers (unit = pass * batch + buffer)."""
        starts = run_starts(batch * self.n_pass, n_sm)
        p0 = np.empty((len(self.f), N_FOLD), np.int64)
        for i, (f0, f1) in enumerate(passes(len(self.f))):
            p0[f0:f1] = starts[i * batch + b]
        return p0

    def single(self, cu8, p0=None):
        return self.fold(self.powers(cu8), p0)
