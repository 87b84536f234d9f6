"""The PDCCH decoder's contract (DESIGN.md section 4.13, include/lcs_pdcch.h) restated in float64 numpy on the grid of
test_carrier_meas_host, with the searcher oracle's de-rate-matching, tail-biting Viterbi and CRC16 as the channel code,
checked against DCIs planted by lte_dl_synth's full-bandwidth generator; the DCI sizes and control-region tables against
hand-worked anchors and pdcch_plan.cpp (built with AddressSanitizer); the binding of liblcs_pdcch.so; the kernels'
resources; and the CLI's --pdcch argument errors (no device is touched)."""
import functools
import math
import os
import re
import subprocess

import numpy as np
import pytest

from test_spectrum_host import exported
from test_channelizer_host import cellsearch
from test_carrier_meas_host import FS, OFFSET, S, carrier_grid, found, n_samples, synth_cell, window_starts
from test_pcfich_host import measure_pcfich

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
CSRC = os.path.join(ROOT, "lte-cell-scanner_b200", "csrc")
N_SF = 61
RBS = (6, 15, 25, 50, 75, 100)
D_OF_R = {6: 2, 15: 2, 25: 4, 50: 8, 75: 8, 100: 16}     # the smallest D with 6 R < 64 D
COMMON = lambda r: r in (0xFFFF, 0xFFFE) or 1 <= r <= 60


# ---- the contract, restated -------------------------------------------------------------------------------------------------
def ceil_log2(x):
    return max(0, math.ceil(math.log2(x)))


def sizes(R):
    """Rule 9 from the field widths of 36.212 5.3.3.1.3-4: (1A, 1C)."""
    n_ra = ceil_log2(R * (R + 1) // 2)
    s1a = 1 + 1 + n_ra + 5 + 3 + 1 + 2 + 2            # flag, localized, RIV, MCS, HARQ, NDI, RV, TPC
    if s1a in (12, 14, 16, 20, 24, 26, 32, 40, 44, 56):
        s1a += 1
    gap = {6: 3, 15: 8, 25: 12, 50: 27, 75: 32, 100: 48}[R]                       # 36.211 Table 6.2.3.2-1, N_gap,1
    n = 2 * min(gap, R - gap) // (2 if R < 50 else 4)
    return s1a, (R >= 50) + ceil_log2(n * (n + 1) // 2) + 5


def pdcch_grid(oracle, x, fs_in, fc_in, d, fs_programmed=FS):
    """Y [61][n_max][12 R]: symbols 0 to n_max - 1 of every even slot of the grid of the found-cell dict d."""
    D = int(round(fs_in / FS))
    cell = oracle.new_cell(**{k: v for k, v in d.items() if k not in ("phich_duration", "phich_resource")})
    n_symb = 7 if d["cp_type"] == 1 else 6
    nm = 4 if d["n_rb_dl"] <= 10 else 3
    ts = window_starts(oracle, cell, x.size, D, fs_programmed)
    rows = [2 * s * n_symb + l for s in range(N_SF) for l in range(nm)]
    return carrier_grid(x, fs_in, fc_in, cell, ts[rows], fs_programmed).reshape(N_SF, nm, -1)


def equalise(Y, s, t, nq, n_id, cp, P, R):
    """Rule 7 on quadruplets j < nq of subframe s: u [8 nq], g [8 nq] and sens [8 nq] (|d u_b| <= delta sens_b to first
    order when every grid element errs by at most delta)."""
    n_symb = 7 if cp == 1 else 6
    rs = S.crs_full(n_id, cp, R)
    _, shift = S.O.rs_dl(n_id, cp)
    sl = (2 * s) % 20

    def hhat(p, k):
        sym = 0 if p < 2 else 1
        sh = int(shift[sl * n_symb + sym, p])
        cols = 6 * np.arange(2 * R) + sh
        h = Y[s, sym, cols] * np.conj(rs[sl, sym])
        return np.interp(k, cols, h.real) + 1j * np.interp(k, cols, h.imag)

    u, g, sens = np.zeros(8 * nq), np.zeros(8 * nq), np.zeros(8 * nq)
    for j in range(nq):
        l, k0 = t["pdcch"][t["quad_reg"][j]]
        k = np.array(S.reg_data_cols(l, k0, n_id, P, cp))
        y = Y[s, l, k]
        if P == 1:
            h = hhat(0, k)
            xh, gg = y * np.conj(h) / np.abs(h) ** 2, np.abs(h) ** 2
            se = (1 + np.abs(xh)) / np.abs(h)
        else:
            xh, gg, se = np.zeros(4, complex), np.zeros(4), np.zeros(4)
            for pr in range(2):
                a, b = (0, 1) if P == 2 else ((0, 2) if pr == 0 else (1, 3))
                ha, hb = hhat(a, k[2 * pr:2 * pr + 2]).mean(), hhat(b, k[2 * pr:2 * pr + 2]).mean()
                gp = abs(ha) ** 2 + abs(hb) ** 2
                y0, y1 = y[2 * pr], y[2 * pr + 1]
                xh[2 * pr] = np.sqrt(2) * (np.conj(ha) * y0 + hb * np.conj(y1)) / gp
                xh[2 * pr + 1] = np.sqrt(2) * (np.conj(ha) * y1 - hb * np.conj(y0)) / gp
                gg[2 * pr:2 * pr + 2] = gp
                hs = abs(ha) + abs(hb)
                for n in (2 * pr, 2 * pr + 1):
                    se[n] = (np.sqrt(2) * (abs(y0) + abs(y1) + hs) + 2 * abs(xh[n]) * hs) / gp
        u[8 * j:8 * j + 8] = np.sqrt(2) * np.stack([xh.real, xh.imag], axis=1).reshape(-1)
        g[8 * j:8 * j + 8] = np.repeat(gg, 2)
        sens[8 * j:8 * j + 8] = np.sqrt(2) * np.repeat(se, 2)
    return u, g, sens


def decode_candidate(u, g, c, L, cce, size):
    """Rules 10-11 on one candidate at one size: (rnti, a, q), q None unless the RNTI and format filters pass."""
    E, K = 72 * L, size + 16
    b = slice(72 * cce, 72 * cce + E)
    v = (1 - 2 * c[b]) * u[b] * g[b]
    a = S.O.conv_decode(S.O.deratematch(v, K)).astype(int)
    p = S.O.crc16(a[:size].astype(np.uint8)).astype(int)
    rnti = int(sum((p[i] ^ a[size + i]) << (15 - i) for i in range(16)))
    if not COMMON(rnti):
        return rnti, a, None
    e = S.O.conv_encode(a.astype(np.uint8)).reshape(-1)[S.ratematch_positions(E, K)] ^ c[b]
    return rnti, a, float(np.sum(u[b] * (1 - 2 * e)) / np.sqrt(E * np.sum(u[b] ** 2)))


def candidates(n_cce):
    """Rule 8: (L, first CCE), L = 8 first."""
    return [(8, 8 * m) for m in range(min(2, n_cce // 8))] + [(4, 4 * m) for m in range(min(4, n_cce // 4))]


def measure_pdcch(Y, cfi, n_id, cp, P, R, dur, res):
    """One lcs_pdcch_meas as a dict of rules 1-12 from pdcch_grid's Y and the CFI decisions: per subframe n_ctrl, n_reg,
    n_cce and `dci`, a list of (format, L, cce, rnti, payload, q); beside them `tried`, every candidate with its q (None
    when a filter failed), and the sensitivities of the soft bits for the device's error bound."""
    s1a, s1c = sizes(R)
    out = dict(cfi=np.array(cfi), n_ctrl=[], n_reg=[], n_cce=[], dci=[], tried=[], u=[], sens=[])
    for s in range(N_SF):
        n_ctrl = S.n_ctrl_of(int(cfi[s]), R, dur)
        t = S.control_regs(R, P, cp, n_id, dur, res, n_ctrl)
        nq = min(144, 9 * t["n_cce"])
        u, g, sens = equalise(Y, s, t, nq, n_id, cp, P, R)
        c = S.O.lte_pn((s % 10) * 512 + n_id, 1152).astype(int)
        tried, acc = [], []
        for L, cce in candidates(t["n_cce"]):
            best = None
            for fmt, size in ((1, s1a), (2, s1c)):
                rnti, a, q = decode_candidate(u, g, c, L, cce, size)
                ok = q is not None and q >= 0.8 and (fmt == 2 or a[0] == 1)
                tried.append((fmt, L, cce, rnti, q if (q is not None and (fmt == 2 or a[0] == 1)) else None))
                pay = int("".join(map(str, a[:size])), 2)
                if ok and (best is None or q > best[5]):
                    best = (fmt, L, cce, rnti, pay, q)
            acc.append(best)
        keep = []
        for i, (L, cce) in enumerate(candidates(t["n_cce"])):
            d = acc[i]
            if d is None:
                continue
            if L == 4 and cce // 8 < len(acc) and candidates(t["n_cce"])[cce // 8][0] == 8:
                p = acc[cce // 8]
                if p is not None and p[0] == d[0] and p[3] == d[3] and p[4] == d[4]:
                    continue
            keep.append(d)
        out["n_ctrl"].append(n_ctrl)
        out["n_reg"].append(t["n_reg"])
        out["n_cce"].append(t["n_cce"])
        out["dci"].append(keep)
        out["tried"].append(tried)
        out["u"].append(u)
        out["sens"].append(sens)
    return out


def measure(oracle, x, fs_in, fc_in, d, dur=1, res=1, fs_programmed=FS):
    Y = pdcch_grid(oracle, x, fs_in, fc_in, d, fs_programmed)
    n_id, P = d["n_id_1"] * 3 + d["n_id_2"], d["n_ports"]
    pc = measure_pcfich(Y[:, :2 if P == 4 else 1], n_id, d["cp_type"], P, d["n_rb_dl"])
    return measure_pdcch(Y, pc["cfi"], n_id, d["cp_type"], P, d["n_rb_dl"], dur, res)


# ---- planted DCIs ---------------------------------------------------------------------------------------------------------------
def plant(R, cfi=(3,), n_ports=2, cp=1, dur=1, res=1, nid=137, seed=0):
    """DCIs on a period-4 schedule: L = 8 and L = 4 at every candidate position the smallest control region of the CFI
    schedule holds, 1A and 1C, SI, P and RA RNTIs; an L = 4 DCI beside empty CCEs of its L = 8 candidate; a quiet
    subframe.  (schedule, n_cce of the smallest region)"""
    n_cce = min(S.control_regs(R, n_ports, cp, nid, dur, res, S.n_ctrl_of(c, R, dur))["n_cce"] for c in cfi)
    s1a, s1c = sizes(R)
    rng = np.random.default_rng(seed + R)

    def dci(ph, rnti, fmt, L, cce):
        bits = rng.integers(0, 2, s1a if fmt == "1A" else s1c)
        if fmt == "1A":
            bits[0] = 1
        return ((4, ph), rnti, fmt, L, cce, [int(b) for b in bits])

    want = [dci(0, 0xFFFF, "1A", 8, 0), dci(0, 0xFFFE, "1C", 4, 8), dci(0, 2, "1A", 4, 12),
            dci(1, 0xFFFF, "1C", 8, 8), dci(1, 60, "1C", 4, 0),
            dci(2, 0xFFFF, "1A", 4, 4), dci(2, 0xFFFE, "1A", 4, 12), dci(2, 17, "1C", 4, 8)]
    return [w for w in want if w[4] + w[3] <= n_cce], n_cce


def expected(sched, s):
    """The records rule 12 gives subframe s of a schedule: (format, L, cce, rnti, payload)."""
    got = [(1 if f == "1A" else 2, L, cce, r, int("".join(map(str, b)), 2)) for (p, ph), r, f, L, cce, b in sched if s % p == ph]
    return sorted(got, key=lambda d: (-d[1], d[2]))


def reported(m, s):
    return [d[:5] for d in m["dci"][s]]


def pdcch_cell(nid, n_ports, cp, R, sched, cfi=(3,), dur=1, res=1, fill=None, **kw):
    c = synth_cell(nid, n_ports, cp, R, cfi=cfi, pdcch=sched, **kw)
    c.update(phich_duration=dur, phich_resource=res)
    if fill is not None:
        c["pdcch_fill"] = fill
    return c


@functools.lru_cache(maxsize=None)
def case(R, n_ports=2, cp=1, dur=1, res=1, cfi=(3,), fill=None, snr_db=30.0, seed=0, paths=None, nid=137):
    """(restatement, schedule, found-cell dict) of one cell sending plant()."""
    import lcs_oracle
    sched, _ = plant(R, cfi, n_ports, cp, dur, res, nid)
    kw = dict(paths=[tuple(p) for p in paths]) if paths else {}
    cell = pdcch_cell(nid, n_ports, cp, R, sched, cfi, dur, res, fill, **kw)
    D = D_OF_R[R]
    x, _ = S.synth_wide_full(n_samples(D), D * FS, 739e6, [(739e6, [cell])], snr_db, seed)
    d = found(cell, 739e6)
    return measure(lcs_oracle, x, D * FS, 739e6, d, dur, res), sched, d


def assert_exact(m, sched, what):
    for s in range(N_SF):
        assert reported(m, s) == expected(sched, s), (what, s, reported(m, s), expected(sched, s))
        for d in m["dci"][s]:
            assert d[5] > 0.9, (what, s, d)


# ---- tables --------------------------------------------------------------------------------------------------------------------
PLAN_DRIVER = r"""
#include <cstdio>
#include "pdcch_plan.hpp"
using namespace lcs::pdcch;
int main() {
  const int rbs[] = {6, 15, 25, 50, 75, 100}, ports[] = {1, 2, 4}, ids[] = {0, 1, 137, 250, 503};
  std::vector<CtrlTable> keep;
  int bad_riv = 0;
  for (int R : rbs) {
    std::printf("S %d %d %d\n", R, size_1a(R), size_1c(R));
    for (int st = 0; st < R; st++)
      for (int len = 1; st + len <= R; len++) {
        int a, b;
        if (!riv_decode(R, riv_encode(R, st, len), a, b) || a != st || b != len) bad_riv++;
      }
    for (int P : ports) for (int cp = 1; cp <= 2; cp++) for (int dur = 1; dur <= 2; dur++) for (int res = 1; res <= 4; res++)
      for (int nid : ids) for (int n = (dur == 2 ? 3 : 1); n <= (R <= 10 ? 4 : 3); n++) {
        const CtrlTable t = control_table(R, P, cp, nid, dur, res, n);
        std::printf("T %d %d %d %d %d %d %d %d %d", R, P, cp, dur, res, nid, n, t.n_reg, t.n_cce);
        for (uint16_t q : t.quad) std::printf(" %d", (int)q);
        std::printf("\n");
        keep.push_back(t);
      }
  }
  std::printf("R %d\n", bad_riv);
  return 0;
}
"""


@pytest.fixture(scope="module")
def plan_out(lcs, tmp_path_factory):
    """pdcch_plan.cpp's sizes, RIV round trips and tables of every configuration, built with AddressSanitizer."""
    tmp = tmp_path_factory.mktemp("pdcch_plan")
    src = tmp / "plan.cpp"
    src.write_text(PLAN_DRIVER)
    exe = str(tmp / "plan")
    libdir = os.path.dirname(lcs.LIB_PATH)
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address", "-fno-omit-frame-pointer", "-I" + CSRC,
                           "-I/usr/local/cuda/include", str(src), os.path.join(CSRC, "pdcch_plan.cpp"),
                           os.path.join(CSRC, "carrier_plan.cpp"), "-o", exe, "-L" + libdir, "-llcs_b200",
                           "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1")
    r = subprocess.run([exe], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout.splitlines()


def test_dci_sizes(plan_out):
    """Rule 9's tables, the field widths of 36.212 and pdcch_plan.cpp agree."""
    t1a = dict(zip(RBS, (21, 22, 25, 27, 27, 28)))
    t1c = dict(zip(RBS, (8, 10, 12, 13, 14, 15)))
    got = {int(l.split()[1]): tuple(map(int, l.split()[2:])) for l in plan_out if l.startswith("S ")}
    for R in RBS:
        assert sizes(R) == (t1a[R], t1c[R]) == got[R] == (S.DCI_SIZES_1A[R], S.DCI_SIZES_1C[R]), R


@pytest.mark.parametrize("R,P,cp,res,cfi,want", [
    (100, 2, 1, 3, 3, 84), (100, 2, 1, 1, 3, 87), (100, 4, 1, 3, 3, 73), (100, 2, 1, 3, 1, 17),
    (50, 2, 1, 3, 3, 41), (25, 2, 1, 3, 3, 20), (6, 2, 1, 3, 3, 6), (6, 2, 2, 3, 3, 5)])
def test_cce_counts_against_hand_worked_anchors(plan_out, R, P, cp, res, cfi, want):
    """Rules 2-5 worked by hand (normal PHICH duration): e.g. 20 MHz, N_g = 1: symbol 0 has 200 - 4 - 3 x 13 REGs, symbols
    1 and 2 300 each, 757 REGs, 84 CCEs."""
    n = S.n_ctrl_of(cfi, R, 1)
    assert S.control_regs(R, P, cp, 137, 1, res, n)["n_cce"] == want
    line = [l for l in plan_out if l.startswith("T %d %d %d 1 %d 137 %d " % (R, P, cp, res, n))]
    assert len(line) == 1 and int(line[0].split()[9]) == want


def test_reg_tables(plan_out):
    """For every R, port count, CP, N_g, duration, n_ctrl and five cell ids: the PCFICH, PHICH and PDCCH REGs are
    disjoint and tile the control region, the quadruplet map is a bijection, and pdcch_plan.cpp equals the restatement."""
    n = 0
    for line in plan_out:
        if not line.startswith("T "):
            continue
        v = list(map(int, line.split()[1:]))
        R, P, cp, dur, res, nid, n_ctrl, n_reg, n_cce = v[:9]
        t = S.control_regs(R, P, cp, nid, dur, res, n_ctrl)
        regs = t["pdcch"]
        cover = [(l, k) for l, k in t["pcfich"] | t["phich"] if l < n_ctrl] + regs
        assert len(cover) == len(set(cover)), v[:9]
        res_cover = sorted((l, k0 + o) for l, k0 in cover for o in range(6 if S.reg_is_six(l, P, cp) else 4))
        assert res_cover == [(l, k) for l in range(n_ctrl) for k in range(12 * R)], v[:9]
        assert len(t["phich"]) == 3 * -(-{1: 1, 2: 3, 3: 6, 4: 12}[res] * R // 48), v[:9]
        assert sorted(t["quad_reg"]) == list(range(len(regs))), v[:9]
        quads = [(l << 12) | k for l, k in (regs[t["quad_reg"][j]] for j in range(min(144, 9 * t["n_cce"])))]
        assert (n_reg, n_cce, v[9:]) == (t["n_reg"], t["n_cce"], quads), v[:9]
        n += 1
    assert n == 3 * 2 * 4 * 5 * (6 + 5 * 4)          # n_ctrl 1-4 and 3-4 at R = 6, 1-3 and 3 otherwise


def test_riv_round_trips(plan_out):
    assert plan_out[-1] == "R 0"


def test_scrambling_words():
    """c of rule 10 from 36.211 7.2's recursions, independently of lte_pn."""
    from test_pcfich_host import gold
    for n_id in (0, 137, 503):
        for u in (0, 5, 9):
            assert np.array_equal(S.O.lte_pn(u * 512 + n_id, 1152).astype(int), gold(u * 512 + n_id, 1152))


# ---- planted DCIs ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", RBS)
def test_every_bandwidth_decodes_exactly(oracle, R):
    m, sched, _ = case(R)
    assert len(sched) == {6: 1, 15: 5}.get(R, 8)
    assert_exact(m, sched, R)


@pytest.mark.parametrize("n_ports,cp,R,dur,res,cfi,fill", [
    (1, 1, 25, 1, 1, (3,), None), (1, 2, 15, 2, 2, (3, 2), 5), (2, 2, 50, 1, 4, (2, 3), None), (4, 1, 50, 2, 3, (3,), 6),
    (4, 2, 6, 1, 2, (3,), 7), (2, 1, 75, 2, 1, (1, 2, 3), 8), (4, 1, 100, 1, 3, (2,), None), (2, 1, 6, 2, 4, (2, 3), 9)])
def test_ports_cp_phich_and_fill(oracle, n_ports, cp, R, dur, res, cfi, fill):
    """1, 2 and 4 ports with unequal gains, both CPs, all four N_g and both durations, changing CFIs, NIL or random
    filled control regions."""
    m, sched, _ = case(R, n_ports, cp, dur, res, cfi, fill)
    assert sched
    assert_exact(m, sched, (n_ports, cp, R, dur, res, cfi, fill))


def test_two_path_channel(oracle):
    m, sched, _ = case(50, 2, paths=((0.0, 1.0), (1.5e-6, 0.6 * np.exp(1j))))
    assert_exact(m, sched, "two paths")


def test_clock_offset_cell(oracle):
    """The clock-offset case of the PCFICH tests."""
    o = OFFSET
    sched, _ = plant(25)
    cell = pdcch_cell(137, 2, 1, 25, sched, t0=o["t0"])
    x, _ = S.synth_wide_offset(o["D"] * (1300 + 122 * 960 + 400), o["D"] * FS, 739e6, o["fc_c"], cell, o["clock_ratio"],
                               o["f_res"], 30.0, 0)
    d = found(cell, o["fc_c"])
    d.update(fc_programmed=(o["fc_c"] - o["f_res"]) / o["clock_ratio"], freq=o["f_res"], freq_fine=o["f_res"],
             freq_superfine=o["f_res"], frame_start=o["t0"] * o["clock_ratio"])
    assert_exact(measure(oracle, x, o["D"] * FS, 739e6, d), sched, "clock offset")


def test_duplicates_are_reported_once(oracle):
    """A true L = 8 DCI also decodes as the L = 4 candidate on its first half: reported once, at L = 8.  A true L = 4 DCI
    beside NIL CCEs also decodes as the L = 8 candidate holding it, with q <= 1/sqrt(2): reported once, at L = 4."""
    m, sched, _ = case(50)
    for s in range(0, N_SF, 4):
        t = {(f, L, c): q for f, L, c, r, q in m["tried"][s]}
        assert t[(1, 4, 0)] is not None and t[(1, 4, 0)] > 0.9          # the SI 1A at L = 8, seen at L = 4
        assert [d[1:3] for d in m["dci"][s]].count((8, 0)) == 1 and (4, 0) not in [d[1:3] for d in m["dci"][s]]
    for s in range(1, N_SF, 4):
        t = {(f, L, c): q for f, L, c, r, q in m["tried"][s]}
        assert t[(2, 8, 0)] is not None and t[(2, 8, 0)] <= 1 / np.sqrt(2) + 0.01   # the RA 1C at L = 4, seen at L = 8
        assert (8, 0) not in [d[1:3] for d in m["dci"][s]] and (4, 0) in [d[1:3] for d in m["dci"][s]]


@pytest.mark.parametrize("n_ports", [1, 2, 4])
def test_low_snr(oracle, n_ports):
    """At 3 dB per RE over a random-filled control region, q of a planted DCI falls to about 0.65, below the threshold:
    every planted DCI still decodes to its RNTI (the Viterbi and CRC hold), every decision whose q is 0.02 or more from
    0.8 is the threshold's, and nothing unplanted is reported."""
    m, sched, _ = case(25, n_ports, snr_db=3.0, seed=4, fill=3)
    n_clear = 0
    for s in range(N_SF):
        want, got = expected(sched, s), reported(m, s)
        assert set(got) <= set(want), (s, got, want)
        t = {(f, L, c): (r, q) for f, L, c, r, q in m["tried"][s]}
        for d in want:
            r, q = t[(d[0], d[1], d[2])]
            assert r == d[3] and q is not None, (s, d, r)
            if abs(q - 0.8) >= 0.02:
                assert (d in got) == (q >= 0.8), (s, d, q)
                n_clear += 1
    assert n_clear > 100


def test_a_cell_without_pdcch_is_unchanged():
    """A cell without "pdcch" gives the same recording as before; one with it changes only its control region."""
    a = synth_cell(137, 2, 1, 6, cfi=(3,))
    sched, _ = plant(6)
    b = pdcch_cell(137, 2, 1, 6, sched)
    ga, _ = S._grid_full(a, 7, np.random.default_rng(1))
    gb, _ = S._grid_full(b, 7, np.random.default_rng(1))
    ctrl = np.zeros(ga.shape[1], bool)
    for u in range(ga.shape[1] // 14):
        ctrl[14 * u:14 * u + 4] = True
    assert np.array_equal(ga[:, ~ctrl], gb[:, ~ctrl]) and not np.array_equal(ga, gb)
    gc, _ = S._grid_full(pdcch_cell(137, 2, 1, 6, sched, fill=3), 7, np.random.default_rng(1))   # its own random stream
    assert np.array_equal(ga[:, ~ctrl], gc[:, ~ctrl]) and not np.array_equal(gb, gc)


# ---- the kernels' resources -----------------------------------------------------------------------------------------------------
def test_pdcch_kernels_compile_without_spills(tmp_path):
    """Every kernel of pdcch.cu compiles for sm_90a with no stack frame and no spills (DESIGN.md section 4.13)."""
    r = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c", os.path.join(CSRC, "pdcch.cu"), "-o",
                        str(tmp_path / "pdcch.o")], capture_output=True, text=True, check=True)
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 6 and len(frames) == 6, r.stderr          # the grid kernel in four formats, PCFICH, PDCCH
    assert sum("carrier_grid_kernel" in e for e in entries) == 4 and sum("pdcch_kernel" in e for e in entries) == 1
    assert all(f == ("0", "0", "0") for f in frames), r.stderr


# ---- binding -------------------------------------------------------------------------------------------------------------------
LAYOUT_DRIVER = r"""
#include <stddef.h>
#include <stdio.h>
#include "lcs_pdcch.h"
#define F(f) printf(#f " %zu\n", offsetof(lcs_pdcch_meas, f));
#define G(f) printf("dci." #f " %zu\n", offsetof(lcs_pdcch_dci, f));
int main(void) {
  printf("size %zu\n", sizeof(lcs_pdcch_meas));
  printf("dci.size %zu\n", sizeof(lcs_pdcch_dci));
  F(dci) F(cfi) F(n_ctrl) F(n_reg) F(n_cce) F(n_dci) F(count) F(si_subframes) F(n_subframes)
  G(quality) G(payload) G(format) G(agg) G(cce) G(rnti) G(n_bits) G(riv) G(rb_start) G(n_rb) G(localized) G(mcs) G(harq)
  G(ndi) G(rv) G(tpc) G(gap) G(tbs_index)
  printf("consts %d %d %d %d %d %d %d %d\n", LCS_PDCCH_CHUNK, LCS_PDCCH_LAUNCHES_PER_CHUNK, LCS_PDCCH_SUBFRAMES,
         LCS_PDCCH_MAX_DCI, LCS_DCI_1A, LCS_DCI_1C, LCS_RNTI_SI, LCS_RNTI_P);
  return 0;
}
"""


def test_pdcch_prototypes_cover_header_and_library(lcs, tmp_path):
    """liblcs_pdcch.so exports exactly the four functions of include/lcs_pdcch.h, all bound with the header's
    prototypes; the other libraries export none of them.  PDCCH_MEAS and PDCCH_DCI have the C layout."""
    import ctypes as C
    header = re.sub(r"/\*.*?\*/", " ", open(lcs.PDCCH_HEADER).read(), flags=re.S)
    names = set(re.findall(r"\b(lcs_\w+)\s*\(", header))
    assert names == {"lcs_pdcch_create", "lcs_pdcch_destroy", "lcs_pdcch_cells", "lcs_pdcch_timing_read"}
    assert set(lcs.prototypes(lcs.PDCCH_HEADER)) == names
    assert exported(lcs.PDCCH_LIB_PATH) == names
    for other in (lcs.LIB_PATH, lcs.MEAS_LIB_PATH, lcs.PSD_LIB_PATH, lcs.CARRIER_LIB_PATH, lcs.CIR_LIB_PATH,
                  lcs.PCFICH_LIB_PATH):
        assert not exported(other) & names
    l = lcs.pdcch_lib()
    V, I, U, D = C.c_void_p, C.c_int, C.c_uint32, C.c_double
    assert l.lcs_pdcch_cells.argtypes == [V, V, I, I, C.c_uint64, D, D, V, U, D, V]
    assert l.lcs_pdcch_create.argtypes == [V, V] and l.lcs_pdcch_timing_read.argtypes == [V, V, V]
    assert l.lcs_pdcch_destroy.restype is None
    src = tmp_path / "layout.c"
    src.write_text(LAYOUT_DRIVER)
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = dict(line.split(" ", 1) for line in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(got["size"]) == lcs.PDCCH_MEAS.itemsize and int(got["dci.size"]) == lcs.PDCCH_DCI.itemsize
    for f in lcs.PDCCH_MEAS.names:
        assert int(got[f]) == lcs.PDCCH_MEAS.fields[f][1], f
    for f in lcs.PDCCH_DCI.names:
        assert int(got["dci." + f]) == lcs.PDCCH_DCI.fields[f][1], f
    assert tuple(map(int, got["consts"].split())) == (lcs.PDCCH_CHUNK, 3, lcs.PDCCH_SUBFRAMES, lcs.PDCCH_MAX_DCI,
                                                      lcs.DCI_1A, lcs.DCI_1C, lcs.RNTI_SI, lcs.RNTI_P) == \
        (32, 3, N_SF, 6, 1, 2, 0xFFFF, 0xFFFE)


# ---- CLI argument errors with --pdcch (no device is touched) ------------------------------------------------------------------
def test_cli_pdcch_argument_errors(lcs, tmp_path):
    f = str(tmp_path / "rec.ci16")
    np.zeros((1000, 2), np.int16).tofile(f)
    wide = ["--wideband", f, "--fc-in", "739e6", "-s", "739e6"]
    cases = [
        (["-s", "739e6", "-l", "-d", str(tmp_path), "--pdcch"], "--pdcch needs --wideband"),
        (wide + ["--fs-in", "7.68e6", "--pdcch-csv", str(tmp_path / "c.csv")], "--pdcch-csv needs --pdcch"),
        (["--wideband", f, "--fc-in", "739e6", "--fs-in", "10e6", "--spectrum", str(tmp_path / "p.csv"), "--pdcch"],
         "--pdcch needs a search (-s)"),
        (wide + ["--fs-in", "11.52e6", "--pdcch"], "--pdcch needs --fs-in = D * 1.92 MHz"),
        (wide + ["--fs-in", "10e6", "--resample", "--pdcch"], "--pdcch needs --fs-in = D * 1.92 MHz"),
        (wide + ["--fs-in", "7.68e6", "--pdcch"], "holds 1000 ci16 samples"),
    ]
    for args, msg in cases:
        out = cellsearch(*args)
        assert out.returncode != 0 and msg in out.stderr, (args, out.stderr)
        assert "lcs_ctx_create" not in out.stderr
