"""The SIB1 decoder's rules (DESIGN.md section 4.14, include/lcs_sib1.h) restated in numpy: the transport block sizes, the
QPP interleaver, the VRB-to-PRB map and the circular buffer of sib1_rules.hpp and the SIB1 parser of sib1_plan.cpp (built
with AddressSanitizer) against lte_dl_synth's own restatement; the turbo code through a float64 max-log-MAP decoder on the
schedule of rule 8; the data REs of rule 5; and the binding of liblcs_sib1.so (no device is touched)."""
import os
import subprocess

import numpy as np
import pytest

from test_carrier_meas_host import FS, S, carrier_grid, found, n_samples, synth_cell, window_starts
from test_spectrum_host import exported

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
CSRC = os.path.join(ROOT, "lte-cell-scanner_b200", "csrc")
RBS = (6, 15, 25, 50, 75, 100)


# ---- rule 8, restated: max-log-MAP in float64 on windows of 32 steps --------------------------------------------------------
def _trellis():
    """For state s = (d1 d2 d3) and input u: (next state, parity)."""
    nxt, par = np.zeros((8, 2), int), np.zeros((8, 2), int)
    for s in range(8):
        d1, d2, d3 = (s >> 2) & 1, (s >> 1) & 1, s & 1
        for u in range(2):
            a = u ^ d2 ^ d3
            nxt[s, u], par[s, u] = (a << 2) | (d1 << 1) | d2, a ^ d1 ^ d3
    return nxt, par


def gam(u, z, lsa, lp):
    return (np.where(u, -lsa, lsa) + np.where(z, -lp, lp)) * 0.5


def turbo_decode(d, K, F, max_iter=8, win=32):
    """Rule 8 on soft inputs d [3][K + 4]: (bits [K], crc_ok, iterations)."""
    f1, f2 = S.qpp_table()[S.turbo_sizes().index(K)]
    pi = (f1 * np.arange(K) + f2 * (np.arange(K) ** 2 % K)) % K
    nxt, par = _trellis()
    nw = -(-K // win)
    beta_k = []
    for dec in range(2):
        t = K + 2 * dec
        xs, zs = [d[0, t], d[2, t], d[1, t + 1]], [d[1, t], d[0, t + 1], d[2, t + 1]]
        b = np.zeros(8)
        for s in range(8):
            sa, us, zz = s, [], []
            for j in range(3):
                a1, a2, a3 = (sa >> 2) & 1, (sa >> 1) & 1, sa & 1
                us.append(a2 ^ a3)
                zz.append(a1 ^ a3)
                sa = (a1 << 1) | a2
            acc = 0.0
            for j in (2, 1, 0):
                acc = float(gam(us[j], zz[j], xs[j], zs[j])) + acc
            b[s] = acc
        beta_k.append(b)
    ext = np.zeros((2, K))
    ab, bb = np.zeros((2, nw + 1, 8)), np.zeros((2, nw + 1, 8))
    # forward: predecessors of state ns
    pred = np.zeros((8, 2), int)
    pu, pz = np.zeros((8, 2), int), np.zeros((8, 2), int)
    for ns in range(8):
        for d3 in range(2):
            p = (((ns >> 1) & 1) << 2) | ((ns & 1) << 1) | d3
            pred[ns, d3] = p
            u = [uu for uu in range(2) if nxt[p, uu] == ns][0]
            pu[ns, d3], pz[ns, d3] = u, par[p, u]
    bits = np.zeros(K, np.uint8)
    it, ok = 0, False
    while it < max_iter and not ok:
        it += 1
        for dec in range(2):
            q = pi if dec else np.arange(K)
            ls_all, lp_all, la_all = d[0, q], d[2 if dec else 1, :K], ext[1 - dec][q]
            a = ab[dec, :nw].copy()
            a[0] = [0.0] + [-np.inf] * 7
            b = bb[dec, :nw].copy()
            b[nw - 1] = beta_k[dec]
            alpha = np.zeros((nw, win, 8))
            for j in range(win):
                t = win * np.arange(nw) + j
                act = t < K
                tt = np.minimum(t, K - 1)
                lsa, lp = (ls_all[tt] + la_all[tt])[:, None], lp_all[tt][:, None]
                alpha[:, j] = a
                c0 = a[:, pred[:, 0]] + gam(pu[:, 0], pz[:, 0], lsa, lp)
                c1 = a[:, pred[:, 1]] + gam(pu[:, 1], pz[:, 1], lsa, lp)
                a = np.where(act[:, None], np.maximum(c0, c1), a)
            a_end = a
            for j in range(win - 1, -1, -1):
                t = win * np.arange(nw) + j
                act = t < K
                tt = np.minimum(t, K - 1)
                ls, la, lp = ls_all[tt][:, None], la_all[tt][:, None], lp_all[tt][:, None]
                lsa = ls + la
                g0 = gam(0, par[:, 0], lsa, lp) + b[:, nxt[:, 0]]
                g1 = gam(1, par[:, 1], lsa, lp) + b[:, nxt[:, 1]]
                m0, m1 = (alpha[:, j] + g0).max(axis=1), (alpha[:, j] + g1).max(axis=1)
                lapp = m0 - m1
                for w in np.nonzero(act)[0]:
                    ext[dec][q[t[w]]] = 0.75 * (lapp[w] - ls[w, 0] - la[w, 0])
                    if dec:
                        bits[q[t[w]]] = lapp[w] < 0
                b = np.where(act[:, None], np.maximum(g0, g1), b)
            ab[dec, 1:nw] = a_end[:nw - 1]
            bb[dec, :nw - 1] = b[1:nw]
        ok = not S.crc24a(bits[F:K - 24]).tolist() != bits[K - 24:].tolist()
    return bits, ok, it


def deratematch(v, K, F, rv):
    """Rule 7: d [3][K + 4] from the soft bits v [E]; filler bits +1e6 in d[0], 0 in d[1]."""
    w = S.circular_buffer(K, F)
    pos = [i for i in range(len(w)) if w[i] is not None]
    k0 = S.k0_position(K, rv)
    order = [i for i in pos if i >= k0] + [i for i in pos if i < k0]
    d = np.zeros((3, K + 4))
    d[0, :F] = 1e6
    for j, x in enumerate(v):
        s, k = w[order[j % len(order)]]
        d[s, k] += x
    return d


# ---- rules 3-8, restated on the grid of test_carrier_meas_host ----------------------------------------------------------------
def occasion_grid(oracle, x, fs_in, fc_in, d, s, fs_programmed=FS):
    """Y [2 n_symb][12 R]: every symbol of grid subframe s of the found-cell dict d."""
    D = int(round(fs_in / FS))
    cell = oracle.new_cell(**{k: v for k, v in d.items() if k not in ("phich_duration", "phich_resource", "sfn")})
    n_symb = 7 if d["cp_type"] == 1 else 6
    ts = window_starts(oracle, cell, x.size, D, fs_programmed)
    return carrier_grid(x, fs_in, fc_in, cell, ts[2 * s * n_symb + np.arange(2 * n_symb)], fs_programmed)


def allocation(R, dci):
    """Rules 3-4 from a parsed DCI record (format, localized, rb_start, n_rb, mcs, tpc, gap, riv, tbs_index): (tbs, PRBs
    of each slot), or None when it is invalid."""
    if dci["format"] == 1:
        if dci["n_rb"] < 1 or dci["mcs"] > 26:
            return None
        s = dict(format="1A", riv=int(dci["riv"]), mcs=int(dci["mcs"]), tpc=int(dci["tpc"]), distributed=int(dci["localized"]))
        if s["distributed"] and dci["rb_start"] + dci["n_rb"] > S.n_vrb(R, 0):
            return None
    else:
        step = 2 if R < 50 else 4
        if S.riv_decode(S.n_vrb(R, int(dci["gap"])) // step, int(dci["riv"])) is None:
            return None
        s = dict(format="1C", riv=int(dci["riv"]), gap=int(dci["gap"]), tbs_index=int(dci["tbs_index"]))
    return S.sib1_allocation(R, s)


def equalise_pdsch(Y, n_id, cp, P, R, res):
    """Rule 6 on the REs res [(l, k)] of an occasion's grid Y: (xhat [n_re], g [n_re])."""
    n_symb = 7 if cp == 1 else 6
    rs = S.crs_full(n_id, cp, R)
    _, shift = S.O.rs_dl(n_id, cp)
    crs_syms = lambda p: [0, n_symb - 3, n_symb, 2 * n_symb - 3] if p < 2 else [1, n_symb + 1]

    def h_at(p, lc, k):
        slot, sym = 10 + lc // n_symb, lc % n_symb
        cols = 6 * np.arange(2 * R) + int(shift[slot * n_symb + sym, p])
        h = Y[lc, cols] * np.conj(rs[slot, sym])
        return np.interp(k, cols, h.real) + 1j * np.interp(k, cols, h.imag)

    def hhat(p, l, k):
        ls = crs_syms(p)
        if l <= ls[0]:
            return h_at(p, ls[0], k)
        if l >= ls[-1]:
            return h_at(p, ls[-1], k)
        i = max(j for j in range(len(ls)) if ls[j] <= l)
        if ls[i] == l:
            return h_at(p, l, k)
        w = (l - ls[i]) / (ls[i + 1] - ls[i])
        return (1 - w) * h_at(p, ls[i], k) + w * h_at(p, ls[i + 1], k)

    xh, g = np.zeros(len(res), complex), np.zeros(len(res))
    for n in range(0, len(res), 2):
        (l, k0), (l1, k1) = res[n], res[n + 1]
        assert l == l1
        y0, y1 = Y[l, k0], Y[l, k1]
        if P == 1:
            for m, (k, y) in enumerate(((k0, y0), (k1, y1))):
                h = hhat(0, l, k)
                xh[n + m], g[n + m] = y * np.conj(h) / abs(h) ** 2, abs(h) ** 2
        else:
            a, b = (0, 1) if P == 2 else ((0, 2) if (n // 2) % 2 == 0 else (1, 3))
            ha, hb = (hhat(a, l, k0) + hhat(a, l, k1)) / 2, (hhat(b, l, k0) + hhat(b, l, k1)) / 2
            gp = abs(ha) ** 2 + abs(hb) ** 2
            xh[n] = np.sqrt(2) * (np.conj(ha) * y0 + hb * np.conj(y1)) / gp
            xh[n + 1] = np.sqrt(2) * (np.conj(ha) * y1 - hb * np.conj(y0)) / gp
            g[n:n + 2] = gp
    return xh, g


def measure_occasion(Y, n_id, cp, P, R, n_ctrl, dci, sfn):
    """Rules 3-8 of one occasion given its DCI record: dict of n_re, sinr, K, F, rv, crc_ok, iterations, tb (bytes)."""
    alloc = allocation(R, dci)
    if alloc is None:
        return dict(n_re=0)
    tbs, prbs = alloc
    res = S.pdsch_res(R, P, cp, n_id, n_ctrl, prbs)
    xh, g = equalise_pdsch(Y, n_id, cp, P, R, res)
    sl = lambda v: np.where(v >= 0, 1, -1) / np.sqrt(2)
    err = np.sum((xh.real - sl(xh.real)) ** 2 + (xh.imag - sl(xh.imag)) ** 2)
    u = np.sqrt(2) * np.stack([xh.real, xh.imag], axis=1).reshape(-1)
    c = S.O.lte_pn(0xFFFF * 16384 + 5 * 512 + n_id, u.size).astype(float)
    v = (1 - 2 * c) * u * np.repeat(g, 2)
    K = min(k for k in S.turbo_sizes() if k >= tbs + 24)
    F, rv = K - tbs - 24, S.sib1_rv(sfn)
    bits, ok, it = turbo_decode(deratematch(v, K, F, rv), K, F)
    return dict(n_re=len(res), sinr=len(res) / err if err > 0 else np.inf, tbs=tbs, K=K, F=F, rv=rv, crc_ok=int(ok),
                iterations=it, tb=bytes(np.packbits(bits[F:F + tbs])), prbs=prbs, err=err, xhat=xh)


# ---- the transport block, the turbo code and the circular buffer ------------------------------------------------------------
def test_tbs_anchors_and_1c_table_ends():
    assert S.TBS_1A[0] == (32, 56) and S.TBS_1A[26] == (1480, 2216)
    assert S.TBS_1C[0] == 40 and S.TBS_1C[-1] == 1736 and len(S.TBS_1C) == 32
    assert max(max(t) for t in S.TBS_1A) + 24 <= 2240


def test_qpp_table_gives_permutations():
    ks, qpp = S.turbo_sizes(), S.qpp_table()
    assert len(ks) == 188 == len(qpp) and ks[0] == 40 and ks[-1] == 6144
    steps = np.diff(ks)
    assert set(steps[:59]) == {8} and set(steps[59:91]) == {16} and set(steps[91:123]) == {32} and set(steps[123:]) == {64}
    assert tuple(qpp[0]) == (3, 10) and tuple(qpp[-1]) == (263, 480)
    for K, (f1, f2) in zip(ks, qpp):
        i = np.arange(K, dtype=np.int64)
        assert np.unique((f1 * i + f2 * i * i) % K).size == K, K


@pytest.mark.parametrize("tbs", [32, 328, 1000, 2216])
@pytest.mark.parametrize("rv", [0, 1, 2, 3])
def test_turbo_round_trip(tbs, rv):
    rng = np.random.default_rng(tbs + rv)
    a = rng.integers(0, 2, tbs).astype(np.uint8)
    b = np.concatenate([a, S.crc24a(a)])
    K = min(k for k in S.turbo_sizes() if k >= b.size)
    F = K - b.size
    c = np.concatenate([np.zeros(F, np.uint8), b])
    d = S.turbo_encode(c)
    E = int(1.6 * 3 * K)
    e = S.rate_match(d, K, F, rv, E)
    v = 1 - 2 * e.astype(float) + 0.3 * rng.standard_normal(E)
    bits, ok, it = turbo_decode(deratematch(v, K, F, rv), K, F)
    assert ok and it == 1 and np.array_equal(bits, c)


def test_circular_buffer_k0_and_nulls():
    for K in (40, 64, 1504, 2240):
        w = S.circular_buffer(K, 0)
        rows = -(-(K + 4) // 32)
        assert len(w) == 96 * rows
        assert sum(x is None for x in w) == 3 * (32 * rows - K - 4)
        assert sorted(x for x in w if x is not None) == [(s, k) for s in range(3) for k in range(K + 4)]
        assert [S.k0_position(K, rv) for rv in range(4)] == [rows * (24 * rv + 2) for rv in range(4)]


# ---- planted SIB1 through the restatement -------------------------------------------------------------------------------------
def planted_dci(R, sib1):
    """The parsed DCI record (as lcs_pdcch_dci's fields) of a "sib1" dict."""
    if sib1["format"] == "1A":
        st, ln = S.riv_decode(R, sib1["riv"])
        return dict(format=1, localized=sib1.get("distributed", 0), rb_start=st, n_rb=ln, mcs=sib1["mcs"],
                    tpc=sib1.get("tpc", 0), riv=sib1["riv"], gap=0, tbs_index=0)
    return dict(format=2, localized=0, rb_start=-1, n_rb=-1, mcs=0, tpc=0, riv=sib1["riv"], gap=sib1.get("gap", 0),
                tbs_index=sib1["tbs_index"])


D_OF_R = {6: 2, 15: 2, 25: 4, 50: 8, 75: 8, 100: 16}
TWO_PATH = [(0.0, 1.0), (0.8e-6, 0.5 * np.exp(1j))]
# (R, ports, cp, cfi of the first occasion, format and DCI fields, SFN of grid frame 0 (its first occasion's RV), two paths)
PLANTED = [
    (6, 1, 1, 3, dict(format="1A", riv=6 * 3 + 1, mcs=4, tpc=1, distributed=0), 0, False),
    (15, 2, 2, 2, dict(format="1A", riv=15 * 4 + 3, mcs=9, tpc=0, distributed=1), 2, True),
    (25, 4, 1, 1, dict(format="1C", riv=12 * 2 + 1, tbs_index=12), 4, True),
    (50, 2, 1, 2, dict(format="1C", riv=9 * 3 + 2, tbs_index=16, gap=1), 6, False),
    (75, 4, 2, 3, dict(format="1A", riv=75 * 7 + 20, mcs=14, tpc=1, distributed=1), 9, True),
    (100, 1, 1, 1, dict(format="1A", riv=100 * 33 + 10, mcs=26, tpc=1, distributed=0), 1, False),
]


@pytest.mark.parametrize("case", PLANTED, ids=lambda c: "%drb-%dport-cp%d-cfi%d-%s" % (c[0], c[1], c[2], c[3], c[4]["format"]))
def test_planted_sib1_decodes_exactly(oracle, case):
    """Every R, 1/2/4 ports, both CPs, CFI 1-3, 1A localized and distributed, 1C with both gaps, every RV, odd and even SFN,
    TBS up to 2216, flat and two-path channels: the restatement returns the planted transport block at 30 dB."""
    R, P, cp, cfi, dci, sfn0, paths = case
    D = D_OF_R[R]
    sib1 = dict(dci, L=4 if R <= 15 or cfi == 1 else 8, cce=0)
    tbs, prbs = S.sib1_allocation(R, sib1)
    sib1["tb"] = bytes((13 * i + R) % 256 for i in range(tbs // 8))
    kw = dict(paths=TWO_PATH) if paths else {}
    cell = synth_cell(137, P, cp, R, cfi=(cfi,), sib1=sib1, **kw)
    cell["sfn0"] = sfn0
    x, _ = S.synth_wide_full(n_samples(D), D * FS, 739e6, [(739e6, [cell])], 30.0, R)
    d = found(cell, 739e6)
    s = 5 if sfn0 % 2 == 0 else 15
    Y = occasion_grid(oracle, x, D * FS, 739e6, d, s)
    m = measure_occasion(Y, 137, cp, P, R, S.n_ctrl_of(cfi, R, 1), planted_dci(R, sib1), sfn0 + s // 10)
    assert m["prbs"] == prbs and m["tbs"] == tbs
    assert m["crc_ok"] == 1 and m["tb"] == sib1["tb"], (case, m["iterations"])
    assert m["sinr"] > 100


def test_a_cell_without_sib1_is_unchanged():
    cell = synth_cell(137, 2, 1, 25, cfi=(2,))
    a, _ = S.synth_wide_full(n_samples(4), 4 * FS, 739e6, [(739e6, [cell])], 30.0, 3)
    b, _ = S.synth_wide_full(n_samples(4), 4 * FS, 739e6, [(739e6, [dict(cell)])], 30.0, 3)
    assert a.tobytes() == b.tobytes()


# ---- allocation and REs ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", RBS)
def test_vrb_to_prb_is_a_bijection_per_slot(R):
    for gap in ((0, 1) if R >= 50 else (0,)):
        n = S.n_vrb(R, gap)
        for slot in (0, 1):
            prbs = [S.vrb_to_prb(R, gap, v, slot) for v in range(n)]
            assert len(set(prbs)) == n and min(prbs) >= 0 and max(prbs) < R, (R, gap, slot)
    # hand-worked: 25 RBs, gap 1 (N_gap 12, N~_VRB 24, N_row 6, no nulls): even slot 6 (v mod 4) + floor(v / 4), odd
    # slot that plus 12 mod 24
    if R == 25:
        assert [S.vrb_to_prb(25, 0, v, 0) for v in range(6)] == [0, 6, 12, 18, 1, 7]
        assert [S.vrb_to_prb(25, 0, v, 1) for v in range(6)] == [12, 18, 0, 6, 13, 19]


@pytest.mark.parametrize("P, cp, n_ctrl, R, want", [
    (1, 1, 1, 6, 12 * 13 - 2 * 3 - 2 * 12),            # 1 PRB: 13 symbols, 3 CRS symbols of port 0 after symbol 0
    (2, 1, 2, 6, 12 * 12 - 4 * 3 - 2 * 12),
    (4, 1, 3, 6, 12 * 11 - 4 * 4 - 2 * 12),            # ports 2 and 3 in symbol 8 as well
    (2, 2, 1, 6, 12 * 11 - 4 * 3 - 2 * 12),
    (1, 1, 3, 15, 12 * 11 - 2 * 3),                     # PRB 0 of 15 lies outside the PSS/SSS columns
])
def test_data_re_counts(P, cp, n_ctrl, R, want):
    assert len(S.pdsch_res(R, P, cp, 1, n_ctrl, [[0], [0]])) == want


def test_pss_sss_prbs_keep_their_outer_res_at_odd_r():
    # R = 25: the 72 central columns are 114 .. 185; PRB 9 (108 .. 119) keeps 6 of its REs in the PSS / SSS symbols
    res = S.pdsch_res(25, 1, 1, 0, 1, [[9], [9]])
    assert sorted(k for l, k in res if l == 5) == list(range(108, 114))


# ---- SIB1 over UPER ----------------------------------------------------------------------------------------------------------
class Bits:
    def __init__(self):
        self.b = []

    def put(self, v, n):
        self.b += [(v >> (n - 1 - i)) & 1 for i in range(n)]
        return self

    def bytes(self, n_bytes=None):
        b = self.b + [0] * (-len(self.b) % 8)
        if n_bytes:
            b += [0] * (8 * n_bytes - len(b))
        return bytes(np.packbits(np.array(b, np.uint8)))


def sib1_bits(plmns, tac, cid, csg_id=None, offset=None, p_max=None, tdd=None, si=((0, [3]),), nce=False, band=7,
              q_rx=-64, win=2, tag=5):
    """UPER BCCH-DL-SCH-Message carrying SIB1 (36.331 Rel-8), field by field.  plmns: (mcc or None, mnc string, reserved)."""
    w = Bits().put(0, 1).put(1, 1)
    w.put(p_max is not None, 1).put(tdd is not None, 1).put(nce, 1)
    w.put(csg_id is not None, 1).put(len(plmns) - 1, 3)
    for mcc, mnc, res in plmns:
        w.put(mcc is not None, 1)
        if mcc is not None:
            for ch in "%03d" % mcc:
                w.put(int(ch), 4)
        w.put(len(mnc) - 2, 1)
        for ch in mnc:
            w.put(int(ch), 4)
        w.put(0 if res else 1, 1)
    w.put(tac, 16).put(cid, 28).put(1, 1).put(0, 1).put(0, 1)
    if csg_id is not None:
        w.put(csg_id, 27)
    w.put(offset is not None, 1).put(q_rx + 70, 6)
    if offset is not None:
        w.put(offset - 1, 3)
    if p_max is not None:
        w.put(p_max + 30, 6)
    w.put(band - 1, 6).put(len(si) - 1, 5)
    for per, sibs in si:
        w.put(per, 3).put(len(sibs), 5)
        for t in sibs:
            w.put(0, 1).put(t - 3, 4)
    if tdd is not None:
        w.put(tdd[0], 3).put(tdd[1], 4)
    w.put(win, 3).put(tag, 5)
    return w


HARNESS = r"""
#include <cstdio>
#include <cstring>
#include <vector>
#include "sib1_plan.hpp"
#include "sib1_rules.hpp"
using namespace lcs::sib1;
int main(int argc, char** argv) {
  for (int i = 0; i < 27; i++) std::printf("A %d %d %d\n", i, tbs_1a(i, 2), tbs_1a(i, 3));
  for (int i = 0; i < 32; i++) std::printf("C %d %d\n", i, tbs_1c(i));
  for (int i = 0; i < N_K; i++) {
    int f1, f2;
    qpp_params(i, f1, f2);
    std::printf("Q %d %d %d\n", k_of(i), f1, f2);
  }
  const int rbs[] = {6, 15, 25, 50, 75, 100};
  for (int R : rbs)
    for (int gap = 0; gap < (R >= 50 ? 2 : 1); gap++)
      for (int ns = 0; ns < 2; ns++) {
        std::printf("V %d %d %d", R, gap, ns);
        for (int n = 0; n < n_vrb_gap(R, gap); n++) std::printf(" %d", vrb_to_prb(R, gap, n, ns));
        std::printf("\n");
      }
  const int ks[] = {40, 64, 1504, 2240};
  for (int K : ks) {
    std::printf("W %d", K);
    for (int i = 0; i < 96 * ((K + 4 + 31) / 32); i++) std::printf(" %d", wbuf_pos(K, 0, i));
    std::printf("\n");
  }
  for (int a = 1; a < argc; a++) {                 // hex strings: parse each as a transport block
    const size_t n = std::strlen(argv[a]) / 2;
    std::vector<uint8_t> tb(n);
    for (size_t i = 0; i < n; i++) std::sscanf(argv[a] + 2 * i, "%2hhx", &tb[i]);
    lcs_sib1_meas m;
    std::memset(&m, 0, sizeof m);
    const bool ok = parse_sib1(tb.data(), (int)n, m);
    std::printf("P %d %u", ok, m.n_plmn);
    for (uint32_t i = 0; i < m.n_plmn && i < 6; i++)
      std::printf(" %u-%u-%u-%u", m.plmn[i].mcc, m.plmn[i].mnc, m.plmn[i].mnc_digits, m.plmn[i].reserved);
    std::printf(" %u %u %u %u %u %d %u %u %d %u %u", m.tac, m.cell_identity, m.csg_identity_present, m.csg_identity,
                m.csg_indication, m.q_rx_lev_min, m.q_rx_lev_min_offset, m.p_max_present, m.p_max,
                m.freq_band_indicator, m.n_si);
    for (uint32_t i = 0; i < m.n_si && i < 32; i++) std::printf(" %u/%u", m.si_periodicity[i], m.si_sib_mask[i]);
    std::printf(" %u %u %u %u %u %u\n", m.tdd_present, m.tdd_subframe_assignment, m.tdd_special_subframe_patterns,
                m.si_window_ms, m.system_info_value_tag, m.non_critical_extension);
  }
  return 0;
}
"""

PARSE_CASES = [
    dict(plmns=[(310, "410", False)], tac=0x1234, cid=0xABCDEF1),
    dict(plmns=[(1, "01", True), (None, "02", False), (262, "123", False)], tac=7, cid=1, csg_id=12345, offset=3, p_max=23,
         tdd=(2, 7), si=((0, [3]), (2, [4, 5, 11]), (6, [])), nce=True, band=64, q_rx=-70, win=6, tag=31),
    dict(plmns=[(100 + i, "%02d" % i, i % 2 == 0) for i in range(6)], tac=0xFFFF, cid=(1 << 28) - 1, p_max=-30, q_rx=-22),
]


@pytest.fixture(scope="module")
def harness(lcs, tmp_path_factory):
    tmp = tmp_path_factory.mktemp("sib1_rules")
    src = tmp / "h.cpp"
    src.write_text(HARNESS)
    exe = str(tmp / "h")
    libdir = os.path.dirname(lcs.LIB_PATH)
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address", "-fno-omit-frame-pointer", "-I" + CSRC,
                           "-I/usr/local/cuda/include", str(src), os.path.join(CSRC, "sib1_plan.cpp"),
                           os.path.join(CSRC, "pdcch_plan.cpp"), os.path.join(CSRC, "carrier_plan.cpp"), "-o", exe,
                           "-L" + libdir, "-llcs_b200", "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64",
                           "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])

    def run(*tbs):
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1")
        r = subprocess.run([exe] + [t.hex() for t in tbs], capture_output=True, text=True, env=env)
        assert r.returncode == 0, r.stderr[-3000:]
        return r.stdout.splitlines()
    return run


def test_rules_header_matches_restatement(harness):
    out = harness()
    rows = lambda tag: [list(map(int, l.split()[1:])) for l in out if l.startswith(tag + " ")]
    assert [tuple(r[1:]) for r in rows("A")] == S.TBS_1A
    assert [r[1] for r in rows("C")] == S.TBS_1C
    assert [r[0] for r in rows("Q")] == S.turbo_sizes()
    assert np.array_equal(np.array([r[1:] for r in rows("Q")]), S.qpp_table())
    for R, gap, ns, *prb in rows("V"):
        assert prb == [S.vrb_to_prb(R, gap, n, ns) for n in range(S.n_vrb(R, gap))], (R, gap, ns)
    for K, *pos in rows("W"):
        want = [-1 if x is None else x[0] * (K + 4) + x[1] for x in S.circular_buffer(K, 0)]
        assert pos == want, K


def expected_parse(c):
    plmns, mcc = [], None
    for m, mnc, res in c["plmns"]:
        mcc = m if m is not None else mcc
        plmns.append("%d-%d-%d-%d" % (mcc, int(mnc), len(mnc), int(res)))
    si = c.get("si", ((0, [3]),))
    mask = lambda sibs: sum(1 << t for t in sibs)
    tdd = c.get("tdd")
    return ("P 1 %d " % len(plmns) + " ".join(plmns)
            + " %d %d %d %d 0 %d %d %d %d %d %d" % (c["tac"], c["cid"], c.get("csg_id") is not None, c.get("csg_id") or 0,
                                                   c.get("q_rx", -64), c.get("offset") or 0, c.get("p_max") is not None,
                                                   c.get("p_max") or 0, c.get("band", 7), len(si))
            + "".join(" %d/%d" % (8 << p, mask(s)) for p, s in si)
            + " %d %d %d %d %d %d" % (tdd is not None, tdd[0] if tdd else 0, tdd[1] if tdd else 0,
                                      [1, 2, 5, 10, 15, 20, 40][c.get("win", 2)], c.get("tag", 5), int(c.get("nce", False))))


def test_sib1_parser(harness):
    tbs = [sib1_bits(**c).bytes() for c in PARSE_CASES]
    out = harness(*tbs)
    for line, c in zip(out[-len(tbs):], PARSE_CASES):
        assert line == expected_parse(c), (line, expected_parse(c))


def test_sib1_parser_rejects_other_messages_and_truncated_input(harness):
    full = sib1_bits(**PARSE_CASES[1])
    tb = full.bytes()
    other = Bits()
    other.b = [0, 0] + full.b[2:]                  # c1: systemInformation
    out = harness(*[tb[:n] for n in (len(tb) - 1, len(tb) // 2, 1)] + [other.bytes()])
    assert [l.split()[1] for l in out if l.startswith("P ")] == ["0"] * 4


def test_sib1_prototypes_cover_header_and_library(lcs):
    names = exported(os.path.join(os.path.dirname(lcs.LIB_PATH), "liblcs_sib1.so"))
    for f in ("lcs_sib1_create", "lcs_sib1_destroy", "lcs_sib1_cells", "lcs_sib1_timing_read"):
        assert f in names
    lcs.sib1_lib()
    assert lcs.SIB1_MEAS.itemsize % 8 == 0 and lcs.SIB1_OCC.fields["tb"][1] + lcs.SIB1_TB_BYTES <= lcs.SIB1_OCC.itemsize


def test_cli_sib1_argument_errors(lcs, tmp_path):
    from test_channelizer_host import cellsearch
    f = str(tmp_path / "rec.ci16")
    np.zeros((1000, 2), np.int16).tofile(f)
    wide = ["--wideband", f, "--fc-in", "739e6", "-s", "739e6"]
    cases = [
        (["-s", "739e6", "-l", "-d", str(tmp_path), "--sib1"], "--sib1 needs --wideband"),
        (wide + ["--fs-in", "7.68e6", "--sib1-csv", str(tmp_path / "c.csv")], "--sib1-csv needs --sib1"),
        (["--wideband", f, "--fc-in", "739e6", "--fs-in", "10e6", "--spectrum", str(tmp_path / "p.csv"), "--sib1"],
         "--sib1 needs a search (-s)"),
        (wide + ["--fs-in", "11.52e6", "--sib1"], "--sib1 needs --fs-in = D * 1.92 MHz"),
        (wide + ["--fs-in", "10e6", "--resample", "--sib1"], "--sib1 needs --fs-in = D * 1.92 MHz"),
        (wide + ["--fs-in", "7.68e6", "--sib1"], "holds 1000 ci16 samples"),
    ]
    for args, msg in cases:
        out = cellsearch(*args)
        assert out.returncode != 0 and msg in out.stderr, (args, out.stderr)
        assert "lcs_ctx_create" not in out.stderr
