"""liblcs_pdcch.so on the device: every reported DCI, n_reg, n_cce and n_dci equal to the float64 restatement of
test_pdcch_host, and q within an FP32 error bound, at every rate and format, from host and device memory; the CFI bitwise
that of lcs_pcfich_cells; many cells in one call, bitwise equal to each decoded alone; launch counts, the carrier, CIR
and PCFICH records untouched by a PDCCH call on their context; and
CellSearch_b200 --pdcch --pdcch-csv end to end."""
import csv
import math

import numpy as np
import pytest

from test_carrier_meas_gpu import FC_IN, many_cells, recording, to_device
from test_carrier_meas_host import FS, S, found, n_samples, synth_cell
from test_channelizer_host import cellsearch
from test_pdcch_host import N_SF, expected, measure, pdcch_cell, plant, sizes

pytestmark = pytest.mark.gpu

# The FP32 error bound, as in test_pcfich_gpu: every grid element errs by at most delta = REL sqrt(128 P_bin), and a soft
# bit u_b by at most delta sens_b to first order (the restatement's `sens`, rule 7's equalisers differentiated).  For
# q = N / sqrt(E S), N = sum u_b s_b (s_b = +-1) and S = sum u_b^2: |dN| <= sum du_b, |dS| <= sum (2 |u_b| + du_b) du_b,
# so |dq| <= |dN| / sqrt(E S) + |q| |dS| / (2 S) (doubled for the second order).
REL = 1e-5


def q_bound(want, s, L, cce, p_bin):
    b = slice(72 * cce, 72 * cce + 72 * L)
    u, du = want["u"][s][b], REL * np.sqrt(128 * p_bin) * want["sens"][s][b]
    S_ = np.sum(u ** 2)
    return 2 * (du.sum() / np.sqrt(72 * L * S_) + np.sum((2 * np.abs(u) + du) * du) / (2 * S_)) + 1e-12


def clear_subframes(want, p_bin):
    """Subframes where no candidate's q lies within its bound of the threshold."""
    ok = []
    for s in range(N_SF):
        ok.append(all(q is None or abs(q - 0.8) > q_bound(want, s, L, c, p_bin) for _, L, c, _, q in want["tried"][s]))
    return np.array(ok)


def assert_matches(got, want, p_bin, R, what):
    s1a, _ = sizes(R)
    n_ra = math.ceil(math.log2(R * (R + 1) // 2))
    assert got["n_subframes"] == N_SF, what
    assert list(got["n_ctrl"]) == want["n_ctrl"] and list(got["n_reg"]) == want["n_reg"], what
    assert list(got["n_cce"]) == want["n_cce"], what
    clear = clear_subframes(want, p_bin)
    assert clear.sum() == N_SF, (what, np.flatnonzero(~clear))
    si = 0
    for s in range(N_SF):
        w = want["dci"][s]
        assert got["n_dci"][s] == len(w), (what, s, got["n_dci"][s], w)
        for i, (f, L, c, r, pay, q) in enumerate(w):
            g = got["dci"][s][i]
            assert (g["format"], g["agg"], g["cce"], g["rnti"], g["payload"]) == (f, L, c, r, pay), (what, s, i)
            assert g["n_bits"] == sizes(R)[f - 1], (what, s)
            assert abs(g["quality"] - q) <= q_bound(want, s, L, c, p_bin), (what, s, g["quality"], q)
            if f == 1:                           # rule 13's fields, read back from the payload
                bits = lambda a, n: (pay >> (s1a - a - n)) & ((1 << n) - 1)
                assert (g["localized"], g["riv"], g["mcs"], g["harq"], g["ndi"], g["rv"], g["tpc"]) == (
                    bits(1, 1), bits(2, n_ra), bits(2 + n_ra, 5), bits(7 + n_ra, 3), bits(10 + n_ra, 1), bits(11 + n_ra, 2),
                    bits(13 + n_ra, 2)), (what, s)
                if g["n_rb"] > 0:
                    st, n = g["rb_start"], g["n_rb"]
                    assert st + n <= R and g["riv"] == (R * (n - 1) + st if n - 1 <= R // 2 else R * (R - n + 1) + R - 1 - st)
            if r == 0xFFFF:
                si |= 1 << (s % 10)
    rn = [d[3] for s in range(N_SF) for d in want["dci"][s]]
    assert list(got["count"]) == [rn.count(0xFFFF), rn.count(0xFFFE), sum(1 <= r <= 60 for r in rn)], what
    assert got["si_subframes"] == si, what


# (D, fmt, on_device, n_ports, cp_type, R, carrier offset in Hz, phich_duration, phich_resource, cfi schedule)
CASES = [(2, "ci16", False, 1, 1, 6, 200_000, 1, 1, (3,)), (4, "cs8", True, 2, 2, 15, -1_000_000, 2, 2, (3, 2)),
         (8, "cu8", False, 4, 1, 25, 3_000_000, 1, 3, (2, 3)), (16, "cf32", True, 2, 1, 50, -5_000_000, 1, 4, (3,)),
         (32, "ci16", True, 4, 2, 100, 12_000_000, 2, 1, (1, 2, 3)), (16, "cu8", True, 1, 2, 75, 0, 1, 2, (3,)),
         (8, "cs8", False, 2, 1, 50, 1_500_000, 2, 3, (2,)), (4, "cf32", False, 4, 2, 25, -600_000, 1, 4, (3, 2))]
PATHS = [(0.0, 1.0), (0.8e-6, 0.5 * np.exp(1j))]


def case_cell(P, cp, R, dur, res, cfi, fill=None):
    nid = 137 if cp == 1 else 52
    sched, _ = plant(R, cfi, P, cp, dur, res, nid)
    return pdcch_cell(nid, P, cp, R, sched, cfi, dur, res, fill, paths=PATHS), sched


def found_pdcch(cell, fc):
    d = found(cell, fc)
    d.update(phich_duration=cell["phich_duration"], phich_resource=cell["phich_resource"])
    return d


@pytest.mark.parametrize("case", CASES, ids=lambda c: "D%d-%s-%s-%dport-cp%d-%drb" % (c[0], c[1], "dev" if c[2] else "host",
                                                                                      c[3], c[4], c[5]))
def test_fields_match_restatement(lcs, oracle, case):
    D, fmt, on_device, P, cp, R, off, dur, res, cfi = case
    cell, sched = case_cell(P, cp, R, dur, res, cfi, fill=D)
    iq, xd, p_bin, _ = recording([(FC_IN + off, [cell])], D, fmt, seed=D)
    d = found_pdcch(cell, FC_IN + off)
    want = measure(oracle, xd, D * FS, FC_IN, d, dur, res)
    for s in range(N_SF):
        assert [w[:5] for w in want["dci"][s]] == expected(sched, s), (case, s)
    ctx = lcs.Context(0)
    cc = lcs.ControlChannel(ctx)
    src = to_device(iq) if on_device else iq
    got = cc.measure(src, fmt, D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
    assert_matches(got, want, p_bin, R, case)
    ms, launches = cc.timing_read()
    assert launches == 3 and ms > 0
    cf = lcs.ControlFormat(ctx)                  # rule 1: the CFI is bitwise that of the PCFICH decoder
    pc = cf.measure(src, fmt, D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
    assert got["cfi"].tobytes() == pc["cfi"].tobytes()
    for h in (cf, cc):
        h.close()
    ctx.close()


def many_pdcch_cells():
    carriers, ds = many_cells()
    k = 0
    for j, (_, cs) in enumerate(carriers):
        for i, c in enumerate(cs):
            c.update(cfi=(3, 2, 3), phich_duration=1 + (i % 2), phich_resource=1 + (i + j) % 4)
            c["pdcch"], _ = plant(25, (3, 2, 3), c["n_ports"], c["cp_type"], c["phich_duration"], c["phich_resource"],
                                  c["n_id_cell"], seed=i)
            ds[k].update(phich_duration=c["phich_duration"], phich_resource=c["phich_resource"])
            k += 1
    return carriers, ds


def test_many_cells_in_one_call_are_bitwise_each_alone(lcs):
    carriers, ds = many_pdcch_cells()
    x, _ = S.synth_wide_full(n_samples(16, 5000), 16 * FS, FC_IN, carriers, 30.0, 11)
    iq = S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    cells = [lcs.new_cell(**d) for d in ds]
    ctx = lcs.Context(0)
    cc = lcs.ControlChannel(ctx)
    n0 = ctx.launches
    a = cc.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    assert ctx.launches - n0 == 3 * math.ceil(len(cells) / lcs.PDCCH_CHUNK) == 6
    assert cc.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS).tobytes() == a.tobytes()
    dev = to_device(iq)
    for k, c in enumerate(cells):
        assert cc.measure(dev, "ci16", 16 * FS, FC_IN, [c], FS).tobytes() == a[k:k + 1].tobytes(), k
        assert a[k]["n_subframes"] == N_SF and np.all(a[k]["n_dci"] <= 6), k
    assert cc.timing_read()[1] == 6 + 6 + 3 * 40
    n0 = ctx.launches
    assert cc.measure(iq, "ci16", 16 * FS, FC_IN, [], FS).size == 0
    assert ctx.launches == n0
    cc.close()
    ctx.close()


def test_other_records_unchanged_by_a_pdcch_call(lcs):
    carriers, ds = many_pdcch_cells()
    x, _ = S.synth_wide_full(n_samples(16, 5000), 16 * FS, FC_IN, carriers, 30.0, 12)
    iq = S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    cells = [lcs.new_cell(**d) for d in ds[:12]]
    ctx = lcs.Context(0)
    hs = [lcs.CarrierMeasure(ctx), lcs.CellImpulse(ctx), lcs.ControlFormat(ctx)]
    cc = lcs.ControlChannel(ctx)
    before = [h.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS) for h in hs]
    cc.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    n0 = ctx.launches
    after = [h.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS) for h in hs]
    assert all(a.tobytes() == b.tobytes() for a, b in zip(after, before)) and ctx.launches - n0 == 6
    for h in hs + [cc]:
        h.close()
    ctx.close()


def test_cli_pdcch_end_to_end(lcs, tmp_path):
    """A 50-RB two-port cell at 737.0 MHz sending SI, P and RA DCIs and a 15-RB cell at 743.5 MHz sending none, in a 15.36
    Msps recording at 739 MHz; without --pdcch the output is that of the search alone."""
    D = 8
    sched = [((5, ph), r, f, L, c, b) for (_, ph), r, f, L, c, b in plant(50, (3,), 2, 1, 1, 1, 277)[0]]
    # period 5: the grid's subframe s is the planted subframe s whichever frame the search starts at
    a = pdcch_cell(277, 2, 1, 50, sched, t0=1234)
    b = synth_cell(100, 1, 1, 15, t0=9000, cfi=(1, 2))
    n = 153600 * D + 1000
    x, _ = S.synth_wide_full(n, D * FS, FC_IN, [(737.0e6, [a]), (743.5e6, [b])], 30.0, 9)
    f = str(tmp_path / "rec.ci16")
    S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2))).tofile(f)
    args = ["--wideband", f, "--fs-in", str(D * FS), "--fc-in", str(FC_IN), "-s", "737e6", "-e", "743.5e6", "-p", "5"]
    plain = cellsearch(*args)
    out_csv = str(tmp_path / "pdcch.csv")
    with_flag = cellsearch(*(args + ["--pdcch", "--pdcch-csv", out_csv]))
    assert plain.returncode == 0 and with_flag.returncode == 0, with_flag.stderr
    t0 = plain.stdout.split("Detected the following cells:")[1].strip().splitlines()
    t1 = with_flag.stdout.split("Detected the following cells:")[1].strip().splitlines()
    assert t1[1] == t0[1] + " SI"
    si = {}
    for r0, r1 in zip(t0[2:], t1[2:]):
        v = r1.split()
        assert " ".join(v[:-1]) == " ".join(r0.split())
        si[int(v[0])] = int(v[-1])
    n_si = sum(1 for s in range(N_SF) for d in expected(sched, s) if d[3] == 0xFFFF)
    assert si == {277: n_si, 100: 0}
    with open(out_csv) as fh:
        lines = list(csv.reader(fh))
    assert lines[0] == ["n_id_cell", "fc_hz", "subframe", "cfi", "format", "agg", "cce", "rnti", "n_bits", "payload_hex",
                        "quality", "rb_start", "n_rb", "mcs", "rv"]
    got = [(int(r[2]), 1 if r[4] == "1A" else 2, int(r[5]), int(r[6]), int(r[7]), int(r[9], 16)) for r in lines[1:]]
    assert all(int(r[0]) == 277 and float(r[10]) > 0.9 and r[3] == "3" for r in lines[1:])
    assert got == [(s,) + d for s in range(N_SF) for d in expected(sched, s)]
