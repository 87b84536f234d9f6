"""liblcs_sib1.so on the device: SIB1 planted by lte_dl_synth decoded exactly at every rate and format, 1A localized and
distributed, 1C with both gaps, 1/2/4 ports, both CPs, odd and even SFN and TBS up to 2216, from host and device memory;
the data RE count of rule 5 and the planted transport block, CRC and fields; the occasions' DCIs, cfi and n_ctrl bitwise
those of lcs_pdcch_cells; 40 cells bitwise each alone; the launch count; and the argument errors."""
import csv
import math

import numpy as np
import pytest

import test_grid_modules_gpu as G
from test_carrier_meas_gpu import FC_IN, many_cells, recording, to_device
from test_carrier_meas_host import FS, S, n_samples, synth_cell
from test_pdcch_gpu import found_pdcch
from test_channelizer_host import cellsearch
from test_sib1_host import PARSE_CASES, TWO_PATH, expected_parse, measure_occasion, occasion_grid, sib1_bits

pytestmark = pytest.mark.gpu


def riv(N, start, length):
    return N * (length - 1) + start if length - 1 <= N // 2 else N * (N - length + 1) + (N - 1 - start)


def sib1_of(R, fmt, tbs_key, alloc, parse, **kw):
    """A cell's "sib1" dict: the DCI and a transport block of the SIB1 of PARSE_CASES[parse], zero-padded to the TBS."""
    s = dict(format=fmt, L=4 if R <= 15 else 8, cce=0, **kw)
    if fmt == "1A":
        s.update(mcs=tbs_key[0], tpc=tbs_key[1], riv=riv(R, *alloc))
    else:
        step = 2 if R < 50 else 4
        s.update(tbs_index=tbs_key, riv=riv(S.n_vrb(R, kw.get("gap", 0)) // step, *alloc))
    tbs, _ = S.sib1_allocation(R, s)
    s["tb"] = sib1_bits(**PARSE_CASES[parse]).bytes(tbs // 8)
    return s


# (D, iq format, on device, ports, cp, R, carrier offset, sfn0, sib1 dict args)
CASES = [
    (2, "ci16", False, 1, 1, 6, 200_000, 0, ("1A", (5, 1), (0, 4), 0, dict(distributed=0))),
    (4, "cs8", True, 2, 2, 15, -1_000_000, 3, ("1A", (8, 0), (2, 6), 1, dict(distributed=1, rv_field=3))),
    (8, "cu8", False, 4, 1, 25, 3_000_000, 1, ("1C", 9, (1, 3), 2, {})),
    (16, "cf32", True, 2, 1, 50, -5_000_000, 6, ("1C", 14, (0, 4), 0, dict(gap=1))),
    (16, "cu8", True, 1, 2, 75, 0, 2, ("1A", (10, 1), (10, 9), 1, dict(distributed=1))),
    (32, "ci16", True, 4, 2, 100, 12_000_000, 1023, ("1A", (26, 1), (40, 36), 2, dict(distributed=0))),
    (8, "cs8", False, 2, 1, 50, 1_500_000, 5, ("1C", 20, (2, 5), 0, dict(gap=0))),
]


def case_cell(case):
    D, fmt, on_device, P, cp, R, off, sfn0, (f, key, alloc, parse, kw) = case
    nid = 137 if cp == 1 else 52
    # a control region with room for the DCI's CCEs at every occasion
    paths = dict(paths=TWO_PATH) if R >= 25 and D != 8 else {}
    c = synth_cell(nid, P, cp, R, cfi=(3,) if R <= 15 else (2, 3, 3), sib1=sib1_of(R, f, key, alloc, parse, **kw), **paths)
    c["sfn0"] = sfn0
    d = found_pdcch(c, FC_IN + off)
    d["sfn"] = sfn0
    return c, d


@pytest.mark.parametrize("case", CASES, ids=lambda c: "D%d-%s-%s-%dport-cp%d-%drb-%s" % (
    c[0], c[1], "dev" if c[2] else "host", c[3], c[4], c[5], c[8][0]))
def test_planted_sib1_is_decoded(lcs, oracle, case):
    D, fmt, on_device, P, cp, R, off, sfn0, (f, key, alloc, parse, kw) = case
    cell, d = case_cell(case)
    iq, xd, _, _ = recording([(FC_IN + off, [cell])], D, fmt, seed=D)
    ctx = lcs.Context(0)
    si = lcs.SystemInfo(ctx)
    src = to_device(iq) if on_device else iq
    n0 = ctx.launches
    got = si.measure(src, fmt, D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
    assert ctx.launches - n0 == lcs_launches(lcs, 1)
    cc = lcs.ControlChannel(ctx)
    pd = cc.measure(src, fmt, D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
    tbs, prbs = S.sib1_allocation(R, cell["sib1"])
    sf = [10 * fr + 5 for fr in range(6) if (sfn0 + fr) % 2 == 0]
    for o in range(3):
        r, s = got["occ"][o], sf[o]
        assert r["subframe"] == s and r["sfn"] == (sfn0 + s // 10) % 1024, (case, o)
        assert r["cfi"] == pd["cfi"][s] and r["n_ctrl"] == pd["n_ctrl"][s], (case, o)
        si_dcis = [x for x in pd["dci"][s][:pd["n_dci"][s]] if x["rnti"] == lcs.RNTI_SI]
        assert r["found"] == 1 and r["dci"].tobytes() == si_dcis[0].tobytes(), (case, o)
        assert r["format"] == (1 if f == "1A" else 2) and r["tbs"] == tbs, (case, o)
        assert [list(r["prb"][sl][:r["n_prb"]]) for sl in (0, 1)] == prbs, (case, o)
        n_ctrl = int(pd["n_ctrl"][s])
        assert r["n_re"] == len(S.pdsch_res(R, P, cp, cell["n_id_cell"], n_ctrl, prbs)), (case, o)
        assert r["rv"] == S.sib1_rv(int(r["sfn"])), (case, o)
        assert r["crc_ok"] == 1 and r["iterations"] >= 1, (case, o, r["iterations"])
        assert bytes(r["tb"][:tbs // 8]) == bytes(cell["sib1"]["tb"]) and not r["tb"][tbs // 8:].any(), (case, o)
        assert r["sinr"] > 10, (case, o, r["sinr"])
        want = measure_occasion(occasion_grid(oracle, xd, D * FS, FC_IN, d, s), cell["n_id_cell"], cp, P, R, n_ctrl,
                                r["dci"], int(r["sfn"]))
        assert_matches(r, want, (case, o))
    assert got["n_found"] == 3 and got["n_crc_ok"] == 3 and got["consistent"] == 1 and got["parse_ok"] == 1
    assert parsed(got) == expected_parse(PARSE_CASES[parse])
    ms, launches = si.timing_read()
    assert launches == 5 and ms > 0
    for h in (cc, si):
        h.close()
    ctx.close()


def sinr_bound(want):
    """|device sinr - restatement| allowed.  Each grid element of the device errs by at most about 1.8e-6 of its window's
    rms bin (test_carrier_meas_gpu); through the channel estimate and combining that moves xhat_n by at most
    delta_n = 1e-4 (1 + |xhat_n|), a margin of more than ten over the grid bound.  Then the error sum err moves by at most
    sum 2 |e_n| delta_n + 2 delta_n^2 (e_n = xhat_n - slice), and sinr = n_re / err by that share of itself."""
    x = want["xhat"]
    sl = lambda v: np.where(v >= 0, 1, -1) / np.sqrt(2)
    e = np.abs(x - (sl(x.real) + 1j * sl(x.imag)))
    dn = 1e-4 * (1 + np.abs(x))
    de = np.sum(2 * e * dn + 2 * dn ** 2)
    return want["sinr"] * de / max(want["err"] - de, 1e-300)


def assert_matches(r, want, what):
    """The device occasion r against the restatement: every field exact but sinr, which is within sinr_bound."""
    assert r["n_re"] == want["n_re"], what
    if not want["n_re"]:
        return
    for k in ("tbs", "K", "F", "rv", "crc_ok", "iterations"):
        assert r[k] == want[k], (what, k, r[k], want[k])
    assert bytes(r["tb"][:want["tbs"] // 8]) == want["tb"], what
    assert abs(r["sinr"] - want["sinr"]) <= sinr_bound(want), (what, r["sinr"], want["sinr"], sinr_bound(want))


def lcs_launches(lcs, n):
    return 5 * math.ceil(n / lcs.SIB1_CHUNK)


def parsed(m):
    """The fields of a record in the form of test_sib1_host.expected_parse."""
    pl = " ".join("%d-%d-%d-%d" % tuple(m["plmn"][i][k] for k in ("mcc", "mnc", "mnc_digits", "reserved"))
                  for i in range(m["n_plmn"]))
    out = "P %d %d %s %d %d %d %d %d %d %d %d %d %d %d" % (
        m["parse_ok"], m["n_plmn"], pl, m["tac"], m["cell_identity"], m["csg_identity_present"], m["csg_identity"],
        m["csg_indication"], m["q_rx_lev_min"], m["q_rx_lev_min_offset"], m["p_max_present"], m["p_max"],
        m["freq_band_indicator"], m["n_si"])
    out += "".join(" %d/%d" % (m["si_periodicity"][i], m["si_sib_mask"][i]) for i in range(m["n_si"]))
    return out + " %d %d %d %d %d %d" % (m["tdd_present"], m["tdd_subframe_assignment"], m["tdd_special_subframe_patterns"],
                                         m["si_window_ms"], m["system_info_value_tag"], m["non_critical_extension"])


def test_no_crc_pass_at_low_snr(lcs):
    case = CASES[2]
    cell, d = case_cell(case)
    ctx = lcs.Context(0)
    si = lcs.SystemInfo(ctx)
    for seed in range(3):
        iq, _, _, _ = recording([(FC_IN + case[6], [cell])], case[0], "ci16", seed=100 + seed, snr_db=-10.0)
        got = si.measure(iq, "ci16", case[0] * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
        assert got["n_crc_ok"] == 0 and got["parse_ok"] == 0 and got["consistent"] == 0 and got["n_plmn"] == 0, seed
        for o in range(3):
            assert got["occ"][o]["crc_ok"] == 0 and got["occ"][o]["iterations"] in (0, 8)
    si.close()
    ctx.close()


@pytest.mark.parametrize("snr_db", [-1.0, 1.0, 3.0])
def test_crc_agrees_with_restatement_at_low_snr(lcs, oracle, snr_db):
    """A fixed seeded set near the decoding threshold: per occasion the device's crc_ok and iterations are the
    restatement's, and no passing transport block differs from the planted one."""
    case = CASES[2]
    D = case[0]
    cell, d = case_cell(case)
    ctx = lcs.Context(0)
    si = lcs.SystemInfo(ctx)
    for seed in range(2):
        iq, xd, _, _ = recording([(FC_IN + case[6], [cell])], D, "ci16", seed=200 + seed, snr_db=snr_db)
        got = si.measure(iq, "ci16", D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
        for o in range(3):
            r = got["occ"][o]
            if not r["found"] or not r["n_re"]:
                continue
            s = int(r["subframe"])
            want = measure_occasion(occasion_grid(oracle, xd, D * FS, FC_IN, d, s), cell["n_id_cell"], case[4], case[3],
                                    case[5], int(r["n_ctrl"]), r["dci"], int(r["sfn"]))
            assert (r["crc_ok"], r["iterations"]) == (want["crc_ok"], want["iterations"]), (snr_db, seed, o)
            if r["crc_ok"] and (r["dci"]["tbs_index"], r["dci"]["riv"]) == (9, cell["sib1"]["riv"]):
                assert bytes(r["tb"][:32]) == bytes(cell["sib1"]["tb"]), (snr_db, seed, o)
    si.close()
    ctx.close()


def many_sib1_cells():
    carriers, ds = many_cells()
    k = 0
    for j, (_, cs) in enumerate(carriers):
        for i, c in enumerate(cs):
            c.update(cfi=(3, 2, 3), sfn0=(17 * k) % 1024,
                     sib1=sib1_of(25, "1A", (5 + i, i % 2), (i, 4 + i % 3), 0, distributed=i % 2))
            ds[k].update(phich_duration=1, phich_resource=1, sfn=c["sfn0"])
            k += 1
    return carriers, ds


def test_many_cells_in_one_call_are_bitwise_each_alone(lcs):
    carriers, ds = many_sib1_cells()
    x, _ = S.synth_wide_full(n_samples(16, 5000), 16 * FS, FC_IN, carriers, 30.0, 11)
    iq = S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    cells = [lcs.new_cell(**d) for d in ds]
    ctx = lcs.Context(0)
    si = lcs.SystemInfo(ctx)
    n0 = ctx.launches
    a = si.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    assert ctx.launches - n0 == lcs_launches(lcs, len(cells)) == 10
    assert si.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS).tobytes() == a.tobytes()
    dev = to_device(iq)
    for k, c in enumerate(cells):
        assert si.measure(dev, "ci16", 16 * FS, FC_IN, [c], FS).tobytes() == a[k:k + 1].tobytes(), k
    n0 = ctx.launches
    assert si.measure(iq, "ci16", 16 * FS, FC_IN, [], FS).size == 0
    assert ctx.launches == n0
    si.close()
    ctx.close()


def test_other_records_unchanged_by_a_sib1_call(lcs):
    carriers, ds = many_sib1_cells()
    x, _ = S.synth_wide_full(n_samples(16, 5000), 16 * FS, FC_IN, carriers, 30.0, 12)
    iq = S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    cells = [lcs.new_cell(**d) for d in ds[:12]]
    ctx = lcs.Context(0)
    hs = [lcs.CarrierMeasure(ctx), lcs.CellImpulse(ctx), lcs.ControlFormat(ctx), lcs.ControlChannel(ctx)]
    before = [h.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS).tobytes() for h in hs]
    si = lcs.SystemInfo(ctx)
    si.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    assert [h.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS).tobytes() for h in hs] == before
    for h in hs + [si]:
        h.close()
    ctx.close()


def test_invalid_arguments_launch_nothing(lcs, monkeypatch):
    """Every invalid case of the grid modules' shared test, on lcs_sib1_cells, then an sfn out of range."""
    monkeypatch.setitem(G.MODULES, "sib1", ("SystemInfo", "sib1_lib", "SIB1_MEAS", 5))
    monkeypatch.setattr(G, "found", lambda cell, fc: dict(found_pdcch(cell, fc), sfn=0))
    G.test_invalid_arguments_launch_nothing(lcs, "sib1")
    D = 8
    cell = synth_cell(137, 2, 1, 25)
    d = dict(found_pdcch(cell, FC_IN + 1e6), sfn=0)
    iq = np.zeros((n_samples(D), 2), np.int16)
    ctx = lcs.Context(0)
    si = lcs.SystemInfo(ctx)
    for sfn in (-1, 1024):
        n0 = ctx.launches
        with pytest.raises(lcs.LcsError, match="lcs_sib1_cells: cell 1: sfn must be 0 to 1023"):
            si.measure(iq, "ci16", D * FS, FC_IN, [lcs.new_cell(**d), lcs.new_cell(**dict(d, sfn=sfn))], FS)
        assert ctx.launches == n0
    si.close()
    ctx.close()


def test_cli_sib1_end_to_end(lcs, tmp_path):
    """A 25-RB cell at 737.0 MHz sending SIB1 and a 15-RB cell at 743.5 MHz sending none, in a 15.36 Msps recording at
    739 MHz: the search's own MIB decode gives the SFN; without --sib1 the output is that of the search alone."""
    D = 8
    a = synth_cell(277, 2, 1, 25, t0=1234, cfi=(2, 3, 3), sib1=sib1_of(25, "1A", (8, 1), (3, 6), 0, distributed=0))
    a["sfn0"] = 301
    b = synth_cell(100, 1, 1, 15, t0=9000, cfi=(1, 2))
    n = 153600 * D + 1000
    x, _ = S.synth_wide_full(n, D * FS, FC_IN, [(737.0e6, [a]), (743.5e6, [b])], 30.0, 9)
    f = str(tmp_path / "rec.ci16")
    S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2))).tofile(f)
    args = ["--wideband", f, "--fs-in", str(D * FS), "--fc-in", str(FC_IN), "-s", "737e6", "-e", "743.5e6", "-p", "5"]
    plain = cellsearch(*args)
    out_csv = str(tmp_path / "sib1.csv")
    with_flag = cellsearch(*(args + ["--sib1", "--sib1-csv", out_csv]))
    assert plain.returncode == 0 and with_flag.returncode == 0, with_flag.stderr
    t0 = plain.stdout.split("Detected the following cells:")[1].strip().splitlines()
    t1 = with_flag.stdout.split("Detected the following cells:")[1].strip().splitlines()
    assert t1[1] == t0[1] + " PLMN TAC CID"
    cols = {}
    for r0, r1 in zip(t0[2:], t1[2:]):
        v = r1.split()
        assert " ".join(v[:-3]) == " ".join(r0.split())
        cols[int(v[0])] = v[-3:]
    c0 = PARSE_CASES[0]
    assert cols == {277: ["%03d-%s" % (c0["plmns"][0][0], c0["plmns"][0][1]), str(c0["tac"]), str(c0["cid"])],
                    100: ["-", "-", "-"]}
    with open(out_csv) as fh:
        lines = list(csv.reader(fh))
    assert lines[0] == ["n_id_cell", "fc_hz", "subframe", "sfn", "format", "rb_start", "n_rb", "tbs", "rv", "crc_ok",
                        "iterations", "sinr_db", "tb_hex"]
    rows = [r for r in lines[1:] if r[0] == "277"]
    assert len(rows) == 3 and all(r[4] == "1A" and r[5:8] == ["3", "6", str(8 * len(a["sib1"]["tb"]))] and r[9] == "1"
                                  and r[12] == a["sib1"]["tb"].hex() for r in rows), rows
    assert all(int(r[3]) % 2 == 0 for r in rows)          # SIB1 goes out in even SFNs: the MIB decode's SFN is right
    assert all(r[4] == "-" for r in lines[1:] if r[0] == "100")
