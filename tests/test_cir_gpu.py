"""liblcs_cir.so on the device: pdp and floor against the float64 restatement of test_cir_host within an FP32 error bound,
at every rate and format, from host and device memory and at every bandwidth; the statistics against the restatement's
on the device's own pdp; many cells in one call, bitwise equal to each measured alone; launch counts,
lcs_carrier_cells untouched by a CIR call on its context; and CellSearch_b200 --cir --cir-csv end to end."""
import csv
import math

import numpy as np
import pytest

from test_carrier_meas_gpu import FC_IN, many_cells, recording, to_device
from test_carrier_meas_host import FS, S, found, n_samples, synth_cell
from test_channelizer_host import cellsearch
from test_cir_host import T_S, TAP0, TAPS, cir_stats, measure_cir

pytestmark = pytest.mark.gpu

# The FP32 error bound.  test_carrier_meas_gpu bounds each grid element's error by eps ~ 1.8e-6 of the rms bin magnitude
# sqrt(128 P_bin) of its window (P_bin = mean |x|^2 / N in the outputs' units), and everything after the grid is FP64
# with exact twiddles.  The transform is linear, so |dc_t(tau)| <= sum_m w[m] |dY| <= R eps sqrt(128 P_bin).  A product
# c_a conj(c_b) then errs by at most |c| 2 R eps sqrt(128 P_bin), which in pdp's units (/ 128 R^2) is
# 2 eps sqrt(P_bin |c|^2 / (128 R^2)); averaged over the pairs (Jensen) at most 2 eps sqrt(P_bin T_j) <= eps (T_j + P_bin),
# T_j = mean (|c_a|^2 + |c_b|^2) / 2 / (128 R^2).  So, as for the carrier's fields,
#   |pdp_j device - pdp_j restatement| <= REL (T_j + P_bin),
# and floor, a mean of T_j - S_j, to 2 REL (mean T_j + P_bin), with REL = 1e-5, a factor 5 above eps.
REL = 1e-5
STATS = ("peak_delay", "first_delay", "mean_delay", "rms_spread")
PATHS = [(0.0, 0.6), (0.8e-6, 1.0), (2.5e-6, 0.3)]


def restate(x, d, D):
    """measure_cir of the found-cell dict d on the recording x (complex, as the device reads it)."""
    import lcs_oracle
    from test_carrier_meas_host import carrier_grid, window_starts
    c = lcs_oracle.new_cell(**d)
    Y = carrier_grid(x, D * FS, FC_IN, c, window_starts(lcs_oracle, c, x.size, D))
    return measure_cir(Y, c.n_id_cell(), c.cp_type, c.n_ports, c.n_rb_dl, D * d["frame_start"] / (D * FS))


def assert_stats_of_own_pdp(got, P, t_frame, what):
    """The statistics of the device's record against rule 5 on the device's own pdp, to 1e-12 (relative, or of T_s)."""
    for p in range(P):
        want = cir_stats(got["pdp"][p])
        for k, w in zip(STATS, want):
            assert abs(got[k][p] - w) <= 1e-12 * max(abs(w), T_S), (what, k, p, got[k][p], w)
        assert got["n_taps"][p] == want[4], (what, p)
    assert abs(got["frame_arrival"] - (t_frame + got["first_delay"][0])) <= 1e-12 * abs(got["frame_arrival"])


def assert_matches(got, want, P, p_bin, what):
    for p in range(4):
        if p < P:
            err = np.abs(got["pdp"][p] - want["pdp"][p])
            bound = REL * (want["t"][p] + p_bin)
            assert np.all(err <= bound), (what, p, (err / bound).max())
            assert abs(got["floor"][p] - want["floor"][p]) <= 2 * REL * (want["t"][p].mean() + p_bin), (what, p)
            assert got["n_pairs"][p] == want["n_pairs"][p] == (240 if p < 2 else 120)
        else:
            assert np.all(np.isnan(got["pdp"][p])) and np.isnan(got["floor"][p]), (what, p)
            assert all(np.isnan(got[k][p]) for k in STATS), (what, p)
            assert got["n_pairs"][p] == 0 and got["n_taps"][p] == 0, (what, p)


# (D, fmt, on_device, n_ports, cp_type, R, carrier offset in Hz)
CASES = [(2, "ci16", False, 1, 1, 6, 200_000), (4, "cs8", True, 2, 2, 15, -1_000_000), (8, "cu8", False, 4, 1, 25, 3_000_000),
         (16, "cf32", True, 2, 1, 50, -5_000_000), (32, "ci16", True, 4, 2, 100, 12_000_000), (16, "cu8", True, 1, 2, 75, 0),
         (8, "cs8", False, 2, 1, 50, 1_500_000), (4, "cf32", False, 4, 2, 25, -600_000)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "D%d-%s-%s-%dport-cp%d-%drb" % (c[0], c[1], "dev" if c[2] else "host",
                                                                                      c[3], c[4], c[5]))
def test_fields_match_restatement(lcs, case):
    D, fmt, on_device, P, cp, R, off = case
    cell = synth_cell(137 if cp == 1 else 52, P, cp, R, paths=PATHS)
    iq, xd, p_bin, _ = recording([(FC_IN + off, [cell])], D, fmt, seed=D)
    d = found(cell, FC_IN + off)
    want = restate(xd, d, D)
    ctx = lcs.Context(0)
    ci = lcs.CellImpulse(ctx)
    got = ci.measure(to_device(iq) if on_device else iq, fmt, D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
    assert_matches(got, want, P, p_bin, case)
    assert_stats_of_own_pdp(got, P, d["frame_start"] / FS, case)
    assert abs(got["first_delay"][0] - want["first_delay"][0]) < 0.05 * T_S
    ms, launches = ci.timing_read()
    assert launches == 2 and ms > 0
    ci.close()
    ctx.close()


def test_many_cells_in_one_call_are_bitwise_each_alone(lcs):
    carriers, ds = many_cells()
    x, _ = S.synth_wide_full(n_samples(16, 5000), 16 * FS, FC_IN, carriers, 30.0, 11)
    iq = S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    cells = [lcs.new_cell(**d) for d in ds]
    ctx = lcs.Context(0)
    ci = lcs.CellImpulse(ctx)
    n0 = ctx.launches
    a = ci.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    assert ctx.launches - n0 == 2 * math.ceil(len(cells) / lcs.CIR_CHUNK) == 4
    assert ci.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS).tobytes() == a.tobytes()
    dev = to_device(iq)
    for i, c in enumerate(cells):
        assert ci.measure(dev, "ci16", 16 * FS, FC_IN, [c], FS).tobytes() == a[i:i + 1].tobytes(), i
        assert_stats_of_own_pdp(a[i], c.n_ports, ds[i]["frame_start"] / FS, i)
        assert np.all(np.isnan(a[i]["pdp"][c.n_ports:])) and np.all(a[i]["n_pairs"][c.n_ports:] == 0)
    assert ci.timing_read()[1] == 4 + 4 + 2 * 40
    n0 = ctx.launches
    assert ci.measure(iq, "ci16", 16 * FS, FC_IN, [], FS).size == 0
    assert ctx.launches == n0
    ci.close()
    ctx.close()


def test_carrier_records_unchanged_by_a_cir_call(lcs):
    carriers, ds = many_cells()
    x, _ = S.synth_wide_full(n_samples(16, 5000), 16 * FS, FC_IN, carriers, 30.0, 12)
    iq = S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    cells = [lcs.new_cell(**d) for d in ds[:12]]
    ctx = lcs.Context(0)
    cm = lcs.CarrierMeasure(ctx)
    ci = lcs.CellImpulse(ctx)
    before = cm.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    ci.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    n0 = ctx.launches
    after = cm.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    assert after.tobytes() == before.tobytes() and ctx.launches - n0 == 2
    ci.close()
    cm.close()
    ctx.close()


def test_cli_cir_end_to_end(lcs, tmp_path):
    """A two-path 50-RB cell at 737.0 MHz and a 15-RB cell at 743.5 MHz in a 15.36 Msps recording at 739 MHz."""
    D = 8
    paths = [(0.0, 0.5), (1.0e-6, 1.0)]
    a = synth_cell(277, 2, 1, 50, t0=1234, paths=paths)
    b = synth_cell(100, 1, 1, 15, t0=9000)
    b["phich_resource"] = 2
    n = 153600 * D + 1000
    x, _ = S.synth_wide_full(n, D * FS, FC_IN, [(737.0e6, [a]), (743.5e6, [b])], 30.0, 9)
    f = str(tmp_path / "rec.ci16")
    S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2))).tofile(f)
    args = ["--wideband", f, "--fs-in", str(D * FS), "--fc-in", str(FC_IN), "-s", "737e6", "-e", "743.5e6", "-p", "5"]
    plain = cellsearch(*args)
    out_csv = str(tmp_path / "cir.csv")
    with_flag = cellsearch(*(args + ["--cir", "--cir-csv", out_csv]))
    assert plain.returncode == 0 and with_flag.returncode == 0, with_flag.stderr
    t0 = plain.stdout.split("Detected the following cells:")[1].strip().splitlines()
    t1 = with_flag.stdout.split("Detected the following cells:")[1].strip().splitlines()
    assert t1[1] == t0[1] + " TOA[us] DS[ns]"
    rows = {}
    for r0, r1 in zip(t0[2:], t1[2:]):
        v = r1.split()
        assert " ".join(v[:-2]) == " ".join(r0.split())
        rows[int(v[0])] = (float(v[-2]), float(v[-1]))
    assert sorted(rows) == [100, 277]
    # the search's frame_start is 2 samples early, so the first path reads about 1.04 us after the frame's start
    for cid, t0_ in ((277, 1234), (100, 9000)):
        toa = rows[cid][0]
        assert abs(toa - (t0_ / FS * 1e6) % 1e4) < 0.1, (cid, toa)
    p1, p2 = 0.25, 1.0
    assert abs(rows[277][1] / (1e9 * np.sqrt(p1 * p2) / (p1 + p2) * 1e-6) - 1) < 0.05, rows[277]
    with open(out_csv) as fh:
        lines = list(csv.reader(fh))
    assert lines[0] == ["n_id_cell", "fc_hz", "port", "delay_ns", "pdp_dbfs"]
    got = {}
    for r in lines[1:]:
        got.setdefault((int(r[0]), int(r[2])), []).append(float(r[3]))
    assert sorted(got) == [(100, 0), (277, 0), (277, 1)]
    for v in got.values():
        assert np.allclose(v, 1e9 * (np.arange(TAPS) - TAP0) * T_S)
