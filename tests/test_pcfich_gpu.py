"""liblcs_pcfich.so on the device: the decided CFI of every subframe equal to the float64 restatement of test_pcfich_host,
and its metrics and SINR within an FP32 error bound, at every rate and format, from host and device memory; the decision
under noise wherever the restatement's margin exceeds that bound; many cells in one call, bitwise equal to each decoded
alone; launch counts, the carrier and CIR records untouched by a PCFICH call on their context; and
CellSearch_b200 --cfi --cfi-csv end to end."""
import csv
import math

import numpy as np
import pytest

from test_carrier_meas_gpu import FC_IN, many_cells, recording, to_device
from test_carrier_meas_host import FS, S, found, n_samples, synth_cell
from test_channelizer_host import cellsearch
from test_pcfich_host import N_SF, SCHED, measure, planted

pytestmark = pytest.mark.gpu

# The FP32 error bound.  As in test_carrier_meas_gpu, each grid element errs by at most eps ~ 1.8e-6 of the rms bin
# magnitude sqrt(128 P_bin) of its window, and everything after the grid is FP64.  A CRS product h = Y conj(r), |r| = 1,
# and every interpolation or pair mean of such products (convex combinations) then err by at most delta = eps
# sqrt(128 P_bin) too.  To first order:
#   one port   xhat = y / h:            |d xhat| <= delta (1 + |xhat|) / |h|;
#   SFBC       xhat = sqrt(2) n / g:    |d n| <= sqrt(2) delta (|y0| + |y1| + |H_a| + |H_b|), |d g| <= 2 delta (|H_a| + |H_b|),
#              so |d xhat| <= delta (sqrt(2) (|y0| + |y1| + |H_a| + |H_b|) + 2 |xhat| (|H_a| + |H_b|)) / g;
# the restatement gives these factors as `sens`.  A metric is a signed sum of the 32 soft bits times sqrt(2) / 32, so it
# errs by at most sqrt(2) / 32 sum_n 2 delta sens_n; sinr = 16 / E, E = sum |xhat - xref|^2, by at most
# dE / (E - dE) relative, dE = sum (2 |xhat_n - xref_n| + delta sens_n) delta sens_n.  delta uses REL = 1e-5, a factor
# 5 above eps.
REL = 1e-5


def bounds(want, p_bin):
    """(metric bound per subframe, relative sinr bound per subframe) of the restatement `want`."""
    dx = REL * np.sqrt(128 * p_bin) * want["sens"]
    b_met = np.sqrt(2) / 32 * 2 * dx.sum(axis=1) + 1e-12
    e = 16 / want["sinr"]
    de = np.sum((2 * (np.abs(want["xhat"]) + 1) + dx) * dx, axis=1)          # |xhat - xref| <= |xhat| + 1
    return b_met, de / np.maximum(e - de, 1e-300)


def assert_matches(got, want, p_bin, what):
    b_met, b_sinr = bounds(want, p_bin)
    assert np.array_equal(got["cfi"], want["cfi"]), (what, np.flatnonzero(got["cfi"] != want["cfi"]))
    err = np.abs(got["metric"] - want["metric"]).max(axis=1)
    assert np.all(err <= b_met), (what, (err / b_met).max())
    rel = np.abs(got["sinr"] / want["sinr"] - 1)
    assert np.all(rel <= b_sinr), (what, (rel / b_sinr).max())
    assert list(got["count"]) == list(want["count"]) and got["cfi_mode"] == want["cfi_mode"], what
    assert got["n_ctrl_symbols"] == want["n_ctrl_symbols"] and got["n_subframes"] == N_SF, what


# (D, fmt, on_device, n_ports, cp_type, R, carrier offset in Hz)
CASES = [(2, "ci16", False, 1, 1, 6, 200_000), (4, "cs8", True, 2, 2, 15, -1_000_000), (8, "cu8", False, 4, 1, 25, 3_000_000),
         (16, "cf32", True, 2, 1, 50, -5_000_000), (32, "ci16", True, 4, 2, 100, 12_000_000), (16, "cu8", True, 1, 2, 75, 0),
         (8, "cs8", False, 2, 1, 50, 1_500_000), (4, "cf32", False, 4, 2, 25, -600_000)]
PATHS = [(0.0, 1.0), (0.8e-6, 0.5 * np.exp(1j))]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "D%d-%s-%s-%dport-cp%d-%drb" % (c[0], c[1], "dev" if c[2] else "host",
                                                                                      c[3], c[4], c[5]))
def test_fields_match_restatement(lcs, oracle, case):
    D, fmt, on_device, P, cp, R, off = case
    cell = synth_cell(137 if cp == 1 else 52, P, cp, R, paths=PATHS, cfi=SCHED)
    iq, xd, p_bin, _ = recording([(FC_IN + off, [cell])], D, fmt, seed=D)
    d = found(cell, FC_IN + off)
    want = measure(oracle, xd, D * FS, FC_IN, d)
    assert np.array_equal(want["cfi"], planted())
    ctx = lcs.Context(0)
    cf = lcs.ControlFormat(ctx)
    got = cf.measure(to_device(iq) if on_device else iq, fmt, D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
    assert_matches(got, want, p_bin, case)
    ms, launches = cf.timing_read()
    assert launches == 2 and ms > 0
    cf.close()
    ctx.close()


@pytest.mark.parametrize("n_ports", [1, 2, 4])
def test_decisions_at_minus_5_db(lcs, oracle, n_ports):
    """At -5 dB per RE the metrics' margins shrink; the device decides as the restatement wherever the restatement's
    margin (best minus second metric) is above twice the metric bound, and its metrics stay within the bound."""
    D, R = 4, 25
    cell = synth_cell(137, n_ports, 1, R, cfi=SCHED)
    iq, xd, p_bin, _ = recording([(FC_IN, [cell])], D, "cf32", seed=20 + n_ports, snr_db=-5.0)
    d = found(cell, FC_IN)
    want = measure(oracle, xd, D * FS, FC_IN, d)
    ctx = lcs.Context(0)
    cf = lcs.ControlFormat(ctx)
    got = cf.measure(iq, "cf32", D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
    b_met, _ = bounds(want, p_bin)
    srt = np.sort(want["metric"], axis=1)
    clear = srt[:, 2] - srt[:, 1] > 2 * b_met
    assert clear.sum() > N_SF // 2
    assert np.array_equal(got["cfi"][clear], want["cfi"][clear]), np.flatnonzero(got["cfi"] != want["cfi"])
    assert np.all(np.abs(got["metric"] - want["metric"]).max(axis=1) <= b_met)
    cf.close()
    ctx.close()


def many_pcfich_cells():
    carriers, ds = many_cells()
    for j, (_, cs) in enumerate(carriers):
        for i, c in enumerate(cs):
            c["cfi"] = SCHED[(i + j) % len(SCHED):] + SCHED[:(i + j) % len(SCHED)]
    return carriers, ds


def test_many_cells_in_one_call_are_bitwise_each_alone(lcs):
    carriers, ds = many_pcfich_cells()
    x, _ = S.synth_wide_full(n_samples(16, 5000), 16 * FS, FC_IN, carriers, 30.0, 11)
    iq = S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    cells = [lcs.new_cell(**d) for d in ds]
    ctx = lcs.Context(0)
    cf = lcs.ControlFormat(ctx)
    n0 = ctx.launches
    a = cf.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    assert ctx.launches - n0 == 2 * math.ceil(len(cells) / lcs.PCFICH_CHUNK) == 4
    assert cf.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS).tobytes() == a.tobytes()
    dev = to_device(iq)
    for k, c in enumerate(cells):            # eight cells share each carrier, so many subframes do not decode
        assert cf.measure(dev, "ci16", 16 * FS, FC_IN, [c], FS).tobytes() == a[k:k + 1].tobytes(), k
        assert a[k]["count"].sum() == N_SF and a[k]["count"][0] == 0 and np.all(np.isin(a[k]["cfi"], (1, 2, 3))), k
    assert cf.timing_read()[1] == 4 + 4 + 2 * 40
    n0 = ctx.launches
    assert cf.measure(iq, "ci16", 16 * FS, FC_IN, [], FS).size == 0
    assert ctx.launches == n0
    cf.close()
    ctx.close()


def test_carrier_and_cir_records_unchanged_by_a_pcfich_call(lcs):
    carriers, ds = many_pcfich_cells()
    x, _ = S.synth_wide_full(n_samples(16, 5000), 16 * FS, FC_IN, carriers, 30.0, 12)
    iq = S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    cells = [lcs.new_cell(**d) for d in ds[:12]]
    ctx = lcs.Context(0)
    cm, ci, cf = lcs.CarrierMeasure(ctx), lcs.CellImpulse(ctx), lcs.ControlFormat(ctx)
    before = cm.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS), ci.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    cf.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    n0 = ctx.launches
    after = cm.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS), ci.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(after, before)) and ctx.launches - n0 == 4
    for h in (cf, ci, cm):
        h.close()
    ctx.close()


def test_cli_cfi_end_to_end(lcs, tmp_path):
    """A 50-RB two-port cell at 737.0 MHz and a 15-RB cell at 743.5 MHz, each with its own CFI schedule, in a 15.36 Msps
    recording at 739 MHz; without --cfi the output is that of the search alone."""
    D = 8
    a = synth_cell(277, 2, 1, 50, t0=1234, cfi=(3, 3, 1, 2, 3))
    b = synth_cell(100, 1, 1, 15, t0=9000, cfi=(1, 2))
    b["phich_resource"] = 2
    n = 153600 * D + 1000
    x, _ = S.synth_wide_full(n, D * FS, FC_IN, [(737.0e6, [a]), (743.5e6, [b])], 30.0, 9)
    f = str(tmp_path / "rec.ci16")
    S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2))).tofile(f)
    args = ["--wideband", f, "--fs-in", str(D * FS), "--fc-in", str(FC_IN), "-s", "737e6", "-e", "743.5e6", "-p", "5"]
    plain = cellsearch(*args)
    out_csv = str(tmp_path / "cfi.csv")
    with_flag = cellsearch(*(args + ["--cfi", "--cfi-csv", out_csv]))
    assert plain.returncode == 0 and with_flag.returncode == 0, with_flag.stderr
    t0 = plain.stdout.split("Detected the following cells:")[1].strip().splitlines()
    t1 = with_flag.stdout.split("Detected the following cells:")[1].strip().splitlines()
    assert t1[1] == t0[1] + " CFI"
    modes = {}
    for r0, r1 in zip(t0[2:], t1[2:]):
        v = r1.split()
        assert " ".join(v[:-1]) == " ".join(r0.split())
        modes[int(v[0])] = int(v[-1])
    assert modes == {277: 3, 100: 1}
    with open(out_csv) as fh:
        lines = list(csv.reader(fh))
    assert lines[0] == ["n_id_cell", "fc_hz", "subframe", "cfi", "metric1", "metric2", "metric3", "sinr_db"]
    got = {}
    for r in lines[1:]:
        got.setdefault(int(r[0]), []).append((int(r[2]), int(r[3])))
        assert float(r[7]) > 10
    assert sorted(got) == [100, 277]
    # schedules of periods 5 and 2: the grid's subframe s is the planted subframe s whichever frame the search starts at
    for cid, sched in ((277, (3, 3, 1, 2, 3)), (100, (1, 2))):
        assert [s for s, _ in got[cid]] == list(range(N_SF))
        assert [c for _, c in got[cid]] == list(planted(sched=sched)), cid
