"""liblcs_carrier.so on the device: every field of lcs_carrier_meas against the float64 restatement of
test_carrier_meas_host within an FP32 error bound, at every rate and format, from host and device memory; many cells on
several carriers in one call, bitwise equal to each measured alone; launch counts; the central six
RBs against lcs_meas_cells on the channelizer's output; and CellSearch_b200 --measure-carrier end to end."""
import csv
import math

import numpy as np
import pytest

from test_carrier_meas_host import FS, GAINS, OFFSET, S, found, measure, n_samples, offset_scenario, synth_cell
from test_channelizer_host import cellsearch

pytestmark = pytest.mark.gpu

FC_IN = 739e6

# The FP32 error bound.  The device computes each grid element with an FP32 FFT of N = 128 D points (log2 N <= 12 stages
# of one rounding each, float twiddles), one float rotation by the mixer and one by the lateness ramp, all from samples
# read exactly; the pair and RSSI sums are FP64.  An element's error is then at most about (2 log2 N + 6) * 2^-24 ~ 1.8e-6
# of the rms bin magnitude of its window, and a product of two elements errs by twice that relative to sqrt(|Y|^2 of the
# element times the window's mean bin power P_bin = mean |x|^2 / N, in the outputs' units).  Sums of such products keep
# the bound.  So every power field (rsrp, noise per port and per RB, rssi per RB) is checked to
#   |device - restatement| <= 1e-5 (T + P_bin),
# T the restatement's rsrp + noise (the mean |h|^2 / 128 of the pairs) or its rssi, a factor 2.7 above the estimate.
REL = 1e-5


def recording(cells_by_carrier, D, fmt, seed, extra=0, snr_db=30.0):
    """(iq [n][2] of fmt, x the samples as the device reads them, P_bin, scale): the synthetic carriers at 0.1 full-scale
    rms."""
    x, _ = S.synth_wide_full(n_samples(D) + extra, D * FS, FC_IN, cells_by_carrier, snr_db, seed)
    scale = 0.1 / np.sqrt(np.mean(np.abs(x) ** 2))
    iq = S.quantise(x, fmt, scale)
    xd = S.dequantise(iq, fmt)
    return iq, xd, np.mean(np.abs(xd) ** 2) / (128 * D), scale


def assert_matches(got, want, P, R, p_bin, what):
    for p in range(4):
        if p < P:
            T = want["rsrp"][p] + want["noise"][p]
            tol = REL * (T + p_bin)
            for k in ("rsrp", "noise"):
                assert abs(got[k][p] - want[k][p]) <= tol, (what, k, p, got[k][p], want[k][p])
            Trb = want["rb_rsrp"][p, :R] + want["rb_noise"][p, :R]
            for k in ("rb_rsrp", "rb_noise"):
                err = np.abs(got[k][p, :R] - want[k][p, :R])
                assert np.all(err <= REL * (Trb + p_bin)), (what, k, p, err.max())
            assert got["n_pairs"][p] == want["n_pairs"][p]
            sinr_want = want["sinr"][p]
            assert np.isinf(got["sinr"][p]) if np.isinf(sinr_want) else got["sinr"][p] == got["rsrp"][p] / got["noise"][p]
        else:
            assert np.isnan(got["rsrp"][p]) and np.isnan(got["noise"][p]) and np.isnan(got["sinr"][p])
            assert got["n_pairs"][p] == 0
    assert np.all(np.isnan(got["rb_rsrp"][P:])) and np.all(np.isnan(got["rb_noise"][:, R:]))
    assert np.all(np.isnan(got["rb_rssi"][R:]))
    assert np.all(np.abs(got["rb_rssi"][:R] - want["rb_rssi"][:R]) <= REL * (want["rb_rssi"][:R] + p_bin)), what
    assert abs(got["rssi"] - want["rssi"]) <= REL * want["rssi"], what
    assert abs(got["rsrq"] / want["rsrq"] - 1) <= 3 * REL, what
    assert got["n_rb"] == R


def to_device(iq):
    import torch
    return torch.from_numpy(np.ascontiguousarray(iq)).cuda()


# (D, fmt, on_device, n_ports, cp_type, R, carrier offset in Hz)
CASES = [(2, "ci16", False, 1, 1, 6, 200_000), (4, "cs8", True, 2, 2, 15, -1_000_000), (8, "cu8", False, 4, 1, 25, 3_000_000),
         (16, "cf32", True, 2, 1, 50, -5_000_000), (32, "ci16", True, 4, 2, 100, 12_000_000), (16, "cu8", True, 1, 2, 75, 0),
         (8, "cs8", False, 2, 1, 50, 1_500_000), (4, "cf32", False, 4, 2, 25, -600_000)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "D%d-%s-%s-%dport-cp%d-%drb" % (c[0], c[1], "dev" if c[2] else "host",
                                                                                      c[3], c[4], c[5]))
def test_fields_match_restatement(lcs, oracle, case):
    D, fmt, on_device, P, cp, R, off = case
    cell = synth_cell(137 if cp == 1 else 52, P, cp, R)
    iq, xd, p_bin, _ = recording([(FC_IN + off, [cell])], D, fmt, seed=D)
    d = found(cell, FC_IN + off)
    want = measure(oracle, xd, D * FS, FC_IN, oracle.new_cell(**d))
    ctx = lcs.Context(0)
    cm = lcs.CarrierMeasure(ctx)
    got = cm.measure(to_device(iq) if on_device else iq, fmt, D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
    assert_matches(got, want, P, R, p_bin, case)
    ms, launches = cm.timing_read()
    assert launches == 2 and ms > 0
    cm.close()
    ctx.close()


@pytest.mark.parametrize("fmt,on_device", [("ci16", False), ("cf32", True)])
def test_clock_offset_matches_restatement(lcs, oracle, fmt, on_device):
    """A clock 25 ppm fast, a carrier 1737.5 Hz off, fc_programmed != fc_requested and a fractional frame start: the
    device's FOC rotation and lateness ramps against the restatement's."""
    x, d, _ = offset_scenario(0)
    D = OFFSET["D"]
    iq = S.quantise(x, fmt, 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    xd = S.dequantise(iq, fmt)
    want = measure(oracle, xd, D * FS, FC_IN, oracle.new_cell(**d))
    ctx = lcs.Context(0)
    cm = lcs.CarrierMeasure(ctx)
    got = cm.measure(to_device(iq) if on_device else iq, fmt, D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
    assert_matches(got, want, 2, 25, np.mean(np.abs(xd) ** 2) / (128 * D), (fmt, on_device))
    cm.close()
    ctx.close()


def many_cells():
    """40 cells on five 25-RB carriers of a 30.72 Msps recording: (carriers, found cell dicts)."""
    carriers, cells = [], []
    for j, off in enumerate((-10_500_000, -4_500_000, 0, 4_500_000, 10_500_000)):
        cs = [synth_cell(3 * (8 * j + i) + i % 3, (1, 2, 4)[i % 3], 1 + (i % 4 == 3), 25, t0=1000 + 517 * i) for i in range(8)]
        for c in cs:
            c["gains"] = [g * (0.3 + 0.1 * (c["n_id_cell"] % 7)) for g in GAINS]
        carriers.append((FC_IN + off, cs))
        cells += [found(c, FC_IN + off) for c in cs]
    return carriers, cells


def test_many_cells_in_one_call_are_bitwise_each_alone(lcs):
    carriers, ds = many_cells()
    x, _ = S.synth_wide_full(n_samples(16, 5000), 16 * FS, FC_IN, carriers, 30.0, 11)
    iq = S.quantise(x, "ci16", 0.1 / np.sqrt(np.mean(np.abs(x) ** 2)))
    cells = [lcs.new_cell(**d) for d in ds]
    ctx = lcs.Context(0)
    cm = lcs.CarrierMeasure(ctx)
    n0 = ctx.launches
    a = cm.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    assert ctx.launches - n0 == 2 * math.ceil(len(cells) / lcs.CARRIER_CHUNK) == 4
    b = cm.measure(iq, "ci16", 16 * FS, FC_IN, cells, FS)
    assert a.tobytes() == b.tobytes()
    dev = to_device(iq)
    for i, c in enumerate(cells):
        alone = cm.measure(dev, "ci16", 16 * FS, FC_IN, [c], FS)
        assert alone.tobytes() == a[i:i + 1].tobytes(), i
    n0 = ctx.launches
    assert cm.measure(iq, "ci16", 16 * FS, FC_IN, cells[:32], FS).tobytes() == a[:32].tobytes()
    assert ctx.launches - n0 == 2
    assert cm.timing_read()[1] == 4 + 4 + 2 * 40 + 2
    n0 = ctx.launches
    assert cm.measure(iq, "ci16", 16 * FS, FC_IN, [], FS).size == 0
    assert ctx.launches == n0
    cm.close()
    ctx.close()


def test_central_six_rbs_agree_with_the_channelized_measurement(lcs):
    """lcs_meas_cells on the channelizer's output of the same recording, divided by gain^2, sees the central six RBs."""
    D, R, off = 8, 50, 2_000_000
    cell = synth_cell(137, 2, 1, R)
    iq, xd, _, _ = recording([(FC_IN + off, [cell])], D, "ci16", seed=5, extra=40 * D * 128, snr_db=40.0)
    d = found(cell, FC_IN + off)
    ctx = lcs.Context(0)
    cm = lcs.CarrierMeasure(ctx)
    full = cm.measure(iq, "ci16", D * FS, FC_IN, [lcs.new_cell(**d)], FS)[0]
    ch = lcs.Channelizer(ctx, D * FS, FC_IN, [FC_IN + off])
    gain = ch.auto_gain(iq)[0]
    out, clip = ch.push_ci16(iq)
    assert not clip.any()
    me = lcs.CellMeasure(ctx)
    six = me.measure(out[0], [lcs.new_cell(**d)], fs_programmed=FS, fmt="cu8")[0]
    for p in range(2):
        centre = full["rb_rsrp"][p, R // 2 - 3:R // 2 + 3].mean()
        db = 10 * np.log10(six["rsrp"][p] / float(gain) ** 2 / centre)
        assert abs(db) < 0.1, (p, db)
    me.close()
    ch.close()
    cm.close()
    ctx.close()


def test_cli_measure_carrier_end_to_end(lcs, tmp_path):
    """A 50-RB two-port cell at 737.0 MHz and a 15-RB one-port cell at 743.5 MHz in a 15.36 Msps recording at 739 MHz."""
    D = 8
    a = synth_cell(277, 2, 1, 50, t0=1234)
    b = synth_cell(100, 1, 1, 15, t0=9000)
    b["phich_resource"] = 2
    n = 153600 * D + 1000
    x, _ = S.synth_wide_full(n, D * FS, FC_IN, [(737.0e6, [a]), (743.5e6, [b])], 30.0, 9)
    scale = 0.1 / np.sqrt(np.mean(np.abs(x) ** 2))
    f = str(tmp_path / "rec.ci16")
    S.quantise(x, "ci16", scale).tofile(f)
    args = ["--wideband", f, "--fs-in", str(D * FS), "--fc-in", str(FC_IN), "-s", "737e6", "-e", "743.5e6", "-p", "5"]
    plain = cellsearch(*args)
    out_csv = str(tmp_path / "carrier.csv")
    with_flag = cellsearch(*(args + ["--measure-carrier", "--carrier-csv", out_csv]))
    assert plain.returncode == 0 and with_flag.returncode == 0, with_flag.stderr
    t0 = plain.stdout.split("Detected the following cells:")[1].strip().splitlines()
    t1 = with_flag.stdout.split("Detected the following cells:")[1].strip().splitlines()
    assert t1[1].endswith(" RSRPc[dBFS] RSRQc[dB] SINRc[dB]") and t1[1][:-len(" RSRPc[dBFS] RSRQc[dB] SINRc[dB]")] == t0[1]
    rows = {}
    for r0, r1 in zip(t0[2:], t1[2:]):
        v = r1.split()
        assert " ".join(v[:-3]) == " ".join(r0.split())
        rows[int(v[0])] = float(v[-3])
    assert sorted(rows) == [100, 277]
    for c, cid in ((a, 277), (b, 100)):
        planted = 10 * np.log10(S.AMP ** 2 * abs(GAINS[0]) ** 2 * scale ** 2 / 128)
        assert abs(rows[cid] - planted) < 0.1, (cid, rows[cid], planted)
    with open(out_csv) as fh:
        lines = list(csv.reader(fh))
    assert lines[0] == ["n_id_cell", "fc_hz", "port", "rb", "rsrp_dbfs", "noise_dbfs", "rssi_dbfs"]
    got = {}
    for r in lines[1:]:
        got.setdefault((int(r[0]), int(r[2])), []).append(int(r[3]))
    assert got == {(277, 0): list(range(50)), (277, 1): list(range(50)), (100, 0): list(range(15))}
