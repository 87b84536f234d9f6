"""CPU checks of the cell tracker's oracle (track_oracle/) and of the synthetic downlink generator it is tested on."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "track_oracle"))

import lte_dl_synth as S  # noqa: E402
import track_oracle as TO  # noqa: E402

FC = 739e6
FS = 1.92e6


def cell_dict(n_id_cell=277, n_ports=2, cp_type=1, t0=1234.0, sfn0=100):
    return dict(n_id_cell=n_id_cell, n_ports=n_ports, cp_type=cp_type, n_rb_dl=25, phich_duration=1, phich_resource=3,
                t0=t0, sfn0=sfn0)


def lcs_cell(d, n_ports=None):
    import lcs_b200 as L
    c = L.Cell()
    c.n_id_1, c.n_id_2 = d["n_id_cell"] // 3, d["n_id_cell"] % 3
    c.cp_type, c.n_ports = d["cp_type"], d["n_ports"] if n_ports is None else n_ports
    c.n_rb_dl, c.phich_duration, c.phich_resource = d["n_rb_dl"], d["phich_duration"], d["phich_resource"]
    return c


def true_frame_timing(tr, d, n, f_true):
    """Frame start in the tracker's own time stamps after n pushed samples: the synthetic t0 (less the 2-sample DFT offset of
    the searcher's frame_start convention) plus the drift of the time stamps, which advance by 1/k of the tracked offset
    while the true sample clock runs at 1/k of f_true."""
    k_true = (FC - f_true) / FC
    n -= n % 10000                   # only complete blocks have been processed
    drift = tr.sample_time() - (-1 + n / k_true)
    return (d["t0"] - 2 + drift) % 19200


@pytest.mark.parametrize("n_ports,cp_type", [(1, 1), (2, 1), (1, 2), (2, 2), (4, 1), (4, 2)])
def test_synthetic_cell_found_by_oracle_search(oracle, n_ports, cp_type):
    d = cell_dict(n_id_cell=277 if cp_type == 1 else 271, n_ports=n_ports, cp_type=cp_type)
    cu8 = S.synth_cu8(153600, [d], f_true=3000.0, snr_db=10, seed=n_ports * 10 + cp_type)
    cells, _ = oracle.cell_search_one(S.to_c128(cu8), np.arange(-10000, 10001, 5000.0), FC, FC, FS)
    assert len(cells) == 1
    c = cells[0]
    assert (c.n_id_cell(), c.cp_type, c.n_ports, c.n_rb_dl, c.phich_duration, c.phich_resource, c.sfn) == \
        (d["n_id_cell"], cp_type, n_ports, 25, 1, 3, 100)
    assert abs(c.freq_superfine - 3000.0) < 5
    assert abs(c.frame_start - (d["t0"] - 2)) < 0.1


def test_pbch_ratematch_round_trip(oracle):
    e = np.random.default_rng(1).standard_normal(1920)
    pos = S.ratematch_positions(1920)
    ref = np.zeros(120)
    cnt = np.zeros(120)
    np.add.at(ref, pos, e)
    np.add.at(cnt, pos, 1)
    ref = np.where(cnt > 1, ref / np.maximum(cnt, 1), ref)
    assert np.array_equal(oracle.deratematch(e, 40).reshape(-1), ref)


def test_oracle_tracker_converges():
    f_true, d = 3000.0, cell_dict()
    cu8 = S.synth_cu8(int(2 * FS), [d], f_true=f_true, snr_db=10, seed=3)
    tr = TO.Tracker(FC, f_true - 300)
    tr.add_cell(0, lcs_cell(d), d["t0"] - 2 + 0.6)
    err = []
    for i in range(0, cu8.shape[0], 192000):
        tr.push_cu8(cu8[i:i + 192000])
        r = tr.read(0)[0]
        err.append((abs(tr.frequency_offset()[0] - f_true),
                    abs((r["frame_timing"] - true_frame_timing(tr, d, i + 192000, f_true) + 9600) % 19200 - 9600)))
        assert r["mib_successes"] == r["mib_attempts"] > 0 and r["mib_decode_failures"] == 0
    err = np.array(err)
    # The FOE loop weighs its estimate against a prior of variance 1e-6 Hz^2 (tracker_thread.cpp:239-242): at 10 dB the
    # 300 Hz start error decays with a time constant of about 1.3 s, so 1 s leaves ~140 Hz and 2 s ~60 Hz.
    assert np.all(np.diff(err[:, 0]) < 0)
    assert err[9, 0] < 160 and err[-1, 0] < 80
    assert err[9:, 1].max() < 0.25
    r = tr.read(0)[0]
    snr0 = 10 * np.log10(r["crs_sp_raw_av"][0] / r["crs_np_av"][0])
    snr1 = 10 * np.log10(r["crs_sp_raw_av"][1] / r["crs_np_av"][1])
    assert abs(snr0 - 10) < 2 and abs(snr1 - (10 + 20 * np.log10(0.8))) < 2
    assert abs(10 * np.log10(r["sync_sp_av"] / r["sync_np_av"]) - 10) < 2


@pytest.mark.parametrize("cp_type", [1, 2])
def test_oracle_tracker_locks_four_port_cell(cp_type):
    """A four-port cell (PBCH in SFBC-FSTD): the MIB locks at the first attempt and stays locked, which needs the channel
    estimates of all four ports (ports 2 and 3 from their CRS at symbol 1)."""
    f_true, d = 3000.0, cell_dict(n_id_cell=277 if cp_type == 1 else 271, n_ports=4, cp_type=cp_type)
    cu8 = S.synth_cu8(int(1.0 * FS), [d], f_true=f_true, snr_db=10, seed=50 + cp_type)
    tr = TO.Tracker(FC, f_true - 300)
    tr.add_cell(0, lcs_cell(d), d["t0"] - 2 + 0.6)
    for i in range(0, cu8.shape[0], 192000):
        tr.push_cu8(cu8[i:i + 192000])
        r = tr.read(0)[0]
        assert r["mib_successes"] == r["mib_attempts"] > 0 and r["mib_decode_failures"] == 0
    assert r["n_ports"] == 4 and r["mib_attempts"] >= 24
    snr = 10 * np.log10(np.asarray(r["crs_sp_raw_av"]) / np.asarray(r["crs_np_av"]))
    assert np.all(np.isfinite(snr))
    # Ports 0 and 1 read their transmitted SNR as in test_oracle_tracker_converges.  Ports 2 and 3 are not held to a
    # value: tracker_thread.cpp gives none.  Their CRS filter spans two slots rather than about half a slot, so the
    # residual frequency error of the FOE loop takes a share of their signal power into the noise estimate (4 to 5 dB
    # here), and port 2's time interpolation uses the port-0/1 CRS spacing (`port_num>2`, tracker_thread.cpp:414).
    assert abs(snr[0] - 10) < 2 and abs(snr[1] - (10 + 20 * np.log10(0.8))) < 2


def test_oracle_drops_unsynchronised_cell_after_1600_attempts():
    rng = np.random.default_rng(5)
    n = int(16.4 * FS)
    cu8 = np.clip(np.round(127 + 128 * 0.1 * rng.standard_normal((n, 2))), 0, 255).astype(np.uint8)
    tr = TO.Tracker(FC, 0.0)
    tr.add_cell(0, lcs_cell(cell_dict()), 100.0)
    tr.push_cu8(cu8)
    r = tr.read(0)
    assert len(r) == 1 and r[0]["dropped"] == 1
    assert r[0]["mib_attempts"] == 1600 and r[0]["mib_successes"] == 0 and r[0]["mib_decode_failures"] == 400
    assert abs(r[0]["drop_sample"] / FS - 16.0) < 0.05
    assert tr.read(0) == []          # reported once, then the slot is free


def test_oracle_drops_locked_cell_400_attempts_after_signal_stops():
    f_true, d = 3000.0, cell_dict()
    stop = int(0.5 * FS)
    # the signal stops at 0.5 s; then noise only, of the same power, until the drop (400 attempts of 40 ms)
    cu8 = np.concatenate([S.synth_cu8(int(0.6 * FS), [d], f_true=f_true, snr_db=10, seed=4, stop_at=stop),
                          S.synth_cu8(int(16.1 * FS), [], f_true=f_true, snr_db=10, seed=5)])
    tr = TO.Tracker(FC, f_true)
    tr.add_cell(0, lcs_cell(d), d["t0"] - 2)
    tr.push_cu8(cu8)
    r = tr.read(0)[0]
    assert r["dropped"] == 1 and r["mib_successes"] > 0
    assert r["mib_attempts"] - r["mib_successes"] == 400
    assert abs((r["drop_sample"] - stop) / FS - 16.0) < 0.1


def test_oracle_push_size_does_not_matter():
    d = cell_dict()
    cu8 = S.synth_cu8(int(0.3 * FS), [d], f_true=2000.0, snr_db=10, seed=6)
    res = []
    for step in (10000, 7, 10 ** 6):
        tr = TO.Tracker(FC, 1900.0)
        tr.add_cell(0, lcs_cell(d), d["t0"] - 2 + 0.3)
        for i in range(0, cu8.shape[0], step):
            tr.push_cu8(cu8[i:i + step])
        r = tr.read(0)[0]
        res.append((tr.frequency_offset()[0], tr.sample_time(), r["frame_timing"], r["n_symbols"], r["ce"].tobytes(),
                    r["crs_np_av"].tobytes(), r["mib_attempts"]))
    assert res[0] == res[1] == res[2]
