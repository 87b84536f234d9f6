"""The device cell tracker (lcs_track_*) against its CPU oracle (track_oracle/), on synthetic and recorded streams."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "track_oracle"))

import lte_dl_synth as S  # noqa: E402
import track_oracle as TO  # noqa: E402
from test_tracker_oracle import FC, FS, cell_dict, lcs_cell  # noqa: E402

DISCRETE = ("n_id_cell", "n_ports", "cp_type", "dropped", "drop_sample", "n_symbols", "last_slice_start", "mib_attempts",
            "mib_successes", "mib_decode_failures")
MEAS = ("crs_tp", "crs_sp_raw", "crs_np", "crs_tp_av", "crs_sp_raw_av", "crs_np_av", "sync_tp", "sync_sp", "sync_np",
        "sync_np_blank", "sync_tp_av", "sync_sp_av", "sync_np_av", "sync_np_blank_av")


def compare(g, o, gfo, ofo):
    assert np.abs(gfo - ofo).max() < 1e-6
    assert len(g) == len(o)
    for a, b in zip(g, o):
        for k in DISCRETE:
            assert a[k] == b[k], k
        assert abs(a["frame_timing"] - b["frame_timing"]) < 1e-9
        for k in MEAS:
            x, y = np.asarray(a[k], float), np.asarray(b[k], float)
            assert np.array_equal(np.isnan(x), np.isnan(y)), k
            m = ~np.isnan(y)
            assert np.all(np.abs(x[m] - y[m]) <= 1e-9 * np.maximum(np.abs(y[m]), 1e-30)), k
        for k in ("ce", "sync_ce"):
            assert np.abs(a[k] - b[k]).max() <= 1e-9 * max(np.abs(b[k]).max(), 1e-30), k


def run_pair(lcs, ctx, cu8s, cells, fo0, step, fc=None, max_cells=4):
    """cu8s: [n_ch][n][2]; cells: per channel list of (lcs_cell, frame_timing).  Compares after every push."""
    n_ch = len(cu8s)
    fc = np.full(n_ch, FC) if fc is None else np.asarray(fc)
    g = lcs.Tracker(ctx, fc, fo0, max_cells=max_cells)
    o = TO.Tracker(fc, fo0, max_cells=max_cells)
    for ch in range(n_ch):
        for c, ft in cells[ch]:
            g.add_cell(ch, c, ft)
            o.add_cell(ch, c, ft)
    n = cu8s.shape[1]
    for i in range(0, n, step):
        blk = np.ascontiguousarray(cu8s[:, i:i + step])
        g.push_cu8(blk)
        o.push_cu8(blk)
        gfo, ofo = g.frequency_offset(), o.frequency_offset()
        for ch in range(n_ch):
            compare(g.read(ch), o.read(ch), gfo, ofo)
    out = [g.read(ch) for ch in range(n_ch)], g.frequency_offset()
    g.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("n_ports,cp_type,declared", [(1, 1, 1), (2, 1, 2), (2, 2, 2), (2, 1, 4)])
def test_tracker_matches_oracle_synthetic(lcs, ctx, n_ports, cp_type, declared):
    d = cell_dict(n_id_cell=277 if cp_type == 1 else 271, n_ports=n_ports, cp_type=cp_type)
    cu8 = S.synth_cu8(int(0.6 * FS), [d], f_true=3000.0, snr_db=10, seed=20 + n_ports + cp_type)
    (cells,), fo = run_pair(lcs, ctx, cu8[None], [[(lcs_cell(d, declared), d["t0"] - 2 + 0.6)]], 2700.0, 96000)
    if declared == n_ports:
        assert cells[0]["mib_successes"] == cells[0]["mib_attempts"] > 0


@pytest.mark.gpu
def test_tracker_real_capture(lcs, ctx, capbuf0000):
    """The recording framed and searched as the searcher cycle does; its cells handed to a tracker of the same stream
    before the first push, so that their frame timing refers to the tracker's own time stamps."""
    fc, fs = capbuf0000["fc"], 1.92e6
    real = capbuf0000["cu8"]
    full, _ = ctx.cell_search(real, lcs.f_search_set(fc, 120.0), fc, fc, fs)
    f_off = float(np.round(full[0].freq_superfine))
    lead = np.random.default_rng(5).integers(100, 156, size=(19200 + 777, 2), dtype=np.uint8)
    stream = np.concatenate([lead, real, lead])
    fr = lcs.Framer(fc, fc, fs, real.shape[0])
    fr.push(stream[:500], f_off)
    fr.request()
    got = None
    for lo in range(500, stream.shape[0], 10000):
        got = got or fr.push(stream[lo:lo + 10000], f_off)
    cap, late = got
    found = ctx.tracker_search_cu8(cap, f_off, fc, fc, fs, late)
    cells = [(c, ft % 19200) for c, ft in found if c.n_id_cell() in (277, 271)]
    assert sorted(c.n_id_cell() for c, _ in cells) == [271, 277]
    (res,), _ = run_pair(lcs, ctx, stream[None], [cells], f_off, 10000, fc=[fc])
    assert [r["n_id_cell"] for r in res] == [c.n_id_cell() for c, _ in cells]
    assert all(r["mib_successes"] > 0 for r in res)


@pytest.mark.gpu
def test_tracker_many_channels_match_single(lcs, ctx):
    rng = np.random.default_rng(9)
    n = int(0.25 * FS)
    n_ch = 16
    fcs = FC + 1e6 * np.arange(n_ch)
    cu8s, cells, fo0 = [], [], []
    for ch in range(n_ch):
        f_true = 1000.0 + 300 * ch
        ds = [cell_dict(n_id_cell=int(i), n_ports=int(rng.integers(1, 3)), cp_type=1, t0=float(rng.uniform(0, 19000)))
              for i in rng.choice(504, size=ch % 5, replace=False)]
        cu8s.append(S.synth_cu8(n, ds, f_true=f_true, fc=fcs[ch], snr_db=8, seed=100 + ch))
        cells.append([(lcs_cell(d), d["t0"] - 2 + 0.2) for d in ds])
        fo0.append(f_true - 100)
    cu8s = np.stack(cu8s)
    multi, fo_multi = run_pair(lcs, ctx, cu8s, cells, np.array(fo0), 48000, fc=fcs)
    for ch in (0, 3, 4, 9, 15):
        (single,), fo_single = run_pair(lcs, ctx, cu8s[ch:ch + 1], [cells[ch]], fo0[ch], 48000, fc=fcs[ch:ch + 1])
        assert fo_single[0] == fo_multi[ch]
        for a, b in zip(single, multi[ch]):
            for k in a:
                assert np.array_equal(np.asarray(a[k]), np.asarray(b[k]), equal_nan=True), k


@pytest.mark.gpu
def test_tracker_push_size_and_time_stamps(lcs, ctx):
    d = cell_dict()
    cu8 = S.synth_cu8(int(0.3 * FS), [d], f_true=2000.0, snr_db=10, seed=6)
    res = []
    for step in (10000, 7777, 10 ** 6):
        g = lcs.Tracker(ctx, FC, 1900.0)
        g.add_cell(0, lcs_cell(d), d["t0"] - 2 + 0.3)
        for i in range(0, cu8.shape[0], step):
            g.push_cu8(cu8[i:i + step])
        r = g.read(0)[0]
        res.append((g.frequency_offset()[0], g.sample_time(), r["frame_timing"], r["n_symbols"], r["ce"].tobytes(),
                    r["crs_np_av"].tobytes(), r["mib_attempts"]))
        g.close()
    assert res[0] == res[1] == res[2]
    # a framer fed block by block with the tracker's offsets keeps the same time stamps
    g = lcs.Tracker(ctx, FC, 1900.0)
    g.add_cell(0, lcs_cell(d), d["t0"] - 2 + 0.3)
    fr = lcs.Framer(FC, FC, 1.92e6)
    for i in range(0, cu8.shape[0] // 10000 * 10000, 10000):
        fo = g.frequency_offset()[0]
        g.push_cu8(cu8[i:i + 10000])
        fr.push(cu8[i:i + 10000], fo)
        assert g.sample_time() == fr.sample_time()


@pytest.mark.gpu
def test_tracker_drop_matches_oracle(lcs, ctx):
    rng = np.random.default_rng(5)
    n = int(16.4 * FS)
    cu8 = np.clip(np.round(127 + 128 * 0.1 * rng.standard_normal((n, 2))), 0, 255).astype(np.uint8)
    g = lcs.Tracker(ctx, FC, 0.0)
    g.add_cell(0, lcs_cell(cell_dict()), 100.0)
    o = TO.Tracker(FC, 0.0)
    o.add_cell(0, lcs_cell(cell_dict()), 100.0)
    for i in range(0, n, 1920000):
        g.push_cu8(cu8[i:i + 1920000])
        o.push_cu8(cu8[i:i + 1920000])
    gr, orr = g.read(0), o.read(0)
    compare(gr, orr, g.frequency_offset(), o.frequency_offset())
    assert gr[0]["dropped"] == 1 and gr[0]["mib_attempts"] == 1600
    assert g.read(0) == []


@pytest.mark.gpu
def test_tracker_bad_arguments(lcs, ctx):
    L = lcs
    g = L.Tracker(ctx, [FC, FC], 0.0, max_cells=1)
    launches = ctx.launches
    good = lcs_cell(cell_dict())
    with pytest.raises(L.LcsError, match="error 1"):
        g.add_cell(2, good, 100.0)
    for field, v in (("n_ports", 3), ("cp_type", 0), ("n_id_1", 168)):
        bad = lcs_cell(cell_dict())
        setattr(bad, field, v)
        with pytest.raises(L.LcsError, match="error 1"):
            g.add_cell(0, bad, 100.0)
    g.add_cell(0, good, 100.0)
    with pytest.raises(L.LcsError, match="error 1"):
        g.add_cell(0, good, 100.0)
    lib = L.lib()
    assert lib.lcs_track_add_cell(g._h, 0, None, 1.0) == 1
    assert lib.lcs_track_push_cu8(g._h, None, 5) == 1
    assert lib.lcs_track_frequency_offset(g._h, None) == 1
    assert lib.lcs_track_read(g._h, 5, None, 0, None) == 1
    assert ctx.launches == launches
    g.close()


@pytest.mark.gpu
def test_stream_search_cli_tracks_cells(lcs, ctx, tmp_path):
    """`StreamSearch_b200 -t N`: kalibrate, then framer + searcher cycles + the cell tracker on one stream; the searcher
    runs at the tracker's (moving) offset, the cell found is tracked with its MIB locked, and the offset stays on f_true."""
    import re
    import subprocess
    host = os.path.join(ROOT, "lte-cell-scanner_b200", "host")
    subprocess.check_call(["make", "-C", host, "-s"])
    f_true, d = 3000.0, cell_dict()
    S.synth_cu8(int(2 * FS), [d], f_true=f_true, snr_db=10, seed=30).tofile(str(tmp_path / "stream.bin"))
    out = subprocess.run([os.path.join(host, "StreamSearch_b200"), "-f", "739000000", "-n", "6", "-t", "50",
                          str(tmp_path / "stream.bin")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "Calibration succeeded!" in out.stdout
    assert re.search(r"cycle 0: new cell 277 ", out.stdout)
    searched = [float(v) for v in re.findall(r"searched at tracker offset ([-0-9.]+) Hz", out.stdout)]
    assert len(searched) == 6 and len(set(searched)) == 6          # the offset moves with the tracker's FOE
    status = [float(v) for v in re.findall(r"frequency offset ([-0-9.]+) Hz", out.stdout)]
    assert len(status) >= 3 and all(abs(f - f_true) < 5 for f in searched + status)
    rows = re.findall(r"cell 277  ports 2 .* MIB (\d+)/(\d+)  failures ([0-9.]+)", out.stdout)
    # the cell starts at slot 0 symbol 0 of the block after its hand-over, so its first MIB windows can straddle two PBCH
    # periods (failures of 0.25 each, tracker_thread.cpp:727-733); once locked no attempt fails
    lost = [int(n) - int(ok) for ok, n, _ in rows]
    assert len(rows) >= 3 and lost[0] <= 3 and len(set(lost)) == 1 and int(rows[-1][0]) > 40
    assert all(float(f) == 0 for _, _, f in rows)
    assert "new cell 277" not in out.stdout.split("cycle 1:", 1)[1]   # a tracked cell is on the skip list
