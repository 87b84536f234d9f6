"""The device cell tracker (lcs_track_*) against its CPU oracle (track_oracle/), on synthetic and recorded streams."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "track_oracle"))

import lte_dl_synth as S  # noqa: E402
import track_oracle as TO  # noqa: E402
from lcs_b200 import TrackCell  # noqa: E402
from test_search_chain_gpu import compare_cells  # noqa: E402
from test_tracker_ac_oracle import STREAMS, crs_estimates, stream  # noqa: E402
from test_tracker_oracle import FC, FS, cell_dict, lcs_cell, true_frame_timing  # noqa: E402

# Every field of lcs_track_cell is in exactly one of these classes, each with its own tolerance.
DISCRETE = ("n_id_cell", "n_ports", "cp_type", "dropped", "drop_sample", "n_symbols", "last_slice_start", "mib_attempts",
            "mib_successes", "mib_decode_failures")
MEAS = ("crs_tp", "crs_sp_raw", "crs_np", "crs_tp_av", "crs_sp_raw_av", "crs_np_av", "sync_tp", "sync_sp", "sync_np",
        "sync_np_blank", "sync_tp_av", "sync_sp_av", "sync_np_av", "sync_np_blank_av")
COMPLEX = ("ce", "sync_ce", "ac_fd", "ac_td")


def compare(g, o, gfo, ofo):
    """Device reads g against oracle reads o, field by field over TrackCell: discrete values exactly, frame_timing to
    1e-9, measurements to 1e-9 relative with the same NaNs, complex arrays to 1e-9 of the oracle array's largest
    magnitude.  A field in no class fails, so that a new field of lcs_track_cell cannot go unchecked."""
    assert np.abs(gfo - ofo).max() < 1e-6
    assert len(g) == len(o)
    for a, b in zip(g, o):
        for k, _ in TrackCell._fields_:
            if k in DISCRETE:
                assert a[k] == b[k], k
            elif k == "frame_timing":
                assert abs(a[k] - b[k]) < 1e-9, k
            elif k in MEAS:
                x, y = np.asarray(a[k], float), np.asarray(b[k], float)
                assert np.array_equal(np.isnan(x), np.isnan(y)), k
                m = ~np.isnan(y)
                assert np.all(np.abs(x[m] - y[m]) <= 1e-9 * np.maximum(np.abs(y[m]), 1e-30)), k
            elif k in COMPLEX:
                assert np.abs(a[k] - b[k]).max() <= 1e-9 * max(np.abs(b[k]).max(), 1e-30), k
            else:
                pytest.fail(f"lcs_track_cell field {k} has no comparison class")


def run_pair(lcs, ctx, cu8s, cells, fo0, step, fc=None, max_cells=4, fc_programmed=None, fs_programmed=1.92e6,
             history=None):
    """cu8s: [n_ch][n][2]; cells: per channel list of (lcs_cell, frame_timing).  Compares after every push; each push's
    device read of every channel is appended to `history` when one is given."""
    n_ch = len(cu8s)
    fc = np.full(n_ch, FC) if fc is None else np.asarray(fc)
    g = lcs.Tracker(ctx, fc, fo0, fs_programmed=fs_programmed, fc_programmed=fc_programmed, max_cells=max_cells)
    o = TO.Tracker(fc, fo0, fs_programmed=fs_programmed, fc_programmed=fc_programmed, max_cells=max_cells)
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
        reads = [g.read(ch) for ch in range(n_ch)]
        for ch in range(n_ch):
            compare(reads[ch], o.read(ch), gfo, ofo)
        if history is not None:
            history.append(reads)
    out = [g.read(ch) for ch in range(n_ch)], g.frequency_offset()
    g.close()
    return out


def read_raw(read_fn, h, ch, m):
    """lcs_track_read / to_read with room for m cells."""
    import ctypes as C
    out = (TrackCell * m)()
    n = C.c_uint32(0)
    assert read_fn(h, ch, out, m, C.byref(n)) == 0
    return [out[i].as_dict() for i in range(n.value)]


# Cells of the tiled stream: one of each kind the tracker distinguishes (1, 2 and 4 ports; normal and extended CP), at
# distinct CRS shifts (n_id_cell % 6).  Cell "a" is the strongest; the others, 3 to 4.5 dB down, still lock their MIB
# under its interference.
TILE_CELLS = dict(
    a=dict(cell_dict(n_id_cell=277, n_ports=2, t0=1234.0), gains=[1.0, 0.8 * np.exp(0.7j)]),
    c=dict(cell_dict(n_id_cell=100, n_ports=1, t0=7000.0), gains=[0.7]),
    d=dict(cell_dict(n_id_cell=431, n_ports=4, t0=15000.0), gains=[0.6, 0.5j, -0.55, 0.45 * np.exp(-2j)]),
    e=dict(cell_dict(n_id_cell=62, n_ports=2, cp_type=2, t0=11000.5), gains=[0.7, -0.5]),
)


@pytest.fixture(scope="module")
def tile():
    """20 frames (five PBCH periods) of the TILE_CELLS at f_true = 0.  With k = 1 every sample falls on the grid of the
    frame, so repeats of the tile form one continuous, exactly periodic stream of any length."""
    return S.synth_cu8(20 * 19200, list(TILE_CELLS.values()), f_true=0.0, snr_db=10, seed=9)


@pytest.mark.gpu
@pytest.mark.parametrize("n_ports,cp_type,declared", [(1, 1, 1), (2, 1, 2), (2, 2, 2), (2, 1, 4), (4, 1, 4), (4, 2, 4)])
def test_tracker_matches_oracle_synthetic(lcs, ctx, n_ports, cp_type, declared):
    """Every autocorrelation lag ends non-zero; with 4 ports declared on a 2-port cell, ports 2 and 3 see no CRS and their
    sp is clamped to 1e-5."""
    d = cell_dict(n_id_cell=277 if cp_type == 1 else 271, n_ports=n_ports, cp_type=cp_type)
    cu8 = S.synth_cu8(int(0.6 * FS), [d], f_true=3000.0, snr_db=10, seed=20 + n_ports + cp_type)
    (cells,), fo = run_pair(lcs, ctx, cu8[None], [[(lcs_cell(d, declared), d["t0"] - 2 + 0.6)]], 2700.0, 96000)
    if declared == n_ports:
        assert cells[0]["mib_successes"] == cells[0]["mib_attempts"] > 0
    assert np.all(cells[0]["ac_td"] != 0) and np.all(cells[0]["ac_fd"] != 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(STREAMS))
def test_ac_matches_oracle_multipath(lcs, ctx, name):
    """The flat, two-path and Doppler streams of test_tracker_ac_oracle.py."""
    d, seconds, seed = STREAMS[name]
    cu8, ft, fo = stream(d, seconds, seed)
    ((r,),), _ = run_pair(lcs, ctx, cu8[None], [[(lcs_cell(d), ft)]], fo, 192000)
    assert r["mib_successes"] == r["mib_attempts"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("cp_type", [1, 2])
def test_cell_search_four_port_cell_matches_oracle(ctx, oracle, cp_type):
    """The searcher's four-port MIB decode (SFBC-FSTD combining, CRC mask) on the captures of
    test_synthetic_cell_found_by_oracle_search, field by field against the oracle."""
    d = cell_dict(n_id_cell=277 if cp_type == 1 else 271, n_ports=4, cp_type=cp_type)
    cu8 = S.synth_cu8(153600, [d], f_true=3000.0, snr_db=10, seed=4 * 10 + cp_type)
    f = np.arange(-10000, 10001, 5000.0)
    o_cells, o_peaks = oracle.cell_search_one(S.to_c128(cu8), f, FC, FC, FS)
    p_cells, p_peaks = ctx.cell_search(cu8, f, FC, FC, FS)
    compare_cells(p_peaks, o_peaks)
    assert [c.n_id_cell() for c in o_cells] == [d["n_id_cell"]]
    compare_cells(p_cells, o_cells)
    assert (p_cells[0].n_ports, p_cells[0].cp_type, p_cells[0].sfn) == (4, cp_type, 100)


@pytest.mark.gpu
def test_tracker_frame_timing_wrap_matches_oracle(lcs, ctx):
    """A frame start 0.2 samples after the wrap, handed over 0.4 samples early (at 19199.8): the timing loop carries it
    across 19200 -> 0 and, as the time stamps drift, back across 0 -> 19200."""
    d = cell_dict(t0=2.2)
    cu8 = S.synth_cu8(int(0.6 * FS), [d], f_true=3000.0, snr_db=10, seed=8)
    hist = []
    (cells,), _ = run_pair(lcs, ctx, cu8[None], [[(lcs_cell(d), (d["t0"] - 2 - 0.4) % 19200)]], 2700.0, 48000,
                           history=hist)
    ft = np.array([h[0][0]["frame_timing"] for h in hist])
    first_low = np.flatnonzero(ft < 1)
    assert first_low.size and np.any(ft[first_low[0]:] > 19199.9)
    assert cells[0]["mib_successes"] == cells[0]["mib_attempts"] > 0


@pytest.mark.gpu
def test_tracker_programmed_rates_match_oracle(lcs, ctx):
    """A tuner that reports a programmed carrier and sample rate other than the requested ones: both enter the time
    stamps and get_fd through k = (fc_requested - f) / fc_programmed."""
    fcp, fsp = FC - 2500.0, 1.92e6 * (1 + 4e-6)
    d = cell_dict()
    cu8 = S.synth_cu8(int(0.6 * FS), [d], f_true=3000.0, fc_programmed=fcp, fs_programmed=fsp, snr_db=10, seed=7)
    (cells,), _ = run_pair(lcs, ctx, cu8[None], [[(lcs_cell(d), d["t0"] - 2 + 0.6)]], 2700.0, 96000,
                           fc_programmed=[fcp], fs_programmed=fsp)
    assert cells[0]["mib_successes"] == cells[0]["mib_attempts"] > 0


@pytest.mark.gpu
def test_tracker_full_channel_matches_oracle(lcs, ctx, tile):
    """max_cells = 32: channel 0 fills all 32 slots (the four cells on the air, spread over the slots so that every pass
    of the kernel's warp loop has one, between absent ids declaring 1, 2 and 4 ports), channel 1 tracks three."""
    rng = np.random.default_rng(11)
    on_air = {3: "a", 12: "d", 21: "e", 30: "c"}
    absent = [int(i) for i in rng.permutation(504) if i not in (277, 100, 431, 62, 271)]
    cells0 = []
    for slot in range(32):
        if slot in on_air:
            d = TILE_CELLS[on_air[slot]]
            cells0.append((lcs_cell(d), d["t0"] - 2 + 0.6))
        else:
            d = cell_dict(n_id_cell=absent.pop(), n_ports=(1, 2, 4)[slot % 3], cp_type=1 + (slot % 5 == 0))
            cells0.append((lcs_cell(d), float(rng.uniform(0, 19200))))
    d1 = cell_dict(n_id_cell=271, n_ports=4, cp_type=2, t0=3333.0)
    ch1 = S.synth_cu8(2 * tile.shape[0], [d1], f_true=1500.0, fc=FC + 5e6, snr_db=10, seed=12)
    cells1 = [(lcs_cell(d1), d1["t0"] - 2 + 0.6), (lcs_cell(cell_dict(n_id_cell=5, n_ports=1)), 4000.0),
              (lcs_cell(cell_dict(n_id_cell=6, n_ports=2, cp_type=2)), 19100.0)]
    cu8s = np.stack([np.concatenate([tile, tile]), ch1])
    res, _ = run_pair(lcs, ctx, cu8s, [cells0, cells1], np.array([-300.0, 1200.0]), 96000, fc=[FC, FC + 5e6],
                      max_cells=32)
    assert [r["n_id_cell"] for r in res[0]] == [c.n_id_cell() for c, _ in cells0]
    for slot, r in enumerate(res[0]):
        assert r["mib_attempts"] > 0
        assert (r["mib_successes"] == r["mib_attempts"]) == (slot in on_air)
    assert len(res[1]) == 3 and res[1][0]["mib_successes"] == res[1][0]["mib_attempts"] > 0


@pytest.mark.gpu
def test_tracker_drop_in_the_middle_then_reuse_slot(lcs, ctx, tile):
    """Cells a, b, c where b is not on the air: b drops after 1600 attempts while a and c stay locked.  A read with room
    for one cell leaves the unreported drop in place; the next full read reports it and frees its slot, c moves down,
    and d (four ports) is added into the freed slot and tracked for about a second."""
    n_tiles = int(np.ceil(18.0 * FS / tile.shape[0]))
    cu8 = np.concatenate([tile] * n_tiles)
    a, c, d = TILE_CELLS["a"], TILE_CELLS["c"], TILE_CELLS["d"]
    b = cell_dict(n_id_cell=11, n_ports=2)
    g = lcs.Tracker(ctx, FC, -200.0, max_cells=3)
    o = TO.Tracker(FC, -200.0, max_cells=3)
    for x, ft in ((a, a["t0"] - 2 + 0.6), (b, 5000.0), (c, c["t0"] - 2 - 0.5)):
        g.add_cell(0, lcs_cell(x), ft)
        o.add_cell(0, lcs_cell(x), ft)
    added_at = None
    step = 1920000
    for i in range(0, cu8.shape[0], step):
        g.push_cu8(cu8[i:i + step])
        o.push_cu8(cu8[i:i + step])
        gfo, ofo = g.frequency_offset(), o.frequency_offset()
        first = read_raw(lcs.lib().lcs_track_read, g._h, 0, 1)
        compare(first, read_raw(TO.lib().to_read, o._h, 0, 1), gfo, ofo)
        assert [r["n_id_cell"] for r in first] == [277]
        gr, orr = g.read(0), o.read(0)
        compare(gr, orr, gfo, ofo)
        ids = [r["n_id_cell"] for r in gr]
        if added_at is None:
            assert ids == [277, 11, 100]
            assert gr[0]["mib_successes"] == gr[0]["mib_attempts"] and gr[2]["mib_successes"] == gr[2]["mib_attempts"]
            if gr[1]["dropped"]:
                assert gr[1]["mib_attempts"] == 1600 and gr[1]["mib_successes"] == 0
                ft = true_frame_timing(g, d, i + step, 0.0)
                g.add_cell(0, lcs_cell(d), ft)
                o.add_cell(0, lcs_cell(d), ft)
                added_at = i + step
            else:
                assert gr[1]["mib_attempts"] < 1600
        else:
            assert ids == [277, 100, 431] and not any(r["dropped"] for r in gr)
    assert added_at is not None and cu8.shape[0] - added_at >= 0.9 * FS
    assert all(r["mib_successes"] == r["mib_attempts"] > 0 for r in gr)
    g.close()


@pytest.fixture(scope="module")
def real_capture_handover(lcs, ctx, capbuf0000):
    """The recording framed and searched as the searcher cycle does; cells 277 and 271 with their frame timing in the
    time stamps of a tracker that starts on the same stream.  (stream, cells, f_off, fc)."""
    fc, fs = capbuf0000["fc"], 1.92e6
    real = capbuf0000["cu8"]
    full, _ = ctx.cell_search(real, lcs.f_search_set(fc, 120.0), fc, fc, fs)
    f_off = float(np.round(full[0].freq_superfine))
    lead = np.random.default_rng(5).integers(100, 156, size=(19200 + 777, 2), dtype=np.uint8)
    st = np.concatenate([lead, real, lead])
    fr = lcs.Framer(fc, fc, fs, real.shape[0])
    fr.push(st[:500], f_off)
    fr.request()
    got = None
    for lo in range(500, st.shape[0], 10000):
        got = got or fr.push(st[lo:lo + 10000], f_off)
    cap, late = got
    found = ctx.tracker_search_cu8(cap, f_off, fc, fc, fs, late)
    cells = [(c, ft % 19200) for c, ft in found if c.n_id_cell() in (277, 271)]
    assert sorted(c.n_id_cell() for c, _ in cells) == [271, 277]
    return st, cells, f_off, fc


@pytest.mark.gpu
def test_tracker_real_capture(lcs, ctx, real_capture_handover):
    """The recording's cells handed to a tracker of the same stream before the first push."""
    st, cells, f_off, fc = real_capture_handover
    (res,), _ = run_pair(lcs, ctx, st[None], [cells], f_off, 10000, fc=[fc])
    assert [r["n_id_cell"] for r in res] == [c.n_id_cell() for c, _ in cells]
    assert all(r["mib_successes"] > 0 for r in res)
    assert all(np.any(r["ac_fd"]) for r in res)


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
    # a framer fed block by block with the tracker's offsets keeps the same time stamps; every push completes a block,
    # so it is one kernel launch, which a timing read reports once
    g = lcs.Tracker(ctx, FC, 1900.0)
    g.add_cell(0, lcs_cell(d), d["t0"] - 2 + 0.3)
    fr = lcs.Framer(FC, FC, 1.92e6)
    for i in range(0, cu8.shape[0] // 10000 * 10000, 10000):
        fo = g.frequency_offset()[0]
        g.push_cu8(cu8[i:i + 10000])
        fr.push(cu8[i:i + 10000], fo)
        assert g.sample_time() == fr.sample_time()
        ms, launches = g.timing_read()
        assert launches == 1 and ms > 0
    g.push_cu8(cu8[:9999])                          # completes no block: no launch
    assert g.timing_read() == (0.0, 0)


@pytest.mark.gpu
def test_tracker_drop_matches_oracle(lcs, ctx):
    """A cell on noise drops with a full CE history and non-zero autocorrelations.  A cell added into the freed slot
    reads zero arrays, keeps ac_fd 0 until its first estimate and ac_td exactly 0 until its own 72nd (so no entry of the
    old history is used)."""
    rng = np.random.default_rng(5)

    def noise(n):
        return np.clip(np.round(127 + 128 * 0.1 * rng.standard_normal((n, 2))), 0, 255).astype(np.uint8)

    n = int(16.4 * FS)
    cu8 = noise(n)
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
    assert np.all(gr[0]["ac_td"] != 0) and np.all(gr[0]["ac_fd"] != 0)
    assert g.read(0) == []
    for t in (g, o):
        t.add_cell(0, lcs_cell(cell_dict(n_id_cell=11)), 5000.0)
    (r,) = g.read(0)
    compare([r], o.read(0), g.frequency_offset(), o.frequency_offset())
    assert r["n_symbols"] == 0 and not np.any(r["ac_fd"]) and not np.any(r["ac_td"])
    more = noise(int(0.2 * FS))
    seen = set()
    for i in range(0, more.shape[0], 10000):
        g.push_cu8(more[i:i + 10000])
        o.push_cu8(more[i:i + 10000])
        (r,) = g.read(0)
        compare([r], o.read(0), g.frequency_offset(), o.frequency_offset())
        u = crs_estimates(r["n_symbols"]) - 71
        seen.add(u > 0)
        assert np.any(r["ac_fd"]) == (crs_estimates(r["n_symbols"]) > 0)   # the first symbols may come in later blocks
        if u <= 0:
            assert not np.any(r["ac_td"]), r["n_symbols"]
        else:
            assert np.all(r["ac_td"] != 0)
    assert seen == {False, True}
    g.close()


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
    runs at the tracker's (moving) offset, the cell found is tracked with its MIB locked, and the offset stays on f_true.
    `-x` adds under each status line of cell 277 the UOS power, one SP/NP/SNR + coherence bandwidth line per port and
    the PSS/SSS line, and changes nothing else."""
    host = os.path.join(ROOT, "lte-cell-scanner_b200", "host")
    subprocess.check_call(["make", "-C", host, "-s"])
    f_true, d = 3000.0, cell_dict()
    S.synth_cu8(int(2 * FS), [d], f_true=f_true, snr_db=10, seed=30).tofile(str(tmp_path / "stream.bin"))

    def run(*opts):
        r = subprocess.run([os.path.join(host, "StreamSearch_b200"), "-f", "739000000", "-n", "6", "-t", "50", *opts,
                            str(tmp_path / "stream.bin")], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr + r.stdout
        return r.stdout

    out, expert = run(), run("-x")
    assert "Calibration succeeded!" in out
    assert re.search(r"cycle 0: new cell 277 ", out)
    searched = [float(v) for v in re.findall(r"searched at tracker offset ([-0-9.]+) Hz", out)]
    assert len(searched) == 6 and len(set(searched)) == 6          # the offset moves with the tracker's FOE
    status = [float(v) for v in re.findall(r"frequency offset ([-0-9.]+) Hz", out)]
    assert len(status) >= 3 and all(abs(f - f_true) < 5 for f in searched + status)
    rows = re.findall(r"cell 277  ports 2 .* MIB (\d+)/(\d+)  failures ([0-9.]+)", out)
    # the cell starts at slot 0 symbol 0 of the block after its hand-over, so its first MIB windows can straddle two PBCH
    # periods (failures of 0.25 each, tracker_thread.cpp:727-733); once locked no attempt fails
    lost = [int(n) - int(ok) for ok, n, _ in rows]
    assert len(rows) >= 3 and lost[0] <= 3 and len(set(lost)) == 1 and int(rows[-1][0]) > 40
    assert all(float(f) == 0 for _, _, f in rows)
    assert "new cell 277" not in out.split("cycle 1:", 1)[1]   # a tracked cell is on the skip list
    blocks = re.findall(r"  cell 277  ports 2 .*\n    UOS pwr +[-0-9.]+ dB\n((?:    P\d .*\n)+)    S  SP/NP/SNR .*\n",
                        expert)
    assert len(blocks) >= 3, expert
    for b in blocks:
        ports = re.findall(r"    P(\d) SP/NP/SNR +[-0-9.]+/ *[-0-9.]+/ *[-0-9.]+ dB  CB (\d+ kHz|>990 kHz)\n", b)
        assert [p for p, _ in ports] == ["0", "1"], b
    plain = [ln for ln in expert.splitlines() if not re.match(r"    (UOS pwr|P\d SP/NP/SNR|S  SP/NP/SNR) ", ln)]
    assert plain == out.splitlines()
