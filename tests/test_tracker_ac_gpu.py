"""The device tracker's channel autocorrelations (ac_fd / ac_td of lcs_track_cell) against the CPU oracle, after every
push, together with every other output."""
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
from test_tracker_ac_oracle import STREAMS, crs_estimates, stream  # noqa: E402
from test_tracker_gpu import compare  # noqa: E402
from test_tracker_oracle import FC, FS, cell_dict, lcs_cell  # noqa: E402


def compare_ac(g, o, gfo, ofo):
    """Every field of test_tracker_gpu.compare, and ac_fd / ac_td to 1e-9 of the oracle array's largest magnitude."""
    compare(g, o, gfo, ofo)
    for a, b in zip(g, o):
        for k in ("ac_fd", "ac_td"):
            assert np.abs(a[k] - b[k]).max() <= 1e-9 * max(np.abs(b[k]).max(), 1e-30), k


def run_pair_ac(lcs, ctx, cu8, cells, fo0, step, fc=FC):
    """One channel, device and oracle side by side, compared after every push; returns the last device read."""
    g = lcs.Tracker(ctx, fc, fo0)
    o = TO.Tracker(fc, fo0)
    for c, ft in cells:
        g.add_cell(0, c, ft)
        o.add_cell(0, c, ft)
    for i in range(0, cu8.shape[0], step):
        g.push_cu8(cu8[i:i + step])
        o.push_cu8(cu8[i:i + step])
        res = g.read(0)
        compare_ac(res, o.read(0), g.frequency_offset(), o.frequency_offset())
    g.close()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("n_ports,cp_type,declared", [(1, 1, 1), (2, 1, 2), (2, 2, 2), (2, 1, 4), (4, 1, 4), (4, 2, 4)])
def test_ac_matches_oracle_synthetic(lcs, ctx, n_ports, cp_type, declared):
    """The streams of test_tracker_matches_oracle_synthetic; with 4 ports declared on a 2-port cell, ports 2 and 3 see
    no CRS and their sp is clamped to 1e-5."""
    d = cell_dict(n_id_cell=277 if cp_type == 1 else 271, n_ports=n_ports, cp_type=cp_type)
    cu8 = S.synth_cu8(int(0.6 * FS), [d], f_true=3000.0, snr_db=10, seed=20 + n_ports + cp_type)
    (r,) = run_pair_ac(lcs, ctx, cu8, [(lcs_cell(d, declared), d["t0"] - 2 + 0.6)], 2700.0, 96000)
    assert np.all(r["ac_td"] != 0) and np.all(r["ac_fd"] != 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(STREAMS))
def test_ac_matches_oracle_multipath(lcs, ctx, name):
    """The flat, two-path and Doppler streams of test_tracker_ac_oracle.py."""
    d, seconds, seed = STREAMS[name]
    cu8, ft, fo = stream(d, seconds, seed)
    (r,) = run_pair_ac(lcs, ctx, cu8, [(lcs_cell(d), ft)], fo, 192000)
    assert r["mib_successes"] == r["mib_attempts"] > 0


@pytest.mark.gpu
def test_ac_matches_oracle_real_capture(lcs, ctx, capbuf0000):
    """The recording with cells 277 and 271, set up as in test_tracker_real_capture."""
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
    res = run_pair_ac(lcs, ctx, st, cells, f_off, 10000, fc=fc)
    assert all(np.any(r["ac_fd"]) for r in res)


@pytest.mark.gpu
def test_ac_reset_in_reused_slot(lcs, ctx):
    """A cell dropped on noise leaves its slot with a full CE history and non-zero arrays.  A cell added into the freed
    slot reads zero arrays, keeps ac_fd 0 until its first estimate and ac_td exactly 0 until its own 72nd (so no
    entry of the old history is used)."""
    rng = np.random.default_rng(5)
    n = int(16.4 * FS)
    cu8 = np.clip(np.round(127 + 128 * 0.1 * rng.standard_normal((n, 2))), 0, 255).astype(np.uint8)
    g = lcs.Tracker(ctx, FC, 0.0, max_cells=1)
    g.add_cell(0, lcs_cell(cell_dict(n_ports=1)), 100.0)
    g.push_cu8(cu8)
    (old,) = g.read(0)
    assert old["dropped"] == 1 and np.all(old["ac_td"] != 0) and np.all(old["ac_fd"] != 0)
    assert g.read(0) == []
    g.add_cell(0, lcs_cell(cell_dict(n_id_cell=11, n_ports=1)), 5000.0)
    (new,) = g.read(0)
    assert new["n_symbols"] == 0 and not np.any(new["ac_fd"]) and not np.any(new["ac_td"])
    more = np.clip(np.round(127 + 128 * 0.1 * rng.standard_normal((int(0.2 * FS), 2))), 0, 255).astype(np.uint8)
    seen = set()
    for i in range(0, more.shape[0], 10000):
        g.push_cu8(more[i:i + 10000])
        (r,) = g.read(0)
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
def test_stream_search_cli_expert(lcs, ctx, tmp_path):
    """`StreamSearch_b200 -t 50 -x` on the stream of test_stream_search_cli_tracks_cells: under each status line of
    cell 277 the UOS power, one SP/NP/SNR + coherence bandwidth line per port, and the PSS/SSS line."""
    host = os.path.join(ROOT, "lte-cell-scanner_b200", "host")
    subprocess.check_call(["make", "-C", host, "-s"])
    d = cell_dict()
    S.synth_cu8(int(2 * FS), [d], f_true=3000.0, snr_db=10, seed=30).tofile(str(tmp_path / "stream.bin"))
    out = subprocess.run([os.path.join(host, "StreamSearch_b200"), "-f", "739000000", "-n", "6", "-t", "50", "-x",
                          str(tmp_path / "stream.bin")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    blocks = re.findall(r"  cell 277  ports 2 .*\n    UOS pwr +[-0-9.]+ dB\n((?:    P\d .*\n)+)    S  SP/NP/SNR .*\n",
                        out.stdout)
    assert len(blocks) >= 3, out.stdout
    for b in blocks:
        ports = re.findall(r"    P(\d) SP/NP/SNR +[-0-9.]+/ *[-0-9.]+/ *[-0-9.]+ dB  CB (\d+ kHz|>990 kHz)\n", b)
        assert [p for p, _ in ports] == ["0", "1"], b
