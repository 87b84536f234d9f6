"""CPU checks of the tracker oracle's channel autocorrelations (do_ac_fd / do_ac_td, tracker_thread.cpp:318-370) and of
the synthetic generator's multipath model they are tested on.  The streams are built here and shared with
tests/test_tracker_gpu.py."""
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "track_oracle"))

import lte_dl_synth as S  # noqa: E402
import track_oracle as TO  # noqa: E402
from test_tracker_oracle import FC, FS, cell_dict, lcs_cell  # noqa: E402

CN = np.concatenate([np.arange(-36, 0), np.arange(1, 37)])   # subcarrier of each of the 72 bins
F_TRUE = 3000.0
F_D = 40.0                      # Doppler of the second path of DOPPLER
D_TWO = 3.6                     # delay of the second path of TWO_PATHS, in samples at 1.92 Msps
G = 1 / np.sqrt(2)              # equal path gains, total power 1

# One path: the cell received as transmitted.
FLAT = dict(cell_dict(n_ports=1), paths=[(0.0, 1.0, 0.0)])
# Two equal static paths D_TWO samples apart.  The cell has an extended CP: the timing loop centres the DFT window on the
# paths' centroid, and only the 32-sample CP keeps both paths' symbols around a window that sits 2 samples before the
# CP's end (with the 9-sample normal CP the window would reach 0.8 samples into the next symbol).
TWO_PATHS = dict(cell_dict(n_id_cell=271, n_ports=1, cp_type=2), paths=[(0.0, G, 0.0), (D_TWO / FS, G, 0.0)])
# Two equal paths with the same delay, one Doppler-shifted by F_D: the channel fades to 0 every 1/F_D = 25 ms.
DOPPLER = dict(cell_dict(n_ports=1), paths=[(0.0, G, 0.0), (0.0, G, F_D)])


def stream(d, seconds, seed):
    """(cu8, handed-over frame timing at the paths' centroid, initial offset at the paths' mean Doppler)."""
    cu8 = S.synth_cu8(int(seconds * FS), [d], f_true=F_TRUE, snr_db=30, seed=seed)
    centroid = np.mean([p[0] for p in d["paths"]]) * FS
    return cu8, d["t0"] - 2 + 0.6 + centroid, F_TRUE + np.mean([p[2] for p in d["paths"]])


STREAMS = {"flat": (FLAT, 2.0, 41), "two_paths": (TWO_PATHS, 2.0, 42), "doppler": (DOPPLER, 3.0, 43)}


def coherence_bandwidth(ac_fd):
    """display_thread.cpp:166-177: the first lag k in 1..11 with |ac_fd[k]| <= 0.5 gives k * 90 kHz; None: > 990 kHz."""
    for k in range(1, 12):
        if abs(ac_fd[k]) <= 0.5:
            return 90 * k
    return None


def true_ac_fd(d):
    """The frequency autocorrelation the tracker estimates, from the true channel: at the 12 CRS subcarriers of each of
    the port's two CRS shifts, sum_t conj(H_t) H_{t+k} / (12 - k) over the mean of |H_t|^2, averaged over the shifts.
    The delays are taken relative to their centroid, where the timing loop puts the DFT window."""
    c = np.mean([p[0] for p in d["paths"]])
    out = 0
    for v in (d["n_id_cell"] % 6, (3 + d["n_id_cell"]) % 6):
        f = CN[v + 6 * np.arange(12)] * 15e3
        h = sum(g * np.exp(-2j * np.pi * f * (tau - c)) for tau, g, _ in d["paths"])
        out = out + np.array([np.sum(np.conj(h[:12 - k]) * h[k:]) / (12 - k) for k in range(12)]) / np.mean(abs(h) ** 2)
    return out / 2


def crs_estimates(n_symbols, cp_type=1):
    """Raw CRS estimates of port 0 that have passed do_ac_fd / do_ac_td after n_symbols symbols: the raw FIFO holds 3,
    and its middle entry is processed when the third arrives, so the first CRS symbol's estimate never is."""
    n_symb = 7 if cp_type == 1 else 6
    crs = sum(1 for s in range(n_symbols) if s % n_symb in (0, n_symb - 3))
    return max(crs - 2, 0)


@pytest.fixture(scope="module")
def runs():
    """Oracle reads after every 10000-sample push of each stream."""
    out = {}
    for name, (d, seconds, seed) in STREAMS.items():
        cu8, ft, fo = stream(d, seconds, seed)
        tr = TO.Tracker(FC, fo)
        tr.add_cell(0, lcs_cell(d), ft)
        hist = []
        for i in range(0, cu8.shape[0], 10000):
            tr.push_cu8(cu8[i:i + 10000])
            hist.append(tr.read(0)[0])
        out[name] = hist
    return out


def test_synth_without_paths_unchanged():
    """A cell without `paths`, or with the one path (0, 1, 0), gives the bytes the generator gave before it had a
    multipath model (the SHA-256 of that output)."""
    cells = [cell_dict(n_ports=1), cell_dict(n_id_cell=431, n_ports=4, cp_type=2, t0=7000.5)]
    want = "83bf1229d5a3368da468141d414d8de1a08acb73de3d9bae7edb533689f445f8"
    a = S.synth_cu8(100000, cells, f_true=3000.0, snr_db=10, seed=21)
    b = S.synth_cu8(100000, [dict(c, paths=[(0, 1, 0)]) for c in cells], f_true=3000.0, snr_db=10, seed=21)
    assert hashlib.sha256(a.tobytes()).hexdigest() == want
    assert np.array_equal(a, b)


def test_synth_path_delay_is_exact():
    """A path delayed by a whole number of samples is the undelayed signal shifted by that many samples (t0 off the
    sample grid, so that no sample sits on a symbol boundary, where rounding could pick either symbol)."""
    d = cell_dict(n_ports=2, t0=1234.25)
    t = np.arange(50000) / FS
    rng = np.random.default_rng(1)
    x0 = S._cells_baseband(t, [d], rng)
    rng = np.random.default_rng(1)
    x5 = S._cells_baseband(t, [dict(d, paths=[(5 / FS, 1.0, 0.0)])], rng)
    assert np.abs(x5[5:] - x0[:-5]).max() < 1e-9


def test_ac_flat_channel(runs):
    """One path at 30 dB: every lag of ac_fd is about 1 and the coherence bandwidth is > 990 kHz.  ac_td stays exactly 0
    until the port's 72nd estimate; from then on each estimate adds one update of weight 1 against 1/.00001, so
    1e5 * |ac_td[0]| counts the updates (each about 1 here)."""
    hist = runs["flat"]
    r = hist[-1]
    # At 30 dB np/sp is about 1e-3, so each CRS symbol moves ac_fd[k] by 500 (12 - k) / 1e5 of the way: converged after
    # 2 s (4000 updates).  The per-lag estimates scatter by 0.3 % in the oracle run; 2 % leaves room for other seeds.
    assert np.all(np.abs(np.abs(r["ac_fd"]) - 1) < 0.02), np.abs(r["ac_fd"])
    assert coherence_bandwidth(r["ac_fd"]) is None
    assert r["mib_successes"] == r["mib_attempts"] > 0
    seen_zero = seen_update = False
    for h in hist:
        u = crs_estimates(h["n_symbols"]) - 71
        if u <= 0:
            assert not np.any(h["ac_td"]), h["n_symbols"]
            seen_zero = True
        else:
            assert np.all(h["ac_td"] != 0)
            assert abs(1e5 * abs(h["ac_td"][0]) / u - 1) < 0.05 or u > 1000
            seen_update = True
    assert seen_zero and seen_update


def test_ac_fd_two_paths(runs):
    """Two equal static paths 3.6 samples (1.875 us) apart.  The reference's rule on the true channel gives 180 kHz with
    both deciding lags clear of the 0.5 threshold; the oracle's ac_fd gives the same, and its shape follows the true
    channel's."""
    ref = true_ac_fd(TWO_PATHS)
    assert coherence_bandwidth(ref) == 180
    assert abs(abs(ref[1]) - 0.5) >= 0.1 and abs(abs(ref[2]) - 0.5) >= 0.1
    r = runs["two_paths"][-1]
    assert coherence_bandwidth(r["ac_fd"]) == 180
    # The tracker normalises by sp = tp - np/7 of the filtered estimate.  On this frequency-selective channel filter_ce
    # smooths away part of the power, so sp is low by a constant factor and every lag reads high by it (the oracle run:
    # ac_fd[0] = 1.14); relative to lag 0 the oracle follows the true shape within 0.007 (at lag 11, which has one
    # product per symbol).  0.03 leaves room for other seeds.
    got = np.abs(r["ac_fd"]) / abs(r["ac_fd"][0])
    assert np.abs(got - np.abs(ref)).max() < 0.03, (got, np.abs(ref))
    assert 1 < abs(r["ac_fd"][0]) < 1.25
    assert r["mib_successes"] == r["mib_attempts"] > 0


def test_ac_td_doppler(runs):
    """Two equal paths, one Doppler-shifted by 40 Hz: over even lags t (whole slots, 0.5 ms per 2 lags) the magnitude of
    ac_td relative to lag 0 follows |cos(pi f_d t 0.25 ms)|, the normalised autocorrelation of the channel, which reaches
    0 at lag 50.  The MIB stays locked through the fades."""
    r = runs["doppler"][-1]
    assert r["mib_successes"] == r["mib_attempts"] > 0 and r["mib_decode_failures"] == 0
    t = np.arange(0, 72, 2)
    got = np.abs(r["ac_td"][t]) / abs(r["ac_td"][0])
    want = np.abs(np.cos(np.pi * F_D * t * 0.25e-3))
    # The reference divides each symbol's correlation by that symbol's own signal power, so each update is about
    # h(t - tau) / h(t).  For two equal paths that ratio is singular at the fades, where only the noise bounds it: the
    # fades add noise-over-signal terms to lag 0 (lag 2 reads 0.92 instead of 1.00) and a bias that moves the first
    # minimum from lag 50 to lag 66.  The fades fall on the same symbols every 25 ms (50 slots), so the bias does not
    # average out.  Largest error over the even lags: 0.50 in this run (0.36 with another seed), at lags 50 to 60.  The
    # tolerance holds that shape and no more; the flat start and the minimum are checked on their own.
    assert np.abs(got - want).max() < 0.6, np.round(got, 3)
    assert np.all(got[t <= 20] > 0.85)                              # about flat over the first 5 ms
    assert got.min() < 0.15 and 50 <= t[np.argmin(got)] <= 70      # a minimum at or after the cosine's first zero
