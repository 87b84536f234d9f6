"""The wideband channelizer's contract without a GPU: the prototype filter, a float64 restatement of the channelizer (the
oracle the GPU tests compare against), the wideband test generator and the CLI's argument checks."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "track_oracle"))

import lte_dl_synth as S  # noqa: E402

FS_CH = 1920000
PASS_HZ, STOP_HZ, PASS_DB, STOP_DB = 0.70e6, 1.22e6, 0.01, 70.0


# ---- the oracle: section 1 of the channelizer contract in float64 -------------------------------------------------------
def n_outputs(n, D, M):
    return max(0, (n - 1 - M) // D + 1)


def mix(iq, fs_in, fc_in, fc):
    """x[m] exp(-j2pi p[m]/fs_in), p[m] = (m * delta) mod fs_in in exact integers."""
    fs = int(round(fs_in))
    delta = int(round(fc - fc_in))
    x = (iq[:, 0].astype(np.float64) + 1j * iq[:, 1].astype(np.float64)) / 32768
    p = (np.arange(iq.shape[0], dtype=np.int64) * delta) % fs
    return x * np.exp(-2j * np.pi * p / fs)


def chan_oracle(iq, fs_in, fc_in, fc_ch, h):
    """y [n_ch][n_out] complex128: y_c[n] = sum_k h[k+M] x~_c[nD-k], x~ = 0 before the stream."""
    D = int(round(fs_in / FS_CH))
    M = (h.size - 1) // 2
    n_out = n_outputs(iq.shape[0], D, M)
    hd = h.astype(np.float64)
    ys = []
    for fc in np.atleast_1d(fc_ch):
        xm = np.concatenate([np.zeros(M, complex), mix(iq, fs_in, fc_in, fc)])   # index i <-> stream sample i - M
        y = np.zeros(n_out, complex)
        base = np.arange(n_out) * D + 2 * M                  # stream sample nD + M - t at padded index nD + 2M - t
        for t in range(h.size):
            y += hd[t] * xm[base - t]
        ys.append(y)
    return np.array(ys).reshape(len(ys), n_out)


def auto_gain_oracle(y):
    ms = np.mean(np.abs(y) ** 2, axis=-1)
    return np.where(ms > 0, 0.25 / np.sqrt(np.where(ms > 0, ms, 1)), 1.0).astype(np.float32)


def quantise(y, gain):
    """(cu8 [n_ch][n][2], n_clipped [n_ch], v float64 [n_ch][n][2])."""
    g = np.asarray(gain, np.float64).reshape(-1, 1, 1)
    v = 127 + 128 * g * np.stack([y.real, y.imag], axis=-1)
    r = np.rint(v)
    clipped = ((r < 0) | (r > 255)).sum(axis=(1, 2))
    return np.clip(r, 0, 255).astype(np.uint8), clipped, v


class OracleStream:
    """The oracle fed push by push: output n is emitted once sample nD+M has arrived."""

    def __init__(self, fs_in, fc_in, fc_ch, h):
        self.args = (fs_in, fc_in, fc_ch, h)
        self.D = int(round(fs_in / FS_CH))
        self.M = (h.size - 1) // 2
        self.iq = np.zeros((0, 2), np.int16)
        self.done = 0

    def push(self, iq):
        self.iq = np.concatenate([self.iq, iq])
        k = n_outputs(self.iq.shape[0], self.D, self.M)
        y = chan_oracle(self.iq, *self.args)[:, self.done:k]
        self.done = k
        return y


# ---- the prototype filter ------------------------------------------------------------------------------------------------
def response_db(h, fs):
    """|H| in dB on the grid of lcs_chan_design_taps: every fs/(64L) in [0, 0.70 MHz] and [1.22 MHz, fs/2], band edges
    included.  Returns (passband dB, stopband dB)."""
    L = h.size
    M = (L - 1) // 2
    step = fs / (64.0 * L)
    fp = np.append(np.arange(0, PASS_HZ, step), PASS_HZ)
    fsb = np.append(np.arange(STOP_HZ, fs / 2, step), fs / 2)
    m = np.arange(L) - M
    hd = h.astype(np.float64)

    def H(f):
        out = []
        for i in range(0, f.size, 2048):
            out.append(np.cos(2 * np.pi * np.outer(f[i:i + 2048], m) / fs) @ hd)
        return 20 * np.log10(np.abs(np.concatenate(out)) + 1e-300)
    return H(fp), H(fsb)


def meets_spec(h, fs):
    p, s = response_db(h, fs)
    return np.abs(p).max() <= PASS_DB and s.max() <= -STOP_DB


def kaiser_sinc(L, fs):
    """The design method: Kaiser window (beta for 70 dB), sinc with cutoff 0.96 MHz, DC gain 1, kept as float."""
    M = (L - 1) // 2
    m = np.arange(L) - M
    h = 2 * 0.96e6 / fs * np.sinc(2 * 0.96e6 / fs * m) * np.kaiser(L, 0.1102 * (70 - 8.7))
    return (h / h.sum()).astype(np.float32)


@pytest.mark.parametrize("D", [2, 4, 8, 16, 32, 64])
def test_design_taps_meet_spec_and_are_shortest(lcs, D):
    fs = D * 1.92e6
    h = lcs.chan_design_taps(fs)
    L = h.size
    assert L % 2 == 1
    assert np.array_equal(h, h[::-1])
    assert abs(h.astype(np.float64).sum() - 1) < 1e-6
    assert 15 * D < L < 17 * D + 8                     # about 16D + 1: 0.52 MHz transition band at 70 dB
    p, s = response_db(h, fs)
    assert np.abs(p).max() <= PASS_DB, np.abs(p).max()
    assert s.max() <= -STOP_DB, s.max()
    # it is the design method's output, and the length below it fails
    assert np.abs(kaiser_sinc(L, fs) - h).max() <= 1e-7
    assert not meets_spec(kaiser_sinc(L - 2, fs), fs)


def test_design_taps_reject_bad_rates(lcs):
    for fs in (1.92e6, 10e6, 65 * 1.92e6, 0.0, float("nan")):
        with pytest.raises(lcs.LcsError, match="error 1"):
            lcs.chan_design_taps(fs)


# ---- the oracle against an independent form -------------------------------------------------------------------------------
def scipy_form(iq, fs_in, fc_in, fc, h):
    """Exact-phase mixing, scipy's upfirdn (filter + keep every D-th sample), then the filter's delay removed."""
    from scipy.signal import upfirdn
    D = int(round(fs_in / FS_CH))
    M = (h.size - 1) // 2
    r = (-M) % D
    z = np.concatenate([np.zeros(r, complex), mix(iq, fs_in, fc_in, fc)])
    y = upfirdn(h.astype(np.float64), z, 1, D)
    s = (M + r) // D
    return y[s:s + n_outputs(iq.shape[0], D, M)]


@pytest.mark.parametrize("D", [2, 5, 16])
def test_oracle_matches_scipy_and_push_sizes(lcs, D):
    rng = np.random.default_rng(D)
    fs_in, fc_in = D * 1.92e6, 739e6
    h = lcs.chan_design_taps(fs_in)
    n = 40 * D + 3 * h.size
    iq = rng.integers(-3000, 3000, (n, 2)).astype(np.int16)
    half = (fs_in / 2 - 960e3) // 100e3 * 100e3
    fcs = fc_in + np.array([-half, 0.0, 100e3, half, 123457.0])
    y = chan_oracle(iq, fs_in, fc_in, fcs, h)
    for c, fc in enumerate(fcs):
        ref = scipy_form(iq, fs_in, fc_in, fc, h)
        assert ref.size == y.shape[1]
        assert np.abs(y[c] - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-30)
    st = OracleStream(fs_in, fc_in, fcs, h)
    parts, i = [], 0
    for k in (1, 7, h.size // 3, 1, 2 * h.size, n):
        parts.append(st.push(iq[i:i + k]))
        i += k
    assert np.array_equal(np.concatenate(parts, axis=1), y)


# ---- generator + oracle + the searcher's oracle, end to end on the CPU ---------------------------------------------------------
def test_wideband_synthetic_cell_found_by_oracle(lcs, oracle):
    fs_in, fc_in, f_true = 7.68e6, 739e6, 1000.0
    D = 4
    h = lcs.chan_design_taps(fs_in)
    M = (h.size - 1) // 2
    n = 153599 * D + M + 1
    a = dict(n_id_cell=277, n_ports=2, cp_type=1, n_rb_dl=25, phich_duration=1, phich_resource=3, t0=1234.0, sfn0=100)
    b = dict(n_id_cell=100, n_ports=1, cp_type=1, n_rb_dl=50, phich_duration=2, phich_resource=2, t0=9000.0, sfn0=7)
    fa, fb = fc_in + 2.1e6, fc_in - 1.9e6
    iq = S.synth_wide_ci16(n, fs_in, fc_in, [(fa, [a], 1.0), (fb, [b], 1.0)], f_true=f_true, snr_db=10, seed=3)
    k = (fc_in - f_true) / fc_in
    for fc, d in ((fa, a), (fb, b)):
        y = chan_oracle(iq, fs_in, fc_in, [fc], h)
        assert y.shape[1] == 153600
        cu8, clipped, _ = quantise(y, auto_gain_oracle(y))
        assert clipped[0] < 10
        cells, _ = oracle.cell_search_one(S.to_c128(cu8[0]), np.arange(-10000, 10001, 5000.0), fc, fc, 1.92e6)
        assert len(cells) == 1
        c = cells[0]
        assert (c.n_id_cell(), c.n_ports, c.cp_type, c.n_rb_dl, c.phich_duration, c.phich_resource, c.sfn) == \
            (d["n_id_cell"], d["n_ports"], 1, d["n_rb_dl"], d["phich_duration"], d["phich_resource"], d["sfn0"])
        assert abs(c.freq_superfine - fc * (1 - k)) < 50


# ---- CLI argument errors (no device is touched) -------------------------------------------------------------------------------
def cellsearch(*args):
    host = os.path.join(ROOT, "lte-cell-scanner_b200", "host")
    exe = os.path.join(host, "CellSearch_b200")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", host, "-s"])
    return subprocess.run([exe] + list(args), capture_output=True, text=True, timeout=60)


def test_cli_wideband_argument_errors(lcs, tmp_path):
    f = str(tmp_path / "none.ci16")
    np.zeros((1000, 2), np.int16).tofile(f)
    out = cellsearch("--wideband", f, "--fs-in", "10e6", "--fc-in", "739e6", "-s", "739e6")
    assert out.returncode != 0 and "--fs-in must be D * 1.92 MHz" in out.stderr
    out = cellsearch("--wideband", f, "--fs-in", "7.68e6", "--fc-in", "739e6", "-s", "735e6", "-e", "739e6")
    assert out.returncode != 0 and "raster point 735 MHz lies outside the input band" in out.stderr
    out = cellsearch("--wideband", f, "--fs-in", "7.68e6", "--fc-in", "739e6", "-s", "739e6", "-e", "742e6")
    assert out.returncode != 0 and "raster point 741.9 MHz lies outside" in out.stderr
    out = cellsearch("--wideband", f, "--fs-in", "7.68e6", "--fc-in", "739e6", "-s", "739e6")
    assert out.returncode != 0 and "153600 outputs per channel need" in out.stderr
    for o in (out,):
        assert "lcs_ctx_create" not in o.stderr
