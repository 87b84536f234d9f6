"""The rational channelizer's contract without a GPU (DESIGN.md section 4.7): the allowed rates and their up / down, the
prototype filters, a float64 restatement of the resampling channelizer for every input format (the oracle the GPU tests
compare against), and the CLI's argument checks with --resample."""
import numpy as np
import pytest

from test_channelizer_host import PASS_DB, PASS_HZ, STOP_DB, STOP_HZ, cellsearch

# fs_in -> (up, down, about L) for the rates SDRs record at
RATES = {2.048e6: (15, 16, 257), 2.4e6: (4, 5, 81), 2.5e6: (96, 125, 2000), 6e6: (8, 25, 400), 10e6: (24, 125, 2000),
         12.5e6: (96, 625, 10000), 20e6: (12, 125, 2000), 25e6: (48, 625, 10000), 56e6: (6, 175, 2800),
         100e6: (12, 625, 10000)}


# ---- the oracle: section 4.7 in float64 ------------------------------------------------------------------------------------
def n_outputs(n, up, down, M):
    return max(0, (n * up - M - 1) // down + 1)


def to_complex(iq, fmt):
    """The contract's x[m] of [n][2] samples in each format."""
    v = iq.astype(np.float64)
    if fmt == "ci16":
        v = v / 32768
    elif fmt == "cs8":
        v = v / 128
    elif fmt == "cu8":
        v = (v - 127) / 128
    return v[:, 0] + 1j * v[:, 1]


def mix(x, fs_in, fc_in, fc):
    """x[m] exp(-j2pi p[m]/fs_in), p[m] = (m * delta) mod fs_in in exact integers."""
    fs = int(round(fs_in))
    delta = int(round(fc - fc_in))
    p = (np.arange(x.size, dtype=np.int64) * delta) % fs
    return x * np.exp(-2j * np.pi * p / fs)


def rchan_oracle(x, fs_in, fc_in, fc_ch, h, up, down):
    """y [n_ch][n_out] complex128: y_c[n] = sum_i h[n*down - i*up + M] x~_c[i] over 0 <= n*down - i*up + M <= 2M, with
    x~ = 0 before the stream."""
    M = (h.size - 1) // 2
    n_out = n_outputs(x.size, up, down, M)
    q = np.arange(n_out, dtype=np.int64) * down + M
    ih, phi = q // up, q % up                       # newest input and branch of each output
    J = 2 * M // up + 1
    hd = np.concatenate([h.astype(np.float64), np.zeros(up)])
    ys = []
    for fc in np.atleast_1d(fc_ch):
        xm = np.concatenate([np.zeros(J, complex), mix(x, fs_in, fc_in, fc)])   # index i + J <-> stream sample i
        y = np.zeros(n_out, complex)
        for j in range(J):
            k = phi + j * up
            y += np.where(k <= 2 * M, hd[np.minimum(k, 2 * M + 1)], 0.0) * xm[ih - j + J]
        ys.append(y)
    return np.array(ys).reshape(len(ys), n_out)


class RationalOracleStream:
    """The oracle fed push by push: output n is emitted once sample floor((n*down + M)/up) has arrived."""

    def __init__(self, fs_in, fc_in, fc_ch, h, up, down, fmt):
        self.args = (fs_in, fc_in, fc_ch, h, up, down)
        self.up, self.down, self.M, self.fmt = up, down, (h.size - 1) // 2, fmt
        self.x = np.zeros(0, complex)
        self.done = 0

    def push(self, iq):
        self.x = np.concatenate([self.x, to_complex(iq, self.fmt)])
        k = n_outputs(self.x.size, self.up, self.down, self.M)
        y = rchan_oracle(self.x, *self.args)[:, self.done:k]
        self.done = k
        return y


def random_iq(rng, n, fmt):
    if fmt == "ci16":
        return rng.integers(-3000, 3000, (n, 2)).astype(np.int16)
    if fmt == "cs8":
        return rng.integers(-128, 128, (n, 2)).astype(np.int8)
    if fmt == "cu8":
        return rng.integers(0, 256, (n, 2)).astype(np.uint8)
    return rng.standard_normal((n, 2)).astype(np.float32)


# ---- the prototype filter on the FFT grid ----------------------------------------------------------------------------------
def fft_response_db(h, F, gain):
    """|H|/gain in dB on the grid of an FFT of the zero-padded taps (every F/N, N the power of two >= 64L) plus the band
    edges: (passband dB, stopband dB)."""
    L = h.size
    M = (L - 1) // 2
    N = 1 << (64 * L - 1).bit_length()
    hd = h.astype(np.float64)
    a = np.abs(np.fft.rfft(hd, N)) / gain
    f = np.arange(N // 2 + 1) * F / N
    m = np.arange(1, M + 1)
    edge = [abs(hd[M] + 2 * np.cos(2 * np.pi * fe * m / F) @ hd[M + 1:]) / gain for fe in (PASS_HZ, STOP_HZ)]
    p = np.append(a[f <= PASS_HZ], edge[0])
    s = np.append(a[f >= STOP_HZ], edge[1])
    return 20 * np.log10(p), 20 * np.log10(s + 1e-300)


def meets_spec(h, F, gain):
    p, s = fft_response_db(h, F, gain)
    return np.abs(p).max() <= PASS_DB and s.max() <= -STOP_DB


def kaiser_sinc(L, F, gain):
    """The design method: Kaiser window (beta for 70 dB), sinc with cutoff 0.96 MHz, DC gain `gain`, kept as float."""
    M = (L - 1) // 2
    m = np.arange(L) - M
    h = 2 * 0.96e6 / F * np.sinc(2 * 0.96e6 / F * m) * np.kaiser(L, 0.1102 * (70 - 8.7))
    return (gain * h / h.sum()).astype(np.float32)


@pytest.mark.parametrize("fs_in", sorted(RATES))
def test_rational_design(lcs, fs_in):
    up, down, L0 = RATES[fs_in]
    u, d, h = lcs.chan_design_rational(fs_in)
    assert (u, d) == (up, down)
    L = h.size
    assert L % 2 == 1 and 0.9 * L0 < L < 1.1 * L0
    assert np.array_equal(h, h[::-1])
    assert abs(h.astype(np.float64).sum() / up - 1) < 1e-6
    F = up * fs_in
    p, s = fft_response_db(h, F, up)
    assert np.abs(p).max() <= PASS_DB, np.abs(p).max()
    assert s.max() <= -STOP_DB, s.max()
    assert np.abs(kaiser_sinc(L, F, up) - h).max() <= 1e-7 * up
    assert not meets_spec(kaiser_sinc(L - 2, F, up), F, up)


@pytest.mark.parametrize("D", [2, 16, 64])
def test_rational_design_integer_d_is_design_taps(lcs, D):
    u, d, h = lcs.chan_design_rational(D * 1.92e6)
    assert (u, d) == (1, D)
    assert np.array_equal(h, lcs.chan_design_taps(D * 1.92e6))


def test_rational_design_rejects_bad_rates(lcs):
    # 31 MHz = 1.92 MHz * 775/48: down > 640
    for fs in (1.92e6, 1.9e6, 10.5e6 + 0.5, 123e6, 31e6, 0.0, -10e6, float("nan"), float("inf")):
        with pytest.raises(lcs.LcsError, match="error 1"):
            lcs.chan_design_rational(fs)


# ---- the oracle against an independent form -------------------------------------------------------------------------------
def scipy_form(x, fs_in, fc_in, fc, h, up, down):
    """Exact-phase mixing, scipy's upfirdn upsampling by up and filtering, sampled at n*down + M."""
    from scipy.signal import upfirdn
    M = (h.size - 1) // 2
    z = upfirdn(h.astype(np.float64), mix(x, fs_in, fc_in, fc), up)
    return z[np.arange(n_outputs(x.size, up, down, M)) * down + M]


@pytest.mark.parametrize("fs_in,fmt", [(2.4e6, "cu8"), (2.5e6, "cf32"), (10e6, "cs8"), (6e6, "ci16"), (56e6, "ci16")])
def test_oracle_matches_scipy_and_push_sizes(lcs, fs_in, fmt):
    rng = np.random.default_rng(int(fs_in) % 1000 + 1)
    up, down, h = lcs.chan_design_rational(fs_in)
    M = (h.size - 1) // 2
    n = 30 * down // up + 3 * h.size // up + 50
    iq = random_iq(rng, n, fmt)
    x = to_complex(iq, fmt)
    fc_in = 739e6
    half = (fs_in / 2 - 960e3) // 100e3 * 100e3
    fcs = fc_in + np.array([-half, 0.0, half, 123457.0])
    y = rchan_oracle(x, fs_in, fc_in, fcs, h, up, down)
    assert y.shape[1] == n_outputs(n, up, down, M) > 20
    for c, fc in enumerate(fcs):
        ref = scipy_form(x, fs_in, fc_in, fc, h, up, down)
        assert np.abs(y[c] - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-30)
    st = RationalOracleStream(fs_in, fc_in, fcs, h, up, down, fmt)
    parts, i = [], 0
    for k in (1, 1, max(1, M // up // 2), 7, 1, 2 * h.size // up, n):   # pushes of 1 and shorter than M/up
        parts.append(st.push(iq[i:i + k]))
        i += k
    assert np.array_equal(np.concatenate(parts, axis=1), y)


# ---- CLI argument errors with --resample (no device is touched) -------------------------------------------------------------
def test_cli_resample_argument_errors(lcs, tmp_path):
    f = str(tmp_path / "none.cs8")
    np.zeros((1000, 2), np.int8).tofile(f)
    base = ["--wideband", f, "--fc-in", "739e6"]
    out = cellsearch(*base, "--fs-in", "31e6", "--resample", "--format", "cs8", "-s", "739e6")
    assert out.returncode != 0 and "--fs-in must be an integer number of Hz" in out.stderr
    out = cellsearch(*base, "--fs-in", "10e6", "--resample", "--format", "cs8", "-s", "734e6", "-e", "739e6")
    assert out.returncode != 0 and "raster point 734 MHz lies outside the input band" in out.stderr
    out = cellsearch(*base, "--fs-in", "10e6", "--resample", "--format", "cs8", "-s", "739e6")
    assert out.returncode != 0 and "cs8 samples; 153600 outputs per channel need" in out.stderr
    out = cellsearch(*base, "--fs-in", "10e6", "--resample", "--format", "ci8", "-s", "739e6")
    assert out.returncode != 0 and "--format must be ci16, cs8, cu8 or cf32" in out.stderr
    out = cellsearch(*base, "--fs-in", "10e6", "-s", "739e6")                  # without --resample: as before, with a hint
    assert out.returncode != 0 and "--fs-in must be D * 1.92 MHz" in out.stderr and "--resample" in out.stderr
    for o in (out,):
        assert "lcs_ctx_create" not in o.stderr
