"""The Welch spectrum's contract (DESIGN.md section 4.8) restated in float64 numpy: equal to scipy.signal.welch followed by
fftshift, invariant to push sizes, and the CLI's --spectrum argument errors (no device is touched)."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from test_channelizer_host import cellsearch
from test_rchan_host import random_iq, to_complex


def hann(N):
    """The periodic Hann window, w[n] = 0.5 - 0.5 cos(2 pi n / N)."""
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N)


def n_segments(n, N):
    """Segments completed by n samples: segment s covers [s N/2, s N/2 + N)."""
    return (n - N) // (N // 2) + 1 if n >= N else 0


class WelchOracle:
    """The contract restated: each segment's |X_s[k]|^2 added to a float64 accumulator per bin in segment order, the
    stream pushed in pieces of any size (at most N - 1 samples of carry)."""

    def __init__(self, fs, N):
        self.fs, self.N = fs, N
        self.w = hann(N)
        self.ws = np.sum(self.w ** 2)                          # the normalisation's sum of w[n]^2
        self.carry = np.zeros(0, complex)
        self.acc = np.zeros(N)
        self.S = 0

    def push(self, x):
        x = np.concatenate([self.carry, np.asarray(x, complex)])
        N, hop = self.N, self.N // 2
        k = n_segments(x.size, N)
        for s in range(k):
            self.acc += np.abs(np.fft.fft(self.w * x[s * hop:s * hop + N])) ** 2
        self.S += k
        self.carry = x[k * hop:]
        assert self.carry.size < N or k == 0

    def read(self):
        """(P in fftshift order, S); the accumulator restarts."""
        P = np.fft.fftshift(self.acc / (self.S * self.fs * self.ws)) if self.S else np.zeros(self.N)
        S, self.acc, self.S = self.S, np.zeros(self.N), 0
        return P, S


def welch_oracle(x, fs, N):
    o = WelchOracle(fs, N)
    o.push(x)
    return o.read()


def scipy_welch(x, fs, N):
    from scipy.signal import welch
    _, P = welch(x, fs, window="hann", nperseg=N, noverlap=N // 2, detrend=False, return_onesided=False,
                 scaling="density")
    return np.fft.fftshift(P)


@pytest.mark.parametrize("N", [64, 4096, 65536])
@pytest.mark.parametrize("fmt", ["ci16", "cs8", "cu8", "cf32"])
def test_oracle_matches_scipy_welch(N, fmt):
    rng = np.random.default_rng(N + len(fmt))
    fs = 30.72e6
    n = 5 * N // 2 + N // 3                                    # four segments and a partial one
    x = to_complex(random_iq(rng, n, fmt), fmt)
    x = x + 0.3 * np.exp(2j * np.pi * 0.137 * np.arange(n))   # a tone off the bin grid
    P, S = welch_oracle(x, fs, N)
    assert S == 4
    ref = scipy_welch(x, fs, N)
    assert np.abs(P - ref).max() <= 1e-12 * ref.max()
    from scipy.signal import get_window
    assert np.abs(hann(N) - get_window("hann", N)).max() < 1e-15     # equal up to the last bit of the cosine


@pytest.mark.parametrize("N", [64, 4096])
def test_oracle_push_sizes_are_bitwise_one_push(N):
    rng = np.random.default_rng(N)
    x = to_complex(random_iq(rng, 7 * N + 5, "ci16"), "ci16")
    whole, S = welch_oracle(x, 1e6, N)
    for k in (1, N // 2 - 1, N + 3):
        o = WelchOracle(1e6, N)
        for i in range(0, x.size, k):
            o.push(x[i:i + k])
        P, S2 = o.read()
        assert S2 == S and np.array_equal(P, whole)


def test_read_before_n_samples_has_no_segment():
    N = 1024
    o = WelchOracle(1e6, N)
    o.push(np.ones(N - 1))
    P, S = o.read()
    assert S == 0 and not P.any()
    o.push(np.ones(1))                                         # the carry completes segment 0
    assert o.read()[1] == 1


def exported(path):
    nm = subprocess.run(["nm", "-D", "--defined-only", path], check=True, capture_output=True, text=True).stdout
    return {line.split()[-1] for line in nm.splitlines() if line.split() and line.split()[-1].startswith("lcs_")}


def test_psd_prototypes_cover_header_and_library(lcs):
    """liblcs_psd.so exports exactly the five functions of include/lcs_psd.h, all bound with the header's prototypes;
    liblcs_b200.so exports none of them."""
    header = re.sub(r"/\*.*?\*/", " ", open(lcs.PSD_HEADER).read(), flags=re.S)
    names = set(re.findall(r"\b(lcs_\w+)\s*\(", header))
    assert names == {"lcs_psd_create", "lcs_psd_destroy", "lcs_psd_push", "lcs_psd_read", "lcs_psd_timing_read"}
    assert set(lcs.prototypes(lcs.PSD_HEADER)) == names
    assert exported(lcs.PSD_LIB_PATH) == names
    assert not exported(lcs.LIB_PATH) & names
    l = lcs.psd_lib()
    assert l.lcs_psd_create.argtypes == [C.c_void_p, C.c_double, C.c_int, C.c_uint32, C.c_void_p]
    assert l.lcs_psd_push.argtypes == [C.c_void_p, C.c_void_p, C.c_uint32]
    assert l.lcs_psd_destroy.restype is None


# ---- CLI argument errors with --spectrum (no device is touched) -------------------------------------------------------------
def test_cli_spectrum_argument_errors(lcs, tmp_path):
    f = str(tmp_path / "rec.ci16")
    np.zeros((1000, 2), np.int16).tofile(f)
    out_csv = str(tmp_path / "psd.csv")
    base = ["--wideband", f, "--fc-in", "739e6", "--fs-in", "10e6", "--spectrum", out_csv]
    cases = [
        (["--spectrum", out_csv, "--fs-in", "10e6", "--fc-in", "739e6"], "--spectrum needs --wideband"),
        (base + ["--nfft", "100"], "--nfft must be a power of two in [64, 65536]"),
        (base + ["--nfft", "32"], "--nfft must be a power of two in [64, 65536]"),
        (base + ["--nfft", "131072"], "--nfft must be a power of two in [64, 65536]"),
        (base + ["--nfft", "4k"], "could not parse --nfft"),
        (base + ["--fs-in", "10000000.5"], "--spectrum needs --fs-in, an integer number of Hz in (0, 250] MHz"),
        (base + ["--fs-in", "251e6"], "--spectrum needs --fs-in, an integer number of Hz in (0, 250] MHz"),
        (["--wideband", f, "--fc-in", "739e6", "--spectrum", out_csv], "--spectrum needs --fs-in"),
        (["--wideband", f, "--fs-in", "10e6", "--spectrum", out_csv], "--wideband needs --fc-in"),
        (base + ["--format", "ci8"], "--format must be ci16, cs8, cu8 or cf32"),
        (["--wideband", str(tmp_path / "missing.ci16"), "--fc-in", "739e6", "--fs-in", "10e6", "--spectrum", out_csv],
         "cannot read"),
        (["--wideband", f, "--fc-in", "739e6", "--fs-in", "10e6", "--spectrum", str(tmp_path / "no" / "psd.csv")],
         "cannot write"),
        (base + ["-s", "739e6"], "--fs-in must be D * 1.92 MHz"),       # with a search its own rules hold as before
    ]
    for args, msg in cases:
        out = cellsearch(*args)
        assert out.returncode != 0 and msg in out.stderr, (args, out.stderr)
        assert "lcs_ctx_create" not in out.stderr
