"""The Welch spectrum (DESIGN.md section 4.8) held to FP32 error bounds and to its accumulation contract bit for bit.

P_ref restates the contract at the kernel's own precision: the exactly converted samples times the float window, each
segment transformed in float64, normalised by the double window's sum of w^2.  Against it the device must meet, at every
N from 64 to 65 536 and in every format,
- a norm bound that holds for any input: sqrt(sum_k (sqrt P_dev - sqrt P_ref)^2) <= beta(N) sqrt(sum_k P_ref), and
- a per-bin bound that holds for broadband input: |P_dev[k] - P_ref[k]| <= 2 tau sqrt(P_ref[k] Pbar) + tau^2 Pbar.
The accumulation is checked exactly: one push equals the in-order float64 sum of the float32 rows |X_s|^2 that a
spectrogram read after every segment exposes, scaled and fftshifted as lcs_psd_read does.  Samples of equal value in
different formats give bitwise the same PSD."""
import functools
import math

import numpy as np
import pytest

from test_rchan_host import random_iq, to_complex
from test_spectrum_gpu import recording
from test_spectrum_host import WelchOracle, hann, n_segments, welch_oracle

U = 2.0 ** -24                        # unit roundoff of float32
FS = 30.72e6                          # an integer number of Hz, so lcs_psd_read's scale is modelled exactly
NS = [1 << lg for lg in range(6, 17)]
FORMATS = ["ci16", "cs8", "cu8", "cf32"]
TILE = 4096                           # points per CTA of psd.cu; larger N runs four-step
# recording() is broadband in these formats: its uniform noise carries 94 % of the power.  In ci16 the noise is drawn
# within +-3000 of 32 767 and the strong tone carries 88 % of the power, a concentrated spectrum (see per_bin_bound).
BROADBAND_RECORDING = ("cs8", "cu8", "cf32")


@functools.lru_cache(maxsize=None)
def window_ss(N):
    """sum_n w[n]^2 over the double window, computed as lcs_psd_create computes it: each term with libm's cos (which
    math.cos calls), added in n order."""
    ws = 0.0
    for n in range(N):
        w = 0.5 - 0.5 * math.cos(2 * math.pi * n / N)
        ws += w * w
    return ws


def window32(N):
    """The window as the kernels read it: the double window rounded to float."""
    return hann(N).astype(np.float32).astype(np.float64)


class PsdRef(WelchOracle):
    """P_ref: the contract at the kernel's precision.  The float window and float64 transforms; normalised by the double
    window's sum of w^2, as the device is."""

    def __init__(self, fs, N):
        super().__init__(fs, N)
        self.w = window32(N)
        self.ws = window_ss(N)


def psd_ref(x, fs, N):
    o = PsdRef(fs, N)
    o.push(x)
    return o.read()


def norm_beta(N):
    """The norm bound's beta for the kernels' FFT of length N: Higham, Accuracy and Stability of Numerical Algorithms,
    Thm 24.2, with L radix-2 stages of float twiddles computed in double (one more for the four-step inter-pass
    twiddle), carried through |.| and the sum over segments by the triangle and Minkowski inequalities."""
    L = int(math.log2(N)) + (1 if N > TILE else 0)
    g4 = 4 * U / (1 - 4 * U)
    eta = U + g4 * (math.sqrt(2) + U)
    return L * eta / (1 - L * eta) + U


def norm_ratio(got, ref, N):
    """sqrt(sum_k (sqrt P_dev - sqrt P_ref)^2) / (beta sqrt(sum_k P_ref)): at most 1 for any input."""
    return math.sqrt(np.sum((np.sqrt(got) - np.sqrt(ref)) ** 2) / np.sum(ref)) / norm_beta(N)


def per_bin_tau(N):
    return 8 * U * math.log2(N)


def per_bin_bound(ref, N):
    """2 tau sqrt(P_ref[k] Pbar) + tau^2 Pbar, Pbar the mean of P_ref over the bins.  A statistical bound, not a proven
    one: the FFT's rounding errors spread over the bins like noise of about Pbar u^2 log2 N, which it allows eight
    times in amplitude.  It holds for broadband input (recording() in cs8, cu8 and cf32, full-scale random samples) and
    fails for concentrated spectra, whose strongest bins carry a relative error far above Pbar's share (a pure
    bin-centred tone exceeds it at large N)."""
    tau, Pm = per_bin_tau(N), ref.mean()
    return 2 * tau * np.sqrt(ref * Pm) + tau ** 2 * Pm


def per_bin_ratio(got, ref, N):
    """(max_k |P_dev[k] - P_ref[k]| / bound[k], the k where it is largest)."""
    r = np.abs(got - ref) / per_bin_bound(ref, N)
    k = int(np.argmax(r))
    return float(r[k]), k


# each format's extreme values and their probabilities, which keep the mean (a DC line) near zero
FULL_SCALE = {"ci16": (np.int16, [-32768, -32767, 32767], [0.25, 0.25, 0.5]), "cs8": (np.int8, [-128, 127], None),
              "cu8": (np.uint8, [0, 255], None), "cf32": (np.float32, [-1.0, 1.0], None)}


def full_scale(rng, n, fmt):
    """Random samples at the format's extreme values only: a white spectrum at the largest amplitude the format holds."""
    dt, v, p = FULL_SCALE[fmt]
    return rng.choice(np.array(v, dt), (n, 2), p=p)


def sweep_segments(N):
    """A segment count that leaves the last CTA of psd_fft_kernel (TILE/N segments each) partly filled."""
    return 2 * max(TILE // N, 1) + 5


def device_psd(lcs, ctx, iq, fmt, N):
    sp = lcs.Spectrum(ctx, FS, fmt, N)
    sp.push(iq)
    _, P, S = sp.read()
    sp.close()
    return P, S


def check_bounds(record_property, name, P, ref, N, per_bin):
    """Both bounds (the per-bin one only if per_bin); the ratios go to the test's report."""
    rn, (rb, k) = norm_ratio(P, ref, N), per_bin_ratio(P, ref, N)
    record_property(name, "norm %.4f per-bin %.4f at output bin %d" % (rn, rb, k))
    assert rn <= 1, (name, rn)
    if per_bin:
        assert rb <= 1, (name, rb)


# ---- the reference and the bounds themselves (CPU) --------------------------------------------------------------------------
@pytest.mark.parametrize("N", [64, 128, 8192, 65536])
def test_reference_is_the_oracle_up_to_the_float_window(N):
    """P_ref and the float64 oracle differ only by the window's rounding to float, |w32 - w| <= u w: by Parseval their
    norm distance is at most u sqrt(sum_k P), and it is not zero."""
    rng = np.random.default_rng(N)
    x = to_complex(recording(rng, 3 * N + N // 3, "cs8", FS), "cs8")
    ref, S = psd_ref(x, FS, N)
    oracle, S_or = welch_oracle(x, FS, N)
    assert S == S_or == 5
    d = math.sqrt(np.sum((np.sqrt(ref) - np.sqrt(oracle)) ** 2) / np.sum(oracle))
    assert 0 < d <= U * (1 + 1e-6)
    assert abs(window_ss(N) / np.sum(hann(N) ** 2) - 1) < 1e-14


@pytest.mark.parametrize("N", [64, 4096])
def test_reference_push_sizes_are_bitwise_one_push(N):
    rng = np.random.default_rng(N + 1)
    x = to_complex(random_iq(rng, 7 * N + 5, "cu8"), "cu8")
    whole, S = psd_ref(x, 1e6, N)
    for k in (1, N // 2 - 1, N + 3):
        o = PsdRef(1e6, N)
        for i in range(0, x.size, k):
            o.push(x[i:i + k])
        P, S2 = o.read()
        assert S2 == S and np.array_equal(P, whole)


def test_bounds_at_hand_computed_sizes():
    # beta = L eta / (1 - L eta) + u, eta = u + gamma_4 (sqrt 2 + u), gamma_4 = 4u / (1 - 4u), u = 2^-24
    assert norm_beta(64) == pytest.approx(2.44029e-6, rel=1e-5)       # L = 6
    assert norm_beta(128) == pytest.approx(2.83707e-6, rel=1e-5)      # L = 7
    assert norm_beta(4096) == pytest.approx(4.82098e-6, rel=1e-5)     # L = 12, one pass
    assert norm_beta(8192) == pytest.approx(5.61455e-6, rel=1e-5)     # L = 13 + 1, four-step
    assert norm_beta(65536) == pytest.approx(6.80490e-6, rel=1e-5)    # L = 16 + 1
    assert per_bin_tau(1024) == 80 * 2.0 ** -24
    # P_ref = (0, 1, 4, 9), Pbar = 3.5, tau = 48 u at N = 64
    t = 48 * 2.0 ** -24
    b = per_bin_bound(np.array([0.0, 1.0, 4.0, 9.0]), 64)
    assert np.allclose(b, [t * t * 3.5, 2 * t * math.sqrt(3.5) + t * t * 3.5, 4 * t * math.sqrt(3.5) + t * t * 3.5,
                           6 * t * math.sqrt(3.5) + t * t * 3.5], rtol=1e-14, atol=0)
    # an error of exactly the bound has ratio 1: sqrt P grown by beta in every bin, P grown by the bound in one bin
    ref = np.full(64, 2.0)
    assert norm_ratio(ref * (1 + norm_beta(64)) ** 2, ref, 64) == pytest.approx(1.0, rel=1e-8)
    one = ref.copy()
    one[5] += per_bin_bound(ref, 64)[5]
    assert per_bin_ratio(one, ref, 64) == (pytest.approx(1.0, rel=1e-12), 5)
    # the periodic Hann window's sum of squares is 3N/8
    for N in NS:
        assert window_ss(N) == pytest.approx(3 * N / 8, rel=1e-13)


# ---- both bounds at every N and format (GPU) ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_bounds_every_size_and_format(lcs, ctx, record_property, N, fmt):
    """recording() over S segments (the last CTA partly filled) and over one segment, and full-scale random samples:
    the norm bound on all, the per-bin bound on the broadband ones."""
    rng = np.random.default_rng(N + 11 * len(fmt))
    S = sweep_segments(N)
    n = (S + 1) * (N // 2) + N // 3                          # S segments and part of another
    for name, iq, S_want in (("recording", recording(rng, n, fmt, FS), S),
                             ("recording_S1", recording(rng, N + N // 2 - 1, fmt, FS), 1),
                             ("full_scale", full_scale(rng, n, fmt), S)):
        P, S_dev = device_psd(lcs, ctx, iq, fmt, N)
        ref, S_ref = psd_ref(to_complex(iq, fmt), FS, N)
        assert S_dev == S_ref == S_want == n_segments(iq.shape[0], N)
        check_bounds(record_property, name, P, ref, N,
                     per_bin=name == "full_scale" or fmt in BROADBAND_RECORDING)


@pytest.mark.gpu
@pytest.mark.parametrize("N", NS)
def test_norm_bound_holds_for_a_bin_centred_tone(lcs, ctx, record_property, N):
    """The norm bound holds for any input, a spectrum concentrated in one bin included."""
    S = 5
    m = np.arange((S + 1) * N // 2)
    x = 0.9 * np.exp(2j * np.pi * (N // 3) * m / N)
    iq = np.stack([x.real, x.imag], axis=1).astype(np.float32)
    P, S_dev = device_psd(lcs, ctx, iq, "cf32", N)
    ref, _ = psd_ref(to_complex(iq, "cf32"), FS, N)
    assert S_dev == S
    check_bounds(record_property, "tone", P, ref, N, per_bin=False)


# ---- the accumulation, bit for bit (GPU) --------------------------------------------------------------------------------------
def launch_chunk(N):
    """Segments per launch as lcs_psd_create sizes them: 64 MB of |X|^2 rows, and of four-step rows above TILE."""
    return (64 << 20) // (N * (4 + (8 if N > TILE else 0)))


def segment_powers(x, N, s0, s1):
    """|X_s[k]|^2 of P_ref's transform for segments s0 <= s < s1, [s1 - s0][N] in bin order k."""
    hop = N // 2
    seg = np.lib.stride_tricks.sliding_window_view(x[s0 * hop:(s1 - 1) * hop + N], N)[::hop]
    return np.abs(np.fft.fft(seg * window32(N), axis=1)) ** 2


# formats vary so that the carry of each sample size crosses launch-chunk boundaries
@pytest.mark.gpu
@pytest.mark.parametrize("N,fmt", [(4096, "cs8"), (8192, "cu8"), (16384, "cf32"), (32768, "cs8"), (65536, "cf32")])
def test_accumulation_is_the_in_order_sum_of_segment_rows(lcs, ctx, record_property, N, fmt):
    """Handle A takes the stream in one push, over at least three launch chunks; handle B takes it one hop at a time and
    is read after every segment, which gives each segment's float32 row f_s = |X_s|^2 exactly (B's read is
    f_s / (fs sum w^2), one rounding of a double, which cannot move a float).  A's read must be, bit for bit,
    sum_s f_s in float64 in segment order, times 1 / ((S fs) sum w^2), in fftshift order.  Every f_s meets the per-bin
    bound; the stream is the format's random noise, broadband in every segment (one segment of recording() puts its
    strong tone some 30 dB above the mean bin, where that bound is not meant to hold)."""
    chunk = launch_chunk(N)
    S = 2 * chunk + chunk // 2 + 1
    hop = N // 2
    rng = np.random.default_rng(N + 3)
    iq = random_iq(rng, (S + 1) * hop, fmt)
    ws = window_ss(N)
    A = lcs.Spectrum(ctx, FS, fmt, N)
    A.push(iq)
    _, P_one, S_one = A.read()
    _, launches = A.timing_read()
    A.close()
    assert S_one == S
    assert launches >= 3 * (3 if N > TILE else 2)              # at least three launch chunks
    B = lcs.Spectrum(ctx, FS, fmt, N)
    rows = np.empty((S, N), np.float32)
    scale1 = 1.0 / ((1 * FS) * ws)
    B.push(iq[:hop])
    for s in range(S):
        B.push(iq[(s + 1) * hop:(s + 2) * hop])
        _, P, k = B.read()
        assert k == 1
        rows[s] = np.fft.ifftshift(P * FS * ws)
        assert np.array_equal(np.fft.fftshift(rows[s].astype(np.float64)) * scale1, P)   # f_s is B's row exactly
    B.close()
    acc = np.zeros(N)
    for r in rows:                                               # in segment order
        acc += r
    model = np.fft.fftshift(acc) * (1.0 / ((S * FS) * ws))
    assert np.array_equal(P_one, model), np.abs(P_one / model - 1).max()
    x = to_complex(iq, fmt)
    worst = (0.0, 0, 0)
    for s0 in range(0, S, 256):
        s1 = min(S, s0 + 256)
        ref = segment_powers(x, N, s0, s1)
        for s, (g, r) in enumerate(zip(rows[s0:s1].astype(np.float64), ref), s0):
            worst = max(worst, per_bin_ratio(g, r, N) + (s,))
    record_property("rows", "per-bin %.4f at bin %d of segment %d" % worst)
    assert worst[0] <= 1, worst


# ---- equal values in every format (GPU) ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N", [2048, 32768])
def test_equal_values_in_every_format_give_the_same_psd(lcs, ctx, N):
    """cs8 v = ci16 256 v = cf32 v / 128, and cu8 w = ci16 256 (w - 127) = cf32 (w - 127) / 128, bitwise.  cu8 255 is
    +1.0, beyond ci16, so it is compared with cf32 alone."""
    rng = np.random.default_rng(N + 5)
    n = 9 * N // 2 + 17
    v = recording(rng, n, "cs8", FS)
    v[:2] = [[-128, 127], [127, -128]]
    w = recording(rng, n, "cu8", FS)
    w[:2] = [[0, 255], [255, 0]]
    w254 = np.minimum(w, 254)
    groups = [
        [("cs8", v), ("ci16", v.astype(np.int16) * 256), ("cf32", v.astype(np.float32) / 128)],
        [("cu8", w254), ("ci16", (w254.astype(np.int16) - 127) * 256), ("cf32", (w254.astype(np.float32) - 127) / 128)],
        [("cu8", w), ("cf32", (w.astype(np.float32) - 127) / 128)],
    ]
    for g in groups:
        psds = [device_psd(lcs, ctx, iq, fmt, N) for fmt, iq in g]
        for (fmt, _), (P, S) in zip(g[1:], psds[1:]):
            assert S == psds[0][1] == n_segments(n, N)
            assert np.array_equal(P, psds[0][0]), (g[0][0], fmt)
