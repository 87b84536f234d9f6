"""A bit-exact model of the channelizer's byte path (chan_kernel and rchan_kernel, chan.cu; DESIGN.md sections 4.6 and
4.7), channel by channel.

The accumulation is a fixed sequence of correctly rounded float32 operations, so every accumulator is determined to
the last bit:
- samples: load_iq's ci16 / 32768, cs8 / 128, (cu8 - 127) / 128 and cf32, all exact; exact zeros before the stream;
- complex taps, built on the host (build_taps) as a = 2 * pi * p / fs in double, left to right, then h * cos(a) and
  h * sin(a) in double, each rounded once to float32:
  chan_kernel  [ch][L], referred to the centre tap, p = ((t - M) * delta) mod fs;
  rchan_kernel [ch][up][J], referred to the newest input, p = (j * delta) mod fs, branch taps past 2M zero;
- one cmac per tap, oldest input first (chan_kernel u = 0..L-1 with tap t = 2M - u on sample nD - M + u; rchan_kernel
  j = J-1..0 on sample ih - j of branch phi, ih = (n down + M) / up, phi = (n down + M) mod up), each cmac four fmaf:
  re = fma(gx, xr, re), re = fma(-gy, xi, re), im = fma(gx, xi, im), im = fma(gy, xr, im).
The epilogue (rotate_quantise) runs in FP64: the exact integer phase p = ((k mod fs) * step) mod fs of the output
(chan_kernel k = n, step = D delta mod fs; rchan_kernel k = ih, step = delta mod fs), the rotation by
exp(-j 2 pi p / fs), v = 127 + 128 gain y, round to nearest even, clamp to [0, 255].  CUDA's sincospi and nvcc's
contraction differ from the host by about 1e-13 in v, so the model's v is compared with a band (compare()).
Auto gain is the same sums with the double taps (fma in double), then (float)(0.25 / sqrt(sum / n_out)), or 1 when the
sum is 0.

The accumulation is a small C++ library (std::fma, -ffp-contract=off), built like xcorr_fp32_model's."""
import ctypes
import math

import numpy as np

from xcorr_fp32_model import compile_model

BAND = 1e-9            # |v - (k + 1/2)| within which the device's byte may differ by one from the model's
GAIN_BAND = 1e-12      # relative distance of the double gain from a float32 rounding boundary that allows one ulp
# variants of the accumulation (the comparison must resolve each of them from the kernel's)
DROP_OLDEST, NEWEST_FIRST, SWAP_FMA, UNFUSED = 1, 2, 4, 8

SRC = r"""
#include <cmath>
#include <cstdint>
enum { DROP_OLDEST = 1, NEWEST_FIRST = 2, SWAP_FMA = 4, UNFUSED = 8 };
// x: float32 [..][2], stream sample s at x[x0 + s]; taps: T [rows][K][2]; output o sums cmac(taps[row[o]][K-1-u],
// x[x0 + start[o] + u]) over u = 0..K-1 (oldest input first); out: T [n][2]
template <class T>
static void acc(const float* x, int64_t x0, const T* taps, int K, const int64_t* start, const int32_t* row, int64_t n,
                int flags, T* out) {
#pragma omp parallel for schedule(static)
  for (int64_t o = 0; o < n; o++) {
    const T* g = taps + (int64_t)row[o] * K * 2;
    const float* xs = x + (x0 + start[o]) * 2;
    T re = 0, im = 0;
    for (int i = 0; i < K; i++) {
      const int u = (flags & NEWEST_FIRST) ? K - 1 - i : i;
      if ((flags & DROP_OLDEST) && u == 0) continue;
      const T gx = g[2 * (K - 1 - u)], gy = g[2 * (K - 1 - u) + 1];
      const T xr = (T)xs[2 * u], xi = (T)xs[2 * u + 1];
      if (flags & UNFUSED) {
        re = re + gx * xr; re = re + -gy * xi; im = im + gx * xi; im = im + gy * xr;
      } else if (flags & SWAP_FMA) {
        re = std::fma(-gy, xi, re); re = std::fma(gx, xr, re); im = std::fma(gy, xr, im); im = std::fma(gx, xi, im);
      } else {
        re = std::fma(gx, xr, re); re = std::fma(-gy, xi, re); im = std::fma(gx, xi, im); im = std::fma(gy, xr, im);
      }
    }
    out[2 * o] = re;
    out[2 * o + 1] = im;
  }
}
extern "C" void acc_f32(const float* x, int64_t x0, const float* taps, int K, const int64_t* start, const int32_t* row,
                        int64_t n, int flags, float* out) { acc<float>(x, x0, taps, K, start, row, n, flags, out); }
extern "C" void acc_f64(const float* x, int64_t x0, const double* taps, int K, const int64_t* start, const int32_t* row,
                        int64_t n, int flags, double* out) { acc<double>(x, x0, taps, K, start, row, n, flags, out); }
// sum over the taps of |g| |x| per output (double taps)
extern "C" void abs_sum(const float* x, int64_t x0, const double* taps, int K, const int64_t* start, const int32_t* row,
                        int64_t n, double* out) {
#pragma omp parallel for schedule(static)
  for (int64_t o = 0; o < n; o++) {
    const double* g = taps + (int64_t)row[o] * K * 2;
    const float* xs = x + (x0 + start[o]) * 2;
    double s = 0;
    for (int u = 0; u < K; u++)
      s += std::hypot(g[2 * (K - 1 - u)], g[2 * (K - 1 - u) + 1]) * std::hypot((double)xs[2 * u], (double)xs[2 * u + 1]);
    out[o] = s;
  }
}
"""

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = compile_model(SRC, "chan_model")
    return _lib


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def samples(iq, fmt):
    """float32 [n][2]: load_iq of [n][2] samples in fmt (every format exact)."""
    if fmt == "cf32":
        assert iq.dtype == np.float32
        return np.ascontiguousarray(iq)
    v = iq.astype(np.float64)
    v = {"ci16": v / 32768, "cs8": v / 128, "cu8": (v - 127) / 128}[fmt]
    return v.astype(np.float32)


def n_outputs(n, up, down, M):
    """Outputs of a fresh channelizer after n input samples."""
    return max(0, (n * up - M - 1) // down + 1)


class ChanModel:
    """The byte path of one channelizer: rate fs_in = 1.92 MHz * down / up, input format fmt, prototype h (float32 [L]),
    channels fc_ch about fc_in.  chan_kernel serves ci16 at up = 1, rchan_kernel everything else."""

    def __init__(self, fs_in, fc_in, fc_ch, fmt, up, down, h):
        self.fs = int(round(fs_in))
        self.fmt, self.up, self.down = fmt, up, down
        self.h = np.asarray(h, np.float32)
        self.L = self.h.size
        self.M = (self.L - 1) // 2
        self.J = 2 * self.M // up + 1
        self.centre = up == 1 and fmt == "ci16"
        self.K = self.L if self.centre else self.J
        self.delta = [int(round(f - fc_in)) for f in np.atleast_1d(fc_ch)]
        self.n_ch = len(self.delta)
        self._taps = {}

    # ---- taps ----------------------------------------------------------------------------------------------------------
    def taps(self, c, float_angle=False):
        """(float32 [rows][K][2], float64 [rows][K][2]) of channel c as build_taps makes them; float_angle=True rounds the
        angle to float32 before the cosine and sine (a variant the tests must resolve)."""
        key = (c, float_angle)
        if key not in self._taps:
            fs, d, M = self.fs, self.delta[c], self.M
            ks = np.arange(self.L) - M if self.centre else np.arange(self.J)
            ca, sa = np.empty(ks.size), np.empty(ks.size)
            for i, k in enumerate(ks):
                p = (int(k) * d) % fs
                a = 2 * math.pi * p / fs
                if float_angle:
                    a = float(np.float32(a))
                ca[i], sa[i] = math.cos(a), math.sin(a)
            h = self.h.astype(np.float64)
            if self.centre:
                hk = h[None]                                                  # [1][L], tap t
            else:
                k = np.arange(self.up)[:, None] + np.arange(self.J)[None] * self.up   # [up][J], branch phi, tap j
                hk = np.where(k <= 2 * M, np.concatenate([h, np.zeros(self.up)])[np.minimum(k, 2 * M + 1)], 0.0)
            t64 = np.ascontiguousarray(np.stack([hk * ca, hk * sa], axis=-1))
            self._taps[key] = (t64.astype(np.float32), t64)
        return self._taps[key]

    # ---- geometry ------------------------------------------------------------------------------------------------------
    def geometry(self, n_out):
        """(start, row, phase index) of outputs 0..n_out-1: the stream index of the oldest input, the tap row, and the
        k of the epilogue's phase ((k mod fs) * step) mod fs."""
        n = np.arange(n_out, dtype=np.int64)
        if self.centre:
            return n * self.down - self.M, np.zeros(n_out, np.int32), n
        q = n * self.down + self.M
        ih = q // self.up
        return ih - (self.J - 1), (q % self.up).astype(np.int32), ih

    def pad(self):
        """Zeros before stream sample 0 that output 0 reads."""
        return self.M if self.centre else self.J - 1

    def stream(self, x32):
        return np.ascontiguousarray(np.concatenate([np.zeros((self.pad(), 2), np.float32), x32]))

    # ---- accumulation --------------------------------------------------------------------------------------------------
    def acc(self, xs, c, n_out, flags=0, float_angle=False, double=False):
        """Accumulators [n_out][2] of channel c (float32, or float64 with the double taps of auto gain); xs = stream()."""
        start, row, _ = self.geometry(n_out)
        assert start.min() + self.pad() >= 0 and start.max() + self.pad() + self.K <= xs.shape[0]
        t32, t64 = self.taps(c, float_angle)
        t = t64 if double else t32
        out = np.zeros((n_out, 2), t.dtype)
        fn = lib().acc_f64 if double else lib().acc_f32
        fn(_p(xs), ctypes.c_int64(self.pad()), _p(t), self.K, _p(start), _p(row), ctypes.c_int64(n_out), flags, _p(out))
        return out

    def abs_sum(self, xs, c, n_out):
        """sum |g| |x| per output of channel c (double taps)."""
        start, row, _ = self.geometry(n_out)
        out = np.zeros(n_out)
        t64 = self.taps(c)[1]
        lib().abs_sum(_p(xs), ctypes.c_int64(self.pad()), _p(t64), self.K, _p(start), _p(row), ctypes.c_int64(n_out),
                      _p(out))
        return out

    # ---- epilogue ------------------------------------------------------------------------------------------------------
    def phase(self, c, n_out):
        """The exact mixer phase p (cycles * fs) of outputs 0..n_out-1 of channel c."""
        step = (self.down * self.delta[c]) % self.fs if self.centre else self.delta[c] % self.fs
        k = self.geometry(n_out)[2]
        return ((k % self.fs) * step) % self.fs

    def rotate(self, acc, c, f32=False):
        """y [n][2] float64: the accumulators rotated by exp(-j 2 pi p / fs) in float64 (f32=True: in float32, a variant
        the tests must resolve)."""
        p = self.phase(c, acc.shape[0])
        if f32:
            th = np.float32(-2.0) * p.astype(np.float32) / np.float32(self.fs)
            cs, sn = np.cos(np.float32(np.pi) * th), np.sin(np.float32(np.pi) * th)
            a = acc.astype(np.float32)
            return np.stack([a[:, 0] * cs - a[:, 1] * sn, a[:, 0] * sn + a[:, 1] * cs], axis=-1)
        th = np.pi * (-2.0 * p / self.fs)
        cs, sn = np.cos(th), np.sin(th)
        a = acc.astype(np.float64)
        return np.stack([a[:, 0] * cs - a[:, 1] * sn, a[:, 0] * sn + a[:, 1] * cs], axis=-1)

    def levels(self, y, gain, f32=False):
        """v = 127 + 128 gain y (float64; in float32 for the float32-rotation variant)."""
        if f32:
            return (np.float32(127) + np.float32(gain) * (np.float32(128) * y.astype(np.float32))).astype(np.float64)
        return 127.0 + (128.0 * float(np.float32(gain))) * y

    # ---- whole streams -------------------------------------------------------------------------------------------------
    def accumulators(self, x32, n_out=None, channels=None, **kw):
        """float32 [len(channels)][n_out][2] of a fresh stream x32 (float32 [n][2])."""
        n_out = n_outputs(x32.shape[0], self.up, self.down, self.M) if n_out is None else n_out
        xs = self.stream(x32)
        chs = range(self.n_ch) if channels is None else channels
        return np.stack([self.acc(xs, c, n_out, **kw) for c in chs]).reshape(len(chs), n_out, 2)

    def v(self, accs, gains, channels=None, f32=False):
        """v [len(channels)][n][2] of the accumulators accs at per-channel gains."""
        chs = range(self.n_ch) if channels is None else channels
        return np.stack([self.levels(self.rotate(a, c, f32), g, f32) for a, c, g in zip(accs, chs, gains)])

    def auto_gain(self, x32, channels=None):
        """(gain float32 [ch], near bool [ch]): lcs_chan_auto_gain over x32 from a fresh stream, and whether the double
        before the float rounding lies within GAIN_BAND of a float32 rounding boundary."""
        n_out = n_outputs(x32.shape[0], self.up, self.down, self.M)
        xs = self.stream(x32)
        chs = range(self.n_ch) if channels is None else channels
        g, near = [], []
        for c in chs:
            a = self.acc(xs, c, n_out, double=True)
            ms = float(np.sum(a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1])) / n_out
            gd = 0.25 / math.sqrt(ms) if ms > 0 else 1.0
            g.append(np.float32(gd))
            near.append(near_float_boundary(gd))
        return np.array(g, np.float32), np.array(near)


def near_float_boundary(d, rel=GAIN_BAND):
    """Whether the double d lies within rel * |d| of a midpoint between two adjacent float32 values."""
    f = np.float32(d)
    for nb in (np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))):
        mid = (float(f) + float(nb)) / 2
        if abs(d - mid) <= rel * abs(d):
            return True
    return False


def quantise(v):
    """(bytes uint8 [..][2], clipped per channel [n_ch]) of levels v [n_ch][n][2], as rotate_quantise."""
    r = np.rint(v)
    return np.clip(r, 0, 255).astype(np.uint8), ((r < 0) | (r > 255)).sum(axis=(1, 2))


def in_band(v):
    """Components whose level lies within BAND of a rounding boundary k + 1/2 (the clamp boundaries included)."""
    return np.abs(v - (np.floor(v) + 0.5)) <= BAND


def compare(got, clip_got, v, what):
    """Device bytes and clip counts against the model's levels v: equal outside the band, off by at most one inside it,
    clip counts off by at most the components in the band of a clamp boundary.  Returns the in-band count."""
    ref, clip_ref = quantise(v)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    band = in_band(v)
    d = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    bad = np.argwhere((d > 0) & ~band)
    assert not bad.size, "%s: %d bytes differ outside the band; first (ch, n, part, device, model, v): %s" % (
        what, len(bad), [(int(c), int(n), int(k), int(got[c, n, k]), int(ref[c, n, k]), float(v[c, n, k]))
                         for c, n, k in bad[:6]])
    assert d.max(initial=0) <= 1, what
    edge = (band & ((np.abs(v + 0.5) <= BAND) | (np.abs(v - 255.5) <= BAND))).sum(axis=(1, 2))
    dc = np.abs(np.asarray(clip_got, np.int64) - clip_ref)
    assert np.all(dc <= edge), (what, np.asarray(clip_got), clip_ref)
    return int(band.sum())


def resolves(v_model, v_variant):
    """Bytes of a variant that differ from the model's where the model's level lies outside the band."""
    a, _ = quantise(v_model)
    b, _ = quantise(v_variant)
    return int(((a != b) & ~in_band(v_model)).sum())
