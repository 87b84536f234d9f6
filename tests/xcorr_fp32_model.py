"""A bit-exact model of the FP32 correlator's xc_incoherent_single (xcorr_fold_fp32_kernel) and of sp_fold_kernel's
sp_incoherent for float input (xcorr_fp32.cu, planset.cu).

The kernel is a fixed sequence of correctly rounded float32 operations, so `single` is determined to the last bit:
- templates: W = conj(fshift(pss_td))/137 in double (plan_build_kernel), each component rounded once to float32; taps
  137-139 are zero;
- samples: cf32 and cu8 (v - 127)/128 exactly, c128 rounded once to float32, 0 at and past n_cap;
- per half frame m, hypothesis f, root t and fold position idx the taps multiply x[soff[m][f] + idx + k] for k = 0..139
  in ascending k with cmac's four fmaf: re = fma(wx, xr, re), re = fma(-wy, xi, re), im = fma(wx, xi, im),
  im = fma(wy, xr, im); they run in five blocks of 28, each from zero, and the block sums are added in block order;
- the power RN(RN(re^2) + RN(im^2)) is added into pw in ascending m, and the result is RN(pw / n_comb).
The arithmetic is a small C++ library (std::fmaf, -ffp-contract=off) compiled once per process; it computes any subset
of hypotheses and fold positions.

sp_fold_kernel runs FP64: per block of 1024 positions and half frame, a 1536-element scan (6 samples per thread, a
Hillis-Steele warp scan, the warp offsets in order), sp = (ps[i+274] - ps[i]) / 274, the fold in ascending m, / n_comb_sp
and the shift by 137.  Its sample power is fma(x, x, RN(y^2)) in double (one DMUL, one DFMA in the SASS)."""
import ctypes
import math
import os
import subprocess
import tempfile

import numpy as np

from xcorr_tc_model import fma32, fold_offsets, n_comb_xc, pss_td  # noqa: F401  (fma32: what one fused rounding means)

N_FOLD, N_TAPS, NTAP_PAD, TAP_BLOCK = 9600, 137, 140, 28
TI, FW = 224, 8                                  # fold positions per CTA (32 lanes x 7), hypotheses per CTA
SMEM_CAP = 100 * 1024                            # planset_build's shared-memory limit for the FP32 correlator
# variants of the arithmetic (the comparison must resolve each of them from the kernel's)
ONE_CHAIN, FUSED_POWER, DESCENDING_M = 1, 2, 4

SRC = r"""
#include <cmath>
#include <cstdint>
extern "C" void fma_f32(const float* a, const float* b, const float* c, float* out, int64_t n) {
  for (int64_t i = 0; i < n; i++) out[i] = std::fmaf(a[i], b[i], c[i]);
}
// x: float32 [n_x][2] (zero past n_cap); w: float32 [n_f][3][140][2]; soff: int64 [n_comb][n_f]
// out: float32 [3][n_fsel][n_isel]
extern "C" void xc_single(const float* x, int64_t n_x, const float* w, const int64_t* soff, int n_comb, int n_f,
                          const int* fsel, int n_fsel, const int* isel, int n_isel, int flags, float* out) {
  const int n_work = 3 * n_fsel;
#pragma omp parallel for schedule(dynamic, 1)
  for (int job = 0; job < n_work; job++) {
    const int t = job / n_fsel, fi = job % n_fsel, f = fsel[fi];
    const float* wt = w + ((int64_t)f * 3 + t) * 140 * 2;
    float* o = out + ((int64_t)t * n_fsel + fi) * n_isel;
    constexpr int CH = 256;
    float pw[CH], sr[CH], si[CH], re[CH], im[CH];
    int64_t base[CH];
    for (int i0 = 0; i0 < n_isel; i0 += CH) {
      const int n = n_isel - i0 < CH ? n_isel - i0 : CH;
      for (int i = 0; i < n; i++) pw[i] = 0.f;
      for (int mm = 0; mm < n_comb; mm++) {
        const int m = (flags & 4) ? n_comb - 1 - mm : mm;
        for (int i = 0; i < n; i++) base[i] = soff[(int64_t)m * n_f + f] + isel[i0 + i];   // in range: checked by the caller
        const int block = (flags & 1) ? 140 : 28;
        for (int b0 = 0; b0 < 140; b0 += block) {
          for (int i = 0; i < n; i++) re[i] = im[i] = 0.f;
          for (int k = b0; k < b0 + block; k++) {
            const float wx = wt[2 * k], wy = wt[2 * k + 1];
            for (int i = 0; i < n; i++) {
              const float xr = x[2 * (base[i] + k)], xi = x[2 * (base[i] + k) + 1];
              re[i] = std::fmaf(wx, xr, re[i]);
              re[i] = std::fmaf(-wy, xi, re[i]);
              im[i] = std::fmaf(wx, xi, im[i]);
              im[i] = std::fmaf(wy, xr, im[i]);
            }
          }
          for (int i = 0; i < n; i++) {
            if (b0 == 0) { sr[i] = re[i]; si[i] = im[i]; }
            else { sr[i] = sr[i] + re[i]; si[i] = si[i] + im[i]; }
          }
        }
        for (int i = 0; i < n; i++) {
          const float p = (flags & 2) ? std::fmaf(si[i], si[i], sr[i] * sr[i]) : sr[i] * sr[i] + si[i] * si[i];
          pw[i] = pw[i] + p;
        }
      }
      for (int i = 0; i < n; i++) o[i0 + i] = pw[i] / (float)n_comb;
    }
  }
}
"""

_lib = None


def compile_model(source, name):
    """A model's C++ arithmetic compiled into a temporary directory and loaded: -ffp-contract=off keeps every product
    and sum separately rounded; std::fmaf is the one fused rounding (checked against fma32 by the tests)."""
    d = tempfile.mkdtemp(prefix=name + "_")
    src, so = os.path.join(d, "model.cpp"), os.path.join(d, "model.so")
    with open(src, "w") as fh:
        fh.write(source)
    subprocess.check_call(["g++", "-O3", "-march=native", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC",
                           "-shared", "-std=c++17", src, "-o", so])
    return ctypes.CDLL(so)


def lib():
    """The compiled arithmetic of `single` (compile_model)."""
    global _lib
    if _lib is None:
        _lib = compile_model(SRC, "xcorr_fp32_model")
    return _lib


def fmaf(a, b, c):
    """The compiled std::fmaf on float32 arrays."""
    a, b, c = (np.ascontiguousarray(v, np.float32) for v in (a, b, c))
    out = np.empty_like(a)
    P = ctypes.c_void_p
    lib().fma_f32(P(a.ctypes.data), P(b.ctypes.data), P(c.ctypes.data), P(out.ctypes.data), ctypes.c_int64(a.size))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# inputs as the kernel sees them
# ---------------------------------------------------------------------------------------------------------------------
def samples(iq, fmt):
    """float32 [n_cap][2]: load_iq of one buffer (cu8 uint8 [n][2], cf32 float32 [n][2], c128 float64 [n][2])."""
    if fmt == "cu8":
        return ((iq.astype(np.float64) - 127) / 128).astype(np.float32)       # exact
    if fmt == "cf32":
        assert iq.dtype == np.float32
        return iq
    assert iq.dtype == np.float64
    return iq.astype(np.float32)                                             # rounded once


_td = None


def templates(f, fc_req, fc_prog, fs_prog, exact=True):
    """float32 [n_f][3][140][2]: (Re W, Im W) of plan_build_kernel's d_w01 / d_w2, W = conj(td * rot) / 137 rounded once.
    exact=False divides the float32-rounded product by 137 in float32 instead (a variant the tests must resolve)."""
    global _td
    if _td is None:
        _td = pss_td()
    tap = np.arange(N_TAPS, dtype=np.float64)
    w = np.zeros((len(f), 3, NTAP_PAD, 2), np.float32)
    for j, fo in enumerate(np.asarray(f, np.float64)):
        k_factor = (fc_req - fo) / fc_prog
        k = (math.pi * fo) / ((fs_prog * k_factor) / 2.0)
        ph = k * tap
        cs, sn = np.cos(ph), np.sin(ph)
        re = _td.real * cs - _td.imag * sn
        im = _td.real * sn + _td.imag * cs
        if exact:
            w[j, :, :N_TAPS, 0] = (re / 137.0).astype(np.float32)
            w[j, :, :N_TAPS, 1] = (-im / 137.0).astype(np.float32)
        else:
            w[j, :, :N_TAPS, 0] = re.astype(np.float32) / np.float32(137)
            w[j, :, :N_TAPS, 1] = (-im).astype(np.float32) / np.float32(137)
    return w


class Fp32Model:
    """Templates, fold offsets and tile geometry of one plan (n_cap, f, fc_requested, fc_programmed, fs_programmed)."""

    def __init__(self, n_cap, f, fc_req, fc_prog, fs_prog):
        self.n_cap, self.f = n_cap, np.asarray(f, np.float64)
        self.cfg = (fc_req, fc_prog, fs_prog)
        self.n_f = len(self.f)
        self.n_comb = n_comb_xc(n_cap)
        self.off = fold_offsets(self.f, fc_req, fc_prog, fs_prog, self.n_comb)
        self.fw = 1 if self.n_f == 1 else FW
        self.n_fchunk = -(-self.n_f // self.fw)
        # planset_build: minimum and spread of the offsets per half frame and chunk (the unused tail repeats the last
        # hypothesis), the tile a CTA stages per half frame, and the range check
        pad = np.concatenate([self.off, np.repeat(self.off[:, -1:], self.n_fchunk * self.fw - self.n_f, axis=1)], axis=1)
        chunks = pad.reshape(self.n_comb, self.n_fchunk, self.fw)
        self.smin = chunks.min(axis=2)
        self.spread = int((chunks.max(axis=2) - self.smin).max())
        self.ti_blk = TI * (FW // self.fw)
        self.tile_len = self.ti_blk + NTAP_PAD + self.spread + 8
        self.smem = self.fw * NTAP_PAD * 24 + self.tile_len * 8 + 256 * 42 * 4
        self.in_range = bool((self.off >= 0).all() and (self.off + N_FOLD - 1 < n_cap - 136).all())
        self.accepted = self.in_range and self.smem <= SMEM_CAP
        self._w = {}

    def w(self, exact=True):
        if exact not in self._w:
            self._w[exact] = templates(self.f, *self.cfg, exact=exact)
        return self._w[exact]

    def last_tile_end(self):
        """One past the last sample the last CTA stages in the last half frame (zero-filled past n_cap)."""
        i0 = (-(-N_FOLD // self.ti_blk) - 1) * self.ti_blk
        return int(i0 + self.smin[-1].max() + self.tile_len)

    def single(self, x32, fs=None, idx=None, flags=0, exact_w=True):
        """float32 [3][len(fs)][len(idx)] of `single` for the samples x32 (float32 [n_cap][2]); all by default."""
        fs = np.arange(self.n_f) if fs is None else np.asarray(fs)
        idx = np.arange(N_FOLD) if idx is None else np.asarray(idx)
        assert x32.dtype == np.float32 and x32.shape == (self.n_cap, 2)
        x = np.zeros((self.n_cap + 256, 2), np.float32)
        x[:self.n_cap] = x32
        assert idx.min() >= 0 and self.off.min() >= 0 and self.off.max() + idx.max() + NTAP_PAD <= x.shape[0]
        w = np.ascontiguousarray(self.w(exact_w))
        off = np.ascontiguousarray(self.off, np.int64)
        fsel = np.ascontiguousarray(fs, np.int32)
        isel = np.ascontiguousarray(idx, np.int32)
        out = np.zeros((3, len(fsel), len(isel)), np.float32)
        P = ctypes.c_void_p
        lib().xc_single(P(x.ctypes.data), ctypes.c_int64(x.shape[0]), P(w.ctypes.data), P(off.ctypes.data), self.n_comb,
                        self.n_f, P(fsel.ctypes.data), len(fsel), P(isel.ctypes.data), len(isel), flags,
                        P(out.ctypes.data))
        return out


# ---------------------------------------------------------------------------------------------------------------------
# sp_fold_kernel for cf32 and c128
# ---------------------------------------------------------------------------------------------------------------------
SP_TILE, SP_THREADS, SP_ITEMS, SP_WIN = 1024, 256, 6, 274


def fma64(a, b, c):
    """RN_float64(a * b + c) with one rounding for non-negative c and |a b| far from under- and overflow: the exact
    product as p + e (Dekker), the exact sum p + c as s + t (TwoSum), then RN(s + RO(t + e)) with RO rounding to odd
    (Boldo and Melquiond's emulation of FMA)."""
    a, b, c = (np.asarray(v, np.float64) for v in (a, b, c))
    split = 134217729.0                                            # 2^27 + 1

    def halves(v):
        g = split * v
        hi = g - (g - v)
        return hi, v - hi

    p = a * b
    ah, al = halves(a)
    bh, bl = halves(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    s = p + c
    bb = s - p
    t = (p - (s - bb)) + (c - bb)
    u = t + e
    bb = u - t
    err = (t - (u - bb)) + (e - bb)
    odd = (u.view(np.int64) & 1) == 1
    fix = (err != 0) & ~odd
    u = np.where(fix, np.nextafter(u, np.where(err > 0, np.inf, -np.inf)), u)
    return s + u


def sample_power(iq, fmt):
    """pwr<FMT> of sp_fold_kernel: float64 [n]; fma(x, x, RN(y^2)) (exact products for cf32)."""
    v = iq.astype(np.float64)
    return fma64(v[:, 0], v[:, 0], v[:, 1] * v[:, 1])


def sp_model(pw, n_cap, block_scan=True):
    """sp_incoherent [9600] from the sample powers pw [n_cap] in sp_fold_kernel's order; block_scan=False takes a plain
    sequential prefix sum per block instead (a variant the tests must resolve)."""
    n_comb_sp = (n_cap - 136 - 137) // N_FOLD
    n_blk = -(-N_FOLD // SP_TILE)
    n_el = SP_THREADS * SP_ITEMS
    padded = np.zeros(n_comb_sp * N_FOLD + n_blk * SP_TILE + n_el)
    padded[:n_cap] = pw
    e = np.arange(n_el)
    base = np.arange(n_blk) * SP_TILE
    n_need = np.minimum(SP_TILE, N_FOLD - base) + SP_WIN - 1
    acc = None
    for m in range(n_comb_sp):
        v = np.where(e[None] < n_need[:, None], padded[m * N_FOLD + base[:, None] + e[None]], 0.0)   # [blk][1536]
        if block_scan:
            v = v.reshape(n_blk, SP_THREADS, SP_ITEMS)
            run = v[..., 0].copy()
            for k in range(1, SP_ITEMS):
                run = run + v[..., k]
            incl = run.reshape(n_blk, SP_THREADS // 32, 32).copy()
            for o in (1, 2, 4, 8, 16):
                prev = incl.copy()
                incl[..., o:] = incl[..., o:] + prev[..., :-o]
            wsum = incl[..., 31]
            woff = np.zeros_like(wsum)
            for w in range(1, SP_THREADS // 32):
                woff[:, w] = woff[:, w - 1] + wsum[:, w - 1]
            a = ((woff[..., None] + incl) - run.reshape(incl.shape)).reshape(n_blk, SP_THREADS)
            ps = np.empty((n_blk, n_el + 1))
            for k in range(SP_ITEMS):
                ps[:, k:n_el:SP_ITEMS] = a
                a = a + v[..., k]
            ps[:, n_el] = a[:, -1]
        else:
            ps = np.concatenate([np.zeros((n_blk, 1)), np.cumsum(v, axis=1)], axis=1)
        i = np.arange(SP_TILE)
        sp = ((ps[:, i + SP_WIN] - ps[:, i]) * 1.0) / SP_WIN
        acc = sp if m == 0 else acc + sp
    out = np.empty(N_FOLD)
    pos = (base[:, None] + np.arange(SP_TILE)[None]).reshape(-1)
    keep = pos < N_FOLD
    out[(pos[keep] + 137) % N_FOLD] = (acc / n_comb_sp).reshape(-1)[keep]
    return out
