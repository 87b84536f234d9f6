"""The channelizer's bytes (chan_kernel and rchan_kernel) bit for bit against chan_model, its FP32 arithmetic restated.

test_channelizer_gpu.py and test_rchan_gpu.py check the contract against the float64 oracle with a 1e-3 band, which
lets small arithmetic slips through (an edge tap dropped, taps summed in another order, a product rounded twice, a
float tap phase).  Here the accumulators are predicted exactly and only the FP64 epilogue, which the host cannot
reproduce to the bit, is given a band of 1e-9 of a level.  On the CPU the model is checked against the oracle, the
comparison is shown to resolve plausible slips on the exact inputs of the device cases, and the SASS is checked for
the absence of flush-to-zero.  On the device, through Channelizer and RationalChannelizer:
- chan_kernel at D = 2, 3, 4, 5, 7, 8, 13, 16, 25, 32 and 64; rchan_kernel at every rate of RATES in ci16, cs8, cu8 and
  cf32, and at up = 1 (D = 5 and 64) in cs8, cu8 and cf32;
- both band edges, DC, DC + 100 kHz (or half the edge where that lies outside the band) and random channels, 1, 5, 33
  or 41 of them (partial warps and CTAs); two tiles of outputs plus a partial one;
- auto gain, then 1x, 3x and 8x auto gain with clipping; pushes of 1, then fewer than M/up samples, then the rest;
- a 1024-channel push that spans two launches, a zero recording and a cf32 recording whose accumulators are
  subnormal, and one large case per kernel (over 2 10^6 byte components) for the slip test."""
import os
import re
import shutil
import subprocess
import zlib

import numpy as np
import pytest

import chan_model as CM
from conftest import ROOT
from test_channelizer_host import auto_gain_oracle, chan_oracle
from test_rchan_host import RATES, rchan_oracle, to_complex
from test_xcorr_fp32_exact_gpu import functions

FC_IN = 739e6
FORMATS = ("ci16", "cs8", "cu8", "cf32")
COUNTS = (1, 5, 33, 41)
CHAN_D = (2, 3, 4, 5, 7, 8, 13, 16, 25, 32, 64)
LEVEL = {"ci16": 1500.0, "cs8": 20.0, "cu8": 20.0, "cf32": 0.05}      # RMS of a noise recording in each format's units
SUBNORMAL_RMS = 2.0 ** -125                                            # RMS of the subnormal cf32 recording


def mhz(fs):
    return ("%.3f" % (fs / 1e6)).rstrip("0").rstrip(".") + "MHz"


# name: (fs_in, fmt, n_ch, kind); kind "noise", "large" (>= 2 10^6 byte components), "zero" or "subnormal"
CASES = {}
for i, D in enumerate(CHAN_D):
    CASES["chan_D%d" % D] = (D * 1.92e6, "ci16", COUNTS[i % 4], "noise")
for i, fs in enumerate(sorted(RATES)):
    for j, fmt in enumerate(FORMATS):
        CASES["rchan_%s_%s" % (mhz(fs), fmt)] = (fs, fmt, COUNTS[(i + j) % 4], "noise")
for i, D in enumerate((5, 64)):
    for j, fmt in enumerate(FORMATS[1:]):
        CASES["up1_D%d_%s" % (D, fmt)] = (D * 1.92e6, fmt, COUNTS[(i + j + 1) % 4], "noise")
CASES.update({
    "chan_D8_large": (8 * 1.92e6, "ci16", 41, "large"),
    "rchan_20MHz_cf32_large": (20e6, "cf32", 41, "large"),
    "chan_D4_zero": (4 * 1.92e6, "ci16", 5, "zero"),
    "rchan_2.4MHz_cu8_zero": (2.4e6, "cu8", 5, "zero"),
    "up1_D5_cf32_subnormal": (5 * 1.92e6, "cf32", 5, "subnormal"),
    "rchan_2.4MHz_cf32_subnormal": (2.4e6, "cf32", 33, "subnormal"),
})
LARGE = [name for name, c in CASES.items() if c[3] == "large"]


# ---------------------------------------------------------------------------------------------------------------------
# the inputs of a case
# ---------------------------------------------------------------------------------------------------------------------
def channel_offsets(rng, fs, n_ch, k):
    """Integer-Hz offsets from fc_in: the band edges, DC, DC + 100 kHz (half the edge if 100 kHz lies outside the band)
    and random ones, n_ch in all (for one channel, the k-th of the four fixed ones)."""
    edge = (fs - 1920000) // 2
    fixed = [-edge, edge, 0, 100000 if 100000 <= edge else edge // 2]
    out = fixed[:n_ch] if n_ch >= 4 else [fixed[k % 4]]
    while len(out) < n_ch:
        d = int(rng.integers(-edge, edge + 1))
        if d not in out:
            out.append(d)
    return np.array(out, np.int64)


def recording(rng, n, fs, fmt, offsets, kind):
    """[n][2] samples in fmt: complex noise plus a tone in each of the first six channels' passbands, at LEVEL RMS
    (SUBNORMAL_RMS for "subnormal"); zeros for "zero"."""
    dtype = {"ci16": np.int16, "cs8": np.int8, "cu8": np.uint8, "cf32": np.float32}[fmt]
    if kind == "zero":
        return np.full((n, 2), 127 if fmt == "cu8" else 0, dtype)
    m = np.arange(n)
    x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    for d in offsets[:6]:
        x += 2 * np.exp(2j * np.pi * ((int(d) + rng.uniform(-5e5, 5e5)) * m / fs))
    x /= np.sqrt(np.mean(np.abs(x) ** 2))
    v = np.stack([x.real, x.imag], axis=1) * (SUBNORMAL_RMS if kind == "subnormal" else LEVEL[fmt])
    if fmt == "cf32":
        return v.astype(np.float32)
    v = np.round(v)
    if fmt == "ci16":
        return np.clip(v, -32768, 32767).astype(np.int16)
    if fmt == "cs8":
        return np.clip(v, -128, 127).astype(np.int8)
    return np.clip(v + 127, 0, 255).astype(np.uint8)


def n_for_outputs(k, up, down, M):
    """The fewest input samples that give k outputs."""
    return ((k - 1) * down + M + 1 + up - 1) // up


class Case:
    """The inputs of a case and its model."""

    def __init__(self, lcs, name, fs_in=None, fmt=None, n_ch=None, kind=None, n_tiles=2):
        if name in CASES:
            fs_in, fmt, n_ch, kind = CASES[name]
        self.name, self.fs_in, self.fmt, self.kind = name, fs_in, fmt, kind
        self.rng = np.random.default_rng(zlib.crc32(name.encode()))
        self.up, self.down, self.h = lcs.chan_design_rational(fs_in)
        fs = int(round(fs_in))
        self.fcs = FC_IN + channel_offsets(self.rng, fs, n_ch, zlib.crc32(name.encode()) >> 3).astype(np.float64)
        self.model = CM.ChanModel(fs_in, FC_IN, self.fcs, fmt, self.up, self.down, self.h)
        self.M = self.model.M
        self.tile = 32 * max(1, -(-4 // self.up)) * self.up             # outputs per CTA
        if kind == "large":
            n_tiles = -(-2 * 10 ** 6 // (2 * n_ch * self.tile))
        self.n_out = n_tiles * self.tile + 37                           # whole tiles plus a partial one
        self.n = n_for_outputs(self.n_out, self.up, self.down, self.M)
        self.iq = recording(self.rng, self.n, fs, fmt, self.fcs - FC_IN, kind)
        self.x32 = CM.samples(self.iq, fmt)
        self.clip_factor = self.rng.choice([1.0, 3.0, 8.0], n_ch)     # 1x, 3x and 8x auto gain; 8x on one at least
        self.clip_factor[self.rng.integers(n_ch)] = 8.0

    @property
    def chan_kernel(self):
        return self.model.centre

    def pushes(self):
        """Push sizes: 1, then fewer than M/up samples, then the rest."""
        a = max(1, self.M // self.up // 2)
        assert 1 + a < self.n and a < self.M / self.up
        return [1, a, self.n - 1 - a]

    def channelizer(self, lcs, ctx, gain=None):
        if self.chan_kernel:
            return lcs.Channelizer(ctx, self.fs_in, FC_IN, self.fcs, gain=gain)
        return lcs.RationalChannelizer(ctx, self.fs_in, FC_IN, self.fcs, fmt=self.fmt, gain=gain)


@pytest.fixture(scope="module")
def cases(lcs):
    made = {}

    def get(name):
        if name not in made:
            made.clear()                                                 # one at a time: the large ones are large
            made[name] = Case(lcs, name)
        return made[name]
    return get


def test_every_case_is_covered(lcs, cases):
    """The case table covers what the device tests claim: every D, every rate x format, up = 1 in the other formats,
    every channel count, both kernels' large cases, the zero and subnormal recordings, partial tiles."""
    chan = sorted(int(round(c[0] / 1.92e6)) for c in CASES.values() if c[1] == "ci16" and c[3] == "noise"
                  and abs(c[0] / 1.92e6 - round(c[0] / 1.92e6)) < 1e-9)
    assert chan == list(CHAN_D)
    assert {(fs, fmt) for fs, fmt, _, k in CASES.values() if k == "noise"} >= {(fs, f) for fs in RATES for f in FORMATS}
    for D in (5, 64):
        assert {f for fs, f, _, _ in CASES.values() if fs == D * 1.92e6} >= {"cs8", "cu8", "cf32"}
    assert {c[2] for c in CASES.values()} >= set(COUNTS)
    for name in ("chan_D2", "rchan_2.048MHz_ci16", "rchan_100MHz_cf32", "up1_D64_cu8"):
        c = cases(name)
        assert c.n_out % c.tile == 37 and c.n_out > 2 * c.tile
    for name in LARGE:
        c = cases(name)
        assert 2 * c.fcs.size * c.n_out >= 2 * 10 ** 6
    assert {cases(name).chan_kernel for name in LARGE} == {True, False}


# ---------------------------------------------------------------------------------------------------------------------
# the model on the CPU
# ---------------------------------------------------------------------------------------------------------------------
def oracle_y(c, channels=None):
    fcs = c.fcs if channels is None else c.fcs[channels]
    if c.chan_kernel:
        return chan_oracle(c.iq, c.fs_in, FC_IN, fcs, c.h)
    return rchan_oracle(to_complex(c.iq, c.fmt), c.fs_in, FC_IN, fcs, c.h, c.up, c.down)


@pytest.mark.parametrize("name", list(CASES))
def test_model_matches_oracle(cases, name):
    """Before quantisation the model's y lies within the FP32 bound (2K + 2) 2^-24 sum |g||x| (+ the subnormal spacing
    per operation) of the float64 oracle, K taps per output; its auto gain is within one ulp of the oracle's."""
    c = cases(name)
    mod = c.model
    y_ref = oracle_y(c)
    xs = mod.stream(c.x32)
    for ch in range(mod.n_ch):
        y = mod.rotate(mod.acc(xs, ch, c.n_out), ch)
        bound = (2 * mod.K + 2) * (2.0 ** -24 * mod.abs_sum(xs, ch, c.n_out) + 2.0 ** -149) + 1e-15 * np.abs(y_ref[ch])
        err = np.maximum(np.abs(y[:, 0] - y_ref[ch].real), np.abs(y[:, 1] - y_ref[ch].imag))
        assert np.all(err <= bound), (name, ch, float((err / bound).max()))
    g, _ = mod.auto_gain(c.x32)
    g_ref = auto_gain_oracle(y_ref)
    assert np.abs(g.view(np.int32).astype(np.int64) - g_ref.view(np.int32)).max() <= 1


def variant_levels(c, accs, gains):
    """{variant: v} of the slips the comparison must resolve; the accumulation variants only for the large cases."""
    mod = c.model
    out = {"rotation in float32": mod.v(accs, gains, f32=True)}
    if c.kind == "large":
        for what, kw in (("oldest tap dropped", dict(flags=CM.DROP_OLDEST)),
                         ("newest input first", dict(flags=CM.NEWEST_FIRST)),
                         ("cmac's fmas reordered", dict(flags=CM.SWAP_FMA)),
                         ("multiply and add rounded separately", dict(flags=CM.UNFUSED)),
                         ("tap phases from a float angle", dict(float_angle=True))):
            out[what] = mod.v(mod.accumulators(c.x32, c.n_out, **kw), gains)
    return out


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c[3] != "zero"])
def test_the_comparison_resolves_plausible_slips(cases, name):
    """On the exact inputs of a device case, at auto gain and at the clipping gains: the float32 rotation moves nine
    levels in ten by more than 100 times the band, so the band cannot hide it; in the large cases it and every
    variant of the accumulation change a byte whose model level lies outside the band.  The variants move v by about 1e-6 to 1e-4 of a level, so a byte changes about ten times per 10^6
    components: the small cases cannot show it.  A zero recording gives 127 whatever the arithmetic; it is left out."""
    c = cases(name)
    mod = c.model
    accs = mod.accumulators(c.x32, c.n_out)
    g, _ = mod.auto_gain(c.x32)
    resolved, moved = {}, []
    for gains in (g, (g * c.clip_factor).astype(np.float32)):
        v = mod.v(accs, gains)
        for what, vv in variant_levels(c, accs, gains).items():
            resolved[what] = resolved.get(what, 0) + CM.resolves(v, vv)
            if what == "rotation in float32":
                moved.append(float(np.mean(np.abs(vv - v) > 100 * CM.BAND)))
    print("\n%s: bytes each variant changes outside the band: %s" % (name, resolved))
    assert min(moved) > 0.9, (name, moved)
    if c.kind == "large":
        assert all(k > 0 for k in resolved.values()), (name, resolved)


def test_subnormal_recordings_reach_subnormal_accumulators(cases):
    """The subnormal recordings' accumulators are mostly below 2^-126 (a flush to zero would zero them) and their auto
    gain is finite."""
    for name in (n for n, c in CASES.items() if c[3] == "subnormal"):
        c = cases(name)
        a = c.model.accumulators(c.x32, c.n_out)
        assert np.mean((a != 0) & (np.abs(a) < 2.0 ** -126)) > 0.5, name
        g, _ = c.model.auto_gain(c.x32)
        assert np.all(np.isfinite(g)) and np.all(g > 2.0 ** 100), name


# ---------------------------------------------------------------------------------------------------------------------
# the SASS: no flush to zero in the accumulation
# ---------------------------------------------------------------------------------------------------------------------
def test_chan_kernels_sass_has_no_ftz(tmp_path):
    """chan.cu compiled with the Makefile's flags: no FP32 instruction of either kernel carries .FTZ, and the byte path
    accumulates with FFMA."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    obj = str(tmp_path / "chan.o")
    subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                    "-lineinfo", "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function", "-c",
                    os.path.join(ROOT, "lte-cell-scanner_b200", "csrc", "chan.cu"), "-o", obj], check=True)
    fns = functions(subprocess.run([exe, "-sass", obj], capture_output=True, text=True, check=True).stdout)
    chan = [k for k in fns if "11chan_kernel" in k]
    rchan = [k for k in fns if "12rchan_kernel" in k]
    assert len(chan) == 2 and len(rchan) == 8                       # POWER x (ci16 / cs8 / cu8 / cf32 for rchan)
    for k in chan + rchan:
        f32 = [(hex(a), op) for a, op, _ in fns[k] if re.match(r"F(FMA|ADD|MUL|MNMX|SETP|SET|CHK)\b", op)]
        ftz = [x for x in f32 if ".FTZ" in x[1]]
        assert not ftz, (k, ftz[:6])
        if re.search(r"ILb0E|Lb0EE", k):                             # the byte path
            assert sum(op.startswith("FFMA") for _, op in f32) >= 16, k


# ---------------------------------------------------------------------------------------------------------------------
# the device against the model
# ---------------------------------------------------------------------------------------------------------------------
IN_BAND = {}                                                        # case -> components in the band, for the report


def check_gain(got, want, near, what):
    """Device gains == the model's bit for bit, one ulp allowed where the model's double lies at a float boundary."""
    d = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32))
    assert np.all(d <= near.astype(np.int64)), (what, got[d > near], want[d > near])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_bytes_match_model(lcs, ctx, cases, name):
    """Auto gain, then the bytes and clip counts of irregular pushes at that gain and, from a second channelizer, at
    1x, 3x and 8x of it, against the model of the whole stream."""
    c = cases(name)
    mod = c.model
    accs = mod.accumulators(c.x32, c.n_out)
    g_model, near = mod.auto_gain(c.x32)
    ch = c.channelizer(lcs, ctx)
    g = ch.auto_gain(c.iq)
    check_gain(g, g_model, near, name)
    parts, clip, i = [], 0, 0
    for k in c.pushes():
        o, cl = ch.push(c.iq[i:i + k])
        parts.append(o)
        clip = clip + cl
        i += k
    ch.close()
    out = np.concatenate(parts, axis=1)
    band = [CM.compare(out, clip, mod.v(accs, g), name + " auto gain")]
    if c.kind == "zero":
        assert np.all(g == 1) and np.all(out == 127) and not clip.any()
    if c.kind == "subnormal":
        assert np.std(out.astype(np.float64) - 127) > 20                # auto gain lifted them to full-scale bytes
    g2 = (g * c.clip_factor).astype(np.float32)
    ch = c.channelizer(lcs, ctx, gain=g2)
    out, clip = ch.push(c.iq)
    ch.close()
    band.append(CM.compare(out, clip, mod.v(accs, g2), name + " clipping gains"))
    if c.kind != "zero":
        assert clip.sum() > 0
    IN_BAND[name] = (band, out.size)
    print("\n%s: components in the band at auto gain / clipping gains: %s of %d each" % (name, band, out.size))
    assert sum(band) <= max(2, 1e-6 * out.size)


@pytest.mark.gpu
def test_push_spanning_launches_matches_model(lcs, ctx):
    """1024 channels at D = 3: a push of 20 037 outputs runs in two launches (16 384 outputs each at most); channels 0-3
    (the band edges, DC, DC + 100 kHz), 31, 32, 500 and 1023 against the model, gains from auto gain."""
    c = Case(lcs, "chan_D3_1024", 3 * 1.92e6, "ci16", 1024, "noise", n_tiles=156)
    assert c.n_out > 16384 and c.chan_kernel
    sel = [0, 1, 2, 3, 31, 32, 500, 1023]
    mod = c.model
    accs = mod.accumulators(c.x32, c.n_out, channels=sel)
    g_model, near = mod.auto_gain(c.x32, channels=sel)
    ch = c.channelizer(lcs, ctx)
    g = ch.auto_gain(c.iq)
    ch.close()
    check_gain(g[sel], g_model, near, c.name)
    ch = c.channelizer(lcs, ctx, gain=g)
    out, clip = ch.push(c.iq)
    assert ch.timing_read()[1] == 2
    ch.close()
    band = CM.compare(out[sel], clip[sel], mod.v(accs, g[sel], channels=sel), c.name)
    print("\n%s: components in the band: %d of %d" % (c.name, band, out[sel].size))
    assert band <= 2
