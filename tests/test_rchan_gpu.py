"""The rational channelizer (lcs_chan_create_rational, lcs_chan_push) against its float64 oracle at the rates SDRs record
at, in every input format, and recordings at those rates driving the sweep, the cell tracker and the CLI."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "track_oracle"))

import lte_dl_synth as S  # noqa: E402
from test_channelizer_gpu import cells_by_id, check_bytes, mib, noise_and_tones, raster  # noqa: E402
from test_channelizer_host import auto_gain_oracle  # noqa: E402
from test_rchan_host import n_outputs, rchan_oracle, to_complex  # noqa: E402

N_CAP = 153600
FC_IN = 739e6


def requantise(iq16, fmt, rms=20.0):
    """A ci16 recording in another format: cs8 / cu8 scaled to an RMS of `rms` levels, cf32 as iq16 / 32768."""
    if fmt == "ci16":
        return iq16
    if fmt == "cf32":
        return (iq16.astype(np.float64) / 32768).astype(np.float32)
    v = np.round(iq16.astype(np.float64) * (rms / np.sqrt(np.mean(iq16.astype(np.float64) ** 2))))
    if fmt == "cs8":
        return np.clip(v, -128, 127).astype(np.int8)
    return np.clip(v + 127, 0, 255).astype(np.uint8)


def from_complex(x, fmt, scale):
    """Complex samples x as a recording: round(x * scale) in ci16 / cs8, + 127 in cu8, x as is in cf32."""
    if fmt == "cf32":
        return np.stack([x.real, x.imag], axis=1).astype(np.float32)
    v = np.round(np.stack([x.real, x.imag], axis=1) * scale)
    if fmt == "ci16":
        return np.clip(v, -32768, 32767).astype(np.int16)
    if fmt == "cs8":
        return np.clip(v, -128, 127).astype(np.int8)
    return np.clip(v + 127, 0, 255).astype(np.uint8)


def n_for_outputs(k, up, down, M):
    """The fewest input samples that give k outputs."""
    return ((k - 1) * down + M + 1 + up - 1) // up


def band_channels(rng, fs_in, fc_in, n_rand):
    edge = int(fs_in / 2 - 960e3)
    fcs = [fc_in - edge, fc_in + edge, fc_in, fc_in + 100e3]
    if n_rand:
        fcs += list(fc_in + rng.integers(-edge, edge, n_rand))
    return np.unique(np.array(fcs, np.float64))


# ---- bytes against the oracle ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fs_in,fmt", [(2.4e6, "cu8"), (2.5e6, "cf32"), (10e6, "cs8"), (20e6, "cs8"), (25e6, "ci16"),
                                       (56e6, "ci16")])
def test_rational_channelizer_matches_oracle(lcs, ctx, fs_in, fmt):
    rng = np.random.default_rng(int(fs_in) // 1000 + len(fmt))
    up, down, h = lcs.chan_design_rational(fs_in)
    M = (h.size - 1) // 2
    fcs = band_channels(rng, fs_in, FC_IN, 28)
    T = 32 * max(1, -(-4 // up)) * up                         # outputs per tile
    n = n_for_outputs(2 * T + 37, up, down, M) + 11
    iq16 = noise_and_tones(rng, n, fs_in, FC_IN, fcs[:6], amp=1500)
    iq = requantise(iq16, fmt)
    y = rchan_oracle(to_complex(iq, fmt), fs_in, FC_IN, fcs, h, up, down)
    ch = lcs.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt=fmt)
    assert (ch.up, ch.down) == (up, down) and np.array_equal(ch.taps, h)
    g = ch.auto_gain(iq)
    g_ref = auto_gain_oracle(y)
    assert np.abs(g.view(np.int32).astype(np.int64) - g_ref.view(np.int32)).max() <= 1
    out, clip = ch.push(iq)
    assert out.shape == (fcs.size, n_outputs(n, up, down, M), 2)
    check_bytes(out, clip, y, g)
    ch.close()
    # gains that clip: 1x to 8x the automatic gain
    g2 = (g * rng.choice([1.0, 3.0, 8.0], fcs.size)).astype(np.float32)
    ch = lcs.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt=fmt, gain=g2)
    out, clip = ch.push(iq)
    assert clip.sum() > 0
    check_bytes(out, clip, y, g2)
    ms, launches = ch.timing_read()
    assert launches >= 1 and ms > 0
    ch.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["cs8", "cu8", "cf32"])
def test_rational_channelizer_integer_d_other_formats(lcs, ctx, fmt):
    """At up = 1 the resampling kernel runs the D * 1.92 MHz filter for the formats lcs_chan_create does not take."""
    rng = np.random.default_rng(7)
    fs_in = 8 * 1.92e6
    fcs = band_channels(rng, fs_in, FC_IN, 8)
    h = lcs.chan_design_taps(fs_in)
    n = 5000
    iq = requantise(noise_and_tones(rng, n, fs_in, FC_IN, fcs[:3]), fmt)
    y = rchan_oracle(to_complex(iq, fmt), fs_in, FC_IN, fcs, h, 1, 8)
    ch = lcs.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt=fmt)
    g = ch.auto_gain(iq)
    assert np.abs(g.view(np.int32).astype(np.int64) - auto_gain_oracle(y).view(np.int32)).max() <= 1
    out, clip = ch.push(iq)
    check_bytes(out, clip, y, g)
    ch.close()


# ---- the integer-D identity -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [2, 16])
def test_rational_integer_d_is_lcs_chan_create(lcs, ctx, D):
    rng = np.random.default_rng(30 + D)
    fs_in = D * 1.92e6
    fcs = band_channels(rng, fs_in, FC_IN, 20)
    iq = noise_and_tones(rng, 300 * D + 3000, fs_in, FC_IN, fcs[:4])
    gain = (rng.uniform(1, 40, fcs.size)).astype(np.float32)        # some of them clip
    for g in (None, gain):
        a = lcs.Channelizer(ctx, fs_in, FC_IN, fcs, gain=g)
        b = lcs.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt="ci16", gain=g)
        if g is None:
            assert np.array_equal(a.auto_gain(iq[:2000]), b.auto_gain(iq[:2000]))
        for part in (iq[:1234], iq[1234:]):
            oa, ca = a.push_ci16(part)
            ob, cb = b.push(part)
            assert np.array_equal(oa, ob) and np.array_equal(ca, cb)
        assert np.array_equal(a.gain, b.gain)
        a.close()
        b.close()


# ---- push-size invariance, long pushes, coexistence -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fs_in,fmt", [(20e6, "cs8"), (25e6, "ci16")])
def test_rational_push_size_invariance(lcs, ctx, fs_in, fmt):
    rng = np.random.default_rng(int(fs_in) // 1000)
    fcs = band_channels(rng, fs_in, FC_IN, 5)
    one = lcs.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt=fmt)
    up, down, M = one.up, one.down, one.M
    n = n_for_outputs(5000, up, down, M)
    iq = requantise(noise_and_tones(rng, n, fs_in, FC_IN, fcs), fmt)
    ref, ref_clip = one.push(iq)
    assert ref.shape[1] == n_outputs(n, up, down, M)
    sizes = [1, 1, M // up - 1, 3, M // up, 1, down, 5000, 17, 1, down // up, up]
    sizes += list(rng.integers(1, 6000, 40))
    ch = lcs.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt=fmt)
    parts, clips, i = [], [], 0
    for k in sizes:
        k = min(int(k), n - i)
        expect = n_outputs(i + k, up, down, M) - n_outputs(i, up, down, M)
        assert ch.n_out(k) == expect
        o, c = ch.push(iq[i:i + k])
        assert o.shape[1] == expect
        parts.append(o)
        clips.append(c)
        i += k
    o, c = ch.push(iq[i:])
    parts.append(o)
    clips.append(c)
    assert np.array_equal(np.concatenate(parts, axis=1), ref)
    assert np.array_equal(np.sum(clips, axis=0), ref_clip)
    one.close()
    ch.close()


@pytest.mark.gpu
def test_rational_push_spanning_launches(lcs, ctx):
    """1024 channels at 2.5 Msps (up = 96): a push of 40 000 outputs runs in several launches; its bytes equal those of
    single-launch pushes and, on a sample of channels, the oracle's."""
    rng = np.random.default_rng(12)
    fs_in, fmt = 2.5e6, "cs8"
    edge = int(fs_in / 2 - 960e3)
    fcs = FC_IN + rng.integers(-edge, edge + 1, 1024).astype(np.float64)
    up, down, h = lcs.chan_design_rational(fs_in)
    M = (h.size - 1) // 2
    n = n_for_outputs(40000, up, down, M)
    iq = requantise(noise_and_tones(rng, n, fs_in, FC_IN, fcs[:4]), fmt)
    gain = np.full(fcs.size, 4.0, np.float32)
    big = lcs.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt=fmt, gain=gain)
    whole, clip_whole = big.push(iq)
    assert big.timing_read()[1] >= 2
    split = lcs.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt=fmt, gain=gain)   # a short push first: the long one starts in the carry
    a, _ = split.push(iq[:777])
    b, _ = split.push(iq[777:])
    small = lcs.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt=fmt, gain=gain)
    parts = [small.push(iq[i:i + 3000])[0] for i in range(0, n, 3000)]
    assert small.timing_read()[1] == sum(p.shape[1] > 0 for p in parts)
    assert np.array_equal(np.concatenate([a, b], axis=1), whole)
    assert np.array_equal(np.concatenate(parts, axis=1), whole)
    sel = np.r_[0:4, 500, 1000:1024]
    y = rchan_oracle(to_complex(iq, fmt), fs_in, FC_IN, fcs[sel], h, up, down)
    check_bytes(whole[sel], clip_whole[sel], y, gain[sel])
    for c in (big, split, small):
        c.close()


@pytest.mark.gpu
def test_rational_channelizers_coexist(lcs, ctx):
    """Channelizers at 25 Msps (the largest tile), 2.4 Msps and D = 32 alive together, pushes interleaved."""
    rng = np.random.default_rng(8)
    chans = []
    for fs_in, fmt in ((2.4e6, "cu8"), (25e6, "ci16"), (32 * 1.92e6, "ci16")):
        up, down, h = lcs.chan_design_rational(fs_in)
        fcs = FC_IN + np.array([0.0, -2e5, 2e5])
        iq = requantise(noise_and_tones(rng, n_for_outputs(3000, up, down, (h.size - 1) // 2), fs_in, FC_IN, fcs), fmt)
        y = rchan_oracle(to_complex(iq, fmt), fs_in, FC_IN, fcs, h, up, down)
        chans.append((lcs.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt=fmt), iq, y))
    for ch, iq, _ in chans:
        ch.auto_gain(iq)
    got = [[] for _ in chans]
    for part in range(2):
        for i, (ch, iq, _) in enumerate(chans):
            k = iq.shape[0] // 2
            got[i].append(ch.push(iq[:k] if part == 0 else iq[k:]))
    for (ch, iq, y), g in zip(chans, got):
        out = np.concatenate([o for o, _ in g], axis=1)
        check_bytes(out, g[0][1] + g[1][1], y, ch.gain)
        ch.close()


@pytest.mark.gpu
def test_rational_bad_arguments(lcs, ctx):
    import ctypes as C
    L = lcs
    launches = ctx.launches
    for fs_in, fcs in ((1.92e6, [FC_IN]), (1.9e6, [FC_IN]), (10.5e6 + 0.5, [FC_IN]), (123e6, [FC_IN]), (31e6, [FC_IN]),
                       (10e6, []), (10e6, [FC_IN] * 1025), (10e6, [FC_IN + 0.5]), (10e6, [FC_IN + 4.04e6 + 1]),
                       (10e6, [FC_IN - 4.04e6 - 1])):
        with pytest.raises(L.LcsError, match="error 1"):
            L.RationalChannelizer(ctx, fs_in, FC_IN, fcs, fmt="cs8")
    for g in (0.0, -1.0, float("nan")):
        with pytest.raises(L.LcsError, match="error 1"):
            L.RationalChannelizer(ctx, 10e6, FC_IN, [FC_IN], fmt="cs8", gain=[g])
    lib = L.lib()
    h = C.c_void_p()
    fc = np.array([FC_IN])
    for fmt in (L.IQ_C128, 5, -1):
        assert lib.lcs_chan_create_rational(ctx._h, C.c_double(10e6), fmt, C.c_double(FC_IN), 1, fc.ctypes.data, None,
                                            C.byref(h)) == 1
    ok = L.RationalChannelizer(ctx, 10e6, FC_IN, [FC_IN - 4.04e6, FC_IN + 4.04e6], fmt="cs8")   # the band edges are valid
    iq = np.zeros((4000, 2), np.int8)
    with pytest.raises(ValueError):
        ok.push(iq.astype(np.int16))                                           # the wrong dtype
    out = np.zeros((2, 4000, 2), np.uint8)
    n = C.c_uint32(0)
    k = ok.n_out(4000)
    assert k > 0
    assert lib.lcs_chan_push_ci16(ok._h, iq.ctypes.data, 4000, out.ctypes.data, 4000, 0, C.byref(n), None) == 1
    assert lib.lcs_chan_auto_gain_ci16(ok._h, iq.ctypes.data, 4000) == 1
    assert lib.lcs_chan_push(ok._h, iq.ctypes.data, 4000, out.ctypes.data, k - 1, 0, C.byref(n), None) == 1
    assert lib.lcs_chan_push(ok._h, None, 5, out.ctypes.data, 4000, 0, C.byref(n), None) == 1
    assert lib.lcs_chan_auto_gain(ok._h, iq.ctypes.data, 10) == 1             # fewer samples than one output
    assert ctx.launches == launches
    assert ok.n_out(4000) == k                                                 # nothing was consumed
    ok.close()


# ---- end to end -------------------------------------------------------------------------------------------------------------
def channelize_to_device(lcs, ctx, iq, fs_in, fc_in, fcs, fmt):
    import torch
    ch = lcs.RationalChannelizer(ctx, fs_in, fc_in, fcs, fmt=fmt)
    ch.auto_gain(iq)
    out = torch.empty((len(fcs), N_CAP, 2), dtype=torch.uint8, device="cuda")
    k, _ = ch.push_device(iq, out)
    assert k == N_CAP
    ch.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fs_in,fmt,shift", [(20e6, "cs8", 3.1e6), (2.4e6, "cu8", 0.2e6)])
def test_rational_real_recording(lcs, ctx, capbuf0000, fs_in, fmt, shift):
    """The recorded capture resampled to an SDR rate, moved off centre and requantised, swept over every raster channel:
    cells 277 and 271 come back as the search on the original bytes finds them."""
    from fractions import Fraction
    from scipy.signal import resample_poly
    fc = capbuf0000["fc"]
    fc_in = fc - shift
    ref_cells, _ = ctx.cell_search(capbuf0000["cu8"], lcs.f_search_set(fc, 120.0), fc, fc, 1.92e6)
    ref = cells_by_id(ref_cells)
    assert {271, 277} <= set(ref)
    r = Fraction(int(fs_in), 1920000)
    x = resample_poly(capbuf0000["capbuf"], r.numerator, r.denominator)
    x *= np.exp(2j * np.pi * shift * np.arange(x.size) / fs_in)
    up, down, h = lcs.chan_design_rational(fs_in)
    n = n_for_outputs(N_CAP, up, down, (h.size - 1) // 2)
    rng = np.random.default_rng(11)
    pad = max(0, n - x.size)
    x = np.concatenate([x, 0.01 * (rng.standard_normal(pad) + 1j * rng.standard_normal(pad))])[:n]
    iq = from_complex(x, fmt, 100.0)
    fcs = raster(fs_in, fc_in)
    out = channelize_to_device(lcs, ctx, iq, fs_in, fc_in, fcs, fmt)
    sw = lcs.Sweep(ctx, N_CAP)
    per_ch = sw.search_cu8_device(out, fcs, lcs.f_search_set(fcs[0], 120.0), max_cells=16)
    sw.close()
    at_fc = cells_by_id(per_ch[int(np.argmin(np.abs(fcs - fc)))])
    for cid in (271, 277):
        assert mib(at_fc[cid]) == mib(ref[cid])
        assert abs(at_fc[cid].freq_superfine - ref[cid].freq_superfine) < 50


SWEEP_CARRIERS = [   # (offset from fc_in, cell, relative power)
    (-9.5e6, dict(n_id_cell=101, n_ports=1, cp_type=1, n_rb_dl=25, phich_duration=1, phich_resource=3, t0=500.0, sfn0=10), 1.0),
    (-3.0e6, dict(n_id_cell=277, n_ports=2, cp_type=1, n_rb_dl=50, phich_duration=2, phich_resource=1, t0=7000.0, sfn0=500), 100.0),
    (6.2e6, dict(n_id_cell=350, n_ports=2, cp_type=2, n_rb_dl=15, phich_duration=1, phich_resource=4, t0=12000.0, sfn0=1000), 1.0),
]


@pytest.mark.gpu
def test_rational_synthetic_sweep(lcs, ctx):
    """A 25 Msps cf32 recording with three carriers and an 8 ppm clock error, every raster channel swept: after dedup
    exactly the planted cells, with their MIB."""
    fs_in = 25e6
    f_true = 8e-6 * FC_IN
    k = (FC_IN - f_true) / FC_IN
    up, down, h = lcs.chan_design_rational(fs_in)
    n = n_for_outputs(N_CAP, up, down, (h.size - 1) // 2)
    carriers = [(FC_IN + off, [d], p) for off, d, p in SWEEP_CARRIERS]
    iq = requantise(S.synth_wide_ci16(n, fs_in, FC_IN, carriers, f_true=f_true, snr_db=10, seed=21, scale=2048.0), "cf32")
    fcs = raster(fs_in, FC_IN)
    assert fcs.size == 231
    out = channelize_to_device(lcs, ctx, iq, fs_in, FC_IN, fcs, "cf32")
    sw = lcs.Sweep(ctx, N_CAP)
    per_ch = sw.search_cu8_device(out, fcs, lcs.f_search_set(fcs[0], 15.0), max_cells=16)
    sw.close()
    final = lcs.dedup([c for cs in per_ch for c in cs])
    assert sorted(c.n_id_cell() for c in final) == sorted(d["n_id_cell"] for _, d, _ in SWEEP_CARRIERS)
    ids = cells_by_id(final)
    for off, d, _ in SWEEP_CARRIERS:
        c = ids[d["n_id_cell"]]
        fc_c = FC_IN + off
        assert mib(c) == (d["n_id_cell"], d["n_ports"], d["cp_type"], d["n_rb_dl"], d["phich_duration"], d["phich_resource"],
                          d["sfn0"])
        assert abs(c.fc_requested + c.freq_superfine - (fc_c + fc_c * (1 - k))) < 100


@pytest.mark.gpu
def test_tracker_fed_by_rational_channelizer(lcs, ctx):
    """The cell tracker on a 2.4 Msps cu8 recording channelized in odd-sized chunks: device and oracle agree and every
    MIB locks from the first attempt, so the fractional output timing survives push boundaries."""
    from test_tracker_gpu import run_pair
    from test_tracker_oracle import lcs_cell
    fs_in, fc_in, f_true = 2.4e6, 739e6, 3000.0
    k = (fc_in - f_true) / fc_in
    a = dict(n_id_cell=277, n_ports=2, cp_type=1, n_rb_dl=6, phich_duration=1, phich_resource=3, t0=1234.0, sfn0=100)
    n = int(0.6 * fs_in)
    iq = requantise(S.synth_wide_ci16(n, fs_in, fc_in, [(fc_in, [a], 1.0)], f_true=f_true, snr_db=10, seed=31), "cu8")
    ch = lcs.RationalChannelizer(ctx, fs_in, fc_in, [fc_in], fmt="cu8")
    ch.auto_gain(iq[:int(0.08 * fs_in)])
    parts = [ch.push(iq[i:i + 123457])[0] for i in range(0, n, 123457)]
    ch.close()
    cu8s = np.ascontiguousarray(np.concatenate(parts, axis=1))
    up, down, h = lcs.chan_design_rational(fs_in)
    assert cu8s.shape[1] == n_outputs(n, up, down, (h.size - 1) // 2)
    fo0 = np.array([fc_in * (1 - k) - 300])
    res, _ = run_pair(lcs, ctx, cu8s, [[(lcs_cell(a), a["t0"] - 2 + 0.6)]], fo0, 96000, fc=[fc_in])
    for (r,) in res:
        assert r["mib_successes"] == r["mib_attempts"] > 0


@pytest.mark.gpu
def test_cli_resample_search(lcs, ctx, tmp_path):
    """`CellSearch_b200 --wideband ... --resample --format cs8` on a 20 Msps recording: the cell table holds the planted
    cell once, at its raster channel."""
    host = os.path.join(ROOT, "lte-cell-scanner_b200", "host")
    subprocess.check_call(["make", "-C", host, "-s"])
    fs_in = 20e6
    up, down, h = lcs.chan_design_rational(fs_in)
    n = n_for_outputs(N_CAP, up, down, (h.size - 1) // 2)
    d = dict(n_id_cell=211, n_ports=2, cp_type=1, n_rb_dl=75, phich_duration=1, phich_resource=3, t0=3000.0, sfn0=12)
    iq16 = S.synth_wide_ci16(n, fs_in, FC_IN, [(FC_IN + 1.5e6, [d], 1.0)], f_true=2000.0, snr_db=10, seed=41)
    requantise(iq16, "cs8").tofile(str(tmp_path / "wide.cs8"))
    out = subprocess.run([os.path.join(host, "CellSearch_b200"), "--wideband", str(tmp_path / "wide.cs8"), "--fs-in", "20e6",
                          "--fc-in", "739e6", "--resample", "--format", "cs8", "-s", "739.5e6", "-e", "741.5e6", "-p", "15"],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "Channelizing and examining 21 center frequencies" in out.stdout
    rows = re.findall(r"^\s*(\d+)\s+(\d)\s+([0-9.]+)M", out.stdout, re.M)
    assert rows == [("211", "2", "740.5")]
