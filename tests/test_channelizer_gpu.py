"""The device channelizer (lcs_chan_*) against its float64 oracle, and wideband recordings driving the sweep and the
cell tracker."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "track_oracle"))

import lte_dl_synth as S  # noqa: E402
from test_channelizer_host import auto_gain_oracle, chan_oracle, n_outputs, quantise  # noqa: E402
from test_search_chain_gpu import same_cells  # noqa: E402

N_CAP = 153600


def near_boundary(v, tol=1e-3):
    """Components whose float64 value lies within tol of a rounding (k + 1/2) or clamp boundary."""
    return np.abs(v - (np.floor(v) + 0.5)) < tol


def check_bytes(got, clip_got, y, gain):
    ref, clip_ref, v = quantise(y, gain)
    d = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    amb = near_boundary(v)
    assert d.max() <= 1
    assert not np.any((d > 0) & ~amb), np.argwhere((d > 0) & ~amb)[:5]
    edge = ((np.abs(v + 0.5) < 1e-3) | (np.abs(v - 255.5) < 1e-3)).sum(axis=(1, 2))
    assert np.all(np.abs(clip_got.astype(np.int64) - clip_ref) <= edge)


def noise_and_tones(rng, n, fs_in, fc_in, fcs, amp=2000):
    m = np.arange(n)
    x = amp * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    for fc in fcs:                                        # one tone inside each channel's passband
        x += 4 * amp * np.exp(2j * np.pi * ((fc - fc_in) + rng.uniform(-5e5, 5e5)) * m / fs_in)
    return np.clip(np.round(np.stack([x.real, x.imag], axis=1)), -32768, 32767).astype(np.int16)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [2, 8, 16, 32])
def test_channelizer_matches_oracle(lcs, ctx, D):
    rng = np.random.default_rng(100 + D)
    fs_in, fc_in = D * 1.92e6, 2140e6
    edge = fs_in / 2 - 960e3
    fcs = np.unique(np.concatenate([[fc_in - edge, fc_in + edge, fc_in, fc_in + 100e3],
                                    fc_in + rng.integers(-int(edge), int(edge), 36)])).astype(np.float64)
    h = lcs.chan_design_taps(fs_in)
    n = 2 * 128 * D + 3 * h.size + 17
    iq = noise_and_tones(rng, n, fs_in, fc_in, fcs[:8])
    y = chan_oracle(iq, fs_in, fc_in, fcs, h)
    # auto gain: the mean over the outputs of a fresh channelizer, to one float ulp
    ch = lcs.Channelizer(ctx, fs_in, fc_in, fcs)
    assert np.array_equal(ch.taps, h)
    g = ch.auto_gain(iq)
    g_ref = auto_gain_oracle(y)
    assert np.abs(g.view(np.int32).astype(np.int64) - g_ref.view(np.int32)).max() <= 1
    out, clip = ch.push_ci16(iq)
    assert out.shape == (fcs.size, n_outputs(n, D, h.size // 2), 2)
    check_bytes(out, clip, y, g)
    ch.close()
    # gains that clip: 1x to 8x the automatic gain
    g2 = (g * rng.choice([1.0, 3.0, 8.0], fcs.size)).astype(np.float32)
    ch = lcs.Channelizer(ctx, fs_in, fc_in, fcs, gain=g2)
    out, clip = ch.push_ci16(iq)
    assert clip.sum() > 0
    check_bytes(out, clip, y, g2)
    ms, launches = ch.timing_read()
    assert launches >= 1 and ms > 0
    ch.close()


@pytest.mark.gpu
def test_channelizer_push_size_invariance(lcs, ctx):
    rng = np.random.default_rng(4)
    D, fc_in = 8, 739e6
    fs_in = D * 1.92e6
    fcs = fc_in + np.array([-3.1e6, -2e5, 0.0, 1.7e6, 6.72e6])
    n = 20000
    iq = noise_and_tones(rng, n, fs_in, fc_in, fcs)
    one = lcs.Channelizer(ctx, fs_in, fc_in, fcs)
    M = one.M
    ref, ref_clip = one.push_ci16(iq)
    assert ref.shape[1] == n_outputs(n, D, M)
    sizes = [1, 1, M - 1, 3, M, 1, D, 5000, 17, 1]
    sizes += list(rng.integers(1, 3000, 40))
    ch = lcs.Channelizer(ctx, fs_in, fc_in, fcs)
    parts, i, total = [], 0, 0
    for k in sizes:
        k = min(int(k), n - i)
        expect = n_outputs(i + k, D, M) - n_outputs(i, D, M)
        assert ch.n_out(k) == expect
        o, _ = ch.push_ci16(iq[i:i + k])
        assert o.shape[1] == expect
        parts.append(o)
        i += k
        total += expect
    o, _ = ch.push_ci16(iq[i:])
    parts.append(o)
    assert np.array_equal(np.concatenate(parts, axis=1), ref)
    one.close()
    ch.close()


@pytest.mark.gpu
def test_channelizers_of_different_rates_coexist(lcs, ctx):
    """A channelizer with a large input tile (D = 32) keeps working after one with a small tile (D = 2) is created, and
    both match the oracle with their pushes interleaved."""
    rng = np.random.default_rng(8)
    chans = []
    for D in (32, 2):
        fs_in, fc_in = D * 1.92e6, 739e6
        fcs = fc_in + np.array([0.0, -3e5, 7e5])
        h = lcs.chan_design_taps(fs_in)
        iq = noise_and_tones(rng, 300 * D + 2 * h.size, fs_in, fc_in, fcs)
        chans.append((lcs.Channelizer(ctx, fs_in, fc_in, fcs), iq, chan_oracle(iq, fs_in, fc_in, fcs, h)))
    for ch, iq, y in chans:
        ch.auto_gain(iq)
    got = [[] for _ in chans]
    for part in range(2):                            # interleaved pushes, halves of each recording
        for i, (ch, iq, _) in enumerate(chans):
            h = iq.shape[0] // 2
            got[i].append(ch.push_ci16(iq[:h] if part == 0 else iq[h:]))
    for (ch, iq, y), g in zip(chans, got):
        out = np.concatenate([o for o, _ in g], axis=1)
        check_bytes(out, g[0][1] + g[1][1], y, ch.gain)
        ch.close()


@pytest.mark.gpu
def test_channelizer_push_spanning_launches(lcs, ctx):
    """1024 channels at D = 2: a push of 20 000 outputs runs in two launches (16 384 outputs each at most).  The bytes
    equal those of single-launch pushes and, on a sample of channels, the oracle's."""
    rng = np.random.default_rng(12)
    D, fc_in = 2, 739e6
    fs_in = D * 1.92e6
    fcs = fc_in + rng.integers(-960000, 960001, 1024).astype(np.float64)
    h = lcs.chan_design_taps(fs_in)
    n = 40000 + 2 * h.size
    iq = noise_and_tones(rng, n, fs_in, fc_in, fcs[:4])
    gain = np.full(fcs.size, 4.0, np.float32)
    big = lcs.Channelizer(ctx, fs_in, fc_in, fcs, gain=gain)
    whole, clip_whole = big.push_ci16(iq)
    assert big.timing_read()[1] == 2
    assert whole.shape[1] == n_outputs(n, D, h.size // 2) > 16384
    split = lcs.Channelizer(ctx, fs_in, fc_in, fcs, gain=gain)   # a short push first: the long one starts in the carry
    a, _ = split.push_ci16(iq[:777])
    b, _ = split.push_ci16(iq[777:])
    assert split.timing_read()[1] == 3
    small = lcs.Channelizer(ctx, fs_in, fc_in, fcs, gain=gain)
    parts = [small.push_ci16(iq[i:i + 3000])[0] for i in range(0, n, 3000)]
    assert small.timing_read()[1] == len(parts)
    assert np.array_equal(np.concatenate([a, b], axis=1), whole)
    assert np.array_equal(np.concatenate(parts, axis=1), whole)
    sel = np.r_[0:4, 500, 1000:1024]
    check_bytes(whole[sel], clip_whole[sel], chan_oracle(iq, fs_in, fc_in, fcs[sel], h), gain[sel])
    for c in (big, split, small):
        c.close()


@pytest.mark.gpu
def test_channelizer_bad_arguments(lcs, ctx):
    L = lcs
    fc_in = 739e6
    launches = ctx.launches
    for fs_in, fcs in ((10e6, [fc_in]), (65 * 1.92e6, [fc_in]), (1.92e6, [fc_in]),
                       (7.68e6, []), (7.68e6, [fc_in] * 1025),
                       (7.68e6, [fc_in + 0.5]), (7.68e6, [fc_in + 2.88e6 + 1]), (7.68e6, [fc_in - 2.88e6 - 1])):
        with pytest.raises(L.LcsError, match="error 1"):
            L.Channelizer(ctx, fs_in, fc_in, fcs)
    for g in (0.0, -1.0, float("nan")):
        with pytest.raises(L.LcsError, match="error 1"):
            L.Channelizer(ctx, 7.68e6, fc_in, [fc_in], gain=[g])
    ok = L.Channelizer(ctx, 7.68e6, fc_in, [fc_in - 2.88e6, fc_in + 2.88e6])   # the band edges themselves are valid
    iq = np.zeros((1000, 2), np.int16)
    lib = L.lib()
    import ctypes as C
    out = np.zeros((2, 1000, 2), np.uint8)
    n = C.c_uint32(0)
    k = ok.n_out(1000)
    assert k > 0
    assert lib.lcs_chan_push_ci16(ok._h, iq.ctypes.data, 1000, out.ctypes.data, k - 1, 0, C.byref(n), None) == 1
    assert lib.lcs_chan_push_ci16(ok._h, None, 5, out.ctypes.data, 1000, 0, C.byref(n), None) == 1
    assert lib.lcs_chan_auto_gain_ci16(ok._h, iq.ctypes.data, 10) == 1       # fewer samples than one output
    assert ctx.launches == launches
    assert ok.n_out(1000) == k                                                # nothing was consumed
    ok.close()


def cells_by_id(cells):
    return {c.n_id_cell(): c for c in cells}


def mib(c):
    return (c.n_id_cell(), c.n_ports, c.cp_type, c.n_rb_dl, c.phich_duration, c.phich_resource, c.sfn)


def channelize_to_device(lcs, ctx, iq, fs_in, fc_in, fcs):
    import torch
    ch = lcs.Channelizer(ctx, fs_in, fc_in, fcs)
    ch.auto_gain(iq)
    out = torch.empty((len(fcs), N_CAP, 2), dtype=torch.uint8, device="cuda")
    k, _ = ch.push_ci16_device(iq, out)
    assert k == N_CAP
    ch.close()
    return out


def raster(fs_in, fc_in):
    edge = fs_in / 2 - 960e3
    return fc_in + 100e3 * np.arange(-int(edge // 100e3), int(edge // 100e3) + 1)


@pytest.mark.gpu
def test_wideband_real_recording(lcs, ctx, capbuf0000):
    from scipy.signal import resample_poly
    fc = capbuf0000["fc"]
    fs_in, D = 15.36e6, 8
    fc_in = fc - 3.1e6
    real = capbuf0000["cu8"]
    ref_cells, _ = ctx.cell_search(real, lcs.f_search_set(fc, 120.0), fc, fc, 1.92e6)
    ref = cells_by_id(ref_cells)
    assert {271, 277} <= set(ref)
    x = resample_poly(capbuf0000["capbuf"], D, 1)
    x *= np.exp(2j * np.pi * 3.1e6 * np.arange(x.size) / fs_in)
    h = lcs.chan_design_taps(fs_in)
    n = 153599 * D + h.size // 2 + 1
    rng = np.random.default_rng(11)
    pad = n - x.size + 1000
    x = np.concatenate([x, 0.1 * (rng.standard_normal(pad) + 1j * rng.standard_normal(pad))])
    syn = dict(n_id_cell=123, n_ports=2, cp_type=1, n_rb_dl=50, phich_duration=1, phich_resource=2, t0=4000.0, sfn0=300)
    w = S.synth_wide_ci16(x.size, fs_in, fc_in, [(fc_in - 4.0e6, [syn], 1.0)], snr_db=25, seed=12, scale=8192.0)
    iq = np.clip(np.round(np.stack([x.real, x.imag], axis=1) * 8192) + w, -32768, 32767).astype(np.int16)[:n]
    fcs = raster(fs_in, fc_in)
    out = channelize_to_device(lcs, ctx, iq, fs_in, fc_in, fcs)
    sw = lcs.Sweep(ctx, N_CAP)
    per_ch = sw.search_cu8_device(out, fcs, lcs.f_search_set(fcs[0], 120.0), max_cells=16)
    sw.close()
    at_fc = cells_by_id(per_ch[int(np.argmin(np.abs(fcs - fc)))])
    for cid in (271, 277):
        assert mib(at_fc[cid]) == mib(ref[cid])
        assert abs(at_fc[cid].freq_superfine - ref[cid].freq_superfine) < 50
    final = lcs.dedup([c for cs in per_ch for c in cs])
    ids = cells_by_id(final)
    assert {271, 277, 123} <= set(ids)
    assert mib(ids[123]) == (123, 2, 1, 50, 1, 2, 300) and ids[123].fc_requested == fc_in - 4.0e6


SWEEP_CARRIERS = [   # (offset from fc_in, cell, relative power)
    (-4.5e6, dict(n_id_cell=101, n_ports=1, cp_type=1, n_rb_dl=25, phich_duration=1, phich_resource=3, t0=500.0, sfn0=10), 1.0),
    (-3.0e6, dict(n_id_cell=277, n_ports=2, cp_type=1, n_rb_dl=50, phich_duration=2, phich_resource=1, t0=7000.0, sfn0=500), 100.0),
    (4.2e6, dict(n_id_cell=350, n_ports=2, cp_type=2, n_rb_dl=15, phich_duration=1, phich_resource=4, t0=12000.0, sfn0=1000), 1.0),
]


@pytest.fixture(scope="module")
def synthetic_sweep(lcs, ctx):
    fs_in, fc_in, D = 15.36e6, 739e6, 8
    f_true = 8e-6 * fc_in
    h = lcs.chan_design_taps(fs_in)
    n = 153599 * D + h.size // 2 + 1
    carriers = [(fc_in + off, [d], p) for off, d, p in SWEEP_CARRIERS]
    iq = S.synth_wide_ci16(n, fs_in, fc_in, carriers, f_true=f_true, snr_db=10, seed=21, scale=2048.0)
    fcs = raster(fs_in, fc_in)
    out = channelize_to_device(lcs, ctx, iq, fs_in, fc_in, fcs)
    return dict(fs_in=fs_in, fc_in=fc_in, f_true=f_true, fcs=fcs, out=out, f_set=lcs.f_search_set(fcs[0], 15.0))


@pytest.mark.gpu
def test_wideband_synthetic_sweep(lcs, ctx, synthetic_sweep):
    s = synthetic_sweep
    k = (s["fc_in"] - s["f_true"]) / s["fc_in"]
    sw = lcs.Sweep(ctx, N_CAP)
    per_ch = sw.search_cu8_device(s["out"], s["fcs"], s["f_set"], max_cells=16)
    sw.close()
    found = [c for cs in per_ch for c in cs]
    fcc = [s["fc_in"] + off for off, _, _ in SWEEP_CARRIERS]
    for c in found:
        assert min(abs(c.fc_requested + c.freq_superfine - f) for f in fcc) < 1e6
    final = lcs.dedup(found)
    assert sorted(c.n_id_cell() for c in final) == sorted(d["n_id_cell"] for _, d, _ in SWEEP_CARRIERS)
    ids = cells_by_id(final)
    for off, d, _ in SWEEP_CARRIERS:
        c = ids[d["n_id_cell"]]
        fc_c = s["fc_in"] + off
        assert mib(c) == (d["n_id_cell"], d["n_ports"], d["cp_type"], d["n_rb_dl"], d["phich_duration"], d["phich_resource"],
                          d["sfn0"])
        assert abs(c.fc_requested + c.freq_superfine - (fc_c + fc_c * (1 - k))) < 100


@pytest.mark.gpu
def test_device_sweep_equals_host_sweep(lcs, ctx, synthetic_sweep):
    s = synthetic_sweep
    sel = slice(0, 64)             # one correlator chunk holds the weak and the strong carrier
    fcs = s["fcs"][sel]
    dev = s["out"][sel].contiguous()
    host = dev.cpu().numpy()
    sw = lcs.Sweep(ctx, N_CAP)
    a = sw.search_cu8_device(dev, fcs, s["f_set"], max_cells=16)
    b = sw.search_cu8(host, fcs, s["f_set"], max_cells=16)
    sw.close()
    assert sum(len(x) for x in a) >= 2
    for x, y in zip(a, b, strict=True):
        same_cells(x, y)


@pytest.mark.gpu
def test_cli_wideband_search(lcs, ctx, tmp_path):
    """`CellSearch_b200 --wideband`: every raster point of a 7.68 Msps recording channelized and searched; the cell table
    holds the planted cell once, at its raster channel."""
    import re
    import subprocess
    host = os.path.join(ROOT, "lte-cell-scanner_b200", "host")
    subprocess.check_call(["make", "-C", host, "-s"])
    fs_in, fc_in, D = 7.68e6, 739e6, 4
    n = 153599 * D + lcs.chan_design_taps(fs_in).size // 2 + 1
    d = dict(n_id_cell=211, n_ports=2, cp_type=1, n_rb_dl=75, phich_duration=1, phich_resource=3, t0=3000.0, sfn0=12)
    S.synth_wide_ci16(n, fs_in, fc_in, [(fc_in + 1.5e6, [d], 1.0)], f_true=2000.0, snr_db=10,
                      seed=41).tofile(str(tmp_path / "wide.ci16"))
    out = subprocess.run([os.path.join(host, "CellSearch_b200"), "--wideband", str(tmp_path / "wide.ci16"), "--fs-in", "7.68e6",
                          "--fc-in", "739e6", "-s", "736.2e6", "-e", "741.8e6", "-p", "15"], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "Channelizing and examining 57 center frequencies" in out.stdout
    rows = re.findall(r"^\s*(\d+)\s+(\d)\s+([0-9.]+)M", out.stdout, re.M)
    assert rows == [("211", "2", "740.5")]


@pytest.mark.gpu
def test_tracker_fed_by_channelizer(lcs, ctx):
    from test_tracker_gpu import run_pair
    from test_tracker_oracle import lcs_cell
    fs_in, fc_in, f_true, D = 7.68e6, 739e6, 3000.0, 4
    k = (fc_in - f_true) / fc_in
    a = dict(n_id_cell=277, n_ports=1, cp_type=1, n_rb_dl=25, phich_duration=1, phich_resource=3, t0=1234.0, sfn0=100)
    b = dict(n_id_cell=100, n_ports=2, cp_type=1, n_rb_dl=50, phich_duration=1, phich_resource=2, t0=15000.0, sfn0=40)
    fcs = np.array([fc_in + 1.5e6, fc_in - 2.0e6])
    n = int(0.6 * fs_in)
    iq = S.synth_wide_ci16(n, fs_in, fc_in, [(fcs[0], [a], 1.0), (fcs[1], [b], 1.0)], f_true=f_true, snr_db=10, seed=31)
    ch = lcs.Channelizer(ctx, fs_in, fc_in, fcs)
    ch.auto_gain(iq[:int(0.08 * fs_in)])
    parts = []
    for i in range(0, n, 123457):            # pushed in chunks
        parts.append(ch.push_ci16(iq[i:i + 123457])[0])
    ch.close()
    cu8s = np.ascontiguousarray(np.concatenate(parts, axis=1))
    assert cu8s.shape[1] == n_outputs(n, D, (lcs.chan_design_taps(fs_in).size - 1) // 2)
    fo0 = fcs * (1 - k) - 300
    cells = [[(lcs_cell(a), a["t0"] - 2 + 0.6)], [(lcs_cell(b), b["t0"] - 2 + 0.6)]]
    res, _ = run_pair(lcs, ctx, cu8s, cells, fo0, 96000, fc=fcs)
    for (r,) in res:
        assert r["mib_successes"] == r["mib_attempts"] > 0
