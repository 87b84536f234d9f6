"""The Welch spectrum on the device (lcs_psd_*, Spectrum) against its float64 oracle in every format and at N from 64 to
65 536, push invariance, spectrogram reads, dynamic range, an independent torch.fft comparison, coexistence with the
channelizer, argument validation and the CLI's --spectrum end to end."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "track_oracle"))

import lte_dl_synth as S  # noqa: E402
from test_rchan_gpu import requantise  # noqa: E402
from test_rchan_host import random_iq, to_complex  # noqa: E402
from test_spectrum_host import WelchOracle, hann, n_segments, welch_oracle  # noqa: E402

FC_IN = 739e6


def check_psd(got, ref):
    """The FP32-FFT tolerance: |P_dev - P_ref| <= 1e-5 max P_ref + 1e-4 P_ref in every bin."""
    err = np.abs(got - ref) - (1e-5 * ref.max() + 1e-4 * ref)
    assert (err <= 0).all(), (int(np.argmax(err)), err.max())


def recording(rng, n, fmt, fs):
    """Uniform noise of the format plus two tones, one strong, one 40 dB below it."""
    x = to_complex(random_iq(rng, n, fmt), fmt)
    m = np.arange(n)
    x = x + 0.2 * np.exp(2j * np.pi * 0.1234 * m) + 0.002 * np.exp(-2j * np.pi * 0.31 * m)
    scale = {"ci16": 32768, "cs8": 128, "cu8": 128}.get(fmt)
    if fmt == "cf32":
        return np.stack([x.real, x.imag], axis=1).astype(np.float32)
    v = np.round(np.stack([x.real, x.imag], axis=1) * 0.5 * scale)
    if fmt == "ci16":
        return np.clip(v, -32768, 32767).astype(np.int16)
    if fmt == "cs8":
        return np.clip(v, -128, 127).astype(np.int8)
    return np.clip(v + 127, 0, 255).astype(np.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [64, 1024, 4096, 65536])
@pytest.mark.parametrize("fmt", ["ci16", "cs8", "cu8", "cf32"])
def test_spectrum_matches_oracle(lcs, ctx, N, fmt):
    rng = np.random.default_rng(N + 7 * len(fmt))
    fs = 30.72e6
    n = max(6 * N, 40000) + N // 3
    iq = recording(rng, n, fmt, fs)
    sp = lcs.Spectrum(ctx, fs, fmt, N, fc_in=FC_IN)
    sp.push(iq)
    f, P, S_dev = sp.read()
    ref, S_ref = welch_oracle(to_complex(iq, fmt), fs, N)
    assert S_dev == S_ref == n_segments(n, N)
    assert np.array_equal(f, FC_IN + (np.arange(N) - N // 2) * fs / N)
    check_psd(P, ref)
    sp.close()


@pytest.mark.gpu
@pytest.mark.parametrize("N,fmt", [(64, "cu8"), (4096, "ci16"), (65536, "cs8")])
def test_spectrum_push_invariance(lcs, ctx, N, fmt):
    """Pushes of 1 sample, below N/2, odd sizes and one spanning several launches give bitwise the single-push PSD."""
    rng = np.random.default_rng(N)
    fs = 15.36e6
    n = {64: 9 * 2 ** 20, 4096: 9 * 2 ** 20, 65536: 6 * 2 ** 20}[N]          # several launches in every case
    iq = recording(rng, n, fmt, fs)
    one = lcs.Spectrum(ctx, fs, fmt, N)
    one.push(iq)
    _, whole, S_whole = one.read()
    _, launches = one.timing_read()
    assert launches > (3 if N > 4096 else 2)                                 # the single push ran in several launches
    sizes = [1, 1, N // 2 - 1, 7, 1, N + 3, N // 3, n // 2, 12345]
    parts = lcs.Spectrum(ctx, fs, fmt, N)
    i = 0
    while i < n:
        for k in sizes:
            parts.push(iq[i:i + k])
            i += k
    _, P, S = parts.read()
    assert S == S_whole == n_segments(n, N)
    assert np.array_equal(P, whole)
    ref, _ = welch_oracle(to_complex(iq, fmt), fs, N)
    check_psd(whole, ref)
    one.close()
    parts.close()


@pytest.mark.gpu
def test_spectrogram_reads(lcs, ctx):
    """Reading after every push gives rows that equal the oracle over the same segments; a read before N samples has
    S = 0 and zeros."""
    N, fs = 1024, 7.68e6
    rng = np.random.default_rng(3)
    iq = recording(rng, 40 * N, "ci16", fs)
    x = to_complex(iq, "ci16")
    sp = lcs.Spectrum(ctx, fs, "ci16", N)
    o = WelchOracle(fs, N)
    launches = ctx.launches
    sp.push(iq[:N - 1])
    o.push(x[:N - 1])
    _, P, S = sp.read()
    assert S == 0 and not P.any() and ctx.launches == launches
    o.read()
    i = N - 1
    for k in (1, 5 * N, 3 * N + 17, N // 2, 7 * N, 40 * N):
        sp.push(iq[i:i + k])
        o.push(x[i:i + k])
        i += k
        _, P, S = sp.read()
        ref, S_ref = o.read()
        assert S == S_ref
        if S:
            check_psd(P, ref)
        else:
            assert not P.any()


@pytest.mark.gpu
def test_spectrum_dynamic_range(lcs, ctx):
    """A near-full-scale LTE-like carrier and a tone 90 dB below it, far from the carrier, in ci16 at N = 65 536: the tone's
    peak bin is within 0.1 dB of the oracle, so the FP32 FFT's error floor lies below what 16-bit input resolves."""
    N, fs = 65536, 30.72e6
    n = 5 * N
    d = dict(n_id_cell=101, n_ports=2, cp_type=1, n_rb_dl=25, phich_duration=1, phich_resource=3, t0=500.0, sfn0=10)
    iq16 = S.synth_wide_ci16(n, fs, FC_IN, [(FC_IN - 6e6, [d], 1.0)], snr_db=200, seed=5, scale=8192.0)
    x = iq16.astype(np.float64)
    x = np.fft.fft(x[:, 0] + 1j * x[:, 1])
    x[np.abs(np.fft.fftfreq(n, 1 / fs) + 6e6) > 2.5e6] = 0              # band-limited: no OFDM sidelobes near the tone
    x = np.fft.ifft(x)
    x *= 24000 / np.abs(x).max()                                         # near full scale
    p_carrier = np.mean(np.abs(x) ** 2)
    f_tone = 9e6 + 0.37 * fs / N                                         # off the bin grid, 15 MHz from the carrier
    x = x + np.sqrt(p_carrier * 1e-9) * np.exp(2j * np.pi * f_tone / fs * np.arange(n))
    iq = np.clip(np.round(np.stack([x.real, x.imag], axis=1)), -32768, 32767).astype(np.int16)
    sp = lcs.Spectrum(ctx, fs, "ci16", N, fc_in=FC_IN)
    sp.push(iq)
    f, P, _ = sp.read()
    ref, _ = welch_oracle(to_complex(iq, "ci16"), fs, N)
    near = np.abs(f - (FC_IN + f_tone)) < 3 * fs / N
    k = np.flatnonzero(near)[np.argmax(ref[near])]
    floor = np.median(ref[np.abs(f - (FC_IN + f_tone)) < 200e3])
    assert ref[k] > 10 * floor                                           # the tone stands out of its surroundings
    assert abs(10 * np.log10(P[k] / ref[k])) < 0.1
    check_psd(P, ref)
    sp.close()


@pytest.mark.gpu
def test_spectrum_agrees_with_torch_fft(lcs, ctx):
    """An independent comparator: torch.fft in float64 over the same windowed segments."""
    import torch
    N, fs = 8192, 20e6
    rng = np.random.default_rng(9)
    iq = recording(rng, 20 * N, "cs8", fs)
    x = torch.from_numpy(to_complex(iq, "cs8"))
    w = torch.from_numpy(hann(N))
    segs = x.unfold(0, N, N // 2) * w
    P = torch.fft.fftshift((torch.fft.fft(segs, dim=1).abs() ** 2).mean(0) / (fs * (w ** 2).sum())).numpy()
    sp = lcs.Spectrum(ctx, fs, "cs8", N)
    sp.push(iq)
    _, got, S = sp.read()
    assert S == segs.shape[0]
    check_psd(got, P)
    sp.close()


@pytest.mark.gpu
def test_spectrum_and_channelizer_coexist(lcs, ctx):
    """A Spectrum and a RationalChannelizer fed the same stream alternately: the channelizer's bytes equal those of a
    channelizer used alone, and the PSD that of a Spectrum used alone."""
    fs = 20e6
    rng = np.random.default_rng(12)
    iq = requantise(recording(rng, 1_600_000, "ci16", fs), "cs8")
    fcs = FC_IN + np.array([-3e6, 0.0, 2.5e6])
    alone = lcs.RationalChannelizer(ctx, fs, FC_IN, fcs, fmt="cs8", gain=[2.0] * 3)
    ref_bytes, ref_clip = alone.push(iq)
    sp_alone = lcs.Spectrum(ctx, fs, "cs8", 16384)
    sp_alone.push(iq)
    _, ref_psd, _ = sp_alone.read()
    ch = lcs.RationalChannelizer(ctx, fs, FC_IN, fcs, fmt="cs8", gain=[2.0] * 3)
    sp = lcs.Spectrum(ctx, fs, "cs8", 16384)
    outs, clips = [], 0
    for i in range(0, iq.shape[0], 300_001):
        o, c = ch.push(iq[i:i + 300_001])
        sp.push(iq[i:i + 300_001])
        outs.append(o)
        clips = clips + c
    assert np.array_equal(np.concatenate(outs, axis=1), ref_bytes)
    assert np.array_equal(clips, ref_clip)
    _, psd, _ = sp.read()
    assert np.array_equal(psd, ref_psd)
    for h in (alone, sp_alone, ch, sp):
        h.close()


@pytest.mark.gpu
def test_spectrum_bad_arguments(lcs, ctx):
    import ctypes as C
    L = lcs
    lib = L.psd_lib()
    launches = ctx.launches
    h = C.c_void_p()
    for fs, fmt, nfft in ((0.0, L.IQ_CI16, 1024), (-1e6, L.IQ_CI16, 1024), (250e6 + 1, L.IQ_CI16, 1024),
                          (10e6 + 0.5, L.IQ_CI16, 1024), (float("nan"), L.IQ_CI16, 1024), (float("inf"), L.IQ_CI16, 1024),
                          (10e6, L.IQ_C128, 1024), (10e6, 5, 1024), (10e6, -1, 1024),
                          (10e6, L.IQ_CS8, 0), (10e6, L.IQ_CS8, 32), (10e6, L.IQ_CS8, 100), (10e6, L.IQ_CS8, 131072),
                          (10e6, L.IQ_CS8, 3 * 2 ** 14), (10e6, L.IQ_CS8, 2 ** 31)):
        assert lib.lcs_psd_create(ctx._h, fs, fmt, nfft, C.byref(h)) == 1, (fs, fmt, nfft)
    assert lib.lcs_psd_create(None, 10e6, L.IQ_CS8, 1024, C.byref(h)) == 1
    assert lib.lcs_psd_create(ctx._h, 10e6, L.IQ_CS8, 1024, None) == 1
    ok = L.Spectrum(ctx, 250e6, "cs8", 64)                                   # the limits are valid
    ok.close()
    ok = L.Spectrum(ctx, 1.0, "cf32", 65536)
    ok.close()
    sp = L.Spectrum(ctx, 10e6, "cs8", 1024)
    with pytest.raises(ValueError):
        sp.push(np.zeros((4000, 2), np.int16))                               # the wrong dtype
    assert lib.lcs_psd_push(sp._h, None, 5) == 1
    assert lib.lcs_psd_push(sp._h, None, 0) == 0
    out = np.zeros(1024)
    n = C.c_uint64(0)
    assert lib.lcs_psd_read(sp._h, None, C.byref(n)) == 1
    assert lib.lcs_psd_read(sp._h, out.ctypes.data, None) == 1
    ms = C.c_double(0)
    assert lib.lcs_psd_timing_read(sp._h, None, C.byref(n)) == 1
    assert lib.lcs_psd_push(None, out.ctypes.data, 5) == 1
    with pytest.raises(ValueError):
        L.Spectrum(ctx, 10e6, "c128", 1024)
    assert ctx.launches == launches
    assert lib.lcs_psd_timing_read(sp._h, C.byref(ms), C.byref(n)) == 0 and n.value == 0
    sp.close()


# ---- CLI end to end ---------------------------------------------------------------------------------------------------------
CLI_CARRIERS = [   # (offset from fc_in, cell, relative power); each signal (72 subcarriers) lies in no other's n_rb_dl * 180 kHz
    (-5.5e6, dict(n_id_cell=101, n_ports=1, cp_type=1, n_rb_dl=25, phich_duration=1, phich_resource=3, t0=500.0, sfn0=10), 1.0),
    (0.0, dict(n_id_cell=277, n_ports=2, cp_type=1, n_rb_dl=50, phich_duration=2, phich_resource=1, t0=7000.0, sfn0=500), 0.3),
    (5.5e6, dict(n_id_cell=350, n_ports=2, cp_type=2, n_rb_dl=15, phich_duration=1, phich_resource=4, t0=12000.0, sfn0=1000), 3.0),
]


@pytest.mark.gpu
def test_cli_spectrum_end_to_end(lcs, ctx, tmp_path):
    """`CellSearch_b200 --wideband ... --spectrum` on a 15.36 Msps recording with three planted carriers: the CSV equals
    lcs_psd_read on the file, each cell's carrier power is within 0.5 dB of what the generator put into its n_rb_dl * 180
    kHz, and the cell columns equal those of the same command without --spectrum."""
    host = os.path.join(ROOT, "lte-cell-scanner_b200", "host")
    subprocess.check_call(["make", "-C", host, "-s"])
    fs_in = 15.36e6
    h = lcs.chan_design_taps(fs_in)
    n = 153599 * 8 + (h.size - 1) // 2 + 1 + 50_000                  # the search's prefix and 50 000 samples more
    parts, p_gen = [], []
    for i, (off, d, rel) in enumerate(CLI_CARRIERS):                  # each carrier alone, noise-free
        c = S.synth_wide_ci16(n, fs_in, FC_IN, [(FC_IN + off, [d], rel)], snr_db=300, seed=60 + i, scale=8192.0)
        c = c.astype(np.float64)
        parts.append(c)
        p_gen.append(10 * np.log10(np.mean(c[:, 0] ** 2 + c[:, 1] ** 2) / 32768.0 ** 2))
    rng = np.random.default_rng(66)
    x = sum(parts)
    sigma2 = 1e-2 * 10 ** (min(p_gen) / 10) * 32768.0 ** 2           # the whole band's noise 20 dB below the weakest carrier
    x = x + rng.standard_normal(x.shape) * np.sqrt(sigma2 / 2)
    iq = np.clip(np.round(x), -32768, 32767).astype(np.int16)
    rec = str(tmp_path / "wide.ci16")
    iq.tofile(rec)
    csv = str(tmp_path / "psd.csv")
    exe = os.path.join(host, "CellSearch_b200")
    search = ["--wideband", rec, "--fs-in", "15.36e6", "--fc-in", "739e6", "-s", "733.5e6", "-e", "744.5e6", "-p", "15"]
    with_spec = subprocess.run([exe] + search + ["--spectrum", csv], capture_output=True, text=True, timeout=600)
    assert with_spec.returncode == 0, with_spec.stderr + with_spec.stdout
    without = subprocess.run([exe] + search, capture_output=True, text=True, timeout=600)
    assert without.returncode == 0, without.stderr + without.stdout
    # the CSV is lcs_psd_read over the whole file
    sp = lcs.Spectrum(ctx, fs_in, "ci16", 4096, fc_in=FC_IN)
    sp.push(iq)
    f, P, S_dev = sp.read()
    sp.close()
    assert S_dev == n_segments(n, 4096)
    lines = open(csv).read().splitlines()
    assert lines[0] == "freq_hz,psd_dbfs_per_hz" and len(lines) == 4097
    tab = np.array([[float(v) for v in l.split(",")] for l in lines[1:]])
    assert np.array_equal(tab[:, 0], f)
    assert np.abs(tab[:, 1] - 10 * np.log10(P)).max() < 1e-9
    # cell table: the same cells and columns, plus the carrier power
    row = re.compile(r"^\s*(\d+)\s+(\d)\s+([0-9.]+)M\s.*$", re.M)
    rows_with = row.findall(with_spec.stdout)
    rows_without = [m.group(0) for m in row.finditer(without.stdout)]
    assert sorted(int(r[0]) for r in rows_with) == sorted(d["n_id_cell"] for _, d, _ in CLI_CARRIERS)
    assert "CrystalCorrectionFactor CarrierPower[dBFS]" in with_spec.stdout
    full_with = [m.group(0) for m in row.finditer(with_spec.stdout)]
    assert len(full_with) == len(rows_without) == 3
    for a, b in zip(full_with, rows_without):
        head, pwr = a.rsplit(" ", 1)
        assert head == b
        cid = int(a.split()[0])
        i = [d["n_id_cell"] for _, d, _ in CLI_CARRIERS].index(cid)
        assert abs(float(pwr) - p_gen[i]) < 0.5, (cid, pwr, p_gen[i])
    assert "CarrierPower" not in without.stdout
    # --spectrum alone: no search, the same CSV
    csv2 = str(tmp_path / "psd2.csv")
    alone = subprocess.run([exe, "--wideband", rec, "--fs-in", "15.36e6", "--fc-in", "739e6", "--spectrum", csv2],
                           capture_output=True, text=True, timeout=600)
    assert alone.returncode == 0, alone.stderr
    assert "Detected" not in alone.stdout and "No LTE cells" not in alone.stdout
    assert open(csv2).read() == open(csv).read()
