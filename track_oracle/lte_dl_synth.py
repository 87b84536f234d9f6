"""Synthetic LTE downlink (6 centre RBs) as raw rtl-sdr bytes.  TEST INFRASTRUCTURE ONLY.

Built on numpy and the searcher oracle's tables (oracle/lcs_oracle.py): PSS, SSS, CRS for 1 or 2 ports, PBCH carrying
a chosen MIB (SFN advancing every frame, each frame carrying its quarter of the rate-matched bits), random QPSK on the
other resource elements, normal or extended CP.

Oscillator model (the reference's crystal model): one oscillator error moves both the carrier and the sample clock.
Sample n is taken at t_n = n / (fs_programmed * k), k = (fc - f_true) / fc_programmed, and every OFDM symbol's 72
subcarriers are evaluated directly at those instants (no resampling error); the carrier rotation for f_true is
applied, then AWGN at a stated per-resource-element SNR, then 8-bit quantisation as capbuf.cpp:172-175 reads it back.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle"))
import lcs_oracle as O  # noqa: E402

FS_LTE16 = 1.92e6
FRAME = 19200
AMP = 0.35                     # resource-element amplitude before the channel (keeps the 8-bit range unclipped)
_PERM = [1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23, 15, 31, 0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22,
         14, 30]
_BW = {6: 0, 15: 1, 25: 2, 50: 3, 75: 4, 100: 5}


def ratematch_positions(n_e, n_c=40):
    """Position in the 3 x n_c coded block of every rate-matched bit (36.212 5.1.4.2), the inverse of deratematch."""
    R = -(-n_c // 32)
    nd = 32 * R - n_c
    w = []
    for s in range(3):
        for col in range(32):
            for r in range(R):
                y = r * 32 + _PERM[col]
                w.append(-1 if y < nd else s * n_c + (y - nd))
    w = [v for v in w if v >= 0]
    return np.array([w[k % len(w)] for k in range(n_e)])


def mib_bits(n_rb_dl, phich_duration, phich_resource, sfn):
    """24 MIB bits (36.331): bandwidth, PHICH duration / resource (lcs_cell encodings), 8 SFN MSBs, 10 spare."""
    b = [(_BW[n_rb_dl] >> i) & 1 for i in (2, 1, 0)]
    b += [1 if phich_duration == 2 else 0]
    r = phich_resource - 1
    b += [(r >> 1) & 1, r & 1]
    b += [((sfn >> 2) >> i) & 1 for i in range(7, -1, -1)]
    return np.array(b + [0] * 10, np.uint8)


def pbch_bits(cell, sfn):
    """The 4 frames' scrambled PBCH bits of the 40 ms period containing sfn ([n_e])."""
    cp = cell["cp_type"]
    n_e = 1920 if cp == 1 else 1728
    a = mib_bits(cell["n_rb_dl"], cell["phich_duration"], cell["phich_resource"], sfn)
    crc = O.crc16(a).astype(np.uint8)
    if cell["n_ports"] == 2:
        crc ^= 1
    elif cell["n_ports"] == 4:
        crc[1::2] ^= 1
    d = O.conv_encode(np.concatenate([a, crc])).reshape(-1)      # [3][40] row-major
    e = d[ratematch_positions(n_e)]
    return e ^ O.lte_pn(cell["n_id_cell"], n_e).astype(np.uint8)


def _grid(cell, n_frames, sfn0, rng):
    """Transmitted resource grid per port: [n_ports][n_frames*20*n_symb][72] complex."""
    cp, P, nid = cell["cp_type"], cell["n_ports"], cell["n_id_cell"]
    n_symb = 7 if cp == 1 else 6
    n_sym = n_frames * 20 * n_symb
    qpsk = ((1 - 2 * rng.integers(0, 2, (n_sym, 72))) + 1j * (1 - 2 * rng.integers(0, 2, (n_sym, 72)))) / np.sqrt(2)
    X = np.zeros((P, n_sym, 72), complex)
    X[0] = qpsk
    used = np.zeros((n_sym, 72), bool)
    rs, shift = O.rs_dl(nid, cp)
    n_id_1, n_id_2 = nid // 3, nid % 3
    pss = O.pss_fd(n_id_2)
    sss = [O.sss_fd(n_id_1, n_id_2, 0), O.sss_fd(n_id_1, n_id_2, 10)]
    v3 = nid % 3
    for f in range(n_frames):
        sfn = (sfn0 + f) % 1024
        e = pbch_bits(cell, sfn - sfn % 4)
        q = e.size // 8                                   # QPSK symbols per frame
        bits = e[(sfn % 4) * 2 * q:(sfn % 4 + 1) * 2 * q]
        pb = ((1 - 2 * bits[0::2].astype(float)) + 1j * (1 - 2 * bits[1::2].astype(float))) / np.sqrt(2)
        for slot in range(20):
            for sym in range(n_symb):
                g = (f * 20 + slot) * n_symb + sym
                if slot in (0, 10) and sym >= n_symb - 2:   # SSS, PSS
                    X[:, g] = 0
                    X[0, g, 5:67] = sss[slot // 10] if sym == n_symb - 2 else pss
                    used[g] = True
                if slot == 1 and sym < 4:                   # PBCH (REs of 4-port CRS positions left empty)
                    has = sym in (0, 1) or (sym == 3 and cp == 2)
                    sc = np.array([s for s in range(72) if not (has and s % 3 == v3)])
                    k0 = sum(48 if (s in (0, 1) or (s == 3 and cp == 2)) else 72 for s in range(sym))
                    y = pb[k0:k0 + sc.size]
                    X[:, g] = 0
                    if P == 1:
                        X[0, g, sc] = y
                    else:                                   # Alamouti over RE pairs
                        s0, s1 = y[0::2], y[1::2]
                        X[0, g, sc[0::2]], X[0, g, sc[1::2]] = s0 / np.sqrt(2), s1 / np.sqrt(2)
                        X[1, g, sc[0::2]], X[1, g, sc[1::2]] = -np.conj(s1) / np.sqrt(2), np.conj(s0) / np.sqrt(2)
                    used[g, sc] = True
                for p in range(P):                          # CRS
                    sh = shift[slot * n_symb + sym, p]
                    if np.isnan(sh):
                        continue
                    idx = int(sh) + 6 * np.arange(12)
                    X[:, g, idx] = 0
                    X[p, g, idx] = rs[slot * n_symb + sym]
                    for p2 in range(P):                     # the other ports' CRS positions stay empty
                        if p2 != p:
                            X[p2, g, idx] = 0
                    used[g, idx] = True
    return X, n_symb


def synth_cu8(n_samples, cells, f_true=0.0, fc=739e6, fc_programmed=None, fs_programmed=1.92e6, snr_db=10.0,
              seed=0, stop_at=None):
    """cu8 [n][2].  cells: list of dicts with n_id_cell, n_ports (1/2), cp_type (1/2), n_rb_dl, phich_duration,
    phich_resource, t0 (frame start in LTE samples), sfn0, gains (per-port complex channel gains).
    snr_db: per resource element, relative to AMP^2.  stop_at: the cells stop transmitting at that sample."""
    rng = np.random.default_rng(seed)
    fcp = fc if fc_programmed is None else fc_programmed
    k = (fc - f_true) / fcp
    n = np.arange(n_samples)
    t = n / (fs_programmed * k)                            # sampling instants (seconds)
    u = t * FS_LTE16                                       # in LTE samples
    x = np.zeros(n_samples, complex)
    for cell in cells:
        cp = cell["cp_type"]
        rel = u - cell.get("t0", 0.0)
        n_frames = int(np.ceil((rel.max() + 1) / FRAME)) + 1
        X, n_symb = _grid(cell, n_frames, cell.get("sfn0", 0), rng)
        gains = cell.get("gains", [1.0, 0.8 * np.exp(0.7j)])[:cell["n_ports"]]
        Xc = AMP * np.tensordot(np.asarray(gains), X, axes=1)
        fr = np.floor(rel / FRAME)
        p = rel - fr * FRAME
        slot = np.floor(p / 960)
        q = p - slot * 960
        if cp == 1:
            sym = np.where(q < 138, 0, 1 + np.floor((q - 138) / 137))
            start = np.where(sym == 0, 0, 138 + (sym - 1) * 137)
            d = q - start - np.where(sym == 0, 10, 9)
        else:
            sym = np.floor(q / 160)
            d = q - sym * 160 - 32
        g = ((fr + 1) * 20 + slot) * n_symb + sym          # frame index shifted by one: samples before t0
        g = g.astype(np.int64) - 20 * n_symb
        ok = (g >= 0) & (g < X.shape[1])
        cn = np.concatenate([np.arange(-36, 0), np.arange(1, 37)])
        for c0 in range(0, n_samples, 65536):
            sl = slice(c0, min(c0 + 65536, n_samples))
            gg = np.where(ok[sl], g[sl], 0)
            ph = np.exp(2j * np.pi * np.outer(d[sl], cn) / 128)
            v = np.sum(Xc[gg] * ph, axis=1) / np.sqrt(128)
            x[sl] += np.where(ok[sl], v, 0)
    if stop_at is not None:
        x[stop_at:] = 0
    x *= np.exp(2j * np.pi * f_true * t)
    sigma2 = AMP ** 2 / 10 ** (snr_db / 10)
    x += np.sqrt(sigma2 / 2) * (rng.standard_normal(n_samples) + 1j * rng.standard_normal(n_samples))
    iq = np.stack([x.real, x.imag], axis=1)
    return np.clip(np.round(iq * 128 + 127), 0, 255).astype(np.uint8)


def to_c128(cu8):
    return ((cu8.astype(np.float64) - 127) / 128).view(np.complex128).reshape(-1)
