"""Synthetic LTE downlink (6 centre RBs) as raw rtl-sdr bytes.  TEST INFRASTRUCTURE ONLY.

Built on numpy and the searcher oracle's tables (oracle/lcs_oracle.py): PSS, SSS, CRS for 1, 2 or 4 ports, PBCH carrying
a chosen MIB (SFN advancing every frame, each frame carrying its quarter of the rate-matched bits; transmit diversity by
Alamouti for 2 ports and SFBC-FSTD for 4), random QPSK on the other resource elements, normal or extended CP.

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
                    elif P == 4:                            # SFBC-FSTD over RE quadruples (36.211 6.3.4.3)
                        q0, q1, q2, q3 = y[0::4], y[1::4], y[2::4], y[3::4]
                        X[0, g, sc[0::4]], X[0, g, sc[1::4]] = q0 / np.sqrt(2), q1 / np.sqrt(2)
                        X[2, g, sc[0::4]], X[2, g, sc[1::4]] = -np.conj(q1) / np.sqrt(2), np.conj(q0) / np.sqrt(2)
                        X[1, g, sc[2::4]], X[1, g, sc[3::4]] = q2 / np.sqrt(2), q3 / np.sqrt(2)
                        X[3, g, sc[2::4]], X[3, g, sc[3::4]] = -np.conj(q3) / np.sqrt(2), np.conj(q2) / np.sqrt(2)
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
    """cu8 [n][2].  cells: list of dicts with n_id_cell, n_ports (1/2/4), cp_type (1/2), n_rb_dl, phich_duration,
    phich_resource, t0 (frame start in LTE samples), sfn0, gains (per-port complex channel gains).
    snr_db: per resource element, relative to AMP^2.  stop_at: the cells stop transmitting at that sample."""
    rng = np.random.default_rng(seed)
    fcp = fc if fc_programmed is None else fc_programmed
    k = (fc - f_true) / fcp
    n = np.arange(n_samples)
    t = n / (fs_programmed * k)                            # sampling instants (seconds)
    x = _cells_baseband(t, cells, rng)
    if stop_at is not None:
        x[stop_at:] = 0
    x *= np.exp(2j * np.pi * f_true * t)
    sigma2 = AMP ** 2 / 10 ** (snr_db / 10)
    x += np.sqrt(sigma2 / 2) * (rng.standard_normal(n_samples) + 1j * rng.standard_normal(n_samples))
    iq = np.stack([x.real, x.imag], axis=1)
    return np.clip(np.round(iq * 128 + 127), 0, 255).astype(np.uint8)


def synth_wide_ci16(n, fs_in, fc_in, carriers, f_true=0.0, snr_db=10.0, seed=0, scale=4096.0):
    """A wideband recording as interleaved int16 I/Q [n][2]: several LTE carriers seen through one receiver whose LO
    and sample clock share one crystal.  carriers: list of (fc_c, cells, relative power), cells as in synth_cu8.

    One oscillator ratio k = (fc_in - f_true) / fc_in: sample m is taken at t_m = m / (fs_in * k) and every OFDM symbol is
    evaluated directly at those instants; carrier c sits at baseband fc_c - k * fc_in, so a channelizer channel at fc_c
    (whose mixer runs in nominal samples) sees exactly the offset fc_c * (1 - k) a dongle tuned to fc_c would see.
    AWGN of variance D * AMP^2 / 10^(snr_db/10) over the whole band (D = fs_in / 1.92 MHz) gives every 1.92 MHz channel
    the per-resource-element SNR snr_db of synth_cu8 at relative power 1.  The sum is scaled by `scale` and rounded to
    int16 (clamped)."""
    rng = np.random.default_rng(seed)
    k = (fc_in - f_true) / fc_in
    t = np.arange(n) / (fs_in * k)
    x = np.zeros(n, complex)
    for fc_c, cells, rel in carriers:
        x += np.sqrt(rel) * _cells_baseband(t, cells, rng) * np.exp(2j * np.pi * (fc_c - k * fc_in) * t)
    sigma2 = (fs_in / FS_LTE16) * AMP ** 2 / 10 ** (snr_db / 10)
    x += np.sqrt(sigma2 / 2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    iq = np.stack([x.real, x.imag], axis=1)
    return np.clip(np.round(iq * scale), -32768, 32767).astype(np.int16)


def _cells_baseband(t, cells, rng):
    """Sum of the cells' received signals at the instants t (seconds): per-port channel gains, then the cell's
    multipath channel.  A cell's optional `paths` [(delay_s, complex_gain, doppler_hz), ...] sum copies of its signal
    evaluated at t - delay_s (exact for any delay, also inside the cyclic prefix), each times
    complex_gain * exp(j 2 pi doppler_hz t).  Without `paths` the cell is received as transmitted."""
    n_samples = t.size
    u = t * FS_LTE16                                       # in LTE samples
    x = np.zeros(n_samples, complex)
    for cell in cells:
        rel = u - cell.get("t0", 0.0)
        n_frames = int(np.ceil((rel.max() + 1) / FRAME)) + 1
        X, n_symb = _grid(cell, n_frames, cell.get("sfn0", 0), rng)
        gains = cell.get("gains", [1.0, 0.8 * np.exp(0.7j), 0.9 * np.exp(-1.1j), 0.7 * np.exp(2.2j)])[:cell["n_ports"]]
        Xc = AMP * np.tensordot(np.asarray(gains), X, axes=1)
        if "paths" not in cell:
            x += _eval_grid(Xc, n_symb, cell["cp_type"], rel)
            continue
        for delay, gain, doppler in cell["paths"]:
            x += gain * np.exp(2j * np.pi * doppler * t) * _eval_grid(Xc, n_symb, cell["cp_type"], rel - delay * FS_LTE16)
    return x


def _eval_grid(Xc, n_symb, cp, rel):
    """The OFDM signal of the grid Xc [n_sym][72] at rel (LTE samples after the cell's frame start); 0 outside it."""
    n_samples = rel.size
    x = np.zeros(n_samples, complex)
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
    ok = (g >= 0) & (g < Xc.shape[0])
    cn = np.concatenate([np.arange(-36, 0), np.arange(1, 37)])
    for c0 in range(0, n_samples, 65536):
        sl = slice(c0, min(c0 + 65536, n_samples))
        gg = np.where(ok[sl], g[sl], 0)
        ph = np.exp(2j * np.pi * np.outer(d[sl], cn) / 128)
        v = np.sum(Xc[gg] * ph, axis=1) / np.sqrt(128)
        x[sl] += np.where(ok[sl], v, 0)
    return x


def to_c128(cu8):
    return ((cu8.astype(np.float64) - 127) / 128).view(np.complex128).reshape(-1)


# ---- full-bandwidth carriers --------------------------------------------------------------------------------------------
def crs_full(n_id_cell, cp_type, n_rb_dl):
    """The CRS of all n_rb_dl RBs (36.211 6.10.1.1): [20 slots][n_symb][2 n_rb_dl], r(m') with m' = 110 - n_rb_dl + m;
    rows of symbols without CRS are 0.  The subcarrier of r[.., m] for port p is 6 m + shift (O.rs_dl's shift table)."""
    n_symb = 7 if cp_type == 1 else 6
    n_cp = 1 if cp_type == 1 else 0
    m = 110 - n_rb_dl + np.arange(2 * n_rb_dl)
    r = np.zeros((20, n_symb, 2 * n_rb_dl), complex)
    for slot in range(20):
        for sym in (0, 1, n_symb - 3):
            c = O.lte_pn((1 << 10) * (7 * (slot + 1) + sym + 1) * (2 * n_id_cell + 1) + 2 * n_id_cell + n_cp, 440)
            r[slot, sym] = ((1 - 2 * c[2 * m].astype(float)) + 1j * (1 - 2 * c[2 * m + 1].astype(float))) / np.sqrt(2)
    return r


def subcarriers(n_rb_dl):
    """Subcarrier number of each grid column c < 12 n_rb_dl: c - 6R below DC, c - 6R + 1 above (DC skipped)."""
    R = n_rb_dl
    return np.concatenate([np.arange(-6 * R, 0), np.arange(1, 6 * R + 1)])


def pcfich_res(n_id_cell, n_rb_dl):
    """The 16 columns of the PCFICH in symbol 0 (36.211 6.7.4): quadruplet i in the REG at 6 (n_id_cell mod 2R) +
    6 floor(i R / 2) (mod 12 R), on its 4 REs off the CRS of ports 0 and 1."""
    R = n_rb_dl
    cols = []
    for i in range(4):
        k0 = (6 * (n_id_cell % (2 * R)) + 6 * (i * R // 2)) % (12 * R)
        cols += [k0 + o for o in range(6) if o % 3 != n_id_cell % 3]
    return np.array(cols)


def pcfich_symbols(n_id_cell, n_ports, subframe, cfi):
    """The PCFICH of CFI cfi in subframe number `subframe` per port, [n_ports][16]: the codeword of 36.212 Table 5.3.4-1
    scrambled (36.211 6.7.1), QPSK-mapped and precoded for transmit diversity (6.3.4.3), as _grid's PBCH."""
    cw = (np.arange(32) % 3 != cfi - 1).astype(np.uint8)
    c = O.lte_pn((subframe + 1) * (2 * n_id_cell + 1) * 512 + n_id_cell, 32).astype(np.uint8)
    e = (cw ^ c).astype(float)
    d = ((1 - 2 * e[0::2]) + 1j * (1 - 2 * e[1::2])) / np.sqrt(2)
    y = np.zeros((n_ports, 16), complex)
    if n_ports == 1:
        y[0] = d
        return y
    for j in range(8):                                  # pair j: ports (0, 1), or (0, 2) / (1, 3) for four ports
        a, b = (0, 1) if n_ports == 2 else ((0, 2) if j % 2 == 0 else (1, 3))
        y[a, 2 * j], y[a, 2 * j + 1] = d[2 * j] / np.sqrt(2), d[2 * j + 1] / np.sqrt(2)
        y[b, 2 * j], y[b, 2 * j + 1] = -np.conj(d[2 * j + 1]) / np.sqrt(2), np.conj(d[2 * j]) / np.sqrt(2)
    return y


def _grid_full(cell, n_frames, rng):
    """Transmitted grid of all n_rb_dl RBs per port, [n_ports][n_sym][12 R]: the 6-RB content of _grid in the centre,
    full-band CRS, and QPSK times sqrt(cell["load"]) (default 1) on port 0 on every other RE outside the centre.  With
    cell["cfi"], a sequence of CFIs, subframe u (counted from the grid's first) carries the PCFICH of cfi[u mod len] in
    its symbol 0, written last; with cell["pdcch"] as well, its control region carries those DCIs (_write_control); with
    cell["sib1"] as well, its SIB1 occasions carry that SIB1 (_write_sib1)."""
    R, P, cp = cell["n_rb_dl"], cell["n_ports"], cell["cp_type"]
    X6, n_symb = _grid(cell, n_frames, cell.get("sfn0", 0), rng)
    n_sym = X6.shape[1]
    X = np.zeros((P, n_sym, 12 * R), complex)
    load = np.sqrt(cell.get("load", 1.0))
    X[0] = load * ((1 - 2 * rng.integers(0, 2, (n_sym, 12 * R))) + 1j * (1 - 2 * rng.integers(0, 2, (n_sym, 12 * R)))) / np.sqrt(2)
    rs = crs_full(cell["n_id_cell"], cp, R)
    _, shift = O.rs_dl(cell["n_id_cell"], cp)
    for g in range(n_sym):
        slot, sym = (g // n_symb) % 20, g % n_symb
        for p in range(P):
            sh = shift[slot * n_symb + sym, p]
            if np.isnan(sh):
                continue
            idx = int(sh) + 6 * np.arange(2 * R)
            X[:, g, idx] = 0
            X[p, g, idx] = rs[slot, sym]
    X[:, :, 6 * R - 36:6 * R + 36] = X6
    if "sib1" in cell:
        cell = dict(cell, pdcch=list(cell.get("pdcch", [])) + sib1_dcis(cell, n_sym // (2 * n_symb)))
    if "pdcch" in cell:
        _write_control(X, cell, n_symb)
    if "sib1" in cell:
        _write_sib1(X, cell, n_symb)
    if "cfi" in cell:
        cols, seq = pcfich_res(cell["n_id_cell"], R), list(cell["cfi"])
        for u in range(n_sym // (2 * n_symb)):
            X[:, 2 * n_symb * u, cols] = pcfich_symbols(cell["n_id_cell"], P, u % 10, seq[u % len(seq)])
    return X, n_symb


# ---- the control region: PHICH and PDCCH REGs (36.211 6.2.4, 6.8.5, 6.9.3) -------------------------------------------------
DCI_SIZES_1A = {6: 21, 15: 22, 25: 25, 50: 27, 75: 27, 100: 28}      # 36.212 5.3.3.1.3, FDD, with its padding bit
DCI_SIZES_1C = {6: 8, 15: 10, 25: 12, 50: 13, 75: 14, 100: 15}       # 36.212 5.3.3.1.4


def reg_is_six(l, n_ports, cp_type):
    """True when the REGs of control symbol l are 6 REs (2 of them CRS), else 4."""
    return l == 0 or (l == 1 and n_ports == 4) or (l == 3 and cp_type == 2)


def reg_data_cols(l, k0, n_id_cell, n_ports, cp_type):
    """The 4 data columns of the REG of symbol l starting at k0, in increasing k."""
    if reg_is_six(l, n_ports, cp_type):
        return [k0 + o for o in range(6) if (k0 + o) % 3 != n_id_cell % 3]
    return [k0 + o for o in range(4)]


def n_ctrl_of(cfi, R, phich_duration):
    """Symbols of the control region: CFI (+1 at R <= 10), at least 3 with extended PHICH duration."""
    n = cfi + (R <= 10)
    return max(n, 3) if phich_duration == 2 else n


def control_regs(R, n_ports, cp_type, n_id_cell, phich_duration, phich_resource, n_ctrl):
    """The REGs of a control region of n_ctrl symbols: dict with `pcfich` and `phich` (sets of (l, k0)), `pdcch` (the
    PDCCH REGs (l, k0) in the order m' of 6.8.5) and `quad_reg` (quadruplet j is on REG pdcch[quad_reg[j]])."""
    W = 12 * R
    pcf = {(0, (6 * (n_id_cell % (2 * R)) + 6 * (i * R // 2)) % W) for i in range(4)}
    avail = [[k0 for k0 in range(0, W, 6 if reg_is_six(l, n_ports, cp_type) else 4) if (l, k0) not in pcf] for l in range(4)]
    ng = {1: (1, 6), 2: (1, 2), 3: (1, 1), 4: (2, 1)}[phich_resource]
    m_u = -(-ng[0] * R // (8 * ng[1]))
    n0 = len(avail[0])
    phich = set()
    for m in range(m_u):
        for i in range(3):
            l = i if phich_duration == 2 else 0
            nl = len(avail[l])
            phich.add((l, avail[l][(n_id_cell * nl // n0 + m + i * nl // 3) % nl]))
    regs = [(l, k) for k in range(W) for l in range(n_ctrl)
            if k % (6 if reg_is_six(l, n_ports, cp_type) else 4) == 0 and (l, k) not in pcf and (l, k) not in phich]
    n = len(regs)
    rows = -(-n // 32)
    nd = 32 * rows - n
    w = [r * 32 + _PERM[c] - nd for c in range(32) for r in range(rows) if r * 32 + _PERM[c] >= nd]
    quad_reg = np.zeros(n, int)
    for m in range(n):
        quad_reg[w[(m + n_id_cell) % n]] = m
    return dict(pcfich=pcf, phich=phich, pdcch=regs, quad_reg=quad_reg, n_reg=n, n_cce=n // 9)


def dci_codeword(bits, rnti, L):
    """The 72 L rate-matched bits of a DCI (36.212 5.3.3.2-4): CRC16 masked with the RNTI, tail-biting code."""
    a = np.asarray(bits, np.uint8)
    crc = O.crc16(a).astype(np.uint8) ^ np.array([(rnti >> (15 - i)) & 1 for i in range(16)], np.uint8)
    c = np.concatenate([a, crc])
    d = O.conv_encode(c).reshape(-1)
    return d[ratematch_positions(72 * L, c.size)]


def _precode(d, n_ports):
    """Transmit diversity of a symbol sequence (6.3.4.3): [n_ports][len]; four ports: pair 2i on ports 0 and 2, 2i + 1
    on ports 1 and 3."""
    y = np.zeros((n_ports, d.size), complex)
    if n_ports == 1:
        y[0] = d
        return y
    for j in range(d.size // 2):
        a, b = (0, 1) if n_ports == 2 else ((0, 2) if j % 2 == 0 else (1, 3))
        y[a, 2 * j], y[a, 2 * j + 1] = d[2 * j] / np.sqrt(2), d[2 * j + 1] / np.sqrt(2)
        y[b, 2 * j], y[b, 2 * j + 1] = -np.conj(d[2 * j + 1]) / np.sqrt(2), np.conj(d[2 * j]) / np.sqrt(2)
    return y


def _write_control(X, cell, n_symb):
    """cell["pdcch"]: DCIs (sf, rnti, fmt, L, cce, bits), sf a grid subframe or (period, phase) for every subframe u with
    u mod period = phase.  Each subframe's control region (cell["cfi"]) is cleared but for its CRS; its PHICH REGs get a
    fixed PN QPSK sequence on port 0, its DCIs are encoded, placed at their CCEs, scrambled (6.8.2), precoded, permuted and
    mapped (6.8.5), and the rest of its PDCCH quadruplets are NIL (zero), or random QPSK from cell["pdcch_fill"] (a
    seed) when it is given."""
    if "cfi" not in cell:
        raise ValueError('a cell with "pdcch" needs "cfi": the control region is sized by it')
    R, P, cp, nid = cell["n_rb_dl"], cell["n_ports"], cell["cp_type"], cell["n_id_cell"]
    seq, dur, res = list(cell["cfi"]), cell["phich_duration"], cell["phich_resource"]
    fill = np.random.default_rng(cell["pdcch_fill"]) if "pdcch_fill" in cell else None
    _, shift = O.rs_dl(nid, cp)
    for u in range(X.shape[1] // (2 * n_symb)):
        n_ctrl = n_ctrl_of(seq[u % len(seq)], R, dur)
        t = control_regs(R, P, cp, nid, dur, res, n_ctrl)
        g0 = 2 * n_symb * u
        for l in range(n_ctrl):
            keep = np.zeros(12 * R, bool)
            for p in range(P):
                sh = shift[(2 * u % 20) * n_symb + l, p]
                if not np.isnan(sh):
                    keep[int(sh) + 6 * np.arange(2 * R)] = True
            X[:, g0 + l, ~keep] = 0
        ph = sorted(t["phich"])
        b = O.lte_pn(nid + 1, 8 * len(ph)).astype(float)
        for i, (l, k0) in enumerate(ph):
            X[0, g0 + l, reg_data_cols(l, k0, nid, P, cp)] = ((1 - 2 * b[8 * i:8 * i + 8:2]) + 1j * (1 - 2 * b[8 * i + 1:8 * i + 8:2])) / np.sqrt(2)
        n_bits = 8 * t["n_reg"]
        bits = np.zeros(n_bits, np.uint8)
        used = np.zeros(n_bits, bool)
        for sf, rnti, fmt, L, cce, payload in cell["pdcch"]:
            if (sf != u) if isinstance(sf, int) else (u % sf[0] != sf[1]):
                continue
            bits[72 * cce:72 * (cce + L)] = dci_codeword(payload, rnti, L)
            used[72 * cce:72 * (cce + L)] = True
        e = (bits ^ O.lte_pn((u % 10) * 512 + nid, n_bits)).astype(float)
        d = ((1 - 2 * e[0::2]) + 1j * (1 - 2 * e[1::2])) / np.sqrt(2)
        d[~used[0::2]] = 0
        if fill is not None:
            nil = ~used[0::2]
            d[nil] = ((1 - 2 * fill.integers(0, 2, nil.sum())) + 1j * (1 - 2 * fill.integers(0, 2, nil.sum()))) / np.sqrt(2)
        y = _precode(d, P)
        for j in range(t["n_reg"]):
            l, k0 = t["pdcch"][t["quad_reg"][j]]
            X[:, g0 + l, reg_data_cols(l, k0, nid, P, cp)] = y[:, 4 * j:4 * j + 4]


def channel_response(paths, f):
    """H(f) of the paths [(delay_s, complex_gain), ...] at the frequencies f (Hz)."""
    return sum(g * np.exp(-2j * np.pi * np.asarray(f) * d) for d, g in paths)


def synth_wide_full(n, fs_in, fc_in, carriers, snr_db=30.0, seed=0):
    """A wideband recording at the nominal clock as complex128 [n] in full-scale units: LTE carriers of all their RBs.

    carriers: list of (fc_c, cells); fc_c - fc_in an integer number of Hz, fs_in = D * 1.92 MHz.  Each cell as in
    synth_cu8 plus n_rb_dl RBs of content (_grid_full), an integer t0, optional `paths` [(delay_s, gain)] (each symbol's
    subcarriers times H(f); exact while the delays stay inside the cyclic prefix) and an optional `interferer`
    (rb_lo, rb_hi, power): complex Gaussian noise of power power * AMP^2 per RE on RBs [rb_lo, rb_hi) of the cell.
    Every OFDM symbol is built by one N = 128 D point inverse FFT and its cyclic prefix, which is exact at these rates.
    AWGN of variance D * AMP^2 / 10^(snr_db/10) over the band gives each RE the SNR snr_db.  Returns (x, grids):
    grids[i] is the received grid [n_sym][12 R] of the i-th cell (port gains, channel and interferer applied, AMP
    included, noise excluded), row 0 the frame starting at t0."""
    rng = np.random.default_rng(seed)
    D = int(round(fs_in / FS_LTE16))
    N, fs = 128 * D, int(round(fs_in))
    x = np.zeros(n, complex)
    grids = []
    for fc_c, cells in carriers:
        delta = int(round(fc_c - fc_in))
        xc = np.zeros(n, complex)
        for cell in cells:
            R, cp = cell["n_rb_dl"], cell["cp_type"]
            start = D * int(cell["t0"])
            n_frames = -(-(n - start) // (D * FRAME))
            X, n_symb = _grid_full(cell, n_frames, rng)
            gains = cell.get("gains", [1.0, 0.8 * np.exp(0.7j), 0.9 * np.exp(-1.1j), 0.7 * np.exp(2.2j)])[:cell["n_ports"]]
            Y = AMP * np.tensordot(np.asarray(gains), X, axes=1)
            k = subcarriers(R)
            if "paths" in cell:
                Y = Y * channel_response(cell["paths"], k * 15e3)[None, :]
            if "interferer" in cell:
                lo, hi, pw = cell["interferer"]
                cols = slice(12 * lo, 12 * hi)
                sh = (Y.shape[0], 12 * (hi - lo))
                Y[:, cols] += AMP * np.sqrt(pw / 2) * (rng.standard_normal(sh) + 1j * rng.standard_normal(sh))
            grids.append(Y)
            V = np.zeros((Y.shape[0], N), complex)
            V[:, k % N] = Y
            u = np.fft.ifft(V, axis=1) * (N / np.sqrt(128))
            pos = start
            for g in range(Y.shape[0]):
                sym = g % n_symb
                ncp = D * (32 if cp == 2 else (10 if sym == 0 else 9))
                seg = np.concatenate([u[g, N - ncp:], u[g]])
                m = min(seg.size, n - pos)
                if m <= 0:
                    break
                xc[pos:pos + m] += seg[:m]
                pos += seg.size
        p = (np.arange(n, dtype=np.int64) * (delta % fs)) % fs
        x += xc * np.exp(2j * np.pi * p / fs)
    sigma2 = D * AMP ** 2 / 10 ** (snr_db / 10)
    x += np.sqrt(sigma2 / 2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return x, grids


def quantise(x, fmt, scale):
    """x * scale (full-scale units) as [n][2] samples of fmt: ci16 (/32768), cs8 (/128), cu8 ((v - 127) / 128) or cf32."""
    v = np.stack([x.real, x.imag], axis=1) * scale
    if fmt == "ci16":
        return np.clip(np.rint(v * 32768), -32768, 32767).astype(np.int16)
    if fmt == "cs8":
        return np.clip(np.rint(v * 128), -128, 127).astype(np.int8)
    if fmt == "cu8":
        return np.clip(np.rint(v * 128 + 127), 0, 255).astype(np.uint8)
    return v.astype(np.float32)


def dequantise(iq, fmt):
    """The samples of quantise() as complex128 in full-scale units, as the device reads them."""
    v = iq.astype(np.float64)
    v = {"ci16": v / 32768, "cs8": v / 128, "cu8": (v - 127) / 128, "cf32": v}[fmt]
    return v[:, 0] + 1j * v[:, 1]


def _eval_grid_full(Xc, n_symb, cp, rel, n_rb_dl):
    """_eval_grid for a grid of all n_rb_dl RBs, Xc [n_sym][12 R]: the OFDM signal at rel (LTE samples after the cell's
    frame start, any real value), evaluated directly; 0 outside the grid."""
    x = np.zeros(rel.size, complex)
    fr = np.floor(rel / FRAME)
    p = rel - fr * FRAME
    slot = np.floor(p / 960)
    q = p - slot * 960
    if cp == 1:
        sym = np.where(q < 138, 0, 1 + np.floor((q - 138) / 137))
        d = q - np.where(sym == 0, 0, 138 + (sym - 1) * 137) - np.where(sym == 0, 10, 9)
    else:
        sym = np.floor(q / 160)
        d = q - sym * 160 - 32
    g = (((fr + 1) * 20 + slot) * n_symb + sym).astype(np.int64) - 20 * n_symb
    ok = (g >= 0) & (g < Xc.shape[0])
    cn = subcarriers(n_rb_dl)
    for c0 in range(0, rel.size, 8192):
        sl = slice(c0, min(c0 + 8192, rel.size))
        gg = np.where(ok[sl], g[sl], 0)
        v = np.einsum("ij,ij->i", Xc[gg], np.exp(2j * np.pi * np.outer(d[sl], cn) / 128)) / np.sqrt(128)
        x[sl] = np.where(ok[sl], v, 0)
    return x


def synth_wide_offset(n, fs_in, fc_in, fc_c, cell, clock_ratio, f_res, snr_db=30.0, seed=0):
    """One cell of all its RBs in a wideband recording whose sample clock is off, by direct evaluation (the slow path,
    for small cases).  Sample m is taken at t_m = m / (fs_in * clock_ratio); the carrier at fc_c (fc_c - fc_in an integer
    number of Hz) turns by the exact nominal mixer phase (m (fc_c - fc_in) mod fs_in) / fs_in and by f_res t_m, so that
    after the nominal mixer it sits f_res off with its clock clock_ratio times fast.  The search reports such a cell with
    freq_superfine = f_res, fc_programmed = (fc_c - f_res) / clock_ratio (so k_factor = clock_ratio) and frame_start =
    t0 * clock_ratio; t0 may be fractional.  AWGN as in synth_wide_full.  Returns (x complex128 [n], received grid)."""
    rng = np.random.default_rng(seed)
    D = int(round(fs_in / FS_LTE16))
    fs, delta = int(round(fs_in)), int(round(fc_c - fc_in))
    t = np.arange(n) / (fs_in * clock_ratio)
    rel = t * FS_LTE16 - cell["t0"]
    X, n_symb = _grid_full(cell, int(np.ceil((rel.max() + 1) / FRAME)) + 1, rng)
    gains = cell.get("gains", [1.0, 0.8 * np.exp(0.7j), 0.9 * np.exp(-1.1j), 0.7 * np.exp(2.2j)])[:cell["n_ports"]]
    Y = AMP * np.tensordot(np.asarray(gains), X, axes=1)
    p = (np.arange(n, dtype=np.int64) * (delta % fs)) % fs
    x = _eval_grid_full(Y, n_symb, cell["cp_type"], rel, cell["n_rb_dl"]) * np.exp(2j * np.pi * p / fs)
    x *= np.exp(2j * np.pi * f_res * t)
    sigma2 = D * AMP ** 2 / 10 ** (snr_db / 10)
    x += np.sqrt(sigma2 / 2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return x, Y


# ---- SIB1 on the PDSCH (36.211 6.2.3, 6.3, 36.212 5.1.1-5.1.4, 36.213 7.1.6-7.1.7, 36.331 5.2.1.2) --------------------------
_TURBO_PERM = [0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22, 14, 30, 1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23,
               15, 31]                                                          # 36.212 Table 5.1.4-1


def turbo_sizes():
    """The 188 code block sizes K of 36.212 Table 5.1.3-3."""
    return ([40 + 8 * i for i in range(60)] + [512 + 16 * i for i in range(1, 33)] + [1024 + 32 * i for i in range(1, 33)]
            + [2048 + 64 * i for i in range(1, 65)])


_QPP = [
    (3, 10), (7, 12), (19, 42), (7, 16), (7, 18), (11, 20), (5, 22), (11, 24), (7, 26), (41, 84), (103, 90),
    (15, 32), (9, 34), (17, 108), (9, 38), (21, 120), (101, 84), (21, 44), (57, 46), (23, 48), (13, 50), (27, 52),
    (11, 36), (27, 56), (85, 58), (29, 60), (33, 62), (15, 32), (17, 198), (33, 68), (103, 210), (19, 36),
    (19, 74), (37, 76), (19, 78), (21, 120), (21, 82), (115, 84), (193, 86), (21, 44), (133, 90), (81, 46),
    (45, 94), (23, 48), (243, 98), (151, 40), (155, 102), (25, 52), (51, 106), (47, 72), (91, 110), (29, 168),
    (29, 114), (247, 58), (29, 118), (89, 180), (91, 122), (157, 62), (55, 84), (31, 64), (17, 66), (35, 68),
    (227, 420), (65, 96), (19, 74), (37, 76), (41, 234), (39, 80), (185, 82), (43, 252), (21, 86), (155, 44),
    (79, 120), (139, 92), (23, 94), (217, 48), (25, 98), (17, 80), (127, 102), (25, 52), (239, 106), (17, 48),
    (137, 110), (215, 112), (29, 114), (15, 58), (147, 118), (29, 60), (59, 122), (65, 124), (55, 84), (31, 64),
    (17, 66), (171, 204), (67, 140), (35, 72), (19, 74), (39, 76), (19, 78), (199, 240), (21, 82), (211, 252),
    (21, 86), (43, 88), (149, 60), (45, 92), (49, 846), (71, 48), (13, 28), (17, 80), (25, 102), (183, 104),
    (55, 954), (127, 96), (27, 110), (29, 112), (29, 114), (57, 116), (45, 354), (31, 120), (59, 610), (185, 124),
    (113, 420), (31, 64), (17, 66), (171, 136), (209, 420), (253, 216), (367, 444), (265, 456), (181, 468),
    (39, 80), (27, 164), (127, 504), (143, 172), (43, 88), (29, 300), (45, 92), (157, 188), (47, 96), (13, 28),
    (111, 240), (443, 204), (51, 104), (51, 212), (451, 192), (257, 220), (57, 336), (313, 228), (271, 232),
    (179, 236), (331, 120), (363, 244), (375, 248), (127, 168), (31, 64), (33, 130), (43, 264), (33, 134),
    (477, 408), (35, 138), (233, 280), (357, 142), (337, 480), (37, 146), (71, 444), (71, 120), (37, 152),
    (39, 462), (127, 234), (39, 158), (39, 80), (31, 96), (113, 902), (41, 166), (251, 336), (43, 170), (21, 86),
    (43, 174), (45, 176), (45, 178), (161, 120), (89, 182), (323, 184), (47, 186), (23, 94), (47, 190), (263, 480)]  # 36.212 Table 5.1.3-3, (f1, f2) of each K


def qpp_table():
    """(f1, f2) of each K of turbo_sizes()."""
    return np.array(_QPP)


def crc24a(bits):
    """The 24 parity bits of 36.212 5.1.1 (g_CRC24A = 0x864CFB) of a bit sequence."""
    r = 0
    for b in bits:
        fb = ((r >> 23) & 1) ^ int(b)
        r = (r << 1) & 0xFFFFFF
        if fb:
            r ^= 0x864CFB
    return np.array([(r >> (23 - i)) & 1 for i in range(24)], np.uint8)


def _rsc(c):
    """One constituent encoder (36.212 5.1.3.2.1): parity of c, then the 3 termination steps' (x, z)."""
    s1 = s2 = s3 = 0
    z = np.zeros(c.size, np.uint8)
    for k, u in enumerate(c):
        a = int(u) ^ s2 ^ s3
        z[k] = a ^ s1 ^ s3
        s1, s2, s3 = a, s1, s2
    tail = []
    for _ in range(3):
        tail.append((s2 ^ s3, s1 ^ s3))
        s1, s2, s3 = 0, s1, s2
    return z, tail


def turbo_encode(c):
    """d [3][K + 4] of code block c (filler bits as 0), 36.212 5.1.3.2."""
    K = c.size
    f1, f2 = qpp_table()[turbo_sizes().index(K)]
    pi = (f1 * np.arange(K) + f2 * np.arange(K) ** 2) % K
    z1, t1 = _rsc(c)
    z2, t2 = _rsc(c[pi])
    d = np.zeros((3, K + 4), np.uint8)
    d[0, :K], d[1, :K], d[2, :K] = c, z1, z2
    (x0, zz0), (x1, zz1), (x2, zz2) = t1
    (y0, w0), (y1, w1), (y2, w2) = t2
    d[:, K:] = [[x0, zz1, y0, w1], [zz0, x2, w0, y2], [x1, zz2, y1, w2]]
    return d


def circular_buffer(K, F):
    """36.212 5.1.4.1.1-2: for each position of w, (stream, index) of d, or None for a NULL (dummy or filler)."""
    D = K + 4
    rows = -(-D // 32)
    kp, nd = 32 * rows, 32 * rows - D
    y = [None] * nd + list(range(D))
    v = [[], [], []]
    for k in range(kp):
        j = _TURBO_PERM[k // rows] + 32 * (k % rows)
        for s in (0, 1):
            v[s].append(None if y[j] is None or y[j] < F else (s, y[j]))
        j2 = (j + 1) % kp
        v[2].append(None if y[j2] is None else (2, y[j2]))
    # column-by-column read of each stream: v_s[k] for k = column-major index
    w = v[0] + [x for pair in zip(v[1], v[2]) for x in pair]
    return w


def k0_position(K, rv):
    rows = -(-(K + 4) // 32)
    return rows * (2 * -(-(96 * rows) // (8 * rows)) * rv + 2)


def rate_match(d, K, F, rv, E):
    """e [E] of d for redundancy version rv (N_cb = K_w), NULLs skipped."""
    w = circular_buffer(K, F)
    k0, out, j = k0_position(K, rv), [], 0
    while len(out) < E:
        x = w[(k0 + j) % len(w)]
        if x is not None:
            out.append(d[x[0], x[1]])
        j += 1
    return np.array(out, np.uint8)


TBS_1A = [(32, 56), (56, 88), (72, 144), (104, 176), (120, 208), (144, 224), (176, 256), (224, 328), (256, 392),
          (296, 456), (328, 504), (376, 584), (440, 680), (488, 744), (552, 840), (600, 904), (632, 968), (696, 1064),
          (776, 1160), (840, 1288), (904, 1384), (1000, 1480), (1064, 1608), (1128, 1736), (1192, 1800), (1256, 1864),
          (1480, 2216)]                                                       # 36.213 Table 7.1.7.2.1-1, N_PRB 2 and 3
TBS_1C = [40, 56, 72, 120, 136, 144, 176, 208, 224, 256, 280, 296, 328, 336, 392, 488, 552, 600, 632, 696, 776, 840, 904,
          1000, 1064, 1128, 1224, 1288, 1384, 1480, 1608, 1736]                # 36.213 Table 7.1.7.2.3-1
N_GAP = {6: (3, None), 15: (8, None), 25: (12, None), 50: (27, 9), 75: (32, 16), 100: (48, 16)}   # 36.211 Table 6.2.3.2-1
RBG = {6: 1, 15: 2, 25: 2, 50: 3, 75: 4, 100: 4}                                                  # 36.213 Table 7.1.6.1-1


def n_vrb(R, gap):
    g = N_GAP[R][gap]
    return (R // (2 * g)) * 2 * g if gap else 2 * min(g, R - g)


def vrb_to_prb(R, gap, n, slot):
    """36.211 6.2.3.2: the PRB of distributed VRB n in slot parity `slot`."""
    g, P = N_GAP[R][gap], RBG[R]
    nt = 2 * g if gap else n_vrb(R, 0)
    n_row = -(-nt // (4 * P)) * P
    n_null = 4 * n_row - nt
    v, blk = n % nt, nt * (n // nt)
    p1, p2 = 2 * n_row * (v % 2) + v // 2 + blk, n_row * (v % 4) + v // 4 + blk
    if n_null and v >= nt - n_null:
        p = p1 - n_row + (n_null // 2 if v % 2 == 0 else 0)
    elif n_null and v % 4 >= 2:
        p = p2 - n_null // 2
    else:
        p = p2
    if slot:
        p = (p + nt // 2) % nt + blk
    return p if p < nt // 2 else p + g - nt // 2


def riv_decode(N, riv):
    """(start, length) of a RIV on N RBs (36.213 7.1.6.3), None when it is not one."""
    for length in range(1, N + 1):
        for start in range(N - length + 1):
            r = N * (length - 1) + start if length - 1 <= N // 2 else N * (N - length + 1) + (N - 1 - start)
            if r == riv:
                return start, length
    return None


def sib1_allocation(R, s):
    """(tbs, [PRBs of slot 0, of slot 1]) of a cell's "sib1" dict."""
    if s["format"] == "1A":
        start, length = riv_decode(R, s["riv"])
        tbs = TBS_1A[s["mcs"]][s.get("tpc", 0) & 1]
        vrbs = range(start, start + length)
        if not s.get("distributed", 0):
            return tbs, [list(vrbs), list(vrbs)]
        gap = 0
    else:
        step, gap = (2 if R < 50 else 4), s.get("gap", 0)
        start, length = riv_decode(n_vrb(R, gap) // step, s["riv"])
        vrbs = range(step * start, step * (start + length))
        tbs = TBS_1C[s["tbs_index"]]
    return tbs, [sorted(vrb_to_prb(R, gap, n, sl) for n in vrbs) for sl in (0, 1)]


def sib1_dci_bits(R, s):
    """The payload bits of the SI-RNTI DCI of a "sib1" dict (36.212 5.3.3.1.3-4)."""
    bits = lambda v, n: [(v >> (n - 1 - i)) & 1 for i in range(n)]
    if s["format"] == "1A":
        n_ra = int(np.ceil(np.log2(R * (R + 1) // 2)))
        a = [1, s.get("distributed", 0)] + bits(s["riv"], n_ra) + bits(s["mcs"], 5) + [0, 0, 0, 0] + bits(s.get("rv_field", 0), 2) \
            + bits(s.get("tpc", 0), 2)
        return a + [0] * (DCI_SIZES_1A[R] - len(a))
    g = [s.get("gap", 0)] if R >= 50 else []
    n = DCI_SIZES_1C[R] - len(g) - 5
    return g + bits(s["riv"], n) + bits(s["tbs_index"], 5)


def sib1_frames(cell, n_frames):
    """The grid frames a cell sends SIB1 in: cell["sib1"]["frames"], or every frame with an even SFN."""
    s = cell["sib1"]
    return s.get("frames", [f for f in range(n_frames) if (cell.get("sfn0", 0) + f) % 2 == 0])


def sib1_dcis(cell, n_subframes):
    s = cell["sib1"]
    R = cell["n_rb_dl"]
    return [(10 * f + 5, 0xFFFF, s["format"], s.get("L", 8), s.get("cce", 0), sib1_dci_bits(R, s))
            for f in sib1_frames(cell, -(-n_subframes // 10)) if 10 * f + 5 < n_subframes]


def pdsch_res(R, P, cp, nid, n_ctrl, prbs):
    """The data REs (l, k) of a SIB1 occasion in mapping order (36.211 6.3.5): symbols n_ctrl .. 2 n_symb - 1 of subframe
    5, k first, the PRBs of each slot, without CRS of ports < P or the PSS / SSS columns of slot 10."""
    n_symb = 7 if cp == 1 else 6
    _, shift = O.rs_dl(nid, cp)
    out = []
    for l in range(n_ctrl, 2 * n_symb):
        sl, ls = l // n_symb, l % n_symb
        crs = set()
        for p in range(P):
            sh = shift[(10 + sl) * n_symb + ls, p]
            if not np.isnan(sh):
                crs |= set(range(int(sh), 12 * R, 6))
        row = [k for prb in prbs[sl] for k in range(12 * prb, 12 * prb + 12)
               if k not in crs and not (sl == 0 and ls >= n_symb - 2 and 6 * R - 36 <= k < 6 * R + 36)]
        assert len(row) % 2 == 0, "a transmit-diversity pair would cross symbols"
        out += [(l, k) for k in row]
    return out


def sib1_rv(sfn):
    return (-(-3 * ((sfn // 2) % 4) // 2)) % 4


def _write_sib1(X, cell, n_symb):
    """cell["sib1"]: dict of the SIB1 bytes `tb` (TBS / 8 of them), the DCI (format "1A" or "1C", L, cce, riv, and
    distributed, mcs, tpc, rv_field for 1A, gap, tbs_index for 1C) and optionally the grid `frames` it is sent in.  In
    each such frame f, subframe 10 f + 5 carries the transport block with CRC24A, turbo-coded, rate-matched for the RV
    of its SFN, scrambled, QPSK-mapped, precoded over all ports and written over the data REs of its allocation."""
    s, R, P, cp, nid = cell["sib1"], cell["n_rb_dl"], cell["n_ports"], cell["cp_type"], cell["n_id_cell"]
    seq, dur = list(cell["cfi"]), cell["phich_duration"]
    tbs, prbs = sib1_allocation(R, s)
    a = np.unpackbits(np.frombuffer(bytes(s["tb"]), np.uint8))
    assert a.size == tbs, (a.size, tbs)
    b = np.concatenate([a, crc24a(a)])
    K = min(k for k in turbo_sizes() if k >= b.size)
    F = K - b.size
    d = turbo_encode(np.concatenate([np.zeros(F, np.uint8), b]))
    n_sub = X.shape[1] // (2 * n_symb)
    for f in sib1_frames(cell, -(-n_sub // 10)):
        u = 10 * f + 5
        if u >= n_sub:
            continue
        res = pdsch_res(R, P, cp, nid, n_ctrl_of(seq[u % len(seq)], R, dur), prbs)
        e = rate_match(d, K, F, sib1_rv(cell.get("sfn0", 0) + f), 2 * len(res))
        e = e ^ O.lte_pn(0xFFFF * 16384 + 5 * 512 + nid, e.size).astype(np.uint8)
        x = ((1 - 2 * e[0::2].astype(float)) + 1j * (1 - 2 * e[1::2].astype(float))) / np.sqrt(2)
        y = _precode(x, P)
        l, k = np.array(res).T
        X[:, 2 * n_symb * u + l, k] = y
