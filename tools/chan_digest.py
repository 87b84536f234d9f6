"""Bit-exact fingerprint of the wideband channelizer (lcs_chan_*): one SHA-256 per configuration over the auto-gain floats,
the output bytes and the clip counts of every push, from seeded numpy input.

The GPU tests compare against a float64 oracle with a rounding-boundary tolerance, so they cannot show that a change left
every byte alone; two builds that print the same lines here computed the same thing.  The configurations cover both
kernels (lcs_chan_create at D = 2, 16, 32; lcs_chan_create_rational at 2.4, 2.5, 20, 25 Msps and at D = 8 in the formats
chan_kernel does not take), unit, automatic and clipping gains, a 1024-channel D = 32 stream that spans several launches
fed as one push and as uneven pushes (one shorter than the filter's half length), and two channelizers of different
rates alive together with interleaved pushes.

Usage: python tools/chan_digest.py        (needs an H100; a few seconds)
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "lte-cell-scanner_b200"))

import lcs_b200 as L  # noqa: E402

FC_IN = 739e6


def samples(fmt, n, seed):
    """Seeded noise [n][2] in the format's dtype, about a fifth of full scale."""
    x = np.random.default_rng(seed).standard_normal((n, 2))
    if fmt == "cf32":
        return (0.2 * x).astype(np.float32)
    if fmt == "ci16":
        return np.clip(np.round(6000 * x), -32768, 32767).astype(np.int16)
    v = np.clip(np.round(25 * x), -127, 127)
    return v.astype(np.int8) if fmt == "cs8" else (v + 127).astype(np.uint8)


def channels(fs_in, n_ch):
    """n_ch integer-Hz offsets from one band edge to the other (both edges included when n_ch > 1)."""
    edge = fs_in / 2 - 960e3
    return FC_IN + np.round(np.linspace(-edge, edge, n_ch)) if n_ch > 1 else np.array([FC_IN + 12345.0])


def make(ctx, fs_in, fmt, n_ch, gain):
    """fmt None: lcs_chan_create (ci16 at D * 1.92 MHz); otherwise lcs_chan_create_rational with that format."""
    g = None if gain in (None, "auto") else gain
    if fmt is None:
        ch = L.Channelizer(ctx, fs_in, FC_IN, channels(fs_in, n_ch), gain=g)
        return ch, ch.push_ci16
    ch = L.RationalChannelizer(ctx, fs_in, FC_IN, channels(fs_in, n_ch), fmt=fmt, gain=g)
    return ch, ch.push


def feed(h, ch, push, iq, cuts, gain):
    """Auto gain (when asked) and the pushes iq[cuts[i]:cuts[i+1]] into the hash h."""
    if gain == "auto":
        h.update(ch.auto_gain(iq).tobytes())
    for a, b in zip(cuts[:-1], cuts[1:]):
        out, clip = push(iq[a:b])
        h.update(np.int64(out.shape[1]).tobytes() + out.tobytes() + clip.tobytes())
    return int(clip.sum())


def one(ctx, name, fs_in, fmt, n_ch, n, gain, cuts=None):
    ch, push = make(ctx, fs_in, fmt, n_ch, gain)
    iq = samples(fmt or "ci16", n, seed=n_ch + n)
    h = hashlib.sha256()
    clipped = feed(h, ch, push, iq, [0, n] if cuts is None else [0] + cuts + [n], gain)
    launches = ch.timing_read()[1]
    ch.close()
    print("%-34s %s  launches %d  clipped in last push %d" % (name, h.hexdigest(), launches, clipped), flush=True)


def interleaved(ctx):
    """A D = 32 ci16 and a 2.4 Msps cu8 channelizer alive together, pushes alternating."""
    a, push_a = make(ctx, 32 * 1.92e6, None, 40, "auto")
    b, push_b = make(ctx, 2.4e6, "cu8", 5, "auto")
    xa, xb = samples("ci16", 200000, 1), samples("cu8", 30000, 2)
    ha, hb = hashlib.sha256(), hashlib.sha256()
    ha.update(a.auto_gain(xa).tobytes())
    hb.update(b.auto_gain(xb).tobytes())
    for i in range(4):
        feed(ha, a, push_a, xa[i * 50000:(i + 1) * 50000], [0, 50000], None)
        feed(hb, b, push_b, xb[i * 7500:(i + 1) * 7500], [0, 7500], None)
    a.close()
    b.close()
    print("%-34s %s\n%-34s %s" % ("interleaved D=32 ci16", ha.hexdigest(), "interleaved 2.4 Msps cu8", hb.hexdigest()),
          flush=True)


def main():
    ctx = L.Context(0)
    # chan_kernel: lcs_chan_create
    one(ctx, "create D=2 unit gain", 2 * 1.92e6, None, 2, 50000, None)
    one(ctx, "create D=16 auto gain", 16 * 1.92e6, None, 289, 300000, "auto")
    one(ctx, "create D=16 clipping gain 40", 16 * 1.92e6, None, 7, 100000, 40.0)
    n32 = 32 * 40000
    one(ctx, "create D=32 1024 ch one push", 32 * 1.92e6, None, 1024, n32, "auto")
    one(ctx, "create D=32 1024 ch uneven pushes", 32 * 1.92e6, None, 1024, n32, "auto",
        cuts=[100, 101, 777, 600000, 600200, 1100001])
    # rchan_kernel: lcs_chan_create_rational
    one(ctx, "rational 2.4 Msps cu8", 2.4e6, "cu8", 5, 60000, "auto")
    one(ctx, "rational 2.5 Msps cf32", 2.5e6, "cf32", 5, 60000, "auto", cuts=[3, 40000])
    one(ctx, "rational 20 Msps cs8", 20e6, "cs8", 181, 400000, "auto", cuts=[50, 123457])
    one(ctx, "rational 20 Msps cs8 clipping", 20e6, "cs8", 3, 100000, 40.0)
    one(ctx, "rational 25 Msps ci16", 25e6, "ci16", 231, 500000, "auto")
    for fmt in ("cs8", "cu8", "cf32"):
        one(ctx, "rational D=8 %s" % fmt, 8 * 1.92e6, fmt, 30, 100000, "auto", cuts=[10, 33333])
    one(ctx, "rational D=16 ci16 (chan_kernel)", 16 * 1.92e6, "ci16", 289, 300000, "auto")
    interleaved(ctx)
    ctx.close()


if __name__ == "__main__":
    main()
