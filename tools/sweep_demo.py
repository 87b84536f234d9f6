#!/usr/bin/env python
"""Multi-GPU frequency sweep demo (BASELINE config 4 in miniature): N ranks, channels round-robin, each rank
runs its channels through lcs_sweep_search_cu8 on its own GPU, NCCL all_gather of the cell records, dedup on rank 0.
Channel 739.0 MHz carries the reference's real capture (tests/golden/capbuf_0000.npz); the others are synthetic noise.
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tools/sweep_demo.py [n_channels]
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "lte-cell-scanner_b200"))
import torch
import torch.distributed as dist
import lcs_b200 as L
import sweep


def main():
    n_ch = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1")); local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    d = None
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
        d = dist
    g = np.load(os.path.join(ROOT, "tests/golden/capbuf_0000.npz"))
    real = g["cu8"].reshape(-1, 2)
    fc0 = 739e6 - (n_ch // 2) * 100e3
    chans = []
    for i in range(n_ch):
        fc = fc0 + i * 100e3
        if abs(fc - 739e6) < 1:
            cap = real
        else:
            rng = np.random.default_rng(0xC0FFEE + i)
            cap = np.clip(np.round(127.5 + 20 * rng.standard_normal((153600, 2))), 0, 255).astype(np.uint8)
        chans.append((i, fc, cap))
    ctx = L.Context(local)
    sw = L.Sweep(ctx, 153600)
    f = L.f_search_set(fc0, 120.0)                       # CellSearch.cpp:463-464: one grid for the sweep, from freq_start
    fcs = [c[1] for c in chans]
    mine = sweep.shard(n_ch, rank, world)
    iq = np.stack([chans[i][2] for i in mine]) if mine else np.zeros((0, 153600, 2), np.uint8)

    def run():
        return sweep.sweep_batched(fcs, iq, lambda b, fc: sw.search_cu8(b, fc, f), L.new_cell, L.dedup, dist=d, device=dev)

    run()                                       # warm-up (allocations, module load)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = run()
    dt = time.perf_counter() - t0
    if rank == 0:
        print("sweep of %d channels on %d GPU(s): %.3f s (%.1f channels/s), %d cell(s)" % (n_ch, world, dt, n_ch / dt, len(res)))
        for c in res:
            print("  cell %3d  fc %.1f MHz  ports %d  n_rb_dl %d  sfn %d  pss_pow %.2f dB  foff %.1f Hz" %
                  (c.n_id_cell(), c.fc_requested / 1e6, c.n_ports, c.n_rb_dl, c.sfn, 10 * np.log10(c.pss_pow), c.freq_superfine))
        ids = sorted(c.n_id_cell() for c in res)
        assert ids == [271, 277], ids
        print("OK")
    ctx.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
