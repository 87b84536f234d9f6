"""The chunk pipeline of the host-batch calls across chunk and stream boundaries.

130 buffers on a plan of max_batch 64 go through chunks of 64, 64 and 2 buffers on the context's three streams.  Every
buffer differs from every other, so an output written to the wrong place shows.  lcs_xcorr_pss_batch_host, with and
without xc_incoherent_single, must equal lcs_xcorr_pss_device on each buffer bit for bit; the batched peak search and
cell search must equal the single-buffer cell search on each buffer."""
import numpy as np
import pytest

from conftest import synth_cu8
from test_search_chain_gpu import same_cells

pytestmark = pytest.mark.gpu

N_BUF = 130
MAX_BATCH = 64
REAL = (0, 63, 64, 127, 128, 129)       # the first and last buffer of every chunk hold the real capture
FS = 1.92e6
OUTPUTS = ("single", "pow", "frq", "sp_incoherent")


@pytest.fixture(scope="module")
def batch(capbuf0000):
    """(buffers [130][n_cap][2] uint8, f_search_set, fc): the real capture, rolled a little differently in every buffer
    of REAL, and noise of its own seed in every other buffer.  The grid of three offsets covers the capture's cells."""
    real = capbuf0000["cu8"]
    bufs = np.stack([np.roll(real, 7 * b, axis=0) if b in REAL else synth_cu8(0xB00 + b, real.shape[0])
                     for b in range(N_BUF)])
    f = 35228.0 + 5000.0 * np.arange(-1, 2)
    return bufs, f, capbuf0000["fc"]


def test_batch_host_equals_device(ctx, lcs, batch):
    import torch
    bufs, f, fc = batch
    plan = ctx.plan(bufs.shape[1], f, 2, fc, fc, FS, max_batch=MAX_BATCH)
    d_iq = torch.from_numpy(bufs).cuda()
    dev = dict(single=torch.empty((N_BUF, 3, f.size, 9600), dtype=torch.float32, device="cuda"),
               pow=torch.empty((N_BUF, 3, 9600), dtype=torch.float64, device="cuda"),
               frq=torch.empty((N_BUF, 3, 9600), dtype=torch.int32, device="cuda"),
               sp_incoherent=torch.empty((N_BUF, 9600), dtype=torch.float64, device="cuda"))
    for b in range(N_BUF):
        plan.run_device(d_iq[b].data_ptr(), lcs.IQ_CU8, 1, *(dev[k][b].data_ptr() for k in OUTPUTS))
    torch.cuda.synchronize()
    dev = {k: v.cpu().numpy() for k, v in dev.items()}
    for want_single in (True, False):
        host = plan.run_host_np(bufs, lcs.IQ_CU8, want_single=want_single)
        for k in OUTPUTS if want_single else OUTPUTS[1:]:
            for b in range(N_BUF):
                assert host[k][b].tobytes() == dev[k][b].tobytes(), (want_single, k, b)
    plan.close()


def test_batch_search_equals_single_buffer(ctx, lcs, batch):
    bufs, f, fc = batch
    plan = ctx.plan(bufs.shape[1], f, 2, fc, fc, FS, max_batch=MAX_BATCH)
    peaks = plan.peaks_batch(bufs, lcs.IQ_CU8)
    cells = plan.cell_search_batch_cu8(bufs)
    plan.close()
    for b in range(N_BUF):
        ref_cells, ref_peaks = ctx.cell_search(bufs[b], f, fc, fc, FS)
        same_cells(peaks[b], ref_peaks)
        same_cells(cells[b], ref_cells)
        assert (len(ref_peaks) > 0) == (b in REAL), b
    assert len(cells[0]) > 0
