/* lcs_b200.h - C ABI of the GPU-native (H100, sm_90a) LTE cell-search correlator.
 *
 * This is the drop-in boundary for the hot path of Evrytania/LTE-Cell-Scanner: the free
 * functions of the reference's include/searcher.h (compiled into its static lib LTE_MISC,
 * src/CMakeLists.txt:2) and the caller-side glue of src/CellSearch.cpp:471-569.  The reference
 * has no FFI of its own; a maintainer binds these entry points from a ~100-line replacement of
 * src/searcher.cpp that marshals IT++ containers (see INTEGRATION.md and
 * lte-cell-scanner_b200/host/searcher_dropin.hpp).
 *
 * Conventions
 *   - plain C: pointers + sizes, no C++/torch types; every function returns an lcs_status
 *     (0 = LCS_OK) and never throws; lcs_last_error() gives the message for the last failure.
 *   - complex arrays are interleaved (re,im); "c128" = complex<double> (IT++ cvec),
 *     "cf32" = complex<float>, "cu8" = raw rtl-sdr unsigned bytes, sample = (u8-127)/128
 *     (reference src/capbuf.cpp:172-175).
 *   - there is NO CPU fallback: every compute entry point needs a CUDA device (sm_90a) and
 *     fails with LCS_ERR_CUDA when none is usable.
 *   - threading: a context and the plans / sweep handles created from it belong to ONE host thread at a time (they
 *     share the context's three streams and scratch buffers).  Use one context per thread; contexts are independent.
 *   - array layouts are stated per argument; "ref layout" is the reference's own
 *     (vf3d [t][idx][f]; IT++ mat/imat column-major).
 */
#ifndef LCS_B200_H
#define LCS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int lcs_status;
enum {
  LCS_OK = 0,
  LCS_ERR_ARG = 1,      /* bad argument (null pointer, size out of range, ...) */
  LCS_ERR_CUDA = 2,     /* CUDA runtime error or no usable device */
  LCS_ERR_RANGE = 3,    /* the reference would index out of bounds for these inputs */
  LCS_ERR_STATE = 4
};

/* IQ sample formats.  The correlator and search entry points take CF32, CU8 and C128 and reject CI16 and CS8 (LCS_ERR_ARG);
 * CI16 (interleaved little-endian int16) and CS8 (int8) are input formats of lcs_chan_create_rational, which also takes
 * CU8 and CF32. */
enum { LCS_IQ_CF32 = 0, LCS_IQ_CU8 = 1, LCS_IQ_C128 = 2, LCS_IQ_CI16 = 3, LCS_IQ_CS8 = 4 };

/* Which correlator kernel a plan uses.  AUTO picks the fastest one that is exact for the input
 * format (DESIGN.md "kernels"). */
enum { LCS_KERNEL_AUTO = 0, LCS_KERNEL_FP32 = 1, LCS_KERNEL_TC = 2 };

#define LCS_N_FOLD 9600   /* samples per 5 ms half frame at 1.92 Msps (searcher.cpp:289) */
#define LCS_N_TAPS 137    /* 128 + 9 CP samples of the time-domain PSS (lte_lib.cpp:177-188) */

/* POD mirror of class Cell (reference include/common.h.in:101-129); sentinels as in
 * src/common.cpp:36-56: NaN for doubles, -1 for integers, 0 (UNKNOWN) for enums. */
typedef struct lcs_cell {
  double fc_requested, fc_programmed, pss_pow;
  int32_t ind;
  double freq;
  int32_t n_id_2;
  int32_t n_id_1;
  int32_t cp_type;          /* 0 unknown, 1 normal, 2 extended */
  double frame_start, freq_fine, freq_superfine;
  int32_t n_ports, n_rb_dl;
  int32_t phich_duration;   /* 0 unknown, 1 normal, 2 extended */
  int32_t phich_resource;   /* 0 unknown, 1 oneSixth, 2 half, 3 one, 4 two */
  int32_t sfn;
} lcs_cell;

typedef struct lcs_ctx lcs_ctx;
typedef struct lcs_xcorr_plan lcs_xcorr_plan;

/* ---- library / context ------------------------------------------------------------------ */
const char* lcs_version(void);
/* Create a context on CUDA device `device` (one per process per GPU).  Fails with LCS_ERR_CUDA
 * when the device is absent or is not compute capability 9.0 (the kernels are built for sm_90a only). */
lcs_status lcs_ctx_create(int device, lcs_ctx** ctx);
void lcs_ctx_destroy(lcs_ctx* ctx);
const char* lcs_last_error(const lcs_ctx* ctx);   /* ctx may be NULL: last global error */
void lcs_cell_init(lcs_cell* c);                  /* Cell::Cell(), common.cpp:36-56 */
/* number of kernels this library has launched on ctx since creation (bench.py gpu_launches) */
uint64_t lcs_launch_count(const lcs_ctx* ctx);

/* ---- xcorr_pss: replaces searcher.h:22-41 (src/searcher.cpp:389-419) ------------------------ */
/* Drop-in: same inputs/outputs as the reference function, IT++ containers flattened.
 *   capbuf            c128 [n_cap]
 *   pow, frq          ref layout of mat(3,9600)/imat(3,9600): column-major, element (t,k) at [k*3+t]
 *   single, incoherent vf3d ref layout [t][idx][f], float (incoherent may be NULL)
 *   sp_incoherent     [9600]
 *   xc                debug: vcf3d [t][k][f] cf32, (n_cap-136) lags (NULL = skip; 136 MB at n_f=37)
 *   sp                debug: [n_comb_sp*9600] (NULL = skip)
 */
lcs_status lcs_xcorr_pss(lcs_ctx* ctx, const double* capbuf, uint32_t n_cap, const double* f_search_set,
                         uint32_t n_f, uint8_t ds_comb_arm, double fc_requested, double fc_programmed,
                         double fs_programmed, double* pow, int32_t* frq, float* single, float* incoherent,
                         double* sp_incoherent, float* xc, double* sp, uint16_t* n_comb_xc,
                         uint16_t* n_comb_sp);

/* Throughput path.  A plan fixes (n_cap, f_search_set, fc_*, fs, ds_comb_arm): it owns the
 * pre-rotated templates (conj(fshift(pss_td))/137, searcher.cpp:145-151), the k_factor fold
 * offsets (searcher.cpp:298) and device scratch for max_batch capture buffers. */
lcs_status lcs_xcorr_plan_create(lcs_ctx* ctx, uint32_t n_cap, const double* f_search_set, uint32_t n_f,
                                 uint8_t ds_comb_arm, double fc_requested, double fc_programmed,
                                 double fs_programmed, uint32_t max_batch, int kernel, lcs_xcorr_plan** plan);
void lcs_xcorr_plan_destroy(lcs_xcorr_plan* plan);
uint16_t lcs_xcorr_plan_n_comb_xc(const lcs_xcorr_plan* plan);
uint16_t lcs_xcorr_plan_n_comb_sp(const lcs_xcorr_plan* plan);
int lcs_xcorr_plan_kernel(const lcs_xcorr_plan* plan, int iq_format);   /* kernel AUTO resolves to */

/* Device-resident, batched, asynchronous on `stream` (a cudaStream_t; NULL = default stream).
 *   d_iq            [batch][n_cap] samples in iq_format (CF32, CU8 or C128), device memory.  The tensor-core correlator
 *                   stages raw bytes with 16-byte bulk copies: a CU8 pointer that is not 16-byte aligned is served by the
 *                   FP32 correlator under LCS_KERNEL_AUTO and rejected under LCS_KERNEL_TC (buffer strides may be odd)
 *   d_single_planar [batch][3][n_f][9600] float  (xc_incoherent_single, f-major "planar" layout)
 *   d_pow           [batch][3][9600] double,  d_frq [batch][3][9600] int32   (row-major (t,idx))
 *   d_sp_incoherent [batch][9600] double
 *   d_incoherent_planar  optional [batch][3][n_f][9600] float (NULL = skip)
 * Alignment (checked before any launch, LCS_ERR_ARG otherwise): d_iq to its sample size (2 bytes CU8, 8 CF32, 16 C128);
 * d_single_planar, d_pow, d_frq and d_incoherent_planar to 16 bytes; d_sp_incoherent to 8 bytes.  cudaMalloc'd bases
 * qualify; pointers into a tensor or buffer at other offsets may not.
 */
lcs_status lcs_xcorr_pss_device(lcs_xcorr_plan* plan, const void* d_iq, int iq_format, uint32_t batch,
                                float* d_single_planar, double* d_pow, int32_t* d_frq, double* d_sp_incoherent,
                                float* d_incoherent_planar, void* stream);

/* Kernel timing hook for roofline accounting (bench.py): when enabled, every launch of the
 * dominant correlator kernel made through this plan is bracketed by CUDA events on its launch
 * stream.  lcs_xcorr_plan_timing_read synchronises those events, returns the summed kernel time
 * (ms) and launch count since the last read, and resets the accumulator. */
lcs_status lcs_xcorr_plan_timing_enable(lcs_xcorr_plan* plan, int enable);
lcs_status lcs_xcorr_plan_timing_read(lcs_xcorr_plan* plan, double* kernel_ms, uint64_t* launches);

/* Host-buffer batched call (the e2e path): H2D of the IQ, kernels, D2H of the results, all on
 * the plan's own streams, double-buffered over the batch.  h_iq is [batch][n_cap] in iq_format
 * (CU8, CF32 or C128); outputs as in lcs_xcorr_pss_device but host memory (pinned memory gives
 * true overlap).  h_single_planar may be NULL (skips its 3*9600*n_f*4 B D2H per buffer). */
lcs_status lcs_xcorr_pss_batch_host(lcs_xcorr_plan* plan, const void* h_iq, int iq_format, uint32_t batch,
                                    float* h_single_planar, double* h_pow, int32_t* h_frq,
                                    double* h_sp_incoherent);

/* ---- rest of the searcher.h chain --------------------------------------------------------- */
/* Z_th1 of CellSearch.cpp:500-503 (chi2cdf_inv threshold x sp_incoherent) */
lcs_status lcs_calc_z_th1(const double* sp_incoherent, uint32_t n, uint16_t n_comb_xc, uint8_t ds_comb_arm,
                          double* z_th1);
/* peak_search, searcher.h:44-56 (searcher.cpp:422-510).  pow/frq row-major (t,idx) [3][9600];
 * single is the planar [3][n_f][9600] array.  Appends up to max_cells cells; *n_cells = total found. */
lcs_status lcs_peak_search(const double* pow, const int32_t* frq, const double* z_th1, const double* f_search_set,
                           uint32_t n_f, double fc_requested, double fc_programmed, const float* single_planar,
                           uint8_t ds_comb_arm, lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells);
/* sss_detect, searcher.h:59-76 (searcher.cpp:696-761).  Debug outputs may each be NULL:
 * sss_h?_np_est [62], sss_h?_{nrm,ext}_est c128 [62], log_lik_{nrm,ext} mat(168,2) column-major. */
lcs_status lcs_sss_detect(lcs_ctx* ctx, const lcs_cell* cell, const double* capbuf, uint32_t n_cap,
                          double thresh2_n_sigma, double fc_requested, double fc_programmed, double fs_programmed,
                          lcs_cell* cell_out, double* sss_h1_np_est, double* sss_h2_np_est, double* sss_h1_nrm_est,
                          double* sss_h2_nrm_est, double* sss_h1_ext_est, double* sss_h2_ext_est,
                          double* log_lik_nrm, double* log_lik_ext);
/* pss_sss_foe, searcher.h:79-85 (searcher.cpp:767-850) */
lcs_status lcs_pss_sss_foe(lcs_ctx* ctx, const lcs_cell* cell_in, const double* capbuf, uint32_t n_cap,
                           double fc_requested, double fc_programmed, double fs_programmed, lcs_cell* cell_out);
/* extract_tfg, searcher.h:88-98 (searcher.cpp:857-935).  tfg: cmat(n_ofdm,72) column-major c128,
 * tfg_timestamp [n_ofdm]; n_ofdm = 122*n_symb_dl (854 normal CP, 732 extended); *n_ofdm_out is set. */
lcs_status lcs_extract_tfg(lcs_ctx* ctx, const lcs_cell* cell, const double* capbuf, uint32_t n_cap,
                           double fc_requested, double fc_programmed, double fs_programmed, double* tfg,
                           double* tfg_timestamp, uint32_t* n_ofdm_out);
/* tfoec, searcher.h:101-112 (searcher.cpp:952-1069).  RS_DL(n_id_cell,6,cp_type) is built inside. */
lcs_status lcs_tfoec(lcs_ctx* ctx, const lcs_cell* cell, const double* tfg, const double* tfg_timestamp,
                     uint32_t n_ofdm, double fc_requested, double fc_programmed, double* tfg_comp,
                     double* tfg_comp_timestamp, lcs_cell* cell_out);
/* decode_mib, searcher.h:115-119 (searcher.cpp:1526-1692).  tfg = tfg_comp, column-major. */
lcs_status lcs_decode_mib(lcs_ctx* ctx, const lcs_cell* cell, const double* tfg, uint32_t n_ofdm,
                          lcs_cell* cell_out);
/* dedup, CellSearch.cpp:285-319 (cells in detection order; out may alias nothing) */
lcs_status lcs_dedup(const lcs_cell* cells, uint32_t n, lcs_cell* out, uint32_t* n_out);
/* f_search_set of CellSearch.cpp:463-464; out may be NULL to query *n_f */
lcs_status lcs_f_search_set(double freq_start, double ppm, double* out, uint32_t* n_f);

/* One centre frequency of the CellSearch main loop (CellSearch.cpp:471-569): xcorr_pss ->
 * threshold -> peak_search -> per peak sss_detect / pss_sss_foe / extract_tfg / tfoec /
 * decode_mib.  Appends the surviving cells (n_id_1 and MIB found).  peaks/n_peaks optional. */
lcs_status lcs_cell_search(lcs_ctx* ctx, const double* capbuf, uint32_t n_cap, const double* f_search_set,
                           uint32_t n_f, double fc_requested, double fc_programmed, double fs_programmed,
                           lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells, lcs_cell* peaks,
                           uint32_t* n_peaks);
/* Same, raw rtl-sdr bytes (cu8 [n_cap][2]) - the wire format of capbuf.cpp:157-181. */
lcs_status lcs_cell_search_cu8(lcs_ctx* ctx, const uint8_t* capbuf_cu8, uint32_t n_cap, const double* f_search_set,
                               uint32_t n_f, double fc_requested, double fc_programmed, double fs_programmed,
                               lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells, lcs_cell* peaks,
                               uint32_t* n_peaks);

/* kalibrate, src/LTE-Tracker.cpp:565-741: the initial search LTE-Tracker runs to calibrate the oscillator.  The grid of
 * CellSearch.cpp:463-464 for (fc_requested, ppm) is centred on fc_requested*(correction-1) (:586-587); after the chain
 * and dedup the strongest cell is returned in *best with *correction_residual = fc_programmed/(fc_programmed -
 * best->freq_superfine) (:719-724; may be NULL).  *n_cells = cells that survived (0: nothing found in this buffer - the
 * reference then captures the next one). */
lcs_status lcs_kalibrate_cu8(lcs_ctx* ctx, const uint8_t* capbuf_cu8, uint32_t n_cap, double fc_requested,
                             double fc_programmed, double fs_programmed, double ppm, double correction, lcs_cell* best,
                             double* correction_residual, uint32_t* n_cells);

/* ---- batched search (many capture buffers of one centre frequency, e.g. a tracked channel) ---- */
/* xcorr_pss (searcher.cpp:389) + Z_th1 (CellSearch.cpp:500-503) + peak_search (searcher.cpp:422-510) for a batch of HOST
 * capture buffers, everything on the device: only the PSS peaks return.  iq_host is [batch][n_cap] in iq_format;
 * peaks is [batch][max_peaks] (fc_requested, fc_programmed, pss_pow, ind, freq, n_id_2 filled as by peak_search,
 * in the reference's order), n_peaks[batch] the number found per buffer (may exceed max_peaks: list truncated).
 * Chunks of up to 64 buffers rotate over the context's three streams. */
lcs_status lcs_xcorr_peaks_batch_host(lcs_xcorr_plan* plan, const void* iq_host, int iq_format, uint32_t batch,
                                      lcs_cell* peaks, uint32_t max_peaks, uint32_t* n_peaks);
/* The whole chain of CellSearch.cpp:497-558 for every buffer of a batch of raw rtl-sdr byte buffers (cu8
 * [batch][n_cap][2]); cells is [batch][max_cells], n_cells[batch].  lcs_cell_search_cu8 runs the same implementation
 * on a batch of one. */
lcs_status lcs_cell_search_batch_cu8(lcs_xcorr_plan* plan, const uint8_t* iq_host, uint32_t batch, lcs_cell* cells,
                                     uint32_t max_cells, uint32_t* n_cells);

/* ---- many channels at once: frequency sweep and multi-channel tracker search -------------------------------------- */
/* A sweep handle owns one search plan per channel (templates for every channel's k_factor built on the device in one
 * launch) and the device buffers of the pipeline; all channels of a chunk go through ONE correlator launch.  n_cap is
 * the capture-buffer length of every channel. */
typedef struct lcs_sweep lcs_sweep;
lcs_status lcs_sweep_create(lcs_ctx* ctx, uint32_t n_cap, lcs_sweep** sweep);
void lcs_sweep_destroy(lcs_sweep* sweep);
/* The per-centre-frequency loop of CellSearch (src/CellSearch.cpp:465-558) for n_ch capture buffers: iq_host is cu8
 * [n_ch][n_cap][2]; fc_requested[n_ch]; fc_programmed[n_ch] or NULL (= fc_requested); one fs_programmed and one
 * f_search_set for the whole sweep like the reference (:463-464 computes it from freq_start).  cells is
 * [n_ch][max_cells], n_cells[n_ch]; apply lcs_dedup to the concatenation in channel order (CellSearch.cpp:560-562). */
lcs_status lcs_sweep_search_cu8(lcs_sweep* sweep, const uint8_t* iq_host, uint32_t n_ch, const double* fc_requested,
                                const double* fc_programmed, double fs_programmed, const double* f_search_set, uint32_t n_f,
                                lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells);
/* One searcher cycle (src/searcher_thread.cpp:95-232) for n_ch tracked channels: channel c is searched at the single
 * offset frequency_offset[c]; tracked_n_id_cell is [n_ch][tracked_stride] with n_tracked[c] valid entries (both may be
 * NULL); late[n_ch] or NULL; cells / frame_timing are [n_ch][max_cells].  lcs_tracker_search_cu8 runs the same
 * implementation on a single channel. */
lcs_status lcs_sweep_track_cu8(lcs_sweep* sweep, const uint8_t* iq_host, uint32_t n_ch, const double* frequency_offset,
                               const double* fc_requested, const double* fc_programmed, double fs_programmed,
                               const double* late, const int32_t* tracked_n_id_cell, const uint32_t* n_tracked,
                               uint32_t tracked_stride, lcs_cell* cells, double* frame_timing, uint32_t max_cells,
                               uint32_t* n_cells);

/* ---- streaming (tracker) mode: producer framing + one searcher cycle ------------------------------------------ */
/* Host-side framing of a continuous raw IQ byte stream into searcher capture buffers: the searcher part of
 * src/producer_thread.cpp:96-161.  A running time stamp (LTE samples modulo 19200) advances by
 * (FS_LTE/16)/(fs_programmed*k_factor) per sample; after lcs_framer_request the capture of n_cap samples starts at the
 * first sample whose stamp is within +-0.5 of 0 (mod 19200); `late` is that stamp wrapped to [-9600, 9600). */
typedef struct lcs_framer lcs_framer;
lcs_status lcs_framer_create(double fc_requested, double fc_programmed, double fs_programmed, uint32_t n_cap,
                             lcs_framer** out);
void lcs_framer_destroy(lcs_framer* framer);
void lcs_framer_request(lcs_framer* framer);                /* capbuf_sync.request = true (searcher_thread.cpp:88) */
double lcs_framer_sample_time(const lcs_framer* framer);    /* current time stamp (starts at -1) */
/* Feed n_samples (I,Q) byte pairs received while the tracked frequency offset estimate is frequency_offset
 * (global_thread_data.frequency_offset(); the reference re-reads it every 10000 samples).  *ready becomes 1 once a
 * requested capture buffer is complete; *capbuf ([n_cap][2] bytes, owned by the framer, valid until the next request)
 * and *late are then set. */
lcs_status lcs_framer_push(lcs_framer* framer, const uint8_t* iq, uint32_t n_samples, double frequency_offset,
                           int* ready, const uint8_t** capbuf, double* late);
/* One cycle of the searcher thread (src/searcher_thread.cpp:95-232) on such a buffer: xcorr_pss at the single offset
 * frequency_offset, threshold, peak_search, sss_detect, skip cells whose n_id_cell is in tracked_n_id_cell,
 * pss_sss_foe / extract_tfg / tfoec / decode_mib.  For every NEW cell frame_timing = frame_start*(FS_LTE/16)/
 * (fs_programmed*k_factor) + late, the value the reference hands to the cell's tracker (:214). */
lcs_status lcs_tracker_search_cu8(lcs_ctx* ctx, const uint8_t* capbuf_cu8, uint32_t n_cap, double frequency_offset,
                                  double fc_requested, double fc_programmed, double fs_programmed, double late,
                                  const int32_t* tracked_n_id_cell, uint32_t n_tracked, lcs_cell* cells,
                                  double* frame_timing, uint32_t max_cells, uint32_t* n_cells);

/* ---- cell tracking: the per-cell tracker loop of LTE-Tracker for many cells and channels ------------------------- */
/* A track handle follows every detected cell of n_ch channels over time: the per-cell slicer of
 * src/producer_thread.cpp:163-250 and the tracker loop of src/tracker_thread.cpp:856-1067 (get_fd, CRS channel
 * estimation and filtering, FOE / TOE, interpolation, CRS and PSS/SSS measurements, MIB decoding, dropping a cell after
 * CELL_DROP_THRESHOLD = 400 failures).  The schedule is deterministic (DESIGN.md section 4.5): each channel's stream is
 * cut into blocks of LCS_TRACK_BLOCK samples counted from its start; a block is processed once it is complete, in one
 * launch per push for every channel.  The channel's frequency offset (moved by every cell's FOE) and each cell's frame
 * timing (moved by its TOE) are sampled at each block start.  Cells added between pushes take part from the first block
 * not yet processed, starting at slot 0, symbol 0. */
#define LCS_TRACK_BLOCK 10000

typedef struct lcs_track lcs_track;

/* One tracked cell as lcs_track_read reports it (the measurements of the reference's tracked_cell_t).  Measurements
 * start as NaN, channel estimates as 0. */
typedef struct lcs_track_cell {
  int32_t n_id_cell, n_ports, cp_type;
  int32_t dropped;               /* 1: dropped (MIB failures reached 400); reported once, then its slot is freed */
  int64_t drop_sample;           /* stream sample one past the symbol whose MIB attempt dropped the cell (-1: live) */
  int64_t n_symbols;             /* OFDM symbols sliced and processed */
  int64_t last_slice_start;      /* stream sample of the first sample of the latest symbol (-1: none yet) */
  int64_t mib_attempts, mib_successes;
  double frame_timing;           /* LTE samples modulo 19200, in the tracker's time stamps */
  double mib_decode_failures;
  double crs_tp[4], crs_sp_raw[4], crs_np[4];
  double crs_tp_av[4], crs_sp_raw_av[4], crs_np_av[4];
  double sync_tp, sync_sp, sync_np, sync_np_blank;
  double sync_tp_av, sync_sp_av, sync_np_av, sync_np_blank_av;
  double sync_ce[72][2];         /* c128, latest PSS/SSS channel estimate */
  double ce[4][72][2];           /* c128, latest interpolated CRS channel estimate per port */
  /* Channel autocorrelations (do_ac_fd / do_ac_td, tracker_thread.cpp:318-370), c128, 0 until their first update.  Each
   * update is normalised by the CRS signal power sp = max(1e-5, tp - np/7) of the estimate that makes it.  Every port
   * of the cell updates the same arrays, ports in ascending order within a symbol.
   * ac_fd[d]: lag d CRS subcarriers = 6d subcarriers = 90d kHz.  Each CRS symbol is weighted by 1/np_d, np_d =
   *   (np^2/sp^2 + 2 np/sp) / (12 - d), against a prior of weight 1e5, so at high SNR it converges within about a second (ac_fd[0] about 1 on a flat channel).
   * ac_td[t]: lag t CRS symbols of one port (ports 0/1: 4 and 3 OFDM symbols alternately, ports 2/3: one slot),
   *   updated from the port's 72nd processed estimate on, each update with weight 1 against 1e5: after n updates it
   *   is about n * 1e-5 times the mean correlation, so only its shape over t is meaningful for n << 1e5.
   * Coherence bandwidth (display_thread.cpp:166-177): the first d in 1..11 with |ac_fd[d]| <= 0.5 gives 90d kHz,
   * none gives more than 990 kHz. */
  double ac_fd[12][2];
  double ac_td[72][2];
} lcs_track_cell;

/* fc_requested[n_ch]; fc_programmed[n_ch] or NULL (= fc_requested); frequency_offset[n_ch] the initial offsets (the
 * kalibrate result); max_cells per channel, 1 to 32 (one slicing thread per cell slot in the channel's CTA). */
lcs_status lcs_track_create(lcs_ctx* ctx, uint32_t n_ch, const double* fc_requested, const double* fc_programmed,
                            double fs_programmed, const double* frequency_offset, uint32_t max_cells, lcs_track** out);
void lcs_track_destroy(lcs_track* track);
/* Start tracking a cell found by lcs_tracker_search_cu8 on channel ch: cell->n_id_1/n_id_2, cp_type, n_ports (1, 2 or
 * 4), n_rb_dl, phich_duration and phich_resource are used; frame_timing in [0, 19200) is the handed-over timing. */
lcs_status lcs_track_add_cell(lcs_track* track, uint32_t ch, const lcs_cell* cell, double frame_timing);
/* Feed n samples of every channel: iq_host is cu8 [n_ch][n][2].  All complete blocks run in one launch. */
lcs_status lcs_track_push_cu8(lcs_track* track, const uint8_t* iq_host, uint32_t n);
lcs_status lcs_track_frequency_offset(const lcs_track* track, double* frequency_offset /*[n_ch]*/);
/* The cells of channel ch in the order they were added (at most max; *n = number written). */
lcs_status lcs_track_read(lcs_track* track, uint32_t ch, lcs_track_cell* out, uint32_t max, uint32_t* n);
/* Time stamp of the last processed sample of channel ch (the lcs_framer_sample_time recurrence). */
lcs_status lcs_track_sample_time(const lcs_track* track, uint32_t ch, double* sample_time);
/* Summed device time of the tracker kernel (CUDA events around each launch, ms) and the number of launches since the
 * last read; resets both. */
lcs_status lcs_track_timing_read(lcs_track* track, double* kernel_ms, uint64_t* launches);

/* ---- wideband channelizer: many LTE raster channels out of one wideband ci16 recording (DESIGN.md section 4.6) ------ */
/* One digital down-converter per channel, all channels in one launch per push; the output of channel c is the 1.92 Msps
 * cu8 stream a dongle tuned to fc_ch[c] would deliver (fc_requested = fc_programmed = fc_ch[c], fs_programmed =
 * 1.92e6 * correction when the recording's LO and sample clock share one crystal).
 *   fs_in = D * 1 920 000 Hz, D integer in [2, 64]; channel offset delta_c = fc_ch[c] - fc_in an integer number of Hz
 *   (within 1e-6) with |delta_c| <= fs_in/2 - 960 kHz; 1 <= n_ch <= 1024; anything else is LCS_ERR_ARG.
 *   input  x[m] = (I[m] + jQ[m]) / 32768, m counted from the start of the stream (interleaved little-endian int16 I/Q).
 *   mixer  p_c[m] = (m * delta_c) mod fs_in in exact 64-bit integers; x~_c[m] = x[m] exp(-j2pi p_c[m]/fs_in).
 *   filter h: real, symmetric, odd length L = 2M+1, Kaiser-windowed sinc (cutoff 0.96 MHz), designed in double and kept
 *          as float; passband deviation <= 0.01 dB for |f| <= 0.70 MHz, stopband >= 70 dB for |f| >= 1.22 MHz, the
 *          shortest such odd L (37, 73, 133, 263, 523, 1045 taps at D = 2, 4, 8, 16, 32, 64: about 16D+5).  The passband holds the central 72 subcarriers (+-0.54 MHz) plus a carrier
 *          offset of up to +-160 kHz.
 *   output y_c[n] = sum_{k=-M..M} h[k+M] x~_c[nD-k] (x~ = 0 before the stream starts).  Output n is emitted once input
 *          sample nD+M has been pushed: after N input samples there are max(0, floor((N-1-M)/D)+1) outputs; output n
 *          belongs to input instant nD.  Any sequence of pushes gives bitwise the bytes of one push of the whole stream.
 *   bytes  v = 127 + 128 g_c Re(y) (and Im), rounded to nearest (ties to even), clamped to [0, 255] - the (u8-127)/128
 *          convention of capbuf.cpp:172-175; the clamped components are counted per channel.
 *   gain   g_c from lcs_chan_create (NULL: 1.0), or lcs_chan_auto_gain_ci16: 0.25 / sqrt(mean |y_c[n]|^2) over the outputs
 *          a FRESH channelizer would produce from the given samples (1.0 when that is 0); it leaves the stream alone. */
typedef struct lcs_chan lcs_chan;
/* host only, no device needed: the prototype filter h for fs_in; taps may be NULL to query *n_taps (on input, the
 * capacity of taps) */
lcs_status lcs_chan_design_taps(double fs_in, float* taps, uint32_t* n_taps);
lcs_status lcs_chan_create(lcs_ctx* ctx, double fs_in, double fc_in, uint32_t n_ch, const double* fc_ch,
                           const float* gain /*[n_ch] or NULL*/, lcs_chan** out);
void lcs_chan_destroy(lcs_chan* chan);
/* iq_host is ci16 [n][2] */
lcs_status lcs_chan_auto_gain_ci16(lcs_chan* chan, const int16_t* iq_host, uint32_t n);
lcs_status lcs_chan_gain(const lcs_chan* chan, float* gain /*[n_ch]*/);
/* the number of outputs per channel the next push of n_in samples yields */
lcs_status lcs_chan_n_out(const lcs_chan* chan, uint64_t n_in, uint32_t* n_out);
/* Push n_in samples (ci16 [n_in][2], host).  out: cu8 [n_ch][out_capacity][2] in host memory, or device memory when
 * out_on_device; *n_out outputs per channel are written from column 0.  n_clipped[n_ch] (may be NULL): components
 * clamped in this push.  out_capacity < the outputs of this push -> LCS_ERR_ARG and nothing is consumed.  Large pushes
 * run in chunks that bound the device scratch. */
lcs_status lcs_chan_push_ci16(lcs_chan* chan, const int16_t* iq_host, uint32_t n_in, uint8_t* out, uint32_t out_capacity,
                              int out_on_device, uint32_t* n_out, uint64_t* n_clipped);
/* Summed device time of the channelizer kernel (CUDA events around each launch, ms) and the number of launches since
 * the last read; resets both. */
lcs_status lcs_chan_timing_read(lcs_chan* chan, double* kernel_ms, uint64_t* launches);

/* ---- rational resampling: any SDR rate, ci16 / cs8 / cu8 / cf32 input (DESIGN.md section 4.7) ------------------------ */
/* The same lcs_chan, created at any allowed rate and sample format; lcs_chan_n_out, lcs_chan_gain, lcs_chan_timing_read
 * and lcs_chan_destroy serve it unchanged.
 *   fs_in  an integer number of Hz (within 1e-6), 1.92 MHz < fs_in <= 122.88 MHz, with fs_in / 1 920 000 = down / up in
 *          lowest terms, up <= 128, down <= 640 (2.048, 2.4, 2.5, 6, 10, 12.5, 20, 25, 56, 100 Msps and every D * 1.92
 *          MHz, D <= 64, are allowed); channels, offsets and gains as in section 4.6.  Anything else is LCS_ERR_ARG.
 *   input  iq_format LCS_IQ_CI16: (I + jQ)/32768; LCS_IQ_CS8: (I + jQ)/128; LCS_IQ_CU8: ((I-127) + j(Q-127))/128;
 *          LCS_IQ_CF32: I + jQ.  The mixer is that of section 4.6.
 *   filter h: the section 4.6 design at F = up * fs_in (grid every F/(64L) or denser), DC gain up, so each of the up
 *          polyphase branches has unit gain; at up = 1 exactly lcs_chan_design_taps(fs_in).
 *   output y_c[n] = sum_i h[n*down - i*up + M] x~_c[i] over 0 <= n*down - i*up + M <= 2M (x~ = 0 before the stream
 *          starts); output n belongs to input instant n*down/up and is emitted once input floor((n*down + M)/up) has
 *          been pushed: after N samples there are max(0, floor((N*up - M - 1)/down) + 1) outputs.  Any sequence of
 *          pushes gives bitwise the bytes of one push.  Bytes, clip counts, gain and auto gain as in section 4.6.
 *   At up = 1 with CI16 the channelizer is lcs_chan_create's (the same bytes, clip counts and auto gain). */
/* host only: fs_in / 1.92e6 = down / up in lowest terms and the prototype at up * fs_in (taps NULL: query *n_taps; on
 * input, the capacity of taps) */
lcs_status lcs_chan_design_rational(double fs_in, uint32_t* up, uint32_t* down, float* taps, uint32_t* n_taps);
lcs_status lcs_chan_create_rational(lcs_ctx* ctx, double fs_in, int iq_format, double fc_in, uint32_t n_ch,
                                    const double* fc_ch, const float* gain /*[n_ch] or NULL*/, lcs_chan** out);
/* lcs_chan_push_ci16 / lcs_chan_auto_gain_ci16 with the samples in the channelizer's own format ([n][2] of int16, int8,
 * uint8 or float); also valid on an lcs_chan_create channelizer (ci16).  lcs_chan_push_ci16 and lcs_chan_auto_gain_ci16
 * on a channelizer whose format is not CI16 return LCS_ERR_ARG before any launch.  The device output feeds
 * lcs_sweep_search_cu8_device unchanged. */
lcs_status lcs_chan_push(lcs_chan* chan, const void* iq_host, uint32_t n_in, uint8_t* out, uint32_t out_capacity,
                         int out_on_device, uint32_t* n_out, uint64_t* n_clipped);
lcs_status lcs_chan_auto_gain(lcs_chan* chan, const void* iq_host, uint32_t n);

/* lcs_sweep_search_cu8 on capture buffers already in device memory (e.g. a channelizer's output): d_iq is cu8
 * [n_ch][n_cap][2], 16-byte aligned, and is read in place (no copy).  Same arguments and results otherwise. */
lcs_status lcs_sweep_search_cu8_device(lcs_sweep* sweep, const uint8_t* d_iq, uint32_t n_ch, const double* fc_requested,
                                       const double* fc_programmed, double fs_programmed, const double* f_search_set,
                                       uint32_t n_f, lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells);

#ifdef __cplusplus
}
#endif
#endif /* LCS_B200_H */
