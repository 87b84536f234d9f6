// stream_search_main.cpp - the searcher side of LTE-Tracker on a recorded raw IQ stream (rtl_sdr byte dump):
// producer framing (src/producer_thread.cpp:96-161) + searcher cycles (src/searcher_thread.cpp:83-246) through
// lcs_framer_* and lcs_tracker_search_cu8.  Every new cell is printed with the frame timing the reference would hand
// to its tracker thread and then counts as "tracked".
//
// With -t N the whole LTE-Tracker loop runs: every 10000-sample block goes to both the framer and the cell tracker
// (lcs_track_*, the tracker threads of src/tracker_thread.cpp), the framer and the searcher use the tracker's frequency
// offset (global_thread_data.frequency_offset(), moved by every cell's FOE), new cells are handed to the tracker, the
// tracker's live cells are the searcher's skip list (so a dropped cell can be found again), and every N frames one status
// line per cell is printed (id, ports, frame timing, offset, CRS SNR per port, MIB health as in display_thread.cpp:124),
// plus a line for every dropped cell.
//
// Like LTE-Tracker's main (src/LTE-Tracker.cpp:795-798) it first calibrates the oscillator with kalibrate
// (src/LTE-Tracker.cpp:565-741, lcs_kalibrate_cu8) on the first 153600 samples of the stream unless -o gives the offset.
//
//   StreamSearch_b200 -f <fc Hz> [-o <frequency offset Hz>] [-p <ppm>] [-c <correction>] [-n <max cycles>]
//                     [-t <status every N frames>] stream.bin
#include <getopt.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../include/lcs_b200.h"

// The full tracker loop (-t): see the header comment.
static int run_tracking(lcs_ctx* ctx, FILE* fp, double fc, double fc_programmed, double fs_programmed, uint32_t n_cap,
                        double f_off, long max_cycles, long status_frames) {
  const uint32_t max_cells = 16;
  lcs_framer* fr = nullptr;
  lcs_track* tr = nullptr;
  if (lcs_framer_create(fc, fc_programmed, fs_programmed, n_cap, &fr) != LCS_OK) { fprintf(stderr, "Error: framer\n"); return -1; }
  if (lcs_track_create(ctx, 1, &fc, &fc_programmed, fs_programmed, &f_off, max_cells, &tr) != LCS_OK) {
    fprintf(stderr, "Error: %s\n", lcs_last_error(ctx));
    return -1;
  }
  std::vector<uint8_t> block(2 * 10000);
  std::vector<lcs_track_cell> live(max_cells);
  std::vector<int32_t> tracked;
  long cycles = 0, samples = 0, next_status = status_frames * 19200;
  bool searching = true;
  lcs_framer_request(fr);
  for (;;) {
    const size_t n = fread(block.data(), 2, 10000, fp);
    if (n == 0) break;
    double fo = 0;
    if (lcs_track_frequency_offset(tr, &fo) != LCS_OK) { fprintf(stderr, "Error: %s\n", lcs_last_error(ctx)); return -1; }
    int ready = 0;
    const uint8_t* cap = nullptr;
    double late = 0;
    if (lcs_framer_push(fr, block.data(), (uint32_t)n, fo, &ready, &cap, &late) != LCS_OK ||
        lcs_track_push_cu8(tr, block.data(), (uint32_t)n) != LCS_OK) {
      fprintf(stderr, "Error: %s\n", lcs_last_error(ctx));
      return -1;
    }
    samples += (long)n;
    uint32_t n_live = 0;
    if (lcs_track_read(tr, 0, live.data(), max_cells, &n_live) != LCS_OK) { fprintf(stderr, "Error: %s\n", lcs_last_error(ctx)); return -1; }
    tracked.clear();
    for (uint32_t i = 0; i < n_live; i++) {
      const lcs_track_cell& t = live[i];
      if (t.dropped) printf("dropped cell %d at sample %lld after %lld MIB attempts\n", t.n_id_cell, (long long)t.drop_sample, (long long)t.mib_attempts);
      else tracked.push_back(t.n_id_cell);                                     // searcher_thread.cpp:153-174
    }
    if (lcs_track_frequency_offset(tr, &fo) != LCS_OK) { fprintf(stderr, "Error: %s\n", lcs_last_error(ctx)); return -1; }
    if (status_frames > 0 && samples >= next_status) {
      next_status += status_frames * 19200;
      printf("time %.3f s  frequency offset %.3f Hz  %zu cell(s)\n", samples / fs_programmed, fo, tracked.size());
      for (uint32_t i = 0; i < n_live; i++) {
        const lcs_track_cell& t = live[i];
        if (t.dropped) continue;
        printf("  cell %3d  ports %d  frame timing %9.3f  CRS SNR", t.n_id_cell, t.n_ports, t.frame_timing);
        for (int p = 0; p < t.n_ports; p++) printf(" %5.1f", 10 * std::log10(t.crs_sp_raw_av[p] / t.crs_np_av[p]));
        printf(" dB  MIB %lld/%lld  failures %.2f\n", (long long)t.mib_successes, (long long)t.mib_attempts, t.mib_decode_failures);
      }
    }
    if (!searching || !ready) continue;
    lcs_cell cells[16];
    double timing[16];
    uint32_t found = 0;
    if (lcs_tracker_search_cu8(ctx, cap, n_cap, fo, fc, fc_programmed, fs_programmed, late, tracked.data(), (uint32_t)tracked.size(),
                               cells, timing, 16, &found) != LCS_OK) {
      fprintf(stderr, "Error: %s\n", lcs_last_error(ctx));
      return -1;
    }
    printf("cycle %ld: searched at tracker offset %.3f Hz\n", cycles, fo);
    for (uint32_t i = 0; i < found && i < 16; i++) {
      const int id = cells[i].n_id_2 + 3 * cells[i].n_id_1;
      const double ft = timing[i] - 19200.0 * std::floor(timing[i] / 19200.0);
      printf("cycle %ld: new cell %d  ports %d  n_rb_dl %d  sfn %d  frame timing %.3f\n", cycles, id, cells[i].n_ports, cells[i].n_rb_dl,
             cells[i].sfn, ft);
      if (lcs_track_add_cell(tr, 0, &cells[i], ft) != LCS_OK) printf("cycle %ld: cell %d not tracked: %s\n", cycles, id, lcs_last_error(ctx));
    }
    cycles++;
    if (max_cycles >= 0 && cycles >= max_cycles) searching = false;          // keep tracking, stop searching
    else lcs_framer_request(fr);
  }
  printf("%ld searcher cycle(s), %zu cell(s) being tracked\n", cycles, tracked.size());
  lcs_track_destroy(tr);
  lcs_framer_destroy(fr);
  return 0;
}

int main(int argc, char** argv) {
  double fc = -1, f_off = 0, correction = 1, ppm = 120;
  bool have_off = false;
  long max_cycles = -1, status_frames = -1;
  int c;
  while ((c = getopt(argc, argv, "f:o:c:n:p:t:h")) != -1) {
    switch (c) {
      case 'f': fc = strtod(optarg, nullptr); break;
      case 'o': f_off = strtod(optarg, nullptr); have_off = true; break;
      case 'p': ppm = strtod(optarg, nullptr); break;
      case 'c': correction = strtod(optarg, nullptr); break;
      case 'n': max_cycles = strtol(optarg, nullptr, 10); break;
      case 't': status_frames = strtol(optarg, nullptr, 10); break;
      default:
        fprintf(stderr, "usage: %s -f <fc Hz> [-o <offset Hz>] [-p <ppm>] [-c <correction>] [-n <max cycles>] [-t <status frames>] stream.bin\n", argv[0]);
        return c == 'h' ? 0 : -1;
    }
  }
  if (fc <= 0 || optind >= argc) {
    fprintf(stderr, "usage: %s -f <fc Hz> [-o <offset Hz>] [-p <ppm>] [-c <correction>] [-n <max cycles>] [-t <status frames>] stream.bin\n", argv[0]);
    return -1;
  }
  FILE* fp = fopen(argv[optind], "rb");
  if (!fp) { perror(argv[optind]); return -1; }
  const double fs_programmed = 1.92e6 * correction, fc_programmed = fc;          // LTE-Tracker.cpp:791,609
  const uint32_t n_cap = 19200 * 8;                                              // LTE-Tracker.cpp:819
  lcs_ctx* ctx = nullptr;
  if (lcs_ctx_create(0, &ctx) != LCS_OK) { fprintf(stderr, "Error: %s\n", lcs_last_error(nullptr)); return -1; }
  if (!have_off) {
    // kalibrate: "similar to running CellSearch with only one center frequency; all information is discarded except for
    // the frequency offset" (LTE-Tracker.cpp:793-798)
    std::vector<uint8_t> first((size_t)n_cap * 2);
    if (fread(first.data(), 2, n_cap, fp) != n_cap) { fprintf(stderr, "Error: not enough data in file!\n"); return -1; }
    rewind(fp);
    lcs_cell best;
    double resid = 1;
    uint32_t n_found = 0;
    printf("Calibrating local oscillator.\n");
    if (lcs_kalibrate_cu8(ctx, first.data(), n_cap, fc, fc_programmed, fs_programmed, ppm, correction, &best, &resid, &n_found) != LCS_OK) {
      fprintf(stderr, "Error: %s\n", lcs_last_error(ctx));
      return -1;
    }
    if (!n_found) { printf("Calibration failed (no cells detected).\n"); return 1; }
    printf("Calibration succeeded!\n   Residual frequency offset: %g Hz\n   New correction factor: %.20g\n", best.freq_superfine, resid);
    f_off = best.freq_superfine;                                                 // global_thread_data.frequency_offset(initial_freq_offset)
  }
  if (status_frames >= 0) {
    const int rc = run_tracking(ctx, fp, fc, fc_programmed, fs_programmed, n_cap, f_off, max_cycles, status_frames);
    lcs_ctx_destroy(ctx);
    fclose(fp);
    return rc;
  }
  lcs_framer* fr = nullptr;
  if (lcs_framer_create(fc, fc_programmed, fs_programmed, n_cap, &fr) != LCS_OK) { fprintf(stderr, "Error: framer\n"); return -1; }
  std::vector<uint8_t> block(2 * 10000);                                         // BLOCK_SIZE, producer_thread.cpp:95
  std::vector<int32_t> tracked;
  long cycles = 0;
  lcs_framer_request(fr);                                                        // searcher_thread.cpp:88
  for (;;) {
    const size_t n = fread(block.data(), 2, 10000, fp);
    if (n == 0) break;
    int ready = 0;
    const uint8_t* cap = nullptr;
    double late = 0;
    if (lcs_framer_push(fr, block.data(), (uint32_t)n, f_off, &ready, &cap, &late) != LCS_OK) { fprintf(stderr, "Error: framer push\n"); return -1; }
    if (!ready) continue;
    lcs_cell cells[16];
    double timing[16];
    uint32_t found = 0;
    if (lcs_tracker_search_cu8(ctx, cap, n_cap, f_off, fc, fc_programmed, fs_programmed, late, tracked.data(), (uint32_t)tracked.size(),
                               cells, timing, 16, &found) != LCS_OK) {
      fprintf(stderr, "Error: %s\n", lcs_last_error(ctx));
      return -1;
    }
    for (uint32_t i = 0; i < found && i < 16; i++) {
      const int id = cells[i].n_id_2 + 3 * cells[i].n_id_1;
      printf("cycle %ld: new cell %d  ports %d  n_rb_dl %d  sfn %d  residual offset %.1f Hz  frame timing %.3f (late %.3f)\n", cycles, id,
             cells[i].n_ports, cells[i].n_rb_dl, cells[i].sfn, cells[i].freq_superfine, timing[i], late);
      tracked.push_back(id);                                                     // searcher_thread.cpp:153-174, 222
    }
    cycles++;
    if (max_cycles >= 0 && cycles >= max_cycles) break;
    lcs_framer_request(fr);
  }
  printf("%ld searcher cycle(s), %zu cell(s) being tracked\n", cycles, tracked.size());
  lcs_framer_destroy(fr);
  lcs_ctx_destroy(ctx);
  fclose(fp);
  return 0;
}
