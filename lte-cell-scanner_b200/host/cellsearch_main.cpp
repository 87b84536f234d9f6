// cellsearch_main.cpp - the CellSearch command line (reference src/CellSearch.cpp) on top of the
// GPU drop-in: same flags (-s -e -p -c -r -l -d -i -v -b -h, CellSearch.cpp:117-130), same
// per-centre-frequency loop (:471-569), same result table (:576-614).  Capture buffers come from
// recorded files (-l, capbuf_NNNN.it, src/capbuf.cpp:98-115) or raw rtl_sdr byte dumps
// (capbuf_NNNN.bin, --raw); live rtl-sdr capture is out of scope (no radio, no librtlsdr here).
//
// `CellSearch -l` at the reference's HEAD reads fs_programmed/fc_programmed uninitialised
// (CellSearch.cpp:456-458,480); this program defines them the way LTE-Tracker does:
// fs_programmed = 1.92e6*correction, fc_programmed = fc_requested (LTE-Tracker.cpp:791,609).
#include <getopt.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <iomanip>
#include <iostream>
#include <sstream>

#include "it_file_min.hpp"
#include "searcher_dropin.hpp"

using namespace std;
using namespace itpp;

static int verbosity = 1;

static void print_usage() {
  cout << "LTE CellSearch (GPU drop-in) help" << endl << endl;
  cout << "CellSearch -s start_frequency [optional_parameters]" << endl << endl;
  cout << "  -h --help                      print this help screen" << endl;
  cout << "  -v --verbose                   increase status messages from program" << endl;
  cout << "  -b --brief                     reduce status messages from program" << endl;
  cout << "  -s --freq-start fs             frequency where cell search should start" << endl;
  cout << "  -e --freq-end fe               frequency where cell search should end" << endl;
  cout << "  -p --ppm ppm                   crystal remaining PPM error (default 120)" << endl;
  cout << "  -c --correction c              crystal correction factor" << endl;
  cout << "  -l --load                      read captured data from capbuf_XXXX.it files" << endl;
  cout << "  -d --data-dir dir              directory of the capbuf_XXXX.it files" << endl;
  cout << "     --raw                       with -l: read capbuf_XXXX.bin raw rtl_sdr byte dumps instead" << endl;
  cout << "     --sweep                     with -l --raw: all centre frequencies in one batched call (lcs_sweep_search_cu8)" << endl;
  cout << "     --wideband FILE             search every 100 kHz raster point in [fs, fe] in one wideband recording: raw" << endl;
  cout << "                                 little-endian int16 I/Q (ci16, no header), channelized on the GPU" << endl;
  cout << "     --fs-in FS                  with --wideband: the recording's sample rate, D * 1.92 MHz with D in [2, 64]" << endl;
  cout << "     --fc-in FC                  with --wideband: the recording's centre frequency" << endl;
  cout << "     --resample                  with --wideband: resample by up/down to 1.92 Msps, so that --fs-in may be any" << endl;
  cout << "                                 integer number of Hz in (1.92, 122.88] MHz with fs-in/1.92 MHz = down/up," << endl;
  cout << "                                 up <= 128, down <= 640 (e.g. 2.048, 2.4, 2.5, 6, 10, 20, 25, 56, 100 Msps)" << endl;
  cout << "     --format F                  with --resample: the recording's sample format, ci16 (default), cs8 (HackRF)," << endl;
  cout << "                                 cu8 (rtl_sdr) or cf32 (GNU Radio, SigMF cf32_le)" << endl;
  cout << "     --spectrum OUT.csv          with --wideband: Welch power spectrum of the WHOLE recording (periodic Hann," << endl;
  cout << "                                 50 % overlap) written as freq_hz,psd_dbfs_per_hz lines; with a search the cell" << endl;
  cout << "                                 table gains each cell's carrier power in dBFS over n_rb_dl * 180 kHz.  -s may" << endl;
  cout << "                                 then be omitted (no search), and --fs-in may be any integer number of Hz up to" << endl;
  cout << "                                 250 MHz and --format any of the four without --resample" << endl;
  cout << "     --nfft N                    with --spectrum: FFT length, a power of two in [64, 65536] (default 4096)" << endl;
  cout << "     --measure                   add RSRP[dBFS] RSRQ[dB] SINR[dB] columns (antenna port 0) to the cell table," << endl;
  cout << "                                 measured on the GPU from the CRS of each cell's central 6 RBs over 60 ms of the" << endl;
  cout << "                                 capture (with --wideband, RSRP in the recording's full scale)" << endl;
  cout << "     --measure-carrier           with --wideband: add RSRPc[dBFS] RSRQc[dB] SINRc[dB] columns (antenna port 0)," << endl;
  cout << "                                 measured on the GPU from the CRS of all n_rb_dl RBs of each cell, taken from the" << endl;
  cout << "                                 recording itself; --fs-in must be D * 1.92 MHz with D in {2, 4, 8, 16, 32}.  A" << endl;
  cout << "                                 cell whose carrier the recording does not hold whole shows -" << endl;
  cout << "     --carrier-csv OUT.csv       with --measure-carrier: one line per cell, port and RB," << endl;
  cout << "                                 n_id_cell,fc_hz,port,rb,rsrp_dbfs,noise_dbfs,rssi_dbfs (- for a power <= 0:" << endl;
  cout << "                                 an RB's noise estimate can come out zero or negative at high SNR)" << endl;
  cout << "     --cir                       with --wideband: add TOA[us] DS[ns] columns, the arrival of each cell's frame" << endl;
  cout << "                                 (its first path, modulo 10 ms, from the recording's first sample) and the RMS" << endl;
  cout << "                                 delay spread of antenna port 0, from the power delay profile of all n_rb_dl RBs" << endl;
  cout << "                                 of the cell, taken from the recording itself; --fs-in as for --measure-carrier." << endl;
  cout << "                                 A cell whose carrier the recording does not hold whole shows -" << endl;
  cout << "     --cir-csv OUT.csv           with --cir: the power delay profile, one line per cell, port and delay tap," << endl;
  cout << "                                 n_id_cell,fc_hz,port,delay_ns,pdp_dbfs (- for a power <= 0)" << endl;
  cout << "     --cfi                       with --wideband: add a CFI column, the control format indicator each cell sends" << endl;
  cout << "                                 most often, decoded from its PCFICH in every subframe over all n_rb_dl RBs," << endl;
  cout << "                                 taken from the recording itself; --fs-in as for --measure-carrier.  A cell whose" << endl;
  cout << "                                 carrier the recording does not hold whole shows -" << endl;
  cout << "     --cfi-csv OUT.csv           with --cfi: one line per cell and subframe," << endl;
  cout << "                                 n_id_cell,fc_hz,subframe,cfi,metric1,metric2,metric3,sinr_db" << endl;
  cout << "     --pdcch                     with --wideband: add an SI column, the number of System Information DCIs" << endl;
  cout << "                                 (SI-RNTI) decoded from each cell's PDCCH common search space in every subframe" << endl;
  cout << "                                 over all n_rb_dl RBs, taken from the recording itself; --fs-in as for" << endl;
  cout << "                                 --measure-carrier.  A cell whose carrier the recording does not hold whole shows -" << endl;
  cout << "     --pdcch-csv OUT.csv         with --pdcch: one line per decoded DCI (SI-, P- and RA-RNTI, formats 1A and 1C)," << endl;
  cout << "                                 n_id_cell,fc_hz,subframe,cfi,format,agg,cce,rnti,n_bits,payload_hex,quality," << endl;
  cout << "                                 rb_start,n_rb,mcs,rv (- for a field the format does not have)" << endl;
  cout << "     --sib1                      with --wideband: add PLMN (the first MCC-MNC), TAC and CID columns, decoded from" << endl;
  cout << "                                 each cell's SIB1 on the PDSCH of its SIB1 occasions, with the SFN of its MIB;" << endl;
  cout << "                                 --fs-in as for --measure-carrier.  A cell whose SIB1 did not decode shows - - -" << endl;
  cout << "     --sib1-csv OUT.csv          with --sib1: one line per SIB1 occasion, n_id_cell,fc_hz,subframe,sfn,format," << endl;
  cout << "                                 rb_start,n_rb,tbs,rv,crc_ok,iterations,sinr_db,tb_hex (- where nothing was found)" << endl;
  cout << "  -r --record / -i --device-index need a live rtl-sdr dongle: not supported by this build" << endl;
}

static string freq_formatter(const double& freq) {   // CellSearch.cpp:322-341
  stringstream temp;
  if (abs(freq) < 998.0) temp << setw(5) << setprecision(3) << freq << "h";
  else if (abs(freq) < 998000.0) temp << setw(5) << setprecision(3) << freq / 1e3 << "k";
  else if (abs(freq) < 998000000.0) temp << setw(5) << setprecision(3) << freq / 1e6 << "m";
  else if (abs(freq) < 998000000000.0) temp << setw(5) << setprecision(3) << freq / 1e9 << "g";
  else if (abs(freq) < 998000000000000.0) temp << setw(5) << setprecision(3) << freq / 1e12 << "t";
  else temp << freq;
  return temp.str();
}

// ---- --spectrum ----------------------------------------------------------------------------------------------------------
// The checks of --spectrum that need no device: rate, --fc-in and a readable recording.
static bool spectrum_args(const string& wideband, double fs_in, double fc_in) {
  if (!(fs_in > 0 && fs_in <= 250e6) || std::fabs(fs_in - std::round(fs_in)) > 1e-6) {
    cerr << "Error: --spectrum needs --fs-in, an integer number of Hz in (0, 250] MHz" << endl;
    return false;
  }
  if (fc_in <= 0) { cerr << "Error: --wideband needs --fc-in" << endl; return false; }
  FILE* f = std::fopen(wideband.c_str(), "rb");
  if (!f) { cerr << "Error: cannot read " << wideband << endl; return false; }
  std::fclose(f);
  return true;
}

static FILE* open_output(const string& path) {
  FILE* f = std::fopen(path.c_str(), "w");
  if (!f) cerr << "Error: cannot write " << path << endl;
  return f;
}

// Welch PSD of the whole recording (wideband_psd), written to `out` as freq_hz,psd_dbfs_per_hz lines; psd is kept for the
// carrier-power column.
static void write_spectrum(const string& wideband, int fmt, size_t bytes, double fs_in, double fc_in, uint32_t nfft,
                           const string& path, FILE* out, vector<double>& psd) {
  uint64_t n_seg = 0;
  try {
    wideband_psd(wideband, fmt, bytes, fs_in, nfft, psd, n_seg);
  } catch (const char*) {
    std::fclose(out);
    throw;
  }
  std::fprintf(out, "freq_hz,psd_dbfs_per_hz\n");
  for (uint32_t i = 0; i < nfft; i++)
    std::fprintf(out, "%.17g,%.17g\n", fc_in + ((double)i - nfft / 2) * (fs_in / nfft), 10 * std::log10(psd[i]));
  const bool ok = std::fclose(out) == 0;
  if (!ok) throw("cannot write the spectrum file");
  if (verbosity >= 1)
    cout << "Power spectrum of " << wideband << " (" << n_seg << " segments of " << nfft << " samples) written to " << path << endl;
}

// The measurement of a final (deduplicated) cell: that of the detected cell it was copied from, in the list of its
// centre frequency.
static const lcs_cell_meas* measurement_of(const Cell& c, double freq_start, const vector<list<Cell> >& detected,
                                           const vector<vector<lcs_cell_meas> >& meas) {
  const long fci = std::lround((c.fc_requested - freq_start) / 100e3);
  if (fci < 0 || fci >= (long)detected.size() || fci >= (long)meas.size()) return nullptr;
  size_t k = 0;
  for (list<Cell>::const_iterator it = detected[fci].begin(); it != detected[fci].end(); ++it, ++k)
    if (it->n_id_cell() == c.n_id_cell() && it->frame_start == c.frame_start && it->freq_superfine == c.freq_superfine &&
        k < meas[fci].size())
      return &meas[fci][k];
  return nullptr;
}

// A power as dB for the carrier CSV, or "-" when it is not positive: an RB's noise is the difference of two near-equal
// sums and can come out zero or negative at high SNR.
static string csv_db(double v) {
  if (!(v > 0)) return "-";
  char b[32];
  std::snprintf(b, sizeof(b), "%.17g", 10 * std::log10(v));
  return b;
}

// 10 log10 of the power in the bins whose centre lies within n_rb_dl * 90 kHz of the cell's carrier fc_requested +
// freq_superfine, in full-scale^2 (dBFS).
static double carrier_power_dbfs(const vector<double>& psd, double fs_in, double fc_in, const Cell& c) {
  const size_t N = psd.size();
  const double fc = c.fc_requested + c.freq_superfine, half = 90e3 * (int)c.n_rb_dl, df = fs_in / N;
  double p = 0;
  for (size_t i = 0; i < N; i++) {
    const double f = fc_in + ((double)i - (double)(N / 2)) * df;
    if (f >= fc - half && f <= fc + half) p += psd[i] * df;
  }
  return 10 * std::log10(p);
}

int main(int argc, char* const argv[]) {
  double freq_start = -1, freq_end = -1, ppm = 120, correction = 1;
  bool save_cap = false, use_recorded_data = false, raw = false, batched = false;
  string data_dir = ".", wideband, format = "ci16";
  double fs_in = -1, fc_in = -1;
  bool resample = false, measure = false, measure_carrier = false, cir = false, cfi = false, pdcch = false, sib1 = false;
  string spectrum, carrier_csv, cir_csv, cfi_csv, pdcch_csv, sib1_csv;
  long nfft = 4096;
  static struct option long_options[] = {
      {"help", no_argument, 0, 'h'},          {"verbose", no_argument, 0, 'v'},       {"brief", no_argument, 0, 'b'},
      {"freq-start", required_argument, 0, 's'}, {"freq-end", required_argument, 0, 'e'}, {"ppm", required_argument, 0, 'p'},
      {"correction", required_argument, 0, 'c'}, {"record", no_argument, 0, 'r'},        {"load", no_argument, 0, 'l'},
      {"data-dir", required_argument, 0, 'd'},   {"device-index", required_argument, 0, 'i'}, {"raw", no_argument, 0, 'R'}, {"sweep", no_argument, 0, 'W'},
      {"wideband", required_argument, 0, 'B'},   {"fs-in", required_argument, 0, 'F'},   {"fc-in", required_argument, 0, 'C'},
      {"resample", no_argument, 0, 'S'},         {"format", required_argument, 0, 'T'},
      {"spectrum", required_argument, 0, 'P'},   {"nfft", required_argument, 0, 'N'},   {"measure", no_argument, 0, 'M'},
      {"measure-carrier", no_argument, 0, 'K'}, {"carrier-csv", required_argument, 0, 'V'},
      {"cir", no_argument, 0, 'X'},             {"cir-csv", required_argument, 0, 'Y'},
      {"cfi", no_argument, 0, 'Q'},             {"cfi-csv", required_argument, 0, 'Z'},
      {"pdcch", no_argument, 0, 'H'},           {"pdcch-csv", required_argument, 0, 'J'},
      {"sib1", no_argument, 0, 'U'},            {"sib1-csv", required_argument, 0, 'G'},
      {0, 0, 0, 0}};
  for (;;) {
    int idx = 0;
    int c = getopt_long(argc, argv, "hvbs:e:p:c:rld:i:", long_options, &idx);
    if (c == -1) break;
    char* endp;
    switch (c) {
      case 'h': print_usage(); return -1;
      case 'v': verbosity = 2; break;
      case 'b': verbosity = 0; break;
      case 's': freq_start = strtod(optarg, &endp); if (optarg == endp || *endp) { cerr << "Error: could not parse start frequency" << endl; return -1; } break;
      case 'e': freq_end = strtod(optarg, &endp); if (optarg == endp || *endp) { cerr << "Error: could not parse end frequency" << endl; return -1; } break;
      case 'p': ppm = strtod(optarg, &endp); if (optarg == endp || *endp) { cerr << "Error: could not parse ppm value" << endl; return -1; } break;
      case 'c': correction = strtod(optarg, &endp); if (optarg == endp || *endp) { cerr << "Error: could not parse correction factor" << endl; return -1; } break;
      case 'r': save_cap = true; break;
      case 'l': use_recorded_data = true; break;
      case 'd': data_dir = optarg; break;
      case 'R': raw = true; break;
      case 'W': batched = true; break;
      case 'B': wideband = optarg; break;
      case 'F': fs_in = strtod(optarg, &endp); if (optarg == endp || *endp) { cerr << "Error: could not parse --fs-in" << endl; return -1; } break;
      case 'C': fc_in = strtod(optarg, &endp); if (optarg == endp || *endp) { cerr << "Error: could not parse --fc-in" << endl; return -1; } break;
      case 'S': resample = true; break;
      case 'T': format = optarg; break;
      case 'P': spectrum = optarg; break;
      case 'N': nfft = strtol(optarg, &endp, 10); if (optarg == endp || *endp) { cerr << "Error: could not parse --nfft" << endl; return -1; } break;
      case 'M': measure = true; break;
      case 'K': measure_carrier = true; break;
      case 'V': carrier_csv = optarg; break;
      case 'X': cir = true; break;
      case 'Y': cir_csv = optarg; break;
      case 'Q': cfi = true; break;
      case 'Z': cfi_csv = optarg; break;
      case 'H': pdcch = true; break;
      case 'J': pdcch_csv = optarg; break;
      case 'U': sib1 = true; break;
      case 'G': sib1_csv = optarg; break;
      case 'i': break;
      default: return -1;
    }
  }
  if (optind < argc) { cerr << "Error: unknown/extra arguments specified on command line" << endl; return -1; }
  const bool spec = !spectrum.empty(), search = !spec || freq_start != -1;   // --spectrum alone: no search
  if (spec && wideband.empty()) { cerr << "Error: --spectrum needs --wideband" << endl; return -1; }
  if (measure && !search) { cerr << "Error: --measure needs a search (-s)" << endl; return -1; }
  if (!carrier_csv.empty() && !measure_carrier) { cerr << "Error: --carrier-csv needs --measure-carrier" << endl; return -1; }
  if (measure_carrier && wideband.empty()) { cerr << "Error: --measure-carrier needs --wideband" << endl; return -1; }
  if (measure_carrier && !search) { cerr << "Error: --measure-carrier needs a search (-s)" << endl; return -1; }
  if (!cir_csv.empty() && !cir) { cerr << "Error: --cir-csv needs --cir" << endl; return -1; }
  if (cir && wideband.empty()) { cerr << "Error: --cir needs --wideband" << endl; return -1; }
  if (cir && !search) { cerr << "Error: --cir needs a search (-s)" << endl; return -1; }
  if (!cfi_csv.empty() && !cfi) { cerr << "Error: --cfi-csv needs --cfi" << endl; return -1; }
  if (cfi && wideband.empty()) { cerr << "Error: --cfi needs --wideband" << endl; return -1; }
  if (cfi && !search) { cerr << "Error: --cfi needs a search (-s)" << endl; return -1; }
  if (!pdcch_csv.empty() && !pdcch) { cerr << "Error: --pdcch-csv needs --pdcch" << endl; return -1; }
  if (pdcch && wideband.empty()) { cerr << "Error: --pdcch needs --wideband" << endl; return -1; }
  if (pdcch && !search) { cerr << "Error: --pdcch needs a search (-s)" << endl; return -1; }
  if (!sib1_csv.empty() && !sib1) { cerr << "Error: --sib1-csv needs --sib1" << endl; return -1; }
  if (sib1 && wideband.empty()) { cerr << "Error: --sib1 needs --wideband" << endl; return -1; }
  if (sib1 && !search) { cerr << "Error: --sib1 needs a search (-s)" << endl; return -1; }
  if (nfft < 64 || nfft > 65536 || (nfft & (nfft - 1))) { cerr << "Error: --nfft must be a power of two in [64, 65536]" << endl; return -1; }
  const bool wide = !wideband.empty();
  int wide_format = LCS_IQ_CI16;   // --format, for the spectrum and the search
  size_t wide_bytes = 4;           // per sample
  if (wide) {
    if (format == "cs8") { wide_format = LCS_IQ_CS8; wide_bytes = 2; }
    else if (format == "cu8") { wide_format = LCS_IQ_CU8; wide_bytes = 2; }
    else if (format == "cf32") { wide_format = LCS_IQ_CF32; wide_bytes = 8; }
    else if (format != "ci16") { cerr << "Error: --format must be ci16, cs8, cu8 or cf32" << endl; return -1; }
  }
  FILE* spec_file = nullptr;
  vector<double> psd;
  if (spec && !spectrum_args(wideband, fs_in, fc_in)) return -1;
  if (!search) {
    if (!(spec_file = open_output(spectrum))) return -1;
    try {
      write_spectrum(wideband, wide_format, wide_bytes, fs_in, fc_in, (uint32_t)nfft, spectrum, spec_file, psd);
    } catch (const char* msg) {
      cerr << "Error: " << msg << endl;
      return -1;
    }
    return 0;
  }
  if (freq_start == -1) { cerr << "Error: must specify a start frequency. (Try --help)" << endl; return -1; }
  if (freq_start < 1e6) { cerr << "Error: start frequency must be greater than 1MHz" << endl; return -1; }
  if (freq_start / 100e3 != std::round(freq_start / 100e3)) {
    freq_start = std::round(freq_start / 100e3) * 100e3;
    cout << "Warning: start frequency has been rounded to the nearest multiple of 100kHz" << endl;
  }
  if (freq_end == -1) freq_end = freq_start;
  if (freq_end < freq_start) { cerr << "Error: end frequency must be >= start frequency" << endl; return -1; }
  if (freq_end / 100e3 != std::round(freq_end / 100e3)) {
    freq_end = std::round(freq_end / 100e3) * 100e3;
    cout << "Warning: end frequency has been rounded to the nearest multiple of 100kHz" << endl;
  }
  if (ppm < 0) { cerr << "Error: ppm value must be positive" << endl; return -1; }
  if (ppm > 200) cout << "Warning: ppm value appears to be set unreasonably high" << endl;
  if (abs(correction - 1) > 1000e-6) cout << "Warning: crystal correction factor appears to be unreasonable" << endl;
  if (save_cap || (!use_recorded_data && !wide)) {
    cerr << "Error: live capture / recording needs an rtl-sdr dongle, which this build does not support; use -l or --wideband" << endl;
    return -1;
  }
  // wideband recording: every argument and the file length are checked before any device work
  vector<unsigned char> wide_iq;
  uint32_t wide_n = 0;
  if (wide) {
    if (use_recorded_data || batched) { cerr << "Error: --wideband cannot be combined with -l or --sweep" << endl; return -1; }
    if (fc_in <= 0) { cerr << "Error: --wideband needs --fc-in" << endl; return -1; }
    if (!resample && wide_format != LCS_IQ_CI16) { cerr << "Error: --format needs --resample" << endl; return -1; }
    uint32_t n_taps = 0, up = 1, down = 1;
    if (resample) {
      if (lcs_chan_design_rational(fs_in, &up, &down, nullptr, &n_taps) != LCS_OK) {
        cerr << "Error: --fs-in must be an integer number of Hz in (1.92, 122.88] MHz with fs-in / 1.92 MHz = down / up, "
                "up <= 128 and down <= 640" << endl;
        return -1;
      }
    } else if (lcs_chan_design_taps(fs_in, nullptr, &n_taps) != LCS_OK) {
      cerr << "Error: --fs-in must be D * 1.92 MHz with an integer D in [2, 64] (other rates: --resample)" << endl;
      return -1;
    } else {
      down = (uint32_t)std::lround(fs_in / 1.92e6);
    }
    if (measure_carrier || cir || cfi || pdcch || sib1) {
      const long D = std::lround(fs_in / 1.92e6);
      if (!((D == 2 || D == 4 || D == 8 || D == 16 || D == 32) && std::fabs(fs_in - D * 1.92e6) <= 1e-6)) {
        cerr << "Error: " << (measure_carrier ? "--measure-carrier" : (cir ? "--cir" : (cfi ? "--cfi" : (pdcch ? "--pdcch" : "--sib1"))))
             << " needs --fs-in = D * 1.92 MHz with D in {2, 4, 8, 16, 32}" << endl;
        return -1;
      }
    }
    const uint64_t M = (n_taps - 1) / 2;
    const int n_fc = (int)floor((freq_end - freq_start) / 100e3) + 1;                     // the raster of the search loop
    for (int fci = 0; fci < n_fc; fci++) {
      const double fc = freq_start + fci * 100e3, d = fc - fc_in;
      if (std::fabs(d - std::round(d)) > 1e-6 || std::fabs(std::round(d)) > fs_in / 2 - 960e3) {
        cerr << "Error: raster point " << setprecision(10) << fc / 1e6
             << " MHz lies outside the input band of the recording (its 1.92 MHz channel must fit in fc-in +- fs-in/2)" << endl;
        return -1;
      }
    }
    wide_n = (uint32_t)((153599ull * down + M + 1 + up - 1) / up);   // 153 600 outputs per channel
    // only the prefix the search uses is read (a recording may be far longer)
    FILE* f = std::fopen(wideband.c_str(), "rb");
    if (!f) { cerr << "Error: cannot read " << wideband << endl; return -1; }
    wide_iq.resize((size_t)wide_n * wide_bytes);
    const size_t got = std::fread(wide_iq.data(), wide_bytes, wide_n, f);
    std::fclose(f);
    if (got < wide_n) {
      cerr << "Error: " << wideband << " holds " << got << " " << format << " samples; 153600 outputs per channel need "
           << wide_n << endl;
      return -1;
    }
  }
  if (spec && !(spec_file = open_output(spectrum))) return -1;
  FILE* carrier_file = nullptr;
  if (!carrier_csv.empty() && !(carrier_file = open_output(carrier_csv))) return -1;
  FILE* cir_file = nullptr;
  if (!cir_csv.empty() && !(cir_file = open_output(cir_csv))) return -1;
  FILE* cfi_file = nullptr;
  if (!cfi_csv.empty() && !(cfi_file = open_output(cfi_csv))) return -1;
  FILE* pdcch_file = nullptr;
  if (!pdcch_csv.empty() && !(pdcch_file = open_output(pdcch_csv))) return -1;
  FILE* sib1_file = nullptr;
  if (!sib1_csv.empty() && !(sib1_file = open_output(sib1_csv))) return -1;
  if (verbosity >= 1) {
    cout << "LTE CellSearch (GPU drop-in, " << lcs_version() << ") beginning" << endl;
    if (freq_start == freq_end) cout << "  Search frequency: " << freq_start / 1e6 << " MHz" << endl;
    else cout << "  Search frequency range: " << freq_start / 1e6 << "-" << freq_end / 1e6 << " MHz" << endl;
    cout << "  PPM: " << ppm << endl;
    stringstream temp;
    temp << setprecision(20) << correction;
    cout << "  correction: " << temp.str() << endl;
    if (wide)
      cout << "  Captured data will be read from the wideband recording " << wideband << " (" << fs_in / 1e6 << " Msps at "
           << fc_in / 1e6 << " MHz)" << endl;
    else
      cout << "  Captured data will be read from capbufXXXX." << (raw ? "bin" : "it") << " files" << endl;
  }

  try {
    const double fs_programmed = 1.92e6 * correction;                                   // LTE-Tracker.cpp:791
    const uint16 n_extra = (uint16)floor((freq_start * ppm / 1e6 + 2.5e3) / 5e3);       // CellSearch.cpp:463
    vec f_search_set(2 * n_extra + 1);
    for (int i = 0; i < 2 * n_extra + 1; i++) f_search_set(i) = (i - (int)n_extra) * 5000.0;
    const int n_fc = (int)floor((freq_end - freq_start) / 100e3) + 1;                   // :465
    vector<list<Cell> > detected_cells(n_fc);
    vector<vector<lcs_cell_meas> > meas;   // --measure: meas[fci][k] of detected_cells[fci]'s k-th cell
    xcorr_pss_skip_debug_outputs(true);
    if (spec) write_spectrum(wideband, wide_format, wide_bytes, fs_in, fc_in, (uint32_t)nfft, spectrum, spec_file, psd);
    if (wide) {
      // every raster point channelized out of the one recording on the device, then the batched search in place
      vector<double> fcs;
      for (int fci = 0; fci < n_fc; fci++) fcs.push_back(freq_start + fci * 100e3);
      if (verbosity >= 1) cout << "Channelizing and examining " << n_fc << " center frequencies of one wideband recording ..." << endl;
      if (resample)
        wideband_search_rational(wide_iq.data(), wide_format, wide_n, fs_in, fc_in, fcs, f_search_set, fs_programmed,
                                 detected_cells, measure ? &meas : nullptr);
      else
        wideband_search_ci16(reinterpret_cast<const int16_t*>(wide_iq.data()), wide_n, fs_in, fc_in, fcs, f_search_set,
                             fs_programmed, detected_cells, measure ? &meas : nullptr);
    }
    if (batched) {
      // every centre frequency of the sweep in one call: the raw byte dumps are concatenated and handed to the batched
      // search (same per-channel results as the loop below, CellSearch.cpp:465-558)
      if (!raw) { cerr << "Error: --sweep needs --raw capture files" << endl; return -1; }
      vector<unsigned char> all;
      vector<double> fcs;
      uint32_t n_cap = 0;
      for (int fci = 0; fci < n_fc; fci++) {
        stringstream filename;
        filename << data_dir << "/capbuf_" << setw(4) << setfill('0') << fci << ".bin";
        vector<unsigned char> b;
        if (!lcs_it::read_all(filename.str(), b) || b.size() < 2) { cerr << "Error: cannot read " << filename.str() << endl; return -1; }
        if (fci == 0) n_cap = (uint32_t)(b.size() / 2);
        if (b.size() / 2 != n_cap) { cerr << "Error: capture buffers of a batched sweep must have equal length" << endl; return -1; }
        all.insert(all.end(), b.begin(), b.begin() + (size_t)n_cap * 2);
        fcs.push_back(freq_start + fci * 100e3);
      }
      if (verbosity >= 1) cout << "Examining " << n_fc << " center frequencies in one batched sweep ..." << endl;
      sweep_search_cu8(all, n_cap, fcs, f_search_set, fs_programmed, detected_cells);
      if (measure) measure_cells(all.data(), LCS_IQ_CU8, n_cap, detected_cells, fs_programmed, meas);
    }
    if (batched || wide) {
      if (verbosity >= 1)
        for (int fci = 0; fci < n_fc; fci++)
          for (list<Cell>::iterator it = detected_cells[fci].begin(); it != detected_cells[fci].end(); ++it) {
            cout << "  Detected a cell!" << endl;
            cout << "    cell ID: " << (*it).n_id_cell() << endl;
            cout << "    RX power level: " << 10 * log10((*it).pss_pow) << " dB" << endl;
            cout << "    residual frequency offset: " << (*it).freq_superfine << " Hz" << endl;
          }
    }
    for (int fci = 0; fci < (batched || wide ? 0 : n_fc); fci++) {
      const double fc_requested = freq_start + fci * 100e3;
      if (verbosity >= 1) cout << "Examining center frequency " << fc_requested / 1e6 << " MHz ..." << endl;
      cvec capbuf;
      const double fc_programmed = fc_requested;                                         // LTE-Tracker.cpp:609
      stringstream filename;
      filename << data_dir << "/capbuf_" << setw(4) << setfill('0') << fci << (raw ? ".bin" : ".it");
      if (verbosity >= 2) cout << "Reading captured data from file: " << filename.str() << endl;
      if (!raw) {
        int fc_file = 0;
        if (!lcs_it::read_capbuf(filename.str(), capbuf, fc_file)) { cerr << "Error: cannot read " << filename.str() << endl; return -1; }
        if (fc_requested != fc_file) {
          cout << "Warning: while reading capture buffer " << fci << ", the read" << endl;
          cout << "center frequency did not match the expected center frequency." << endl;
        }
      } else {
        vector<unsigned char> b;
        if (!lcs_it::read_all(filename.str(), b) || b.size() < 2) { cerr << "Error: cannot read " << filename.str() << endl; return -1; }
        capbuf.set_size((int)(b.size() / 2));
        for (int i = 0; i < capbuf.length(); i++)                                        // capbuf.cpp:172-175
          capbuf(i) = complex<double>((b[2 * i] - 127.0) / 128.0, (b[2 * i + 1] - 127.0) / 128.0);
      }
      const uint8 DS_COMB_ARM = 2;
      mat pow; imat frq; vf3d single, inc; vec sp_incoherent, sp; vcf3d xc; uint16 n_comb_xc, n_comb_sp;
      if (verbosity >= 2) cout << "  Calculating PSS correlations" << endl;
      xcorr_pss(capbuf, f_search_set, DS_COMB_ARM, fc_requested, fc_programmed, fs_programmed, pow, frq, single, inc,
                sp_incoherent, xc, sp, n_comb_xc, n_comb_sp);
      vec Z_th1 = calc_Z_th1(sp_incoherent, n_comb_xc, DS_COMB_ARM);                     // :500-503
      if (verbosity >= 2) cout << "  Searching for and examining correlation peaks..." << endl;
      list<Cell> peaks;
      peak_search(pow, frq, Z_th1, f_search_set, fc_requested, fc_programmed, single, DS_COMB_ARM, peaks);
      detected_cells[fci] = peaks;
      list<Cell>::iterator it = detected_cells[fci].begin();
      while (it != detected_cells[fci].end()) {
        vec a, b2; cvec c1, c2, c3, c4; mat l1, l2;
        (*it) = sss_detect((*it), capbuf, 3, fc_requested, fc_programmed, fs_programmed, a, b2, c1, c2, c3, c4, l1, l2);
        if ((*it).n_id_1 == -1) { it = detected_cells[fci].erase(it); continue; }
        (*it) = pss_sss_foe((*it), capbuf, fc_requested, fc_programmed, fs_programmed);
        cmat tfg, tfg_comp; vec ts, ts_comp;
        extract_tfg((*it), capbuf, fc_requested, fc_programmed, fs_programmed, tfg, ts);
        RS_DL rs_dl((*it).n_id_cell(), 6, (*it).cp_type);
        (*it) = tfoec((*it), tfg, ts, fc_requested, fc_programmed, rs_dl, tfg_comp, ts_comp);
        (*it) = decode_mib((*it), tfg_comp, rs_dl);
        if ((*it).n_rb_dl == -1) { it = detected_cells[fci].erase(it); continue; }
        if (verbosity >= 1) {
          cout << "  Detected a cell!" << endl;
          cout << "    cell ID: " << (*it).n_id_cell() << endl;
          cout << "    RX power level: " << 10 * log10((*it).pss_pow) << " dB" << endl;
          cout << "    residual frequency offset: " << (*it).freq_superfine << " Hz" << endl;
        }
        ++it;
      }
      if (measure) {   // this centre frequency's cells on its own capture buffer
        vector<vector<lcs_cell_meas> > m;
        measure_cells(capbuf._data(), LCS_IQ_C128, (uint32_t)capbuf.length(), vector<list<Cell> >(1, detected_cells[fci]),
                      fs_programmed, m);
        meas.resize(n_fc);
        meas[fci] = m[0];
      }
    }
    list<Cell> cells_final;
    dedup(detected_cells, cells_final);
    vector<lcs_carrier_meas> cmeas;   // --measure-carrier: that of the k-th final cell, if cok[k]
    vector<bool> cok;
    if (measure_carrier) {
      measure_carriers(wide_iq.data(), wide_format, wide_n, fs_in, fc_in, vector<Cell>(cells_final.begin(), cells_final.end()),
                       fs_programmed, cmeas, cok);
      if (carrier_file) {
        bool ok = std::fprintf(carrier_file, "n_id_cell,fc_hz,port,rb,rsrp_dbfs,noise_dbfs,rssi_dbfs\n") > 0;
        size_t k = 0;
        for (list<Cell>::iterator it = cells_final.begin(); it != cells_final.end(); ++it, ++k)
          for (int p = 0; cok[k] && p < (int)(*it).n_ports; p++)
            for (uint32_t b = 0; b < cmeas[k].n_rb; b++)
              ok = ok && std::fprintf(carrier_file, "%d,%.17g,%d,%u,%s,%s,%s\n", (int)(*it).n_id_cell(), (*it).fc_requested, p,
                                      b, csv_db(cmeas[k].rb_rsrp[p][b]).c_str(), csv_db(cmeas[k].rb_noise[p][b]).c_str(),
                                      csv_db(cmeas[k].rb_rssi[b]).c_str()) > 0;
        ok = std::fclose(carrier_file) == 0 && ok;
        if (!ok) throw("cannot write the carrier CSV file");
      }
    }
    vector<lcs_cir_meas> tmeas;   // --cir: that of the k-th final cell, if tok[k]
    vector<bool> tok;
    if (cir) {
      measure_cirs(wide_iq.data(), wide_format, wide_n, fs_in, fc_in, vector<Cell>(cells_final.begin(), cells_final.end()),
                   fs_programmed, tmeas, tok);
      if (cir_file) {
        bool ok = std::fprintf(cir_file, "n_id_cell,fc_hz,port,delay_ns,pdp_dbfs\n") > 0;
        size_t k = 0;
        for (list<Cell>::iterator it = cells_final.begin(); it != cells_final.end(); ++it, ++k)
          for (int p = 0; tok[k] && p < (int)(*it).n_ports; p++)
            for (int j = 0; j < LCS_CIR_TAPS; j++)
              ok = ok && std::fprintf(cir_file, "%d,%.17g,%d,%.17g,%s\n", (int)(*it).n_id_cell(), (*it).fc_requested, p,
                                      (j - 64) * 1e9 / 30.72e6, csv_db(tmeas[k].pdp[p][j]).c_str()) > 0;
        ok = std::fclose(cir_file) == 0 && ok;
        if (!ok) throw("cannot write the CIR CSV file");
      }
    }
    vector<lcs_pcfich_meas> fmeas;   // --cfi: that of the k-th final cell, if fok[k]
    vector<bool> fok;
    if (cfi) {
      measure_pcfich(wide_iq.data(), wide_format, wide_n, fs_in, fc_in, vector<Cell>(cells_final.begin(), cells_final.end()),
                     fs_programmed, fmeas, fok);
      if (cfi_file) {
        bool ok = std::fprintf(cfi_file, "n_id_cell,fc_hz,subframe,cfi,metric1,metric2,metric3,sinr_db\n") > 0;
        size_t k = 0;
        for (list<Cell>::iterator it = cells_final.begin(); it != cells_final.end(); ++it, ++k)
          for (int s = 0; fok[k] && s < (int)fmeas[k].n_subframes; s++) {
            const lcs_pcfich_meas& m = fmeas[k];
            ok = ok && std::fprintf(cfi_file, "%d,%.17g,%d,%u,%.17g,%.17g,%.17g,%s\n", (int)(*it).n_id_cell(), (*it).fc_requested,
                                    s, m.cfi[s], m.metric[s][0], m.metric[s][1], m.metric[s][2], csv_db(m.sinr[s]).c_str()) > 0;
          }
        ok = std::fclose(cfi_file) == 0 && ok;
        if (!ok) throw("cannot write the CFI CSV file");
      }
    }
    vector<lcs_pdcch_meas> pmeas;   // --pdcch: that of the k-th final cell, if pok[k]
    vector<bool> pok;
    if (pdcch) {
      measure_pdcch(wide_iq.data(), wide_format, wide_n, fs_in, fc_in, vector<Cell>(cells_final.begin(), cells_final.end()),
                    fs_programmed, pmeas, pok);
      if (pdcch_file) {
        bool ok = std::fprintf(pdcch_file, "n_id_cell,fc_hz,subframe,cfi,format,agg,cce,rnti,n_bits,payload_hex,quality,"
                                           "rb_start,n_rb,mcs,rv\n") > 0;
        size_t k = 0;
        for (list<Cell>::iterator it = cells_final.begin(); it != cells_final.end(); ++it, ++k)
          for (int s = 0; pok[k] && s < (int)pmeas[k].n_subframes; s++)
            for (uint32_t i = 0; i < pmeas[k].n_dci[s]; i++) {
              const lcs_pdcch_dci& d = pmeas[k].dci[s][i];
              const bool a = d.format == LCS_DCI_1A;
              const string rb = a && d.n_rb > 0 ? std::to_string(d.rb_start) + "," + std::to_string(d.n_rb) : "-,-";
              const string mr = a ? std::to_string(d.mcs) + "," + std::to_string(d.rv) : "-,-";
              ok = ok && std::fprintf(pdcch_file, "%d,%.17g,%d,%u,%s,%u,%u,%u,%u,%llx,%.17g,%s,%s\n", (int)(*it).n_id_cell(),
                                      (*it).fc_requested, s, pmeas[k].cfi[s], a ? "1A" : "1C", d.agg, d.cce, d.rnti, d.n_bits,
                                      (unsigned long long)d.payload, d.quality, rb.c_str(), mr.c_str()) > 0;
            }
        ok = std::fclose(pdcch_file) == 0 && ok;
        if (!ok) throw("cannot write the PDCCH CSV file");
      }
    }
    vector<lcs_sib1_meas> smeas;    // --sib1: that of the k-th final cell, if sok[k]
    vector<bool> sok;
    if (sib1) {
      measure_sib1(wide_iq.data(), wide_format, wide_n, fs_in, fc_in, vector<Cell>(cells_final.begin(), cells_final.end()),
                   fs_programmed, smeas, sok);
      if (sib1_file) {
        bool ok = std::fprintf(sib1_file, "n_id_cell,fc_hz,subframe,sfn,format,rb_start,n_rb,tbs,rv,crc_ok,iterations,"
                                          "sinr_db,tb_hex\n") > 0;
        size_t k = 0;
        for (list<Cell>::iterator it = cells_final.begin(); it != cells_final.end(); ++it, ++k)
          for (int o = 0; sok[k] && o < LCS_SIB1_OCCASIONS; o++) {
            const lcs_sib1_occasion& x = smeas[k].occ[o];
            string rest = "-,-,-,-,-,-,-,-,-";
            if (x.found && x.n_re) {
              string hex;
              char b[3];
              for (uint32_t i = 0; i < x.tbs / 8; i++) {
                std::snprintf(b, sizeof(b), "%02x", x.tb[i]);
                hex += b;
              }
              rest = string(x.format == LCS_DCI_1A ? "1A" : "1C") + "," + std::to_string(x.vrb_start) + "," +
                     std::to_string(x.n_vrb) + "," + std::to_string(x.tbs) + "," + std::to_string(x.rv) + "," +
                     std::to_string(x.crc_ok) + "," + std::to_string(x.iterations) + "," + csv_db(x.sinr) + "," + hex;
            } else if (x.found) {
              rest = string(x.format == LCS_DCI_1A ? "1A" : "1C") + ",-,-,-,-,-,-,-,-";
            }
            ok = ok && std::fprintf(sib1_file, "%d,%.17g,%u,%u,%s\n", (int)(*it).n_id_cell(), (*it).fc_requested, x.subframe,
                                    x.sfn, rest.c_str()) > 0;
          }
        ok = std::fclose(sib1_file) == 0 && ok;
        if (!ok) throw("cannot write the SIB1 CSV file");
      }
    }
    if (cells_final.size() == 0) {
      cout << "No LTE cells were found..." << endl;
    } else {   // CellSearch.cpp:579-613
      cout << "Detected the following cells:" << endl;
      cout << "A: #antenna ports C: CP type ; P: PHICH duration ; PR: PHICH resource type" << endl;
      cout << "CID A      fc   foff RXPWR C nRB P  PR CrystalCorrectionFactor" << (spec ? " CarrierPower[dBFS]" : "")
           << (measure ? " RSRP[dBFS] RSRQ[dB] SINR[dB]" : "") << (measure_carrier ? " RSRPc[dBFS] RSRQc[dB] SINRc[dB]" : "")
           << (cir ? " TOA[us] DS[ns]" : "") << (cfi ? " CFI" : "") << (pdcch ? " SI" : "") << (sib1 ? " PLMN TAC CID" : "") << endl;
      size_t k = 0;
      for (list<Cell>::iterator it = cells_final.begin(); it != cells_final.end(); ++it, ++k) {
        stringstream ss;
        ss << setw(3) << (*it).n_id_cell();
        ss << setw(2) << (int)(*it).n_ports;
        ss << " " << setw(6) << setprecision(5) << (*it).fc_requested / 1e6 << "M";
        ss << " " << freq_formatter((*it).freq_superfine);
        ss << " " << setw(5) << setprecision(3) << 10 * log10((*it).pss_pow);
        ss << " " << (((*it).cp_type == cp_type_t::NORMAL) ? "N" : (((*it).cp_type == cp_type_t::UNKNOWN) ? "U" : "E"));
        ss << " " << setw(3) << (int)(*it).n_rb_dl;
        ss << " " << (((*it).phich_duration == phich_duration_t::NORMAL) ? "N" : (((*it).phich_duration == phich_duration_t::UNKNOWN) ? "U" : "E"));
        switch ((*it).phich_resource) {
          case phich_resource_t::UNKNOWN: ss << " UNK"; break;
          case phich_resource_t::oneSixth: ss << " 1/6"; break;
          case phich_resource_t::half: ss << " 1/2"; break;
          case phich_resource_t::one: ss << " one"; break;
          case phich_resource_t::two: ss << " two"; break;
        }
        const double crystal_freq_actual = (*it).fc_requested - (*it).freq_superfine;
        const double correction_new = correction * ((*it).fc_requested / crystal_freq_actual);
        ss << " " << setprecision(20) << correction_new;
        if (spec) ss << " " << fixed << setprecision(2) << carrier_power_dbfs(psd, fs_in, fc_in, *it);
        if (measure) {
          const lcs_cell_meas* m = measurement_of(*it, freq_start, detected_cells, meas);
          if (!m) throw("--measure: a listed cell has no measurement");
          ss << " " << fixed << setprecision(2) << 10 * log10(m->rsrp[0]) << " " << 10 * log10(m->rsrq) << " "
             << 10 * log10(m->sinr[0]);
        }
        if (measure_carrier) {
          if (cok[k])
            ss << " " << fixed << setprecision(2) << 10 * log10(cmeas[k].rsrp[0]) << " " << 10 * log10(cmeas[k].rsrq) << " "
               << 10 * log10(cmeas[k].sinr[0]);
          else
            ss << " - - -";
        }
        if (cir) {
          if (tok[k])
            ss << " " << fixed << setprecision(3) << 1e6 * std::fmod(tmeas[k].frame_arrival, 10e-3) << " " << setprecision(1)
               << 1e9 * tmeas[k].rms_spread[0];
          else
            ss << " - -";
        }
        if (cfi) {
          if (fok[k])
            ss << " " << fmeas[k].cfi_mode;
          else
            ss << " -";
        }
        if (pdcch) {
          if (pok[k])
            ss << " " << pmeas[k].count[0];
          else
            ss << " -";
        }
        if (sib1) {
          const lcs_sib1_meas& m = smeas[k];
          if (sok[k] && m.parse_ok) {
            char plmn[32];
            std::snprintf(plmn, sizeof(plmn), "%03u-%0*u", m.plmn[0].mcc, (int)m.plmn[0].mnc_digits, m.plmn[0].mnc);
            ss << " " << plmn << " " << m.tac << " " << m.cell_identity;
          } else {
            ss << " - - -";
          }
        }
        cout << ss.str() << endl;
      }
    }
  } catch (const char* msg) {
    cerr << "Error: " << msg << endl;
    return -1;
  }
  return 0;
}
