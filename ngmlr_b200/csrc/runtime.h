// ngmlr_b200/csrc/runtime.h -- host runtime state shared by the translation units behind the C ABI
// (capi.cu: batch entry points; pipeline.cu: resident read set + the computeAlignment mirror).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <numeric>
#include <stdlib.h>
#include <mutex>
#include <thread>
#include <string>
#include <vector>

#include "../../include/ngmlr_b200.h"
#include "cigar_text.h"
#include "device_types.h"
#include "kernels.h"
#include "stream.h"

namespace nb {

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;  // elements
  // the capacity reserve(n) grows to (n > cap)
  size_t grown(size_t n) const { return borrowed ? n : std::max(n, cap + cap / 2); }
  // bytes of device memory the buffer owns
  size_t owned_bytes() const { return borrowed ? 0 : cap * sizeof(T); }
  cudaError_t reserve(size_t n, bool keep = false, cudaStream_t st = 0) {
    if (n <= cap) return cudaSuccess;
    const size_t want = grown(n);
    if (borrowed) {  // never grow (or free) somebody else's memory: start an own buffer
      p = nullptr;
      cap = 0;
      borrowed = false;
    }
    T* q = nullptr;
    cudaError_t e = cudaMalloc(&q, want * sizeof(T));
    if (e != cudaSuccess) return e;
    if (keep && p && cap) cudaMemcpyAsync(q, p, cap * sizeof(T), cudaMemcpyDeviceToDevice, st);
    if (p) {
      cudaStreamSynchronize(st);
      cudaFree(p);
    }
    p = q;
    cap = want;
    return cudaSuccess;
  }
  bool borrowed = false;  // the memory belongs to another buffer (reference / index shared between contexts)
  void release() {
    if (p && !borrowed) cudaFree(p);
    p = nullptr;
    cap = 0;
    borrowed = false;
  }
  void borrow(const DevBuf& o) {
    release();
    p = o.p;
    cap = o.cap;
    borrowed = p != nullptr;
  }
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
};

template <typename T>
struct PinBuf {
  T* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    size_t want = std::max(n, cap + cap / 2);
    T* q = nullptr;
    cudaError_t e = cudaMallocHost(&q, want * sizeof(T));
    if (e != cudaSuccess) return e;
    if (p) cudaFreeHost(p);
    p = q;
    cap = want;
    return cudaSuccess;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
  PinBuf() = default;
  PinBuf(const PinBuf&) = delete;
  PinBuf& operator=(const PinBuf&) = delete;
  ~PinBuf() { release(); }
};

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

inline double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// Host worker threads for packing and CIGAR/MD text (NGMLR_B200_HOST_THREADS overrides).
int host_threads();

// fn(i) for i in [0, n), dynamically scheduled in chunks over host_threads() threads.
template <typename F>
void parallel_for(int n, int chunk, F fn) {
  const int threads = std::min(host_threads(), (n + chunk - 1) / chunk);
  if (threads <= 1) {
    for (int i = 0; i < n; ++i) fn(i);
    return;
  }
  std::atomic<int> next(0);
  auto work = [&]() {
    for (;;) {
      const int b = next.fetch_add(chunk);
      if (b >= n) break;
      const int e = std::min(n, b + chunk);
      for (int i = b; i < e; ++i) fn(i);
    }
  };
  std::vector<std::thread> pool;
  pool.reserve(threads - 1);
  for (int t = 1; t < threads; ++t) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
}

// bytes readable past the end of every staged sequence (the fill kernel stages whole 64-column
// chunks, see convex_fill.cu) and slack of the per-warp boundary strip
constexpr size_t SEQ_PAD = 192;
constexpr size_t STRIP_SLACK = 192;

// ---- what a convex batch is made of (convex_upload_spec) -----------------------------------
// Reference windows: host text, or positions decoded on the device (DecodeRefSequenceExact).
struct RefWindows {
  const uint8_t* d_enc;
  const unsigned long long* d_ref_starts;
  int n_starts;
  const uint64_t* win_start;  // host, n entries
};
// Reads: host text, or parts of the read set resident in HBM (extractReadSeq).
struct ReadParts {
  const uint8_t* d_reads;
  const uint64_t* d_read_off;
  const int32_t* read_index;   // host, n entries each
  const int32_t* part_start;
  const uint8_t* revcomp;
};
// Corridors: CorridorLine arrays, or the closed form of the reference's builders (AlnDesc::ckind).
struct CorridorForm {
  int32_t kind, c0, cstep, width;
  float d, k, right;
};
inline int corridor_form_offset(const CorridorForm& f, int y) {
  if (f.kind == 0) return f.c0 + f.cstep * y;
  volatile float a = (float)y - f.d;  // volatile: one rounding per operation, no contraction
  volatile float b = a / f.k;
  volatile float c = b - f.right;
  return (int)c;
}
struct UploadSpec {
  int n = 0;
  const char* const* refs = nullptr;
  const RefWindows* win = nullptr;
  const int32_t* ref_lens = nullptr;
  const char* const* qrys = nullptr;
  const ReadParts* parts = nullptr;
  const int32_t* qry_lens = nullptr;
  const int32_t* corridor_offsets = nullptr;
  const int32_t* corridor_lengths = nullptr;
  const int64_t* row_start = nullptr;
  const CorridorForm* forms = nullptr;
  const int32_t* ext_qstart = nullptr;
  const int32_t* ext_qend = nullptr;
};
constexpr int TEXT_SLOTS = 6;  // pinned result arenas: one per attempt of a compute_alignments call

}  // namespace nb

struct ngmlr_b200_ctx {
  int device = 0;
  int num_sms = 0;
  int sm_ids = 0;                   // %nsmid: size of the per-SM slot table of the short-lived fill CTAs
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;   // the big-team fill launch runs beside the ordinary one
  cudaStream_t stream3 = nullptr;   // ... and so does the team launch of the ramp-free schedule's largest problems
  cudaStream_t stream_fill = nullptr;  // lowest priority: the launch of short-lived fill CTAs
  cudaEvent_t ev_fill = nullptr;
  int small_batch_big_teams = 1;    // NGMLR_B200_SMALL_BATCH_BIG_TEAMS=0: batches of <= num_sms problems keep 4-warp teams
  int fill_resident = 0;            // NGMLR_B200_FILL_RESIDENT: resident fill CTAs per SM (0 = what the kernel was tuned for)
  int fill_persistent = 0;          // NGMLR_B200_FILL_PERSISTENT=1: always the capped persistent grid
  bool sm_slots_zeroed = false;
  nb::DevBuf<unsigned int> d_sm_slots;
  cudaEvent_t ev_big = nullptr;
  cudaEvent_t ev_team = nullptr;
  cudaEvent_t ev_sync = nullptr;    // cudaEventBlockingSync: waiting host threads sleep instead of spinning
  bool spin_sync = false;           // NGMLR_B200_SPIN_SYNC=1: cudaStreamSynchronize (lowest latency, one busy CPU per waiter)
  unsigned long long big_cells = 8ull << 20;  // a problem is "big" from this many cells ...
  int big_width = 768;                        // ... in a corridor at least this wide
  int n_big = 0;                    // leading problems of the order that get FILL_BIG_TEAM-warp teams (0: no such launch)
  bool own_stream = true;
  cudaEvent_t ev[8] = {};
  nb::Scoring sc{};
  bool raw = false;  // the batch needs the RAW fill kernel: its scoring, at the magnitude its problems can reach
  int force_raw = -1;
  std::string error;

  // ---- convex batch state ----
  int n = 0;
  size_t seq_bytes = 0, rows = 0, nblocks = 0, tb_ints = 0;
  int max_len = 0;
  int max_ref_len = 0;
  int wide_problems = 0;  // problems whose corridor is >= 352 columns wide
  int force_team = -1;
  bool team_safe = true;  // every corridor of the batch is monotone with non-empty rows
  int rf_wide = 0;        // problems whose corridor is >= RF_MIN_WIDTH columns wide
  bool rf_fits = true;    // every problem's ramp-free step count fits the kernel's int step numbers
  unsigned long long rf_problems = 0;  // problems filled by the ramp-free kernels since the context was created
  unsigned long long rf2_problems = 0; // of those, by the kernel with two rows per lane
  unsigned long long rf2_skew_problems = 0;  // of those, in its skewed schedule
  // Routing counters since the context was created (ngmlr_b200_debug_fill_counts): problems filled by the
  // FILL_BIG_TEAM-warp launch, by the ramp-free schedule's concurrent launch of ramped 4-warp teams, by the ordinary
  // launch's ramped one-warp and ramped 4-warp team kernels, and by the RAW instantiation (whatever the launch); fill
  // launches, those with more than one of the three concurrent launches non-empty, and those with all three.
  unsigned long long big_team_problems = 0, rf_team_problems = 0, ramped_warp_problems = 0, ramped_team_problems = 0;
  unsigned long long raw_problems = 0, fill_launch_count = 0, multi_launch_count = 0, three_way_launch_count = 0;
  int rows_per_lane = 2;  // rows per lane of the ramp-free kernel: 1 or 2 (NGMLR_B200_FILL_ROWS_PER_LANE)
  int rf2_skew = 1;       // two rows per lane: the second row one column behind the first (NGMLR_B200_FILL_RF2_SKEW)
  int rf_team = 0;        // problems after the big ones with >= rf_team_cells cells (they lead the order)
  unsigned long long rf_team_cells = nb::RF_TEAM_CELLS;  // NGMLR_B200_RF_TEAM_CELLS
  int fill_schedule = 1;  // 1: ramp-free row schedule where it applies, 2: for every batch, 0: ramped (NGMLR_B200_FILL_SCHEDULE)
  int fill_ctas_cap = 0;  // 0 = full occupancy
  nb::PinBuf<unsigned long long> h_win;   // decode_windows: start | arena offset | (sequenceLength, span) pairs
  nb::DevBuf<unsigned long long> d_win;
  int64_t upload_d2h_bytes = 0;
  int ctas_per_sm[16] = {};  // occupancy of the fill-kernel variants (raw x team x launch_convex_fill's rampfree)
  long long debug_arena_words = -1;    // test hook: initial direction-arena size
  // Test hook (ngmlr_b200_debug_set_arena_cap, NGMLR_B200_DEBUG_ARENA_CAP): the device arenas of convex batches may
  // hold at most this many bytes (-1: no cap). A reservation beyond it fails the way cudaMalloc does when the device
  // is full ("out of memory"), without asking the driver for anything.
  long long debug_arena_cap = -1;
  size_t arena_bytes = 0;  // bytes the convex-batch device arenas hold (all of them reserve through arena_reserve)
  template <typename T>
  cudaError_t arena_reserve(nb::DevBuf<T>& b, size_t n) {
    if (n <= b.cap) return cudaSuccess;
    const size_t held = b.owned_bytes();
    if (debug_arena_cap >= 0 && arena_bytes - held + b.grown(n) * sizeof(T) > (size_t)debug_arena_cap)
      return cudaErrorMemoryAllocation;
    const cudaError_t e = b.reserve(n);
    if (e == cudaSuccess) arena_bytes += b.owned_bytes() - held;
    return e;
  }
  template <typename T>
  void arena_release(nb::DevBuf<T>& b) {
    arena_bytes -= b.owned_bytes();
    b.release();
  }
  nb::PinBuf<uint8_t> h_seq;
  nb::PinBuf<int32_t> h_coff, h_clen, h_order, h_blkbase;
  nb::PinBuf<int8_t> h_delta;
  std::vector<uint8_t> is_packed;
  int no_corridor_packing = 0;  // NGMLR_B200_NO_CORRIDOR_PACKING=1: always ship raw CorridorLines
  nb::PinBuf<nb::AlnDesc> h_desc;
  nb::PinBuf<nb::FillOut> h_fill;
  nb::PinBuf<nb::TraceOut> h_trace;
  nb::PinBuf<int32_t> h_runs;
  nb::PinBuf<unsigned long long> h_counters;
  std::vector<int32_t> ext_qs, ext_qe;
  nb::DevBuf<uint8_t> d_seq;
  nb::DevBuf<int32_t> d_coff, d_clen, d_order, d_blkbase;
  nb::DevBuf<int8_t> d_delta;
  nb::DevBuf<nb::AlnDesc> d_desc;
  nb::DevBuf<nb::BlockRec> d_blocks;
  nb::DevBuf<uint32_t> d_dir;
  nb::DevBuf<nb::BndEntry> d_bnd;
  nb::DevBuf<nb::FillOut> d_fill;
  nb::DevBuf<int32_t> d_scratch;
  nb::DevBuf<nb::TraceOut> d_trace;
  nb::DevBuf<int32_t> d_runs;
  // [0] dir_alloc, [1] runs_alloc, [2] work counter (as int), [3] big-team and [7] ramp-free team work counters,
  // [4] text_alloc, [5] peaks_alloc, [6] nm_alloc
  nb::DevBuf<unsigned long long> d_counters;
  size_t dir_words_needed = 0;
  size_t dir_words_rf = 0;  // the same for the ramp-free kernel (rows_per_lane rows per lane)
  bool ran = false;
  unsigned long long runs_used = 0, dir_used = 0;
  int fill_grid = 0;
  ngmlr_b200_batch_stats stats{};
  std::vector<nb::AlignText> texts;
  std::vector<std::vector<int32_t>> host_peaks;  // host text mode: low-identity regions per problem
  // ---- device text stage ----
  int text_mode = 0;      // 0: host threads (cigar_text.cpp, full nmPerPosition); 1: device (convex_text.cu)
  int want_nm = 0;        // device text mode: also materialise nmPerPosition (12 B per alignment column)
  int text_slot = 0;      // which pinned result arena the next fetch fills
  bool windows_mode = false, parts_mode = false, forms_mode = false, ref_on_host = true;
  size_t ref_region = 0;
  nb::DevBuf<nb::TextOut> d_textout;
  nb::DevBuf<char> d_text;
  nb::DevBuf<int4> d_peaks;
  nb::DevBuf<int32_t> d_nm;
  nb::PinBuf<nb::TextOut> h_textout;
  nb::PinBuf<char> h_text[nb::TEXT_SLOTS];
  nb::PinBuf<int4> h_peaks[nb::TEXT_SLOTS];
  nb::PinBuf<int32_t> h_nm[nb::TEXT_SLOTS];
  unsigned long long text_used = 0, peaks_used = 0, nm_used = 0;
  size_t text_cap_hint = 0;
  nb::PinBuf<unsigned char> h_aux;   // windows / read parts descriptors of the batch
  nb::DevBuf<unsigned char> d_aux;
  // ---- resident read set (pipeline.cu) ----
  nb::DevBuf<uint8_t> d_reads;
  nb::DevBuf<uint64_t> d_read_off;
  nb::DevBuf<int32_t> d_read_len;
  nb::PinBuf<uint8_t> h_reads;
  std::vector<uint64_t> read_off;
  std::vector<int32_t> read_len;
  int n_reads = 0;
  size_t reads_bytes = 0;
  int64_t reads_h2d_bytes = 0;
  // totals over the device batches of the last compute_alignments call
  int64_t ca_h2d_bytes = 0, ca_d2h_bytes = 0, ca_cells = 0;
  float ca_fill_ms = 0, ca_traceback_ms = 0, ca_text_ms = 0;
  int ca_batches = 0;
  // results of the last ngmlr_b200_map_short_reads call (short_reads.cu): records and the CIGAR / MD strings they
  // point into
  std::vector<ngmlr_b200_sam_aln> sr_alns;
  std::vector<std::string> sr_text;

  // ---- sw state ----
  nb::PinBuf<uint8_t> h_sw_seq;
  nb::PinBuf<uint64_t> h_sw_off;
  nb::PinBuf<int32_t> h_sw_len;
  nb::PinBuf<float> h_sw_out;
  nb::DevBuf<uint8_t> d_sw_seq;
  nb::DevBuf<uint64_t> d_sw_off;
  nb::DevBuf<int32_t> d_sw_len;
  nb::DevBuf<float> d_sw_out;
  nb::DevBuf<int32_t> d_sw_scratch;

  int fail(const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    error = buf;
    return -1;
  }
};

// Wait for the context's stream. By default the waiting thread SLEEPS (event with cudaEventBlockingSync): a process
// drives several contexts per GPU from as many host threads, and on the multi-GPU boxes all ranks share one CPU quota --
// spinning waiters would take it away from the threads that have host work to do.
inline cudaError_t nb_stream_sync(ngmlr_b200_ctx* ctx, cudaStream_t st) {
  if (ctx->spin_sync || !ctx->ev_sync) return cudaStreamSynchronize(st);
  cudaError_t e = cudaEventRecord(ctx->ev_sync, st);
  if (e != cudaSuccess) return e;
  return cudaEventSynchronize(ctx->ev_sync);
}

#define CU(call)                                                                          \
  do {                                                                                    \
    cudaError_t e__ = (call);                                                             \
    if (e__ != cudaSuccess)                                                               \
      return ctx->fail("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)


namespace nb {

// Candidate-search / reference state of a context (side table keyed by the context).
struct CsState {
  DevBuf<uint8_t> d_packed;
  DevBuf<uint32_t> d_tab, d_pos, d_order;
  DevBuf<uint32_t> d_used;  // bitmap
  DevBuf<int8_t> d_rci;     // Index::m_RevCompIndex
  DevBuf<uint8_t> d_seq, d_tables;
  DevBuf<uint64_t> d_off;     // seq_off | table_off | order_off | out_off
  DevBuf<int32_t> d_len, d_count;
  DevBuf<uint32_t> d_cap;
  DevBuf<unsigned long long> d_hits;
  DevBuf<float> d_max;
  DevBuf<CsCandidate> d_out;
  uint32_t index_len = 0, n_pos = 0;
  uint64_t unit_offset = 0;
  int k = 0, bin_shift = 0;
  std::vector<float> scores;
  std::vector<uint64_t> locs;
  std::vector<uint8_t> reverse;
  std::vector<float> sw_scores;
  float last_ms = 0;
  // candidate scoring
  DevBuf<uint8_t> d_enc, d_rev;
  uint64_t enc_bytes = 0, concat_len = 0;
  DevBuf<unsigned long long> d_ref_starts;   // refStartPos (set_ref_starts)
  std::vector<unsigned long long> ref_starts;
  DevBuf<unsigned long long> d_winpos;
  DevBuf<uint64_t> d_qoff;
  DevBuf<int32_t> d_qlen;
  DevBuf<float> d_sw;
  DevBuf<int32_t> d_swscratch;
  std::vector<uint64_t> last_seq_off;  // arena offsets of the reads of the last search
  // resident pipeline
  int rn = 0;                       // (sub-)reads the resident pipeline runs on
  int rmax = 0;                     // the longest of them
  size_t rbytes = 0;
  const uint8_t* seq_base = nullptr;  // their arena: d_seq (cs_upload) or the context's resident read set
  DevBuf<unsigned long long> d_a, d_b, d_c, d_sa, d_sb, d_sc, d_cnt64, d_cstart, d_cloc;
  DevBuf<uint8_t> d_scan_tmp;
  DevBuf<float> d_cscore;
  long long n_cand = 0;
  unsigned long long n_small_tables = 1;  // tables of the last run that live in shared memory
  bool reads_searched = false;  // the candidates on the device are cs_run's for the sub-reads of the last reads_upload
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::vector<int64_t> h_cstart;
  // pinned staging for the resident pipeline's upload / fetch
  PinBuf<uint8_t> p_seq, p_rev;
  PinBuf<float> p_score, p_sw;
  PinBuf<uint64_t> p_loc;
  // short-read scoring (short_reads.cu): pairs (read, location, strand) -> window, query, score
  DevBuf<int32_t> d_sr_ridx, d_sr_winlen, d_sr_qlen;
  DevBuf<unsigned long long> d_sr_loc, d_sr_winpos;
  DevBuf<uint64_t> d_sr_qoff;
  DevBuf<uint8_t> d_sr_rev;
  DevBuf<float> d_sr_sw;
  DevBuf<unsigned int> d_sr_counts;  // general pairs | wide ungapped pairs
  DevBuf<int32_t> d_sr_scratch;
  unsigned int sr_general_pairs = 0;  // pairs of the last short-read scoring that missed the ungapped path
  unsigned int sr_wide_pairs = 0;     // pairs of the last short-read scoring on the wide ungapped instantiation
  DevBuf<unsigned int> d_sub_counts;  // the same two counters for the last sub-read scoring (cs_run, cs_score_batch)
  // the contig table of the last ngmlr_b200_load_reference (reference_load.cu); cleared when another call replaces
  // the reference
  std::vector<std::string> contig_names;
  std::vector<const char*> contig_name_ptrs;
  std::vector<uint64_t> contig_start, contig_len;
  float load_ms[6] = {0, 0, 0, 0, 0, 0};  // read / parse, install, reference write, index, index write, total
  StreamCounters load_inflate;            // the FASTA file's inflate in the last load_reference
};

CsState* cs_state(ngmlr_b200_ctx* ctx, bool create);

// What ngmlr_b200_last_error(NULL) reports (calls that take no context: create, read_file_open).
void set_error_without_context(const std::string& msg);

// The resident read set of ngmlr_b200_reads_upload and ngmlr_b200_reads_load (pipeline.cu): reads back to back,
// 16-byte aligned and NUL padded, and their sub-reads (ReadProvider::splitRead). read_set_layout fills
// ctx->read_off / read_len and sub_start (the first sub-read of every read, n_reads + 1 entries) from the lengths;
// read_set_reserve sizes the device arrays; read_set_install makes the set the one stage 0/2 and stage 4 run on,
// once its bytes, offsets and sub-read table are on the device.
struct ReadSetShape {
  size_t bytes = 0, n_sub = 0;
  int max_sub = 0;  // the longest sub-read
};
int read_set_layout(ngmlr_b200_ctx* ctx, const char* who, int n_reads, const int32_t* lens, int read_part_length,
                    std::vector<uint64_t>& sub_start, ReadSetShape& shape);
int read_set_reserve(ngmlr_b200_ctx* ctx, CsState* cs, int n_reads, const ReadSetShape& shape);
void read_set_install(ngmlr_b200_ctx* ctx, CsState* cs, int n_reads, const ReadSetShape& shape);

int convex_upload_spec(ngmlr_b200_ctx* ctx, const UploadSpec& spec);

// Fill kernel choice (capi.cu): whether a batch under scoring `s` whose scores stay below `magnitude` needs the RAW
// (as-coded SSE) kernel, and the magnitude bound of one problem.
bool scoring_needs_raw(const Scoring& s, double magnitude);
double score_magnitude_bound(const Scoring& s, long long qry_len, long long ref_len);

}  // namespace nb
