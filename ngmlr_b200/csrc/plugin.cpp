// ngmlr_b200/csrc/plugin.cpp -- the IAlignment object behind ngmlr's plugin boundary.
//
// `class B200Alignment : public IAlignment` (interface: src/IAlignment.h:211-247) is what
// CreateAlignment(gpu_id) returns. It serves both construction sites of the reference:
//   * the convex aligner of AlignmentBuffer (src/AlignmentBuffer.h:345-363) -> SingleAlign with
//     CorridorLine[] (ConvexAlignFast::SingleAlign, src/ConvexAlignFast.cpp:452-559), plus a real
//     BatchAlign (the reference throws "Not implemented", :441-450);
//   * the scorer of ScoreBuffer / NGM::CreateAlignment (src/NGM.cpp:350-362) -> BatchScore /
//     SingleScore (StrippedSW, src/StrippedSW.cpp:118-202); GetScoreBatchSize() = 1024 like
//     StrippedSW.h:53-55.
// Argument meaning, buffer ownership and error behaviour follow SURVEY.md section 8(b).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/ngmlr_b200.h"
#include "../../include/ngmlr_b200_ialignment.h"

namespace {

ngmlr_b200_scoring g_scoring = {2.0f, -5.0f, -5.0f, -5.0f, -1.0f, 0.15f};

// ngmlr creates and destroys aligner objects freely (e.g. a fresh StrippedSW per inversion check,
// src/AlignmentBuffer.cpp:1217). A context owns a stream, events and grown device/pinned arenas, so
// retired contexts are parked here and handed to the next object with the same device and scoring.
struct ParkedContext {
  int gpu_id;
  ngmlr_b200_scoring scoring;
  ngmlr_b200_ctx* ctx;
};
std::mutex g_pool_mutex;
std::vector<ParkedContext> g_pool;

// Counters of the cross-thread batchers, printed at exit with NGMLR_B200_STATS=1 (INTEGRATION.md).
struct PluginStats {
  std::atomic<long long> align_calls{0}, align_batches{0}, align_problems{0}, align_batch_us{0};
  std::atomic<long long> score_calls{0}, score_batches{0}, score_pairs{0}, score_batch_us{0};
  // time the calling threads spent blocked inside the batched calls (summed over threads), microseconds
  std::atomic<long long> align_wait_us{0}, score_wait_us{0};
  // batched SingleAlign / BatchAlign launches that ran out of memory and were split in halves
  std::atomic<long long> align_oom_splits{0};
  const std::chrono::steady_clock::time_point t_start = std::chrono::steady_clock::now();
  // phases of the batched SingleAlign launches, microseconds (from ngmlr_b200_convex_stats + the copy back)
  std::atomic<long long> us_pack{0}, us_h2d{0}, us_run{0}, us_fill{0}, us_trace{0}, us_d2h{0}, us_text{0}, us_copy{0};
  ~PluginStats() {
    if (!getenv("NGMLR_B200_STATS")) return;
    fprintf(stderr,
            "[ngmlr_b200] SingleAlign calls %lld in %lld batches (%.1f per batch, %.2f ms per batch); "
            "BatchScore/SingleScore calls %lld in %lld launches (%.0f pairs per launch)\n",
            align_calls.load(), align_batches.load(),
            align_batches ? (double)align_problems / (double)align_batches : 0.0,
            align_batches ? 1e-3 * (double)align_batch_us / (double)align_batches : 0.0, score_calls.load(),
            score_batches.load(), score_batches ? (double)score_pairs / (double)score_batches : 0.0);
    const double nb = align_batches ? (double)align_batches : 1.0;
    fprintf(stderr,
            "[ngmlr_b200] caller threads blocked: %.2f s in SingleAlign (%.2f ms per call), %.2f s in BatchScore/SingleScore "
            "(%.2f ms per call; %.2f ms per scoring launch); process lifetime of the plugin %.2f s\n",
            1e-6 * align_wait_us, align_calls ? 1e-3 * (double)align_wait_us / (double)align_calls : 0.0,
            1e-6 * score_wait_us, score_calls ? 1e-3 * (double)score_wait_us / (double)score_calls : 0.0,
            score_batches ? 1e-3 * (double)score_batch_us / (double)score_batches : 0.0,
            1e-6 * (double)std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t_start).count());
    fprintf(stderr,
            "[ngmlr_b200] per SingleAlign batch (ms): pack %.2f, H2D %.2f, run %.2f (fill kernel %.2f, traceback kernel "
            "%.2f), D2H %.2f, CIGAR/MD/nmPerPosition text %.2f, copy into the callers' Align %.2f\n",
            1e-3 * us_pack / nb, 1e-3 * us_h2d / nb, 1e-3 * us_run / nb, 1e-3 * us_fill / nb, 1e-3 * us_trace / nb,
            1e-3 * us_d2h / nb, 1e-3 * us_text / nb, 1e-3 * us_copy / nb);
    if (align_oom_splits)
      fprintf(stderr, "[ngmlr_b200] alignment batches split after running out of memory: %lld\n", align_oom_splits.load());
  }
} g_stats;

// fn(i) for i in [0, n) on a few host threads (the per-problem copies of a big BatchAlign: CorridorLine[] in,
// nmPerPosition out -- 12 bytes per alignment column into the caller's buffers)
template <typename F>
void plugin_parallel_for(int n, int chunk, F fn) {
  static const int max_threads = [] {
    const char* e = getenv("NGMLR_B200_HOST_THREADS");
    const int v = e ? atoi(e) : 0;
    return v > 0 ? v : (int)std::min(16u, std::max(1u, std::thread::hardware_concurrency()));
  }();
  const int threads = std::min(max_threads, (n + chunk - 1) / chunk);
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
  for (int t = 1; t < threads; ++t) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
}

bool same_scoring(const ngmlr_b200_scoring& a, const ngmlr_b200_scoring& b) {
  return memcmp(&a, &b, sizeof(a)) == 0;
}

// One SingleAlign call parked in the cross-thread batcher (below).
struct AlignRequest {
  char const* ref;
  char const* qry;
  Align* result;
  NgmlrB200BatchAlignArgs args;
  int ret = -1;
  bool threw = false, done = false;
  bool failed = false;
  std::string error;  // owned by the request: the next batch cannot overwrite what a client is still throwing
};
class B200Alignment;
bool score_batcher_submit(int gpu_id, const ngmlr_b200_scoring& scoring, int n, char const* const* refs,
                          char const* const* qrys, float* results);
// what a thrown `const char*` points at must outlive the throw: one string per calling thread
std::string& thread_error() {
  static thread_local std::string e;
  return e;
}
bool batcher_submit(int gpu_id, const ngmlr_b200_scoring& scoring, AlignRequest& r);

class B200Alignment : public IAlignment {
 public:
  explicit B200Alignment(int gpu_id, const ngmlr_b200_scoring& scoring) : gpu_id_(gpu_id), scoring_(scoring) {
    if (const char* e = getenv("NGMLR_B200_MAX_MATRIX_MB")) {  // Config.getMaxMatrixSizeMB() (--max-matrix-size)
      const long v = atol(e);
      if (v > 0) max_matrix_mb_ = (unsigned long)v;
    }
    // fail loudly at construction when there is no usable device; the context itself (stream, events, device
    // and pinned arenas) is made on first direct use -- with the cross-thread batchers on, ngmlr's hundreds of
    // per-thread aligner objects never need one of their own
    device_ok_ = gpu_id >= 0 && gpu_id < ngmlr_b200_device_count();
  }
  ngmlr_b200_ctx* ctx() {
    if (ctx_) return ctx_;
    {
      std::lock_guard<std::mutex> lock(g_pool_mutex);
      for (size_t i = 0; i < g_pool.size(); ++i) {
        if (g_pool[i].gpu_id == gpu_id_ && same_scoring(g_pool[i].scoring, scoring_)) {
          ctx_ = g_pool[i].ctx;
          g_pool.erase(g_pool.begin() + i);
          return ctx_;
        }
      }
    }
    if (ngmlr_b200_create(gpu_id_, &scoring_, &ctx_) != 0) {
      ctx_ = nullptr;
      throw "ngmlr_b200: cannot create a device context (no CUDA device? there is no CPU fallback)";
    }
    return ctx_;
  }
  ~B200Alignment() override {
    if (!ctx_) return;
    std::lock_guard<std::mutex> lock(g_pool_mutex);
    if (g_pool.size() < 256) {
      ParkedContext p = {gpu_id_, scoring_, ctx_};
      g_pool.push_back(p);
    } else {
      ngmlr_b200_destroy(ctx_);
    }
  }
  bool ok() const { return device_ok_; }

  int GetScoreBatchSize() const override { return 1024; }
  int GetAlignBatchSize() const override { return 1024; }

  int BatchScore(int const, int const batchSize, char const* const* const refSeqList,
                 char const* const* const qrySeqList, float* const results, void*) override {
    if (batchSize <= 0) return 0;
    if (score_batcher_submit(gpu_id_, scoring_, batchSize, refSeqList, qrySeqList, results)) return batchSize;
    return score_direct(batchSize, refSeqList, qrySeqList, results);
  }
  int score_direct(int n, char const* const* refs, char const* const* qrys, float* results) {
    int rc = ngmlr_b200_sw_score_batch(ctx(), n, refs, qrys, results);
    if (rc < 0) throw ngmlr_b200_last_error(ctx_);
    return rc;
  }

  int SingleScore(int const, int const, char const* const refSeq, char const* const qrySeq,
                  float& result, void*) override {
    float r = -1.0f;
    if (!score_batcher_submit(gpu_id_, scoring_, 1, &refSeq, &qrySeq, &r)) score_direct(1, &refSeq, &qrySeq, &r);
    result = r;
    return r == -1.0f ? 0 : 1;  // StrippedSW::SingleScore returns 0 for over-long input (:175-178)
  }

  // The (mode, int corridor) overload is "not implemented" in the reference (:561-567).
  int SingleAlign(int const, int const, char const* const, char const* const, Align&, void*) override {
    throw "Not implemented";
  }

  int SingleAlign(int const mode, CorridorLine* corridor, int const corridorHeight,
                  char const* const refSeq, char const* const qrySeq, Align& result,
                  int const externalQStart, int const externalQEnd, void*) override {
    NgmlrB200BatchAlignArgs a = {corridor, corridorHeight, externalQStart, externalQEnd};
    if (corridorHeight >= (int)strlen(qrySeq)) {  // (a malformed call keeps the direct path and its throw)
      AlignRequest req;
      req.ref = refSeq;
      req.qry = qrySeq;
      req.result = &result;
      req.args = a;
      g_stats.align_calls++;
      const auto t_w0 = std::chrono::steady_clock::now();
      const bool batched = batcher_submit(gpu_id_, scoring_, req);
      g_stats.align_wait_us += std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t_w0).count();
      if (batched) {  // false: batching is off -> direct path below
        if (req.failed) {
          thread_error() = req.error;
          throw thread_error().c_str();
        }
        if (req.threw) throw 1;
        return req.ret;
      }
    }
    int ret = -1;
    Align* rp = &result;
    align_many(1, &refSeq, &qrySeq, &rp, &a, &ret, nullptr);
    return ret;
  }

  // extData: NgmlrB200BatchAlignArgs[batchSize]. Returns batchSize; per-problem results (and the
  // SingleAlign return value in Align::alignmentLength's sibling... see below) are in results[i].
  int BatchAlign(int const, int const batchSize, char const* const* const refSeqList,
                 char const* const* const qrySeqList, Align* const results, void* extData) override {
    if (batchSize <= 0) return 0;
    if (!extData) throw "BatchAlign: extData must point to NgmlrB200BatchAlignArgs[batchSize]";
    std::vector<int> rets(batchSize);
    std::vector<Align*> rp(batchSize);
    for (int i = 0; i < batchSize; ++i) rp[i] = results + i;
    align_many(batchSize, refSeqList, qrySeqList, rp.data(),
               static_cast<NgmlrB200BatchAlignArgs*>(extData), rets.data(), nullptr);
    // A failed problem is reported exactly like SingleAlign does: Score == -1.0f.
    return batchSize;
  }

  // n problems through one batched call; results[i] is the caller's Align of problem i. threw_out
  // (optional) receives which problems the reference would have thrown on; without it a throwing
  // single problem throws 1 like SingleAlign.
  void align_many(int n, char const* const* refs, char const* const* qrys, Align* const* results,
                  NgmlrB200BatchAlignArgs* args, int* rets, bool* threw_out) {
    ref_len_.resize(n);
    qry_len_.resize(n);
    qs_.resize(n);
    qe_.resize(n);
    std::vector<char> too_big((size_t)n, 0);  // local: a throw below must not leave state behind
    for (int i = 0; i < n; ++i) {
      ref_len_[i] = (int32_t)strlen(refs[i]);  // lengths by strlen (:463-464)
      qry_len_[i] = (int32_t)strlen(qrys[i]);
      qs_[i] = args[i].externalQStart;
      qe_[i] = args[i].externalQEnd;
      if (args[i].corridorHeight < qry_len_[i]) throw "corridorHeight < read length";
    }
    plugin_parallel_for(n, 16, [&](int i) {
      // matrix->prepare(): rows = qryLen; also publishes offsetInMatrix to the caller's lines
      // (src/AlignmentMatrixFast.cpp:36-43)
      CorridorLine* c = args[i].corridor;
      unsigned long at = 0;
      const int h = args[i].corridorHeight;
      for (int y = 0; y < h; ++y) {
        c[y].offsetInMatrix = at;
        at += (unsigned long)c[y].length;
      }
      // prepare() refuses matrices of >= maxMatrixSizeMB MB -> the alignment fails (:45-58); such a
      // problem never reaches the device
      too_big[i] = (unsigned long)((float)at / 1000.0f / 1000.0f) >= max_matrix_mb_;
    });
    // the problems that go to the device, in order
    keep_.clear();
    for (int i = 0; i < n; ++i)
      if (!too_big[i]) keep_.push_back(i);
    const int m = (int)keep_.size();
    row_start_.resize((size_t)m + 1);
    krefs_.resize(m); kqrys_.resize(m); krl_.resize(m); kql_.resize(m); kqs_.resize(m); kqe_.resize(m);
    size_t rows = 0;
    for (int j = 0; j < m; ++j) {
      const int i = keep_[j];
      row_start_[j] = (int64_t)rows;
      rows += (size_t)qry_len_[i];
      krefs_[j] = refs[i]; kqrys_[j] = qrys[i];
      krl_[j] = ref_len_[i]; kql_[j] = qry_len_[i]; kqs_[j] = qs_[i]; kqe_[j] = qe_[i];
    }
    row_start_[m] = (int64_t)rows;
    off_.resize(rows);
    len_.resize(rows);
    plugin_parallel_for(m, 16, [&](int j) {
      const int i = keep_[j];
      CorridorLine* c = args[i].corridor;
      int32_t* o = off_.data() + row_start_[j];
      int32_t* l = len_.data() + row_start_[j];
      for (int y = 0; y < qry_len_[i]; ++y) {
        o[y] = c[y].offset;
        l[y] = c[y].length;
      }
    });
    res_.resize((size_t)std::max(m, 1));
    for (int i = 0; i < n; ++i) {
      results[i]->svType = 0;  // (:454-457)
      results[i]->Score = -1.0f;
      rets[i] = -1;
      if (threw_out) threw_out[i] = false;
    }
    std::vector<char> threw_j((size_t)std::max(m, 1), 0);
    if (m > 0) align_range(0, m, results, rets, threw_j, false);
    bool threw = false;
    for (int j = 0; j < m; ++j)
      if (threw_j[j]) {
        threw = true;
        if (threw_out) threw_out[keep_[j]] = true;
      }
    if (threw && n == 1 && !threw_out) throw 1;  // caller wraps SingleAlign in try/catch(...) -> unmapped
  }

 private:
  // The kept problems [j0, j1) through one batched call, their results copied into the callers' Align records.
  // A batch that runs out of memory (device arenas or pinned staging) runs again on released arenas (`fresh`), and
  // if it still does not fit, as two halves one after the other: n independent SingleAlign calls would each have
  // fitted where the batch did not. Only a problem that runs out of memory alone on released arenas fails, with
  // Score -1 -- the reference's "matrix too large".
  void align_range(int j0, int j1, Align* const* results, int* rets, std::vector<char>& threw_j, bool fresh) {
    const int m = j1 - j0;
    std::vector<int64_t> rs((size_t)m + 1);
    for (int k = 0; k <= m; ++k) rs[k] = row_start_[j0 + k] - row_start_[j0];
    const int rc = ngmlr_b200_convex_align_batch(ctx(), m, krefs_.data() + j0, krl_.data() + j0, kqrys_.data() + j0,
                                                 kql_.data() + j0, off_.data() + row_start_[j0],
                                                 len_.data() + row_start_[j0], rs.data(), kqs_.data() + j0,
                                                 kqe_.data() + j0, res_.data());
    if (rc != 0) {
      const char* e = ngmlr_b200_last_error(ctx_);
      if (!(e && strstr(e, "out of memory"))) {
        error_ = e ? e : "ngmlr_b200: batched alignment failed";
        throw error_.c_str();
      }
      ngmlr_b200_release_arenas(ctx_);
      if (!fresh) {
        align_range(j0, j1, results, rets, threw_j, true);
        return;
      }
      if (m == 1) return;  // Score -1, ret -1 (set by align_many)
      g_stats.align_oom_splits++;
      const int mid = j0 + m / 2;
      align_range(j0, mid, results, rets, threw_j, true);
      align_range(mid, j1, results, rets, threw_j, false);
      return;
    }
    ngmlr_b200_batch_stats bs;
    if (ngmlr_b200_convex_stats(ctx_, &bs) == 0) {
      g_stats.us_pack += (long long)(1e3 * bs.host_pack_ms);
      g_stats.us_h2d += (long long)(1e3 * bs.host_h2d_ms);
      g_stats.us_run += (long long)(1e3 * bs.host_run_ms);
      g_stats.us_fill += (long long)(1e3 * bs.fill_ms);
      g_stats.us_trace += (long long)(1e3 * bs.traceback_ms);
      g_stats.us_d2h += (long long)(1e3 * bs.host_d2h_ms);
      g_stats.us_text += (long long)(1e3 * bs.host_text_ms);
    }
    // the results point into the context's arenas: copy them out before the next batch call
    const auto t_copy0 = std::chrono::steady_clock::now();
    plugin_parallel_for(m, 16, [&](int jj) {
      const int j = j0 + jj;
      const int i = keep_[j];
      const ngmlr_b200_align_result& r = res_[jj];
      Align& a = *results[i];
      if (a.pBuffer2) a.pBuffer2[0] = '\0';  // (:469)
      if (r.threw) {
        threw_j[j] = 1;
        return;
      }
      if (r.ret < 0) return;
      // caller-owned buffers; grow MD / nmPerPosition like checkMdBufferLength / addPosition do
      if (r.cigar_len + 1 > a.maxBufferLength || !a.pBuffer1) {
        threw_j[j] = 1;  // "CIGAR/MD buffer not long enough" -> throw 1 (:289-294)
        return;
      }
      memcpy(a.pBuffer1, r.cigar, (size_t)r.cigar_len + 1);
      if (r.md_len + 1 > a.maxMdBufferLength || !a.pBuffer2) {
        int cap = a.maxMdBufferLength > 0 ? a.maxMdBufferLength : 1024;
        while (cap < r.md_len + 1) cap *= 2;
        delete[] a.pBuffer2;
        a.pBuffer2 = new char[cap];
        a.maxMdBufferLength = cap;
      }
      memcpy(a.pBuffer2, r.md, (size_t)r.md_len + 1);
      if (r.nm_count > a.nmPerPostionLength || !a.nmPerPosition) {
        int cap = a.nmPerPostionLength > 0 ? a.nmPerPostionLength : 64;
        while (cap < r.nm_count) cap *= 2;
        delete[] a.nmPerPosition;
        a.nmPerPosition = new PositionNM[cap];
        a.nmPerPostionLength = cap;
      }
      for (int k = 0; k < r.nm_count; ++k) {
        a.nmPerPosition[k].refPosition = r.nm_positions[3 * k + 0];
        a.nmPerPosition[k].readPosition = r.nm_positions[3 * k + 1];
        a.nmPerPosition[k].nm = r.nm_positions[3 * k + 2];
      }
      a.QStart = r.qstart;
      a.QEnd = r.qend;
      a.firstPosition.refPosition = r.first_ref;
      a.firstPosition.readPosition = r.first_read;
      a.lastPosition.refPosition = r.last_ref;
      a.lastPosition.readPosition = r.last_read;
      a.Identity = r.identity;
      a.NM = r.nm;
      a.alignmentLength = r.alignment_length;
      a.cigarOpCount = r.cigar_op_count;
      a.PositionOffset = r.position_offset;
      a.Score = r.score;
      a.svType = r.sv_type;
      rets[i] = r.ret;
    });
    g_stats.us_copy += std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t_copy0).count();
  }

  int gpu_id_ = 0;
  bool device_ok_ = false;
  ngmlr_b200_scoring scoring_;
  ngmlr_b200_ctx* ctx_ = nullptr;
  unsigned long max_matrix_mb_ = 10000ul;  // Config.getMaxMatrixSizeMB() default (src/IConfig.h)
  std::vector<int32_t> ref_len_, qry_len_, off_, len_, qs_, qe_, krl_, kql_, kqs_, kqe_;
  std::vector<int64_t> row_start_;
  std::vector<int> keep_;
  std::vector<char const*> krefs_, kqrys_;
  std::vector<ngmlr_b200_align_result> res_;
  std::string error_;
};

// ---- cross-thread batcher (SURVEY section 8(b): "a GPU implementation that batches across threads
// must do its own cross-thread queueing behind these blocking calls") ----------------------------
// ngmlr runs one aligner object per worker thread and every SingleAlign blocks. With
// NGMLR_B200_BATCH_WINDOW_US=<n> (> 0; off by default) the calls of all threads are parked in one
// queue; a dispatcher thread collects what arrives within the window (or NGMLR_B200_BATCH_MAX
// problems, default 256), runs ONE batched launch on its own context and hands every caller its
// result. Results are those of n independent SingleAlign calls; the call sites stay untouched.
class Batcher {
 public:
  Batcher(int gpu_id, const ngmlr_b200_scoring& sc, int window_us, int max_batch)
      : gpu_id_(gpu_id), scoring_(sc), window_us_(window_us), max_batch_(max_batch) {
    server_ = new B200Alignment(gpu_id, sc);  // the server object takes the scoring of its first client
    if (server_->ok()) {
      worker_ = std::thread([this] { loop(); });
      worker_.detach();  // lives for the process: never torn down behind the CUDA runtime's back
    }
  }
  bool usable(int gpu_id, const ngmlr_b200_scoring& sc) const {
    return server_->ok() && gpu_id == gpu_id_ && same_scoring(sc, scoring_);
  }
  void submit(AlignRequest& r) {
    std::unique_lock<std::mutex> lk(m_);
    queue_.push_back(&r);
    cv_work_.notify_one();
    cv_done_.wait(lk, [&] { return r.done; });
  }

 private:
  void loop() {
    std::vector<AlignRequest*> batch;
    std::vector<char const*> refs, qrys;
    std::vector<Align*> results;
    std::vector<NgmlrB200BatchAlignArgs> args;
    std::vector<int> rets;
    std::vector<char> threw;
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(m_);
        cv_work_.wait(lk, [&] { return !queue_.empty(); });
        // linger: give the other worker threads a chance to join this launch
        const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(window_us_);
        while ((int)queue_.size() < max_batch_ &&
               cv_work_.wait_until(lk, deadline) != std::cv_status::timeout) {
        }
        const size_t take = std::min(queue_.size(), (size_t)max_batch_);
        batch.assign(queue_.begin(), queue_.begin() + take);
        queue_.erase(queue_.begin(), queue_.begin() + take);
      }
      const int n = (int)batch.size();
      refs.resize(n); qrys.resize(n); results.resize(n); args.resize(n); rets.assign(n, -1); threw.assign(n, 0);
      for (int i = 0; i < n; ++i) {
        refs[i] = batch[i]->ref;
        qrys[i] = batch[i]->qry;
        results[i] = batch[i]->result;
        args[i] = batch[i]->args;
      }
      bool failed = false;
      std::string error;
      const auto t_b0 = std::chrono::steady_clock::now();
      g_stats.align_batches++;
      g_stats.align_problems += n;
      try {
        server_->align_many(n, refs.data(), qrys.data(), results.data(), args.data(), rets.data(),
                            reinterpret_cast<bool*>(threw.data()));
      } catch (const char* e) {
        failed = true;
        error = e ? e : "batched alignment failed";
      } catch (...) {
        failed = true;
        error = "batched alignment failed";
      }
      g_stats.align_batch_us += std::chrono::duration_cast<std::chrono::microseconds>(
                                    std::chrono::steady_clock::now() - t_b0).count();
      {
        std::lock_guard<std::mutex> lk(m_);
        for (int i = 0; i < n; ++i) {
          batch[i]->ret = rets[i];
          batch[i]->threw = threw[i] != 0;
          batch[i]->failed = failed;
          batch[i]->error = error;
          batch[i]->done = true;
        }
      }
      cv_done_.notify_all();
    }
  }

  int gpu_id_;
  ngmlr_b200_scoring scoring_;
  int window_us_, max_batch_;
  B200Alignment* server_ = nullptr;
  std::thread worker_;
  std::mutex m_;
  std::condition_variable cv_work_, cv_done_;
  std::vector<AlignRequest*> queue_;
};

int batch_window_us() {
  static const int v = [] {
    const char* e = getenv("NGMLR_B200_BATCH_WINDOW_US");
    return e ? atoi(e) : 0;
  }();
  return v;
}

int batch_servers() {  // dispatcher threads (each with its own context) that take batches in turn
  static const int v = [] {
    const char* e = getenv("NGMLR_B200_BATCH_SERVERS");
    const int n = e ? atoi(e) : 2;
    return n < 1 ? 1 : (n > 8 ? 8 : n);
  }();
  return v;
}

bool batcher_submit(int gpu_id, const ngmlr_b200_scoring& scoring, AlignRequest& r) {
  const int window_us = batch_window_us();
  if (window_us <= 0) return false;
  static std::mutex create_mutex;
  static std::vector<Batcher*> batchers;  // leaked on purpose (see the detach above)
  static std::atomic<unsigned> next(0);
  {
    std::lock_guard<std::mutex> lk(create_mutex);
    if (batchers.empty()) {
      const char* e = getenv("NGMLR_B200_BATCH_MAX");
      const int mx = e && atoi(e) > 0 ? atoi(e) : 256;
      for (int i = 0; i < batch_servers(); ++i) batchers.push_back(new Batcher(gpu_id, scoring, window_us, mx));
    }
  }
  Batcher* b = batchers[next.fetch_add(1) % batchers.size()];
  if (!b->usable(gpu_id, scoring)) return false;
  b->submit(r);
  return true;
}

// ---- the same for BatchScore / SingleScore ------------------------------------------------------
// ScoreBuffer calls BatchScore once per read with a few dozen (window, sub-read) pairs, every thread on its
// own; here the calls of all threads that arrive within the window become ONE scoring launch.
struct ScoreRequest {
  int n;
  char const* const* refs;
  char const* const* qrys;
  float* results;
  bool done = false, failed = false;
  std::string error;
};

class ScoreBatcher {
 public:
  ScoreBatcher(int gpu_id, const ngmlr_b200_scoring& sc, int window_us, int max_pairs)
      : gpu_id_(gpu_id), window_us_(window_us), max_pairs_(max_pairs) {
    server_ = new B200Alignment(gpu_id, sc);
    if (server_->ok()) {
      worker_ = std::thread([this] { loop(); });
      worker_.detach();
    }
  }
  bool usable(int gpu_id) const { return server_->ok() && gpu_id == gpu_id_; }
  void submit(ScoreRequest& r) {
    std::unique_lock<std::mutex> lk(m_);
    queue_.push_back(&r);
    pending_pairs_ += r.n;
    cv_work_.notify_one();
    cv_done_.wait(lk, [&] { return r.done; });
  }

 private:
  void loop() {
    std::vector<ScoreRequest*> batch;
    std::vector<char const*> refs, qrys;
    std::vector<float> out;
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(m_);
        cv_work_.wait(lk, [&] { return !queue_.empty(); });
        const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(window_us_);
        while (pending_pairs_ < max_pairs_ && cv_work_.wait_until(lk, deadline) != std::cv_status::timeout) {
        }
        batch.swap(queue_);
        queue_.clear();
        pending_pairs_ = 0;
      }
      refs.clear();
      qrys.clear();
      for (ScoreRequest* r : batch) {
        refs.insert(refs.end(), r->refs, r->refs + r->n);
        qrys.insert(qrys.end(), r->qrys, r->qrys + r->n);
      }
      out.assign(refs.size(), -1.0f);
      bool failed = false;
      std::string error;
      const auto t_s0 = std::chrono::steady_clock::now();
      try {
        server_->score_direct((int)refs.size(), refs.data(), qrys.data(), out.data());
      } catch (const char* e) {
        failed = true;
        error = e ? e : "batched scoring failed";
      } catch (...) {
        failed = true;
        error = "batched scoring failed";
      }
      g_stats.score_batches++;
      g_stats.score_pairs += (long long)refs.size();
      g_stats.score_batch_us += std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t_s0).count();
      {
        std::lock_guard<std::mutex> lk(m_);
        size_t at = 0;
        for (ScoreRequest* r : batch) {
          if (!failed) memcpy(r->results, out.data() + at, (size_t)r->n * sizeof(float));
          at += (size_t)r->n;
          r->failed = failed;
          r->error = error;
          r->done = true;
        }
      }
      batch.clear();
      cv_done_.notify_all();
    }
  }
  int gpu_id_, window_us_, max_pairs_;
  long long pending_pairs_ = 0;
  B200Alignment* server_ = nullptr;
  std::thread worker_;
  std::mutex m_;
  std::condition_variable cv_work_, cv_done_;
  std::vector<ScoreRequest*> queue_;
};

bool score_batcher_submit(int gpu_id, const ngmlr_b200_scoring& scoring, int n, char const* const* refs,
                          char const* const* qrys, float* results) {
  const int window_us = batch_window_us();
  if (window_us <= 0) return false;
  static std::mutex create_mutex;
  static std::vector<ScoreBatcher*> batchers;
  static std::atomic<unsigned> next(0);
  {
    std::lock_guard<std::mutex> lk(create_mutex);
    if (batchers.empty())
      for (int i = 0; i < batch_servers(); ++i) batchers.push_back(new ScoreBatcher(gpu_id, scoring, window_us, 65536));
  }
  ScoreBatcher* b = batchers[next.fetch_add(1) % batchers.size()];
  if (!b->usable(gpu_id)) return false;
  ScoreRequest r;
  r.n = n;
  r.refs = refs;
  r.qrys = qrys;
  r.results = results;
  g_stats.score_calls++;
  const auto t_w0 = std::chrono::steady_clock::now();
  b->submit(r);
  g_stats.score_wait_us += std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t_w0).count();
  if (r.failed) {
    thread_error() = r.error;
    throw thread_error().c_str();
  }
  return true;
}

}  // namespace

extern "C" {

IAlignment* CreateAlignment(int const gpu_id) {
  ngmlr_b200_scoring sc;
  {
    std::lock_guard<std::mutex> lock(g_pool_mutex);
    sc = g_scoring;
  }
  B200Alignment* a = new B200Alignment(gpu_id, sc);
  if (!a->ok()) {  // fail loudly: no CPU fallback
    delete a;
    return nullptr;
  }
  return a;
}

void DeleteAlignment(IAlignment* aligner) { delete aligner; }

void SetAlignmentScoring(float match, float mismatch, float gapOpen, float gapExtend,
                         float gapExtendMin, float gapDecay) {
  std::lock_guard<std::mutex> lock(g_pool_mutex);
  g_scoring.match = match;
  g_scoring.mismatch = mismatch;
  g_scoring.gap_open = gapOpen;
  g_scoring.gap_extend = gapExtend;
  g_scoring.gap_extend_min = gapExtendMin;
  g_scoring.gap_decay = gapDecay;
}

int ngmlr_b200_plugin_cookie(void) { return 0x10201130; }  // cCookie, src/IAlignment.h:193

// Test / diagnostic aid: the device context an object made by CreateAlignment runs its direct calls on (created
// here if it has none yet), so that FFI callers can read its last error and batch statistics or set its test hooks.
// NULL for any other object or when no context can be made.
ngmlr_b200_ctx* ngmlr_b200_plugin_context(IAlignment* aligner) {
  B200Alignment* a = dynamic_cast<B200Alignment*>(aligner);
  if (!a) return nullptr;
  try {
    return a->ctx();
  } catch (...) {
    return nullptr;
  }
}

// Benchmark / test aid for FFI callers that cannot build C++ objects (bench.py): n SingleAlign problems
// given as flat arrays are turned into what ngmlr itself would hold -- caller-allocated `Align` records
// (buffers sized like AlignmentBuffer::computeAlignment does, src/AlignmentBuffer.cpp:271-278) and
// CorridorLine arrays -- and pushed `repeats` times through `aligner->BatchAlign(...)`, i.e. through the
// IAlignment vtable, host buffers in, host buffers out. Only the BatchAlign calls are timed
// (*seconds). rets[i] / score_bits[i] / cigar_crc[i] of the last repeat let the caller verify the results.
int ngmlr_b200_plugin_time_batch_align(IAlignment* aligner, int n, char const* const* refs, char const* const* qrys,
                                       const int32_t* corridor_offsets, const int32_t* corridor_lengths,
                                       const int64_t* row_start, const int32_t* ext_qstart, const int32_t* ext_qend,
                                       int repeats, double* seconds, int32_t* rets, uint32_t* score_bits,
                                       uint32_t* cigar_crc) {
  if (!aligner || n < 0) return -1;
  std::vector<Align> aligns((size_t)n);
  std::vector<std::vector<CorridorLine>> lines((size_t)n);
  std::vector<NgmlrB200BatchAlignArgs> args((size_t)n);
  for (int i = 0; i < n; ++i) {
    const int h = (int)(row_start[i + 1] - row_start[i]);
    lines[i].resize((size_t)h);
    for (int y = 0; y < h; ++y) {
      lines[i][y].offset = corridor_offsets[row_start[i] + y];
      lines[i][y].length = corridor_lengths[row_start[i] + y];
      lines[i][y].offsetInMatrix = 0;
    }
    args[i].corridor = lines[i].data();
    args[i].corridorHeight = h;
    args[i].externalQStart = ext_qstart ? ext_qstart[i] : 0;
    args[i].externalQEnd = ext_qend ? ext_qend[i] : 0;
    Align& a = aligns[i];
    const int read_length = h;
    a.maxBufferLength = read_length * 4 + 8;
    a.maxMdBufferLength = read_length * 4 + 8;
    a.pBuffer1 = new char[a.maxBufferLength];
    a.pBuffer2 = new char[a.maxMdBufferLength];
    a.pBuffer1[0] = a.pBuffer2[0] = '\0';
    a.nmPerPostionLength = (read_length + 1) * 2;
    a.nmPerPosition = new PositionNM[a.nmPerPostionLength];
  }
  double total = 0.0;
  int rc = 0;
  try {
    for (int r = 0; r < repeats; ++r) {
      const auto t0 = std::chrono::steady_clock::now();
      aligner->BatchAlign(0, n, refs, qrys, aligns.data(), args.data());
      total += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    }
  } catch (...) {
    rc = -2;
  }
  for (int i = 0; i < n; ++i) {
    Align& a = aligns[i];
    const bool ok = a.Score != -1.0f;
    if (rets) rets[i] = ok ? a.QStart + a.QEnd : -1;  // BatchAlign reports failure as Score == -1
    if (score_bits) memcpy(score_bits + i, &a.Score, 4);
    if (cigar_crc) {
      uint32_t c = 2166136261u;  // FNV-1a over CIGAR + MD
      if (ok) {
        for (const char* q = a.pBuffer1; *q; ++q) c = (c ^ (uint8_t)*q) * 16777619u;
        for (const char* q = a.pBuffer2; *q; ++q) c = (c ^ (uint8_t)*q) * 16777619u;
      }
      cigar_crc[i] = c;
    }
    delete[] a.pBuffer1;
    delete[] a.pBuffer2;
    delete[] a.nmPerPosition;
    a.pBuffer1 = a.pBuffer2 = nullptr;
    a.nmPerPosition = nullptr;
  }
  if (seconds) *seconds = total;
  return rc;
}

}  // extern "C"
