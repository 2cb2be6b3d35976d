// ngmlr_b200/csrc/pipeline.cu -- the read set resident in HBM and the batched mirror of
// AlignmentBuffer::computeAlignment (C ABI, include/ngmlr_b200.h).
//
// ngmlr hands every read to the hot path several times: its 256-bp pieces to the candidate search
// and the sub-read scorer (stage 0/2), then parts of it -- forward or reverse-complemented -- to the
// convex aligner, once per interval and again for every retry with a wider corridor
// (src/AlignmentBuffer.cpp:226-465). Here the reads of a batch cross PCIe ONCE
// (ngmlr_b200_reads_upload); every later stage names what it needs by index:
//   stage 0/2   sub-read s = (read, k * readPartLength, readPartLength)   ReadProvider::splitRead
//   stage 4     interval   = (read, onReadStart, length, strand) + reference window positions +
//                            the corridor in closed form (device_types.h AlnDesc::ckind)
// so that an alignment costs ~150 bytes of H2D traffic; windows are decoded, read parts gathered and
// corridor rows generated on the device. ngmlr_b200_compute_alignments is computeAlignment for n
// intervals at once: attempt k of all intervals that are still invalid is one device batch.
#include "runtime.h"

using namespace nb;

namespace {

// getChrStart's contract for DecodeRefSequenceExact, as check_windows in capi.cu but per window: a
// window the reference cannot decode makes extractReferenceSequenceForAlignment return 0.
bool window_ok(const CsState* cs, uint64_t p) {
  const auto& rs = cs->ref_starts;
  if (rs.size() < 2) return false;
  if (p >= cs->concat_len || p >= rs.back() || p == 0) return false;
  size_t u = std::upper_bound(rs.begin(), rs.end(), (unsigned long long)p) - rs.begin();
  if (rs[u] - p < 1000ull) ++u;
  if (u >= rs.size() || p > rs[u] - 1000ull) return false;
  return true;
}

struct IvState {
  int ref_seq_len = 0;   // refSeqLen = onRefStop - onRefStart + 1 (the buffer, NUL included)
  int corridor = 0;      // min(corridor, 2 * refSeqLen)
  int retry = 0, mult = 1;
};

// The corridor computeAlignment builds for this attempt (src/AlignmentBuffer.cpp:333-352), in closed form.
CorridorForm corridor_for(const ngmlr_b200_interval& iv, const ngmlr_b200_anchor* anchors, const IvState& s,
                          int read_part_length) {
  CorridorForm f;
  memset(&f, 0, sizeof(f));
  const int qry_len = iv.read_seq_len;
  const int ref_len = s.ref_seq_len - 1;  // strlen(refSeq)
  if (iv.full_alignment) {  // getCorridorFull(refSeqLen, ...) (:84-105): double arithmetic
    const int w = s.ref_seq_len;
    f.kind = 0;
    f.c0 = (int)(w * -0.2);
    f.cstep = 0;
    f.width = w + (int)(w * 0.2);
    return f;
  }
  if (iv.short_read) {  // getCorridorLinear(corridor * multiplier, ...) (:68-82)
    const int w = s.corridor * s.mult;
    f.kind = 0;
    f.c0 = -(w / 2);
    f.cstep = 1;
    f.width = w;
    return f;
  }
  const float k = (float)qry_len * 1.0f / (float)ref_len;
  f.kind = 1;
  f.k = k;
  if (s.mult < 3 && !iv.realign && iv.n_anchors > 0) {  // getCorridorEndpointsWithAnchors (:129-197)
    float left = 0.0f, right = 0.0f;
    const float d_align = 0.0f;
    for (int a = 0; a < iv.n_anchors; ++a) {
      const ngmlr_b200_anchor& an = anchors[iv.anchor_begin + a];
      const int anchor_x = (int)(an.on_ref - (int64_t)iv.on_ref_start);
      const int anchor_y = an.is_reverse ? iv.full_read_length - an.on_read - read_part_length - iv.ext_qstart
                                         : an.on_read - iv.ext_qstart;
      const float x_found = (float)anchor_x;
      const float x_expect = ((float)anchor_y - d_align) / k;
      const float diff = x_expect - x_found;
      if (diff > 0) right = std::max(right, diff);
      else left = std::max(left, diff * -1.0f);
    }
    left += 128;
    right += 128;
    left = left + (left + right) * 0.1f;
    right = right + (left + right) * 0.1f;
    left = left * s.mult;
    right = right * s.mult;
    f.width = (int)(left + right);
    f.d = 0.0f;
    f.right = right;
    return f;
  }
  // getCorridorEndpoints(corridor * multiplier, ..., realign) (:107-127)
  const int w = (s.corridor * s.mult) / (iv.realign ? 1 : 4);
  f.width = w;
  f.d = (float)w / 2.0f;
  f.right = 0.0f;
  return f;
}

// Scratch of one device batch of intervals (attempt k of a compute_alignments call).
struct IntervalBatchBuf {
  std::vector<uint64_t> win_start;
  std::vector<int32_t> ref_lens, qry_lens, ridx, pstart, eqs, eqe;
  std::vector<uint8_t> rc;
  std::vector<const char*> qtext;
  std::vector<CorridorForm> forms;
};

int upload_interval_batch(ngmlr_b200_ctx* ctx, CsState* cs, const ngmlr_b200_interval* intervals,
                          const ngmlr_b200_anchor* anchors, const std::vector<int>& batch,
                          const std::vector<IvState>& st, int read_part_length, bool by_index,
                          IntervalBatchBuf& b) {
  const int m = (int)batch.size();
  b.win_start.resize(m); b.ref_lens.resize(m); b.qry_lens.resize(m); b.ridx.resize(m); b.pstart.resize(m);
  b.eqs.resize(m); b.eqe.resize(m); b.rc.resize(m); b.forms.resize(m); b.qtext.resize(m);
  for (int j = 0; j < m; ++j) {
    const ngmlr_b200_interval& iv = intervals[batch[j]];
    const IvState& s = st[batch[j]];
    b.win_start[j] = iv.on_ref_start;
    b.ref_lens[j] = s.ref_seq_len - 1;
    b.qry_lens[j] = iv.read_seq_len;
    b.ridx[j] = iv.read_index;
    b.pstart[j] = iv.on_read_start;
    b.rc[j] = iv.reverse ? 1 : 0;
    b.qtext[j] = iv.read_seq;
    b.eqs[j] = iv.ext_qstart;
    b.eqe[j] = iv.ext_qend;
    b.forms[j] = corridor_for(iv, anchors, s, read_part_length);
  }
  RefWindows w;
  w.d_enc = cs->d_enc.p;
  w.d_ref_starts = cs->d_ref_starts.p;
  w.n_starts = (int)cs->ref_starts.size();
  w.win_start = b.win_start.data();
  ReadParts rp;
  rp.d_reads = ctx->d_reads.p;
  rp.d_read_off = ctx->d_read_off.p;
  rp.read_index = b.ridx.data();
  rp.part_start = b.pstart.data();
  rp.revcomp = b.rc.data();
  UploadSpec sp;
  sp.n = m;
  sp.win = &w;
  sp.ref_lens = b.ref_lens.data();
  if (by_index) sp.parts = &rp;
  else sp.qrys = b.qtext.data();
  sp.qry_lens = b.qry_lens.data();
  sp.forms = b.forms.data();
  sp.ext_qstart = b.eqs.data();
  sp.ext_qend = b.eqe.data();
  return convex_upload_spec(ctx, sp);
}

// Validates the intervals and initialises their retry state. live = intervals that reach SingleAlign.
int prepare_intervals(ngmlr_b200_ctx* ctx, CsState* cs, int n, const ngmlr_b200_interval* intervals,
                      std::vector<IvState>& st, std::vector<int>& live, bool& by_index) {
  if (!cs || !cs->enc_bytes || cs->ref_starts.empty())
    return ctx->fail("compute_alignments: call cs_set_reference and set_ref_starts first");
  bool any_text = false, any_index = false;
  for (int i = 0; i < n; ++i) {
    if (intervals[i].read_index >= 0) any_index = true;
    else any_text = true;
  }
  if (any_text && any_index)
    return ctx->fail("compute_alignments: intervals must all name resident reads or all carry read_seq");
  if (any_index && ctx->n_reads == 0) return ctx->fail("compute_alignments: call reads_upload first");
  by_index = any_index;
  st.assign((size_t)n, IvState());
  live.clear();
  live.reserve(n);
  for (int i = 0; i < n; ++i) {
    const ngmlr_b200_interval& iv = intervals[i];
    if (iv.read_index < 0 && !iv.read_seq) continue;                       // readSeq == nullptr -> 0 (:237-239)
    if (iv.on_ref_start >= iv.on_ref_stop) continue;                        // (:204-207)
    if (iv.on_ref_stop - iv.on_ref_start > 0x7ffffff0ull) continue;
    if (!window_ok(cs, iv.on_ref_start)) continue;                          // DecodeRefSequenceExact fails
    if (iv.read_seq_len < 0) return ctx->fail("compute_alignments: negative read length at %d", i);
    if (iv.read_index >= 0) {
      if (iv.read_index >= ctx->n_reads) return ctx->fail("compute_alignments: read index out of range at %d", i);
      if (iv.on_read_start < 0 || (int64_t)iv.on_read_start + iv.read_seq_len > ctx->read_len[iv.read_index])
        return ctx->fail("compute_alignments: interval %d leaves its read", i);
    }
    IvState& s = st[i];
    s.ref_seq_len = (int)(iv.on_ref_stop - iv.on_ref_start + 1);
    s.corridor = std::min(iv.corridor, s.ref_seq_len * 2);  // (:266-267)
    s.retry = iv.full_alignment ? 1 : 5;
    s.mult = 1;
    live.push_back(i);
  }
  return 0;
}

}  // namespace

extern "C" {

int ngmlr_b200_reads_upload(ngmlr_b200_ctx* ctx, int n_reads, const char* const* seqs, const int32_t* lens,
                            int read_part_length) {
  if (!ctx) return -1;
  if (n_reads < 0) return ctx->fail("reads_upload: n_reads < 0");
  if (read_part_length < 1) return ctx->fail("reads_upload: read_part_length < 1");
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  CsState* cs = cs_state(ctx, true);
  ctx->read_off.resize((size_t)n_reads + 1);
  ctx->read_len.assign(lens, lens + n_reads);
  size_t bytes = 0, n_sub = 0;
  int max_sub = 0;  // the longest sub-read
  for (int i = 0; i < n_reads; ++i) {
    if (lens[i] < 0) return ctx->fail("reads_upload: negative length at %d", i);
    ctx->read_off[i] = bytes;
    bytes += align_up((size_t)lens[i] + 1, 16);
    const int parts = lens[i] / read_part_length;
    n_sub += parts > 0 ? (size_t)parts : 1;  // a read shorter than one part is its own sub-read (:76-104)
    max_sub = std::max(max_sub, parts > 0 ? read_part_length : lens[i]);
  }
  ctx->read_off[n_reads] = bytes;
  if (n_sub > 0x7fffffffull) return ctx->fail("reads_upload: too many sub-reads");
  // one pinned staging block: read bytes | read offsets | sub-read offsets | sub-read lengths
  const size_t off_at = align_up(bytes + 16, 16), soff_at = off_at + ((size_t)n_reads + 1) * 8,
               slen_at = soff_at + (n_sub + 1) * 8, total = slen_at + (n_sub + 1) * 4;
  CU(ctx->h_reads.reserve(total + 16));
  uint8_t* h = ctx->h_reads.p;
  parallel_for(n_reads, 64, [&](int i) {
    const size_t L = (size_t)lens[i];
    memcpy(h + ctx->read_off[i], seqs[i], L);
    memset(h + ctx->read_off[i] + L, 0, align_up(L + 1, 16) - L);
  });
  memcpy(h + off_at, ctx->read_off.data(), ((size_t)n_reads + 1) * 8);
  uint64_t* soff = reinterpret_cast<uint64_t*>(h + soff_at);
  int32_t* slen = reinterpret_cast<int32_t*>(h + slen_at);
  size_t s = 0;
  for (int i = 0; i < n_reads; ++i) {
    const int parts = lens[i] / read_part_length;
    if (parts == 0) {
      soff[s] = ctx->read_off[i];
      slen[s++] = lens[i];
    } else {
      for (int k = 0; k < parts; ++k) {
        soff[s] = ctx->read_off[i] + (uint64_t)k * (uint64_t)read_part_length;
        slen[s++] = read_part_length;
      }
    }
  }
  CU(ctx->d_reads.reserve(bytes + 64));
  CU(ctx->d_read_off.reserve((size_t)n_reads + 1));
  CU(cs->d_off.reserve(n_sub + 1));
  CU(cs->d_len.reserve(n_sub + 1));
  CU(cudaMemcpyAsync(ctx->d_reads.p, h, bytes, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(ctx->d_read_off.p, h + off_at, ((size_t)n_reads + 1) * 8, cudaMemcpyHostToDevice, st));
  if (n_sub) {
    CU(cudaMemcpyAsync(cs->d_off.p, soff, n_sub * 8, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(cs->d_len.p, slen, n_sub * 4, cudaMemcpyHostToDevice, st));
  }
  CU(nb_stream_sync(ctx, st));
  ctx->n_reads = n_reads;
  ctx->reads_bytes = bytes;
  // stage 0/2 now runs on the sub-reads of the resident set (ngmlr_b200_cs_run / cs_fetch)
  cs->rn = (int)n_sub;
  cs->rmax = max_sub;
  cs->rbytes = bytes;
  cs->seq_base = ctx->d_reads.p;
  cs->n_cand = 0;
  cs->reads_searched = false;
  ctx->reads_h2d_bytes = (int64_t)(bytes + ((size_t)n_reads + 1) * 8 + n_sub * 12);
  return (int)n_sub;
}

int64_t ngmlr_b200_reads_h2d_bytes(const ngmlr_b200_ctx* ctx) { return ctx ? ctx->reads_h2d_bytes : 0; }

int ngmlr_b200_compute_alignments(ngmlr_b200_ctx* ctx, int n, const ngmlr_b200_interval* intervals,
                                  const ngmlr_b200_anchor* anchors, int read_part_length,
                                  ngmlr_b200_align_result* results, int32_t* attempts) {
  if (!ctx) return -1;
  if (n < 0) return ctx->fail("compute_alignments: n < 0");
  CsState* cs = cs_state(ctx, false);
  std::vector<IvState> st;
  std::vector<int> live;
  bool by_index = false;
  if (prepare_intervals(ctx, cs, n, intervals, st, live, by_index)) return -1;
  const int saved_mode = ctx->text_mode, saved_slot = ctx->text_slot;
  ctx->text_mode = 1;  // results of every attempt stay valid in their own pinned arena
  ctx->ca_h2d_bytes = ctx->ca_d2h_bytes = 0;
  ctx->ca_fill_ms = ctx->ca_traceback_ms = ctx->ca_text_ms = 0.0f;
  ctx->ca_cells = 0;
  ctx->ca_batches = 0;
  for (int i = 0; i < n; ++i) {
    ngmlr_b200_align_result& r = results[i];
    memset(&r, 0, sizeof(r));
    r.ret = -1;
    r.score = -1.0f;
    r.cigar = "";
    r.md = "";
    if (attempts) attempts[i] = 0;
  }
  std::vector<int> batch;
  IntervalBatchBuf buf;
  std::vector<ngmlr_b200_align_result> tmp;
  int rcode = 0;
  for (int attempt = 0; !live.empty() && attempt < TEXT_SLOTS; ++attempt) {
    batch.clear();
    for (int i : live) {
      IvState& s = st[i];
      if ((long long)s.corridor * s.mult <= (long long)s.ref_seq_len * 2 && s.retry > 0) {  // (:303-305)
        --s.retry;
        batch.push_back(i);
      }
    }
    if (batch.empty()) break;
    const int m = (int)batch.size();
    ctx->text_slot = attempt;
    tmp.resize(m);
    if ((rcode = upload_interval_batch(ctx, cs, intervals, anchors, batch, st, read_part_length, by_index, buf)) != 0) break;
    if ((rcode = ngmlr_b200_convex_run(ctx)) != 0) break;
    if ((rcode = ngmlr_b200_convex_fetch(ctx, tmp.data())) != 0) break;
    ctx->ca_h2d_bytes += ctx->stats.h2d_bytes;
    ctx->ca_d2h_bytes += ctx->stats.d2h_bytes;
    ctx->ca_fill_ms += ctx->stats.fill_ms;
    ctx->ca_traceback_ms += ctx->stats.traceback_ms;
    ctx->ca_text_ms += ctx->stats.text_ms;
    ctx->ca_cells += ctx->stats.cells;
    ctx->ca_batches++;
    live.clear();
    for (int j = 0; j < m; ++j) {
      const int i = batch[j];
      if (attempts) attempts[i]++;
      if (tmp[j].threw) continue;  // computeAlignment's catch (...) -> 0
      if (tmp[j].ret == intervals[i].full_read_length) {
        results[i] = tmp[j];
      } else {
        st[i].mult++;  // invalid: again with a wider corridor (:436-444)
        live.push_back(i);
      }
    }
  }
  ctx->text_mode = saved_mode;
  ctx->text_slot = saved_slot;
  return rcode ? rcode : n;
}

// The first attempt of ngmlr_b200_compute_alignments only, staged for the phased calls: afterwards
// ngmlr_b200_convex_run / ngmlr_b200_convex_fetch operate on it (benchmarks time the kernels with the
// batch resident in HBM). Every interval must reach SingleAlign (a window and a read part).
// Switches the context to the device text stage.
int ngmlr_b200_intervals_upload(ngmlr_b200_ctx* ctx, int n, const ngmlr_b200_interval* intervals,
                                const ngmlr_b200_anchor* anchors, int read_part_length) {
  if (!ctx) return -1;
  if (n < 0) return ctx->fail("intervals_upload: n < 0");
  CsState* cs = cs_state(ctx, false);
  std::vector<IvState> st;
  std::vector<int> live;
  bool by_index = false;
  if (prepare_intervals(ctx, cs, n, intervals, st, live, by_index)) return -1;
  if ((int)live.size() != n) return ctx->fail("intervals_upload: %d of %d intervals have no reference window or read part",
                                              n - (int)live.size(), n);
  ctx->text_mode = 1;
  ctx->text_slot = 0;
  IntervalBatchBuf buf;
  return upload_interval_batch(ctx, cs, intervals, anchors, live, st, read_part_length, by_index, buf);
}

int ngmlr_b200_compute_alignments_stats(ngmlr_b200_ctx* ctx, ngmlr_b200_batch_stats* out) {
  if (!ctx || !out) return -1;
  *out = ctx->stats;
  out->h2d_bytes = ctx->ca_h2d_bytes;
  out->d2h_bytes = ctx->ca_d2h_bytes;
  out->fill_ms = ctx->ca_fill_ms;
  out->traceback_ms = ctx->ca_traceback_ms;
  out->text_ms = ctx->ca_text_ms;
  out->cells = ctx->ca_cells;
  out->fill_launches = ctx->ca_batches;
  out->traceback_launches = ctx->ca_batches;
  out->text_launches = ctx->ca_batches;
  return 0;
}

}  // extern "C"
