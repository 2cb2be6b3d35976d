// ngmlr_b200/csrc/short_reads.cu -- ngmlr's path for reads of at most --subread-length bases, on the resident
// read set (C ABI, include/ngmlr_b200.h).
//
// ngmlr does not split such a read (ReadProvider::NextRead, src/ReadProvider.cpp:152-156). CS::SendToBuffer
// (src/CS.cpp:307-316) hands it to ScoreBuffer::scoreShortRead (src/ScoreBuffer.cpp:216-286), which drops
// candidates that repeat a location, scores the rest against windows of len + (int)(len * 0.3 + 256) characters,
// orders them by score and computes the MQ; AlignmentBuffer::processShortRead (src/AlignmentBuffer.cpp:2550-2660)
// then aligns the best candidates one by one and hands the read to WriteRead (:3470-3482), which converts the
// positions to contig coordinates. Here:
//   dedupe        host (the reference's std::sort of equal locations decides which strand survives)
//   scoring       device: per-pair window geometry + the StrippedSW kernel's ungapped path (<= 640 columns)
//   order + MQ    host, ngmlr_b200_select_candidates
//   align loop    rounds: round r aligns candidate r of every read still in its loop, one
//                 ngmlr_b200_compute_alignments call (short_read = 1) per round
//   convert       host, upper_bound over refStartPos
#include "runtime.h"

using namespace nb;

namespace {

struct SrPair {
  int32_t read;   // resident read index
  uint64_t loc;   // candidate location (concatenated genome)
  uint8_t rev;
};

int score_pairs(ngmlr_b200_ctx* ctx, CsState* cs, int n, const int32_t* read_index, const uint64_t* locs,
                const uint8_t* reverse, float* scores) {
  cudaStream_t st = ctx->stream;
  cs->sr_general_pairs = 0;
  if (n == 0) return 0;
  const size_t nn = (size_t)n + 1;
  CU(cs->d_sr_ridx.reserve(nn)); CU(cs->d_sr_winlen.reserve(nn)); CU(cs->d_sr_qlen.reserve(nn));
  CU(cs->d_sr_loc.reserve(nn)); CU(cs->d_sr_winpos.reserve(nn)); CU(cs->d_sr_qoff.reserve(nn));
  CU(cs->d_sr_rev.reserve(nn)); CU(cs->d_sr_sw.reserve(nn)); CU(cs->d_sr_general.reserve(1));
  CU(ctx->d_read_len.reserve((size_t)ctx->n_reads + 1));
  CU(cudaMemcpyAsync(ctx->d_read_len.p, ctx->read_len.data(), (size_t)ctx->n_reads * 4, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(cs->d_sr_ridx.p, read_index, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(cs->d_sr_loc.p, locs, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(cs->d_sr_rev.p, reverse, (size_t)n, cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(cs->d_sr_general.p, 0, sizeof(unsigned int), st));
  CU(launch_cs_short_geometry(cs->d_sr_ridx.p, cs->d_sr_loc.p, ctx->d_read_off.p, ctx->d_read_len.p, n,
                              cs->d_sr_winpos.p, cs->d_sr_winlen.p, cs->d_sr_qoff.p, cs->d_sr_qlen.p, st));
  const int warps_per_cta = 4;
  const int grid = std::max(1, std::min(ctx->num_sms * 8, (n + warps_per_cta - 1) / warps_per_cta));
  const size_t stride = 4;  // queries of <= 257 characters never reach the multi-pass strip
  CU(cs->d_sr_scratch.reserve((size_t)grid * warps_per_cta * stride * 2));
  SwParams sp;
  memset(&sp, 0, sizeof(sp));
  sp.seq = ctx->d_reads.p;
  sp.qry_off = cs->d_sr_qoff.p;
  sp.qry_len = cs->d_sr_qlen.p;
  sp.out = cs->d_sr_sw.p;
  sp.n = n;
  sp.scratch = cs->d_sr_scratch.p;
  sp.scratch_stride = stride;
  sp.enc = cs->d_enc.p;
  sp.concat_len = cs->concat_len;
  sp.win_pos = cs->d_sr_winpos.p;
  sp.rev = cs->d_sr_rev.p;
  sp.win_lens = cs->d_sr_winlen.p;
  sp.general_pairs = cs->d_sr_general.p;
  CU(launch_sw_score_gather_short(sp, grid, st));
  CU(cudaMemcpyAsync(scores, cs->d_sr_sw.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(&cs->sr_general_pairs, cs->d_sr_general.p, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  CU(nb_stream_sync(ctx, st));
  return 0;
}

int check_short_ready(ngmlr_b200_ctx* ctx, CsState* cs, const char* who) {
  if (!cs || !cs->enc_bytes || cs->ref_starts.empty())
    return ctx->fail("%s: call cs_set_reference and set_ref_starts first", who);
  if (ctx->n_reads == 0) return ctx->fail("%s: call reads_upload first", who);
  return 0;
}

// One read's processShortRead loop (src/AlignmentBuffer.cpp:2564-2639).
struct SrLoop {
  int read = 0, first = 0, m = 0;  // candidates [first, first + m) of the score-ordered pair list
  int k = 0, last_score = 0;
  std::vector<int> kept;           // pair indices of the mapped alignments, in alignment order
  std::vector<ngmlr_b200_align_result> res;
  std::vector<std::pair<std::string, std::string>> text;  // CIGAR, MD
};

}  // namespace

extern "C" {

// ScoreBuffer::scoreShortRead's duplicate removal (src/ScoreBuffer.cpp:225-239).
int ngmlr_b200_dedupe_short_read_candidates(int n, const int64_t* cand_start, const uint64_t* locs,
                                            int read_part_length, int32_t* kept, int64_t* kept_start) {
  if (n < 0 || (n > 0 && (!cand_start || !locs || !kept || !kept_start))) return -1;
  for (int i = 0; i < n; ++i)
    if (cand_start[i + 1] < cand_start[i] || cand_start[i + 1] - cand_start[i] > 0x7fffffff) return -1;
  std::vector<int32_t> cnt((size_t)n);
  parallel_for(n, 512, [&](int i) {
    struct Item {
      uint64_t loc;
      int32_t idx;
    };
    const int64_t b = cand_start[i];
    const int m = (int)(cand_start[i + 1] - b);
    std::vector<Item> it((size_t)m);
    for (int j = 0; j < m; ++j) it[j] = Item{locs[b + j], (int32_t)(b + j)};
    // the reference's call and comparator (sortLocationScoreLocation, :29-31): equal locations -- the forward and
    // reverse candidate of one bin -- come out in libstdc++'s std::sort order, which decides the surviving strand
    std::sort(it.begin(), it.end(), [](Item x, Item y) { return x.loc < y.loc; });
    uint64_t last = 0;  // uloc arithmetic: after the sort only exact repeats (and a first candidate at 0) are dropped
    int c = 0;
    for (int j = 0; j < m; ++j) {
      if (last - it[j].loc > (uint64_t)(int64_t)read_part_length) kept[b + c++] = it[j].idx;
      last = it[j].loc;
    }
    cnt[i] = c;
  });
  int64_t t = 0;
  for (int i = 0; i < n; ++i) {
    kept_start[i] = t;
    if (t != cand_start[i]) memmove(kept + t, kept + cand_start[i], (size_t)cnt[i] * 4);
    t += cnt[i];
  }
  kept_start[n] = t;
  return n;
}

int ngmlr_b200_score_short_reads(ngmlr_b200_ctx* ctx, int n, const int32_t* read_index, const uint64_t* locs,
                                 const uint8_t* reverse, float* scores) {
  if (!ctx) return -1;
  if (n < 0) return ctx->fail("score_short_reads: n < 0");
  CsState* cs = cs_state(ctx, false);
  if (check_short_ready(ctx, cs, "score_short_reads")) return -1;
  for (int i = 0; i < n; ++i) {
    if (read_index[i] < 0 || read_index[i] >= ctx->n_reads)
      return ctx->fail("score_short_reads: read index out of range at %d", i);
    if (ctx->read_len[read_index[i]] > 256)
      return ctx->fail("score_short_reads: read %d is longer than 256 bases", read_index[i]);
  }
  CU(cudaSetDevice(ctx->device));
  if (score_pairs(ctx, cs, n, read_index, locs, reverse, scores)) return -1;
  return n;
}

unsigned int ngmlr_b200_debug_short_read_general_pairs(ngmlr_b200_ctx* ctx) {
  CsState* cs = ctx ? cs_state(ctx, false) : nullptr;
  return cs ? cs->sr_general_pairs : 0u;
}

int ngmlr_b200_map_short_reads(ngmlr_b200_ctx* ctx, int read_part_length, float min_residues, int32_t* n_aln,
                               int64_t* first_aln, int32_t* mapped, const ngmlr_b200_sam_aln** alns,
                               int64_t* n_alns_total) {
  if (!ctx) return -1;
  if (!n_aln || !first_aln || !mapped || !alns || !n_alns_total) return ctx->fail("map_short_reads: NULL output");
  if (read_part_length < 1 || read_part_length > 256)
    return ctx->fail("map_short_reads: read_part_length must be in 1 .. 256");
  CsState* cs = cs_state(ctx, false);
  if (check_short_ready(ctx, cs, "map_short_reads")) return -1;
  if (!cs->reads_searched) return ctx->fail("map_short_reads: call cs_run on the uploaded reads first");
  CU(cudaSetDevice(ctx->device));
  const int nr = ctx->n_reads;
  const std::vector<int32_t>& len = ctx->read_len;
  // short read -> its (only) sub-read of the resident pipeline (ngmlr_b200_reads_upload's split)
  std::vector<int> sub((size_t)nr, -1), shorts;
  int64_t s = 0;
  for (int i = 0; i < nr; ++i) {
    const int parts = len[i] / read_part_length;
    if (len[i] <= read_part_length) {
      sub[i] = (int)s;
      shorts.push_back(i);
    }
    s += parts > 0 ? parts : 1;
  }
  if (s != cs->rn) return ctx->fail("map_short_reads: read_part_length differs from the one of reads_upload");
  std::vector<int64_t> cstart((size_t)cs->rn + 1);
  const float *cs_scores = nullptr, *sw = nullptr;
  const uint64_t* locs = nullptr;
  const uint8_t* rev = nullptr;
  if (ngmlr_b200_cs_fetch(ctx, cstart.data(), &cs_scores, &locs, &rev, &sw, nullptr) < 0) return -1;

  // (2) duplicate removal on each short read's candidates, in the reference's emission order
  const int ns = (int)shorts.size();
  std::vector<int64_t> sstart((size_t)ns + 1), kstart((size_t)ns + 1);
  std::vector<uint64_t> sloc;
  std::vector<uint8_t> srev;
  for (int j = 0; j < ns; ++j) {
    sstart[j] = (int64_t)sloc.size();
    const int sr = sub[shorts[j]];
    for (int64_t c = cstart[sr]; c < cstart[sr + 1]; ++c) {
      sloc.push_back(locs[c]);
      srev.push_back(rev[c]);
    }
  }
  sstart[ns] = (int64_t)sloc.size();
  std::vector<int32_t> kept(sloc.size() + 1);
  ngmlr_b200_dedupe_short_read_candidates(ns, sstart.data(), sloc.data(), read_part_length, kept.data(), kstart.data());
  const int np = (int)kstart[ns];
  std::vector<SrPair> pairs((size_t)np);
  std::vector<int32_t> pr((size_t)np + 1);
  std::vector<uint64_t> pl((size_t)np + 1);
  std::vector<uint8_t> pv((size_t)np + 1);
  for (int j = 0; j < ns; ++j)
    for (int64_t q = kstart[j]; q < kstart[j + 1]; ++q) {
      pairs[q] = SrPair{shorts[j], sloc[kept[q]], srev[kept[q]]};
      pr[q] = pairs[q].read;
      pl[q] = pairs[q].loc;
      pv[q] = pairs[q].rev;
    }
  // (3) scores against scoreShortRead's windows
  std::vector<float> score((size_t)np + 1);
  if (score_pairs(ctx, cs, np, pr.data(), pl.data(), pv.data(), score.data())) return -1;
  // (4) order by score from the location order + MQ: ScoreBuffer::topNSE's sort and computeMQ (0.75 cut unused)
  std::vector<int32_t> order((size_t)np + 1), kcount((size_t)ns + 1), mq((size_t)ns + 1);
  ngmlr_b200_select_candidates(ns, kstart.data(), score.data(), order.data(), kcount.data(), mq.data());

  // (5) processShortRead's loop as rounds
  std::vector<SrLoop> lp((size_t)ns);
  std::vector<int> live;
  for (int j = 0; j < ns; ++j) {
    lp[j].read = shorts[j];
    lp[j].first = (int)kstart[j];
    lp[j].m = (int)(kstart[j + 1] - kstart[j]);
    if (lp[j].m > 0) live.push_back(j);
  }
  std::vector<ngmlr_b200_interval> ivs;
  std::vector<int> batch;
  std::vector<ngmlr_b200_align_result> res;
  while (!live.empty()) {
    ivs.clear();
    batch.clear();
    for (int j : live) {
      SrLoop& L = lp[j];
      const int alignIndex = (int)L.kept.size();
      if (!(L.k < L.m && ((int)score[order[L.first + L.k]] >= L.last_score || alignIndex < 2))) continue;
      const int p = order[L.first + L.k];
      L.last_score = (int)score[p];
      const int rl = len[L.read];
      const int ref_extend = (int)(rl * 0.15f);
      ngmlr_b200_interval iv;
      memset(&iv, 0, sizeof(iv));
      iv.read_index = L.read;
      iv.on_read_start = 0;
      iv.read_seq_len = rl;
      iv.reverse = pairs[p].rev;
      iv.on_ref_start = pairs[p].loc - (uint64_t)(int64_t)ref_extend;
      iv.on_ref_stop = pairs[p].loc + (uint64_t)rl + (uint64_t)(int64_t)ref_extend;
      iv.corridor = read_part_length + 2 * ref_extend;
      iv.full_read_length = rl;
      iv.short_read = 1;
      ivs.push_back(iv);
      batch.push_back(j);
    }
    if (batch.empty()) break;
    res.resize(ivs.size());
    if (ngmlr_b200_compute_alignments(ctx, (int)ivs.size(), ivs.data(), nullptr, read_part_length, res.data(),
                                      nullptr) < 0)
      return -1;
    live.clear();
    for (size_t b = 0; b < batch.size(); ++b) {
      SrLoop& L = lp[batch[b]];
      const ngmlr_b200_align_result& r = res[b];
      const int rl = len[L.read];
      bool ok = r.ret >= 0 && r.score > 0.0f;
      if (ok) {
        if (min_residues < 1.0) ok = ((rl - r.qstart - r.qend) * 1.0f / rl) > min_residues;
        else ok = (rl - r.qstart - r.qend) > min_residues;
      }
      if (ok) {
        L.kept.push_back(order[L.first + L.k]);
        L.res.push_back(r);
        L.text.emplace_back(std::string(r.cigar ? r.cigar : ""), std::string(r.md ? r.md : ""));
      }
      ++L.k;
      live.push_back(batch[b]);
    }
  }

  // (6) records + SequenceProvider::convert (src/SequenceProvider.cpp:180-205)
  const auto& rs = cs->ref_starts;
  ctx->sr_alns.clear();
  ctx->sr_text.clear();
  for (int i = 0; i < nr; ++i) {
    n_aln[i] = sub[i] < 0 ? -1 : 0;
    first_aln[i] = 0;
    mapped[i] = 0;
  }
  for (int j = 0; j < ns; ++j) {
    SrLoop& L = lp[j];
    const int i = L.read;
    first_aln[i] = (int64_t)ctx->sr_alns.size();
    n_aln[i] = (int32_t)L.kept.size();
    bool is_mapped = false;
    for (size_t a = 0; a < L.kept.size(); ++a) {
      const ngmlr_b200_align_result& r = L.res[a];
      const int rl = len[i];
      const uint64_t loc = pairs[L.kept[a]].loc - (uint64_t)(int64_t)(int)(rl * 0.15f) + (uint64_t)(int64_t)r.position_offset;
      ngmlr_b200_sam_aln x;
      memset(&x, 0, sizeof(x));
      x.ref_pos = loc;
      x.ref_id = 0;  // an unconverted location keeps the candidate's reference id (0)
      const auto up = std::upper_bound(rs.begin(), rs.end(), (unsigned long long)loc);
      is_mapped = up != rs.end() && up != rs.begin() && *up - loc >= 1000ull;
      if (is_mapped) {
        x.ref_pos = loc - *(up - 1);
        x.ref_id = (int32_t)((up - 1) - rs.begin()) * 2;  // SequenceProvider ids count both strands
      }
      x.reverse = pairs[L.kept[a]].rev;
      x.score = r.score;
      x.mq = mq[j];
      x.nm = r.nm;
      x.identity = r.identity;
      x.qstart = r.qstart;
      x.qend = r.qend;
      x.sv_type = r.sv_type;
      x.primary = a == 0 ? 1 : 0;
      x.skip = 0;
      x.cigar_ops = r.cigar_op_count;
      ctx->sr_alns.push_back(x);
      ctx->sr_text.push_back(L.text[a].first);
      ctx->sr_text.push_back(L.text[a].second);
    }
    mapped[i] = is_mapped ? 1 : 0;  // WriteRead: the result of the LAST convert (the reference's "TODO: fix for -n > 1")
  }
  for (size_t a = 0; a < ctx->sr_alns.size(); ++a) {
    ctx->sr_alns[a].cigar = ctx->sr_text[2 * a].c_str();
    ctx->sr_alns[a].md = ctx->sr_text[2 * a + 1].c_str();
  }
  *alns = ctx->sr_alns.data();
  *n_alns_total = (int64_t)ctx->sr_alns.size();
  return nr;
}

}  // extern "C"
