// ngmlr_b200/csrc/convex_host.cu -- upload / run / fetch of a batch of convex alignments (C ABI,
// include/ngmlr_b200.h): packs the batch into the device arenas, launches fill -> traceback (+ the
// device text stage), and turns the results into the reference's `Align` fields.
#include "runtime.h"

using namespace nb;

namespace nb {

// One batch of SingleAlign problems -> device arenas. Every input comes in two forms (UploadSpec):
// reference windows as host text or as positions decoded on the device; reads as host text or as
// parts of the resident read set; corridors as CorridorLine arrays or in closed form. With the
// second form of all three, a problem costs ~150 bytes of H2D traffic and no per-row host work.
int convex_upload_spec(ngmlr_b200_ctx* ctx, const UploadSpec& sp) {
  if (!ctx) return -1;
  const int n = sp.n;
  if (n < 0) return ctx->fail("convex_upload: n < 0");
  CU(cudaSetDevice(ctx->device));
  ctx->ran = false;
  ctx->n = n;
  if (n == 0) return 0;
  const bool windows = sp.refs == nullptr, parts = sp.qrys == nullptr, forms = sp.forms != nullptr;
  if (windows && !sp.win) return ctx->fail("convex_upload: neither reference text nor windows given");
  if (parts && !sp.parts) return ctx->fail("convex_upload: neither read text nor read parts given");
  const int32_t* ref_lens = sp.ref_lens;
  const int32_t* qry_lens = sp.qry_lens;
  const int64_t* row_start = sp.row_start;
  // ---- sizes ----
  size_t seq_bytes = 0, rows = 0, nblocks = 0, tb_ints = 0;
  for (int i = 0; i < n; ++i) {
    if (ref_lens[i] < 0 || qry_lens[i] < 0) return ctx->fail("convex_upload: negative length at %d", i);
    if (!forms && row_start[i + 1] - row_start[i] != (int64_t)qry_lens[i])
      return ctx->fail("convex_upload: problem %d has %lld corridor rows for a %d-base read "
                       "(corridorHeight must equal qryLen)", i,
                       (long long)(row_start[i + 1] - row_start[i]), qry_lens[i]);
    seq_bytes += align_up((size_t)ref_lens[i] + SEQ_PAD, 16) + align_up((size_t)qry_lens[i] + SEQ_PAD, 16);
    if (!forms) rows += (size_t)qry_lens[i];
    nblocks += ((size_t)qry_lens[i] + 31) / 32;
  }
  if (!(windows && parts)) CU(ctx->h_seq.reserve(seq_bytes + 64));
  if (!forms) {
    CU(ctx->h_coff.reserve(rows + 32));
    CU(ctx->h_clen.reserve(rows + 32));
    CU(ctx->h_delta.reserve(rows + 32));
    CU(ctx->h_blkbase.reserve(nblocks + 1));
  }
  ctx->is_packed.assign(n, 0);
  CU(ctx->h_desc.reserve(n));
  CU(ctx->h_order.reserve(n));
  ctx->ext_qs.assign(n, 0);
  ctx->ext_qe.assign(n, 0);
  // ---- pack (parallel over problems) ----
  const double t_pack0 = now_ms();
  const int64_t r0 = forms ? 0 : row_start[0];
  std::vector<size_t> ref_at(n), qry_at(n), blk_at(n), tb_at(n);
  // Layout of the sequence arena: all reference windows first when they are decoded on the device
  // (one contiguous region to bring back for the host text stage), reads after them.
  size_t ref_region = 0;
  if (windows)
    for (int i = 0; i < n; ++i) ref_region += align_up((size_t)ref_lens[i] + SEQ_PAD, 16);
  {
    size_t so_ = 0, ro_ = 0, qo_ = ref_region, bo_ = 0, tb_ = 0;
    for (int i = 0; i < n; ++i) {
      const int rl = ref_lens[i], ql = qry_lens[i];
      const size_t rspan = align_up((size_t)rl + SEQ_PAD, 16), qspan = align_up((size_t)ql + SEQ_PAD, 16);
      if (!windows) {
        ref_at[i] = so_;
        qry_at[i] = so_ + rspan;
        so_ += rspan + qspan;
      } else {
        ref_at[i] = ro_;
        qry_at[i] = qo_;
        ro_ += rspan;
        qo_ += qspan;
      }
      blk_at[i] = bo_;
      bo_ += ((size_t)ql + 31) / 32;
      tb_at[i] = tb_;
      const long long ref_cap = ql > 200000 ? (long long)ql + 1 : 200000;  // maxBinaryCigarLength (:480-485)
      tb_ += (size_t)std::min<long long>((long long)ql + rl + 4, ref_cap);
    }
    tb_ints = tb_;
  }
  std::vector<unsigned long long> est(n);
  std::vector<size_t> dirw(n), dirw_rf(n);
  std::vector<int> maxlen(n);
  std::vector<uint8_t> orderly(n);  // corridor never moves left and rows are never empty in the middle
  parallel_for(n, forms ? 256 : 16, [&](int i) {
    AlnDesc& d = ctx->h_desc.p[i];
    memset(&d, 0, sizeof(d));
    const int rl = ref_lens[i], ql = qry_lens[i];
    d.ref_off = ref_at[i];
    if (!windows) {
      memcpy(ctx->h_seq.p + ref_at[i], sp.refs[i], rl);
      memset(ctx->h_seq.p + ref_at[i] + rl, 0, align_up((size_t)rl + SEQ_PAD, 16) - rl);
    }
    d.qry_off = qry_at[i];
    if (!parts) {
      memcpy(ctx->h_seq.p + qry_at[i], sp.qrys[i], ql);
      memset(ctx->h_seq.p + qry_at[i] + ql, 0, align_up((size_t)ql + SEQ_PAD, 16) - ql);
    }
    d.row_off = forms ? 0 : (uint64_t)(row_start[i] - r0);
    d.blk_off = blk_at[i];
    d.ref_len = rl;
    d.height = ql;
    d.ref_cap = ql > 200000 ? ql + 1 : 200000;
    d.tb_cap = (int)std::min<long long>((long long)ql + rl + 4, d.ref_cap);
    d.tb_off = tb_at[i];
    d.ext_qstart = sp.ext_qstart ? sp.ext_qstart[i] : 0;
    d.ext_qend = sp.ext_qend ? sp.ext_qend[i] : 0;
    int ml = 0;
    unsigned long long sum = 0;
    long long first_off = 0, last_off = 0;
    if (forms) {
      const CorridorForm& f = sp.forms[i];
      d.packed = 2;
      d.const_len = f.width;
      d.ckind = f.kind;
      d.c0 = f.c0;
      d.cstep = f.cstep;
      d.cd = f.d;
      d.ck = f.k;
      d.cright = f.right;
      ml = f.width;
      sum = (unsigned long long)std::max(f.width, 0) * (unsigned long long)ql;
      if (ql > 0) {
        first_off = corridor_form_offset(f, 0);
        last_off = corridor_form_offset(f, ql - 1);
      }
      ctx->is_packed[i] = 2;
      orderly[i] = f.width > 0 && (f.kind == 0 ? f.cstep >= 0 : f.k > 0.0f);
    } else {
      // Corridor rows: one pass that writes the packed form (int8 offset deltas + one base per 32-row
      // block) and finds out whether it is exact for this problem (constant length, |delta| < 128);
      // only problems that fail ship their raw CorridorLines.
      const int32_t* src_off = sp.corridor_offsets + row_start[i];
      const int32_t* src_len = sp.corridor_lengths + row_start[i];
      int8_t* delta = ctx->h_delta.p + d.row_off;
      int32_t* blkbase = ctx->h_blkbase.p + d.blk_off;
      bool packable = !ctx->no_corridor_packing && ql > 0;
      bool mono = true;
      const int len0 = ql ? src_len[0] : 0;
      for (int y = 0; y < ql; ++y) {
        const int ln = src_len[y];
        ml = std::max(ml, ln);
        sum += (unsigned long long)std::max(ln, 0);
        const long long dl = y ? (long long)src_off[y] - (long long)src_off[y - 1] : 0;
        packable = packable && ln == len0 && dl >= -128 && dl <= 127;
        mono = mono && dl >= 0 && ln > 0;
        delta[y] = (int8_t)dl;
        if ((y & 31) == 0) blkbase[y >> 5] = src_off[y];
      }
      if (!packable && ql) {
        memcpy(ctx->h_coff.p + d.row_off, src_off, (size_t)ql * sizeof(int32_t));
        memcpy(ctx->h_clen.p + d.row_off, src_len, (size_t)ql * sizeof(int32_t));
      }
      d.packed = packable ? 1 : 0;
      d.const_len = len0;
      ctx->is_packed[i] = packable ? 1 : 0;
      orderly[i] = mono;
      if (ql > 0) {
        first_off = src_off[0];
        last_off = src_off[ql - 1];
      }
    }
    d.max_len = ml;
    maxlen[i] = std::min(ml, rl);
    est[i] = sum;
    // direction arena estimate: per 32-row block, steps = row width + 31 (stagger) + corridor
    // advance over the block; for the ramp-free kernel at least what its hand-off spacing costs a
    // narrow corridor. The exact figure is computed by the kernel (bump allocation) and an
    // overflow triggers a re-run with a larger arena.
    dirw[i] = dirw_rf[i] = 0;
    if (ql > 0) {
      const long long adv_total = std::max<long long>(0, last_off - first_off);
      const long long adv = (adv_total * 32 + std::max(ql - 1, 1) - 1) / std::max(ql - 1, 1) + 2;
      const long long w = std::min<long long>(ml, (long long)rl);
      const long long steps = w + 31 + adv, steps_rf = std::max<long long>(steps, RF_MIN_BLOCK_STEPS);
      dirw[i] = (size_t)(((size_t)ql + 31) / 32) * (size_t)((steps + 15) / 16 + 1) * 32;
      dirw_rf[i] = (size_t)(((size_t)ql + 31) / 32) * (size_t)((steps_rf + 15) / 16 + 1) * 32;
    }
  });
  int max_len_all = 0;
  size_t dir_words = 0, dir_words_rf = 0, qry_total = 0, ref_total = 0;
  ctx->max_ref_len = 0;
  ctx->wide_problems = 0;
  ctx->team_safe = true;
  ctx->rf_wide = 0;
  ctx->rf_fits = true;
  for (int i = 0; i < n; ++i) {
    // The ramp-free kernel numbers the steps of a problem in an int: a block adds at most its column span
    // (<= refLen + 1) plus the hand-off and placement slack (< 400 steps) -- keep the total below 2^30.
    if ((((long long)qry_lens[i] + 31) / 32) * ((long long)ref_lens[i] + 400) >= (1ll << 30)) ctx->rf_fits = false;
    if (!orderly[i]) ctx->team_safe = false;
    if (maxlen[i] >= 352) ctx->wide_problems++;
    if (maxlen[i] >= RF_MIN_WIDTH) ctx->rf_wide++;
    max_len_all = std::max(max_len_all, maxlen[i]);
    ctx->max_ref_len = std::max(ctx->max_ref_len, ref_lens[i]);
    dir_words += dirw[i];
    dir_words_rf += dirw_rf[i];
    qry_total += (size_t)qry_lens[i];
    ref_total += (size_t)ref_lens[i];
    ctx->ext_qs[i] = ctx->h_desc.p[i].ext_qstart;
    ctx->ext_qe[i] = ctx->h_desc.p[i].ext_qend;
  }
  const size_t so = seq_bytes, bo = nblocks;
  // Largest first (LPT); the few huge and wide matrices of a batch -- realignments, full matrices, corridors
  // widened by the anchors around a long indel -- lead the order: they get FILL_BIG_TEAM-warp teams.
  std::vector<uint8_t> big(n);
  int n_big = 0;
  for (int i = 0; i < n; ++i) {
    big[i] = est[i] >= ctx->big_cells && maxlen[i] >= ctx->big_width;
    n_big += big[i];
  }
  ctx->n_big = n_big;
  ctx->rf_team = 0;
  for (int i = 0; i < n; ++i) ctx->rf_team += !big[i] && est[i] >= ctx->rf_team_cells;
  std::iota(ctx->h_order.p, ctx->h_order.p + n, 0);
  std::stable_sort(ctx->h_order.p, ctx->h_order.p + n,
                   [&](int a, int b) { return big[a] != big[b] ? big[a] > big[b] : est[a] > est[b]; });
  ctx->seq_bytes = so;
  ctx->rows = rows;
  ctx->nblocks = bo;
  ctx->tb_ints = tb_ints;
  ctx->max_len = max_len_all;
  ctx->dir_words_needed = dir_words + dir_words / 16 + 1024;
  ctx->dir_words_rf = dir_words_rf + dir_words_rf / 16 + 1024;
  ctx->windows_mode = windows;
  ctx->parts_mode = parts;
  ctx->forms_mode = forms;
  ctx->ref_region = ref_region;
  ctx->text_cap_hint = 3 * qry_total + ref_total / 4 + 64 * (size_t)n + 4096;
  const double t_pack1 = now_ms();
  // ---- device arenas + H2D ----
  cudaStream_t st = ctx->stream;
  CU(ctx->d_seq.reserve(so + 64));
  CU(ctx->d_coff.reserve(rows + 32));
  CU(ctx->d_clen.reserve(rows + 32));
  CU(ctx->d_desc.reserve(n));
  CU(ctx->d_order.reserve(n));
  CU(ctx->d_blocks.reserve(bo + 1));
  CU(ctx->d_fill.reserve(n));
  CU(ctx->d_trace.reserve(n));
  CU(ctx->d_scratch.reserve(tb_ints + 32));
  CU(ctx->d_runs.reserve(tb_ints / 4 + 4096));
  CU(ctx->d_counters.reserve(8));
  CU(ctx->h_counters.reserve(8));
  CU(ctx->h_fill.reserve(n));
  CU(ctx->h_trace.reserve(n));
  size_t h2d = 0;
  if (!windows && !parts) {
    CU(cudaMemcpyAsync(ctx->d_seq.p, ctx->h_seq.p, so, cudaMemcpyHostToDevice, st));
    h2d += so;
  } else if (windows && !parts) {
    CU(cudaMemcpyAsync(ctx->d_seq.p + ref_region, ctx->h_seq.p + ref_region, so - ref_region, cudaMemcpyHostToDevice, st));
    h2d += so - ref_region;
  } else if (!windows && parts) {  // references interleaved with (device-gathered) reads: ship the arena whole
    CU(cudaMemcpyAsync(ctx->d_seq.p, ctx->h_seq.p, so, cudaMemcpyHostToDevice, st));
    h2d += so;
  }
  if (windows || parts) {
    // descriptors of the windows / read parts -> device, then decode / gather straight into the arena
    const size_t nn = (size_t)n;
    const size_t aux_bytes = nn * (3 * 8 + 6 * 4 + 1) + 64;
    CU(ctx->h_aux.reserve(aux_bytes));
    CU(ctx->d_aux.reserve(aux_bytes));
    unsigned char* ha = ctx->h_aux.p;
    uint64_t* a_win = reinterpret_cast<uint64_t*>(ha);
    uint64_t* a_roff = a_win + nn;
    uint64_t* a_qoff = a_roff + nn;
    int32_t* a_wlen = reinterpret_cast<int32_t*>(a_qoff + nn);
    int32_t* a_rspan = a_wlen + nn;
    int32_t* a_ridx = a_rspan + nn;
    int32_t* a_pstart = a_ridx + nn;
    int32_t* a_plen = a_pstart + nn;
    int32_t* a_qspan = a_plen + nn;
    uint8_t* a_rc = reinterpret_cast<uint8_t*>(a_qspan + nn);
    for (int i = 0; i < n; ++i) {
      a_win[i] = windows ? sp.win->win_start[i] : 0;
      a_roff[i] = ref_at[i];
      a_qoff[i] = qry_at[i];
      a_wlen[i] = ref_lens[i] + 1;                                             // sequenceLength incl. NUL
      a_rspan[i] = (int32_t)align_up((size_t)ref_lens[i] + SEQ_PAD, 16);     // text + zero padding
      a_ridx[i] = parts ? sp.parts->read_index[i] : 0;
      a_pstart[i] = parts ? sp.parts->part_start[i] : 0;
      a_plen[i] = qry_lens[i];
      a_qspan[i] = (int32_t)align_up((size_t)qry_lens[i] + SEQ_PAD, 16);
      a_rc[i] = parts ? sp.parts->revcomp[i] : 0;
    }
    CU(cudaMemcpyAsync(ctx->d_aux.p, ha, aux_bytes - 64, cudaMemcpyHostToDevice, st));
    h2d += aux_bytes - 64;
    const unsigned char* da = ctx->d_aux.p;
    const uint64_t* d_win = reinterpret_cast<const uint64_t*>(da);
    const uint64_t* d_roff = d_win + nn;
    const uint64_t* d_qoff = d_roff + nn;
    const int32_t* d_wlen = reinterpret_cast<const int32_t*>(d_qoff + nn);
    if (windows) {
      RefDecodeParams rp;
      rp.enc = sp.win->d_enc;
      rp.ref_starts = sp.win->d_ref_starts;
      rp.n_starts = sp.win->n_starts;
      rp.n = n;
      rp.win_start = reinterpret_cast<const unsigned long long*>(d_win);
      rp.out_off = d_roff;
      rp.win_len = d_wlen;
      rp.out_span = d_wlen + nn;
      rp.out = ctx->d_seq.p;
      CU(launch_decode_windows(rp, st));
    }
    if (parts) {
      GatherParams gp;
      gp.reads = sp.parts->d_reads;
      gp.read_off = sp.parts->d_read_off;
      gp.n = n;
      gp.read_index = d_wlen + 2 * nn;
      gp.part_start = d_wlen + 3 * nn;
      gp.part_len = d_wlen + 4 * nn;
      gp.out_span = d_wlen + 5 * nn;
      gp.revcomp = reinterpret_cast<const uint8_t*>(d_wlen + 6 * nn);
      gp.out_off = d_qoff;
      gp.out = ctx->d_seq.p;
      CU(launch_gather_reads(gp, st));
    }
  }
  ctx->upload_d2h_bytes = 0;
  ctx->ref_on_host = !windows;
  if (!ctx->text_mode && (windows || parts)) {
    // the host text stage reads the reference windows: bring the device-made part of the arena back
    CU(ctx->h_seq.reserve(so + 64));
    const size_t back = windows ? ref_region : 0;
    if (back) CU(cudaMemcpyAsync(ctx->h_seq.p, ctx->d_seq.p, back, cudaMemcpyDeviceToHost, st));
    ctx->upload_d2h_bytes = (int64_t)back;
    ctx->ref_on_host = true;
  }
  size_t raw_rows = 0;
  if (!forms) {
    int raw_problems = 0;
    for (int i = 0; i < n; ++i)
      if (!ctx->is_packed[i]) {
        raw_rows += (size_t)qry_lens[i];
        ++raw_problems;
      }
    CU(ctx->d_delta.reserve(rows + 32));
    CU(ctx->d_blkbase.reserve(bo + 1));
    if (rows) {
      CU(cudaMemcpyAsync(ctx->d_delta.p, ctx->h_delta.p, rows, cudaMemcpyHostToDevice, st));
      CU(cudaMemcpyAsync(ctx->d_blkbase.p, ctx->h_blkbase.p, bo * sizeof(int32_t), cudaMemcpyHostToDevice, st));
      if (raw_problems > 64 || raw_rows * 2 > rows) {  // many raw problems: ship the arrays whole
        CU(cudaMemcpyAsync(ctx->d_coff.p, ctx->h_coff.p, rows * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(ctx->d_clen.p, ctx->h_clen.p, rows * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        raw_rows = rows;
      } else {
        for (int i = 0; i < n; ++i) {
          if (ctx->is_packed[i] || !qry_lens[i]) continue;
          const size_t ro = (size_t)ctx->h_desc.p[i].row_off, nb = (size_t)qry_lens[i] * sizeof(int32_t);
          CU(cudaMemcpyAsync(ctx->d_coff.p + ro, ctx->h_coff.p + ro, nb, cudaMemcpyHostToDevice, st));
          CU(cudaMemcpyAsync(ctx->d_clen.p + ro, ctx->h_clen.p + ro, nb, cudaMemcpyHostToDevice, st));
        }
      }
    }
    h2d += rows + bo * 4 + raw_rows * 8;
  } else {
    CU(ctx->d_delta.reserve(32));
    CU(ctx->d_blkbase.reserve(bo + 1));
  }
  CU(cudaMemcpyAsync(ctx->d_desc.p, ctx->h_desc.p, (size_t)n * sizeof(AlnDesc), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(ctx->d_order.p, ctx->h_order.p, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  h2d += (size_t)n * (sizeof(AlnDesc) + 4);
  CU(nb_stream_sync(ctx, st));
  ctx->stats = ngmlr_b200_batch_stats();
  ctx->stats.host_pack_ms = (float)(t_pack1 - t_pack0);
  ctx->stats.host_h2d_ms = (float)(now_ms() - t_pack1);
  ctx->stats.host_threads = host_threads();
  ctx->stats.h2d_bytes = (int64_t)h2d;
  ctx->stats.seq_bytes = (int64_t)so;
  return 0;
}

}  // namespace nb

extern "C" {

int ngmlr_b200_convex_upload(ngmlr_b200_ctx* ctx, int n, const char* const* refs,
                             const int32_t* ref_lens, const char* const* qrys,
                             const int32_t* qry_lens, const int32_t* corridor_offsets,
                             const int32_t* corridor_lengths, const int64_t* row_start,
                             const int32_t* ext_qstart, const int32_t* ext_qend) {
  if (ctx && n > 0 && (!refs || !qrys)) return ctx->fail("convex_upload: refs / qrys is NULL");
  UploadSpec sp;
  sp.n = n;
  sp.refs = refs;
  sp.ref_lens = ref_lens;
  sp.qrys = qrys;
  sp.qry_lens = qry_lens;
  sp.corridor_offsets = corridor_offsets;
  sp.corridor_lengths = corridor_lengths;
  sp.row_start = row_start;
  sp.ext_qstart = ext_qstart;
  sp.ext_qend = ext_qend;
  return convex_upload_spec(ctx, sp);
}

// Text stage: 0 = host threads (the reference's convertCigar restated in cigar_text.cpp; results
// carry the full nmPerPosition array), 1 = device (convex_text.cu: strings, scalars and the
// low-identity regions; nmPerPosition only when `want_nm_positions`). Takes effect at the next upload.
int ngmlr_b200_set_text_stage(ngmlr_b200_ctx* ctx, int on_device, int want_nm_positions) {
  if (!ctx) return -1;
  ctx->text_mode = on_device ? 1 : 0;
  ctx->want_nm = want_nm_positions ? 1 : 0;
  ctx->ran = false;
  return 0;
}

int ngmlr_b200_convex_run(ngmlr_b200_ctx* ctx) {
  if (!ctx) return -1;
  if (ctx->n == 0) {
    ctx->ran = true;
    return 0;
  }
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int n = ctx->n;
  const double t_run0 = now_ms();
  const bool raw = ctx->force_raw < 0 ? (ctx->raw || ctx->max_len > 32767) : (ctx->force_raw != 0);
  // Team mode (4 warps pipeline one problem) when the corridors are wide enough for the pipeline to
  // stay full (a warp must still be busy with its block when the fourth warp behind it has produced
  // the first chunk of the next one: ~4 x 100 columns); NGMLR_B200_FILL_TEAM=0/1 overrides.
  // Team mode also assumes what every corridor builder of the reference guarantees -- offsets never
  // decrease and no row is empty: a consumer warp may then skip its wait only behind a block without
  // cells at the very start or end of a problem. Anything else (raw C ABI input) runs one warp per problem.
  bool team = ctx->wide_problems * 2 > n;
  if (ctx->force_team >= 0) team = ctx->force_team != 0;
  team = team && ctx->team_safe;
  // Ramp-free schedule (convex_fill.cu, one warp per problem) when most corridors are at least RF_MIN_WIDTH wide:
  // narrower ones lose more to the schedule's boundary hand-off spacing than the ramp costs them. The largest
  // problems still get 4-warp teams, in a launch of their own (below). NGMLR_B200_FILL_TEAM=1 selects the ramped
  // teams for everything, NGMLR_B200_FILL_SCHEDULE=ramped the ramped kernels everywhere (DESIGN.md section 4.1).
  // (fill_schedule 2, NGMLR_B200_FILL_SCHEDULE=rampfree-all: every batch, whatever its widths -- test / tuning hook)
  const bool rampfree = ctx->fill_schedule >= 1 && ctx->force_team != 1 && ctx->rf_fits &&
                        (ctx->fill_schedule == 2 || ctx->rf_wide * 2 > n);
  if (rampfree) team = false;
  const int variant = (raw ? 1 : 0) | (team ? 2 : 0) | (rampfree ? 4 : 0);
  if (!ctx->ctas_per_sm[variant]) ctx->ctas_per_sm[variant] = std::max(1, fill_max_ctas_per_sm(raw, team, rampfree));
  int per_sm = std::min(ctx->ctas_per_sm[variant], team ? (int)FILL_TEAM_CTAS_PER_SM : (int)FILL_CTAS_PER_SM);
  if (ctx->fill_resident > 0) per_sm = std::min(per_sm, ctx->fill_resident);
  if (ctx->fill_ctas_cap > 0) per_sm = std::min(per_sm, ctx->fill_ctas_cap);
  const int max_grid = ctx->num_sms * per_sm;
  const int want_grid = team ? n : (n + FILL_WARPS_PER_CTA - 1) / FILL_WARPS_PER_CTA;
  // Persistent launch (grid capped at what is resident, CTAs loop over problems) when a cap is set; otherwise
  // short-lived CTAs -- one problem per team / warp -- on a low-priority stream: SM slots keep coming free, and the
  // latency-bound kernels of this and the other contexts (candidate search, traceback, text: high-priority
  // streams) slip in beside the ALU-bound fill instead of queueing behind a grid that never lets go.
  const bool persistent = ctx->fill_ctas_cap > 0 || ctx->fill_persistent;
  const int grid = persistent ? std::max(1, std::min(max_grid, want_grid)) : std::max(1, want_grid);
  ctx->fill_grid = grid;
  const size_t strips = persistent ? (size_t)grid : (size_t)ctx->sm_ids * FILL_SM_SLOTS;
  const size_t warps = strips * (team ? 1 : FILL_WARPS_PER_CTA);  // a team shares one strip
  if (!persistent) {
    CU(ctx->d_sm_slots.reserve((size_t)ctx->sm_ids));
    if (!ctx->sm_slots_zeroed) {
      CU(cudaMemsetAsync(ctx->d_sm_slots.p, 0, (size_t)ctx->sm_ids * sizeof(unsigned int), st));
      ctx->sm_slots_zeroed = true;
    }
  }
  const size_t bnd_stride = align_up((size_t)ctx->max_ref_len + STRIP_SLACK, 8);
  // huge matrices: their own launch with FILL_BIG_TEAM-warp teams, concurrent with the rest (second stream)
  const bool big_ok = ctx->team_safe && ctx->force_team != 0 && !getenv("NGMLR_B200_NO_BIG_TEAMS");
  int n_big = big_ok ? ctx->n_big : 0;
  if (n_big > 2 * ctx->num_sms && n_big * 2 > n) n_big = 0;  // a batch of huge problems only: 4-warp teams fill the GPU
  // A batch smaller than the GPU (the plugin's SingleAlign batches: a handful of blocking callers) is latency, not
  // throughput: every problem gets an SM and a 16-warp team of its own.
  if (big_ok && n <= ctx->num_sms && ctx->small_batch_big_teams) n_big = n;
  const int big_grid = std::min(n_big, ctx->num_sms);
  // ramp-free schedule: the largest problems (they lead the order after the big ones) go to a persistent launch of
  // ramped 4-warp teams beside the one-warp launch, one CTA per SM at most
  const int n_team = rampfree && ctx->team_safe && ctx->force_team != 0 ? std::min(ctx->rf_team, n - n_big) : 0;
  const int team_grid = std::min(n_team, ctx->num_sms);
  CU(ctx->d_bnd.reserve((warps + (size_t)big_grid + (size_t)team_grid) * bnd_stride));
  size_t& words_needed = rampfree ? ctx->dir_words_rf : ctx->dir_words_needed;
  size_t dir_words = std::max(words_needed, (size_t)4096);
  if (ctx->debug_arena_words >= 0) {  // force the overflow -> grow -> re-run path (tests)
    dir_words = (size_t)ctx->debug_arena_words;
    ctx->d_dir.release();
  }
  size_t runs_cap = ctx->d_runs.cap;
  const bool dev_text = ctx->text_mode != 0;
  size_t text_cap = 0, peaks_cap = 0, nm_cap = 0;
  if (dev_text) {
    text_cap = std::max(ctx->d_text.cap, ctx->debug_arena_words >= 0 ? (size_t)256 : ctx->text_cap_hint);
    peaks_cap = std::max(ctx->d_peaks.cap, (size_t)n * 4 + 1024);
    nm_cap = ctx->want_nm ? std::max(ctx->d_nm.cap, (size_t)3 * (ctx->tb_ints + 64)) : 0;
    CU(ctx->d_textout.reserve(n));
    CU(ctx->h_textout.reserve(n));
  }
  bool need_fill = true;

  for (int attempt = 0; attempt < 24; ++attempt) {
    CU(ctx->d_dir.reserve(dir_words));
    CU(ctx->d_runs.reserve(runs_cap));
    if (need_fill) CU(cudaMemsetAsync(ctx->d_counters.p, 0, 8 * sizeof(unsigned long long), st));
    else CU(cudaMemsetAsync(ctx->d_counters.p + 4, 0, 4 * sizeof(unsigned long long), st));
    if (need_fill) {
      FillParams fp;
      fp.seq = ctx->d_seq.p;
      fp.c_off = ctx->d_coff.p;
      fp.c_len = ctx->d_clen.p;
      fp.c_blkbase = ctx->d_blkbase.p;
      fp.c_delta = ctx->d_delta.p;
      fp.desc = ctx->d_desc.p;
      fp.order = ctx->d_order.p;
      fp.n = n;
      fp.first = n_big + n_team;
      fp.last = n;
      fp.sm_slots = persistent ? nullptr : ctx->d_sm_slots.p;
      fp.sm_slot_count = std::min(per_sm, (int)FILL_SM_SLOTS);
      fp.problems_per_cta = 1;
      fp.blocks = ctx->d_blocks.p;
      fp.dir = ctx->d_dir.p;
      fp.dir_capacity = ctx->d_dir.cap;
      fp.dir_alloc = ctx->d_counters.p + 0;
      fp.work_counter = reinterpret_cast<int*>(ctx->d_counters.p + 2);
      fp.bnd = ctx->d_bnd.p;
      fp.bnd_stride = bnd_stride;
      fp.out = ctx->d_fill.p;
      fp.sc = ctx->sc;
      TraceParams tp;
      tp.seq = ctx->d_seq.p;
      tp.c_off = ctx->d_coff.p;
      tp.c_len = ctx->d_clen.p;
      tp.c_blkbase = ctx->d_blkbase.p;
      tp.c_delta = ctx->d_delta.p;
      tp.desc = ctx->d_desc.p;
      tp.order = ctx->d_order.p;
      tp.n = n;
      tp.blocks = ctx->d_blocks.p;
      tp.dir = ctx->d_dir.p;
      tp.fill = ctx->d_fill.p;
      tp.scratch = ctx->d_scratch.p;
      tp.out = ctx->d_trace.p;
      tp.runs = ctx->d_runs.p;
      tp.runs_capacity = ctx->d_runs.cap;
      tp.runs_alloc = ctx->d_counters.p + 1;
      CU(cudaEventRecord(ctx->ev[0], st));
      if (n_big > 0) {
        FillParams fb = fp;
        fb.first = 0;
        fb.last = n_big;
        fb.work_counter = reinterpret_cast<int*>(ctx->d_counters.p + 3);
        fb.sm_slots = nullptr;  // the few huge matrices: one resident 16-warp CTA per SM that loops
        fb.sm_slot_count = 0;
        fb.problems_per_cta = 0;
        fb.bnd = ctx->d_bnd.p + warps * bnd_stride;
        CU(cudaStreamWaitEvent(ctx->stream2, ctx->ev[0], 0));
        CU(launch_convex_fill_big(fb, raw, big_grid, ctx->stream2));
        CU(cudaEventRecord(ctx->ev_big, ctx->stream2));
      }
      if (n_team > 0) {
        FillParams ft = fp;
        ft.first = n_big;
        ft.last = n_big + n_team;
        ft.work_counter = reinterpret_cast<int*>(ctx->d_counters.p + 7);
        ft.sm_slots = nullptr;
        ft.sm_slot_count = 0;
        ft.problems_per_cta = 0;
        ft.bnd = ctx->d_bnd.p + (warps + (size_t)big_grid) * bnd_stride;
        CU(cudaStreamWaitEvent(ctx->stream3, ctx->ev[0], 0));
        CU(launch_convex_fill(ft, raw, true, false, team_grid, ctx->stream3));
        CU(cudaEventRecord(ctx->ev_team, ctx->stream3));
      }
      const int n_rest = n - n_big - n_team;
      if (n_rest > 0) {
        const int g = persistent ? grid : std::max(1, team ? n_rest : (n_rest + FILL_WARPS_PER_CTA - 1) / FILL_WARPS_PER_CTA);
        if (persistent || !ctx->stream_fill) {
          CU(launch_convex_fill(fp, raw, team, rampfree, g, st));
        } else {  // on the low-priority stream, between two events of the context's stream
          CU(cudaStreamWaitEvent(ctx->stream_fill, ctx->ev[0], 0));
          CU(launch_convex_fill(fp, raw, team, rampfree, g, ctx->stream_fill));
          CU(cudaEventRecord(ctx->ev_fill, ctx->stream_fill));
          CU(cudaStreamWaitEvent(st, ctx->ev_fill, 0));
        }
      }
      if (n_big > 0) CU(cudaStreamWaitEvent(st, ctx->ev_big, 0));
      if (n_team > 0) CU(cudaStreamWaitEvent(st, ctx->ev_team, 0));
      CU(cudaEventRecord(ctx->ev[1], st));
      CU(launch_convex_traceback(tp, st));
      CU(cudaEventRecord(ctx->ev[2], st));
      ctx->stats.fill_launches++;
      ctx->stats.traceback_launches++;
    }
    if (dev_text) {
      CU(ctx->d_text.reserve(text_cap));
      CU(ctx->d_peaks.reserve(peaks_cap));
      if (nm_cap) CU(ctx->d_nm.reserve(nm_cap));
      TextParams xp;
      xp.seq = ctx->d_seq.p;
      xp.desc = ctx->d_desc.p;
      xp.order = ctx->d_order.p;
      xp.n = n;
      xp.trace = ctx->d_trace.p;
      xp.runs = ctx->d_runs.p;
      xp.out = ctx->d_textout.p;
      xp.text = ctx->d_text.p;
      xp.text_capacity = ctx->d_text.cap;
      xp.text_alloc = ctx->d_counters.p + 4;
      xp.peaks = ctx->d_peaks.p;
      xp.peaks_capacity = ctx->d_peaks.cap;
      xp.peaks_alloc = ctx->d_counters.p + 5;
      xp.nm = ctx->want_nm ? ctx->d_nm.p : nullptr;
      xp.nm_capacity = ctx->want_nm ? ctx->d_nm.cap : 0;
      xp.nm_alloc = ctx->d_counters.p + 6;
      CU(cudaEventRecord(ctx->ev[6], st));
      CU(launch_convex_text(xp, st));
      CU(cudaEventRecord(ctx->ev[7], st));
      ctx->stats.text_launches++;
    }
    CU(cudaMemcpyAsync(ctx->h_counters.p, ctx->d_counters.p, 8 * sizeof(unsigned long long),
                       cudaMemcpyDeviceToHost, st));
    CU(nb_stream_sync(ctx, st));
    bool again = false;
    if (need_fill) {
      const unsigned long long dir_used = ctx->h_counters.p[0], runs_used = ctx->h_counters.p[1];
      if (dir_used > ctx->d_dir.cap) {
        // the counter under-reports after an overflow (warps stop allocating), so also double and
        // fall back to the host's estimate
        dir_words = std::max({(size_t)dir_used + (size_t)dir_used / 8 + 4096, (size_t)ctx->d_dir.cap * 2,
                              words_needed});
        again = true;
      }
      if (runs_used > ctx->d_runs.cap) {
        runs_cap = (size_t)runs_used + 4096;
        again = true;
      }
      ctx->dir_used = dir_used;
      ctx->runs_used = runs_used;
      need_fill = again;
    }
    if (dev_text && !again) {
      const unsigned long long tu = ctx->h_counters.p[4], pu = ctx->h_counters.p[5], nu = ctx->h_counters.p[6];
      if (tu > ctx->d_text.cap) {
        text_cap = (size_t)tu + (size_t)tu / 8 + 4096;
        again = true;
      }
      if (pu > ctx->d_peaks.cap) {
        peaks_cap = (size_t)pu * 2 + 1024;
        again = true;
      }
      if (ctx->want_nm && nu > ctx->d_nm.cap) {
        nm_cap = (size_t)nu + 4096;
        again = true;
      }
      ctx->text_used = tu;
      ctx->peaks_used = pu;
      ctx->nm_used = ctx->want_nm ? nu : 0;
    }
    if (!again) break;
    if (attempt == 23) return ctx->fail("convex_run: arena sizing did not converge");
  }
  words_needed = std::max(words_needed, (size_t)ctx->dir_used);
  if (rampfree) ctx->rf_problems += (unsigned long long)(n - n_big - n_team);
  float ms = 0;
  cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[1]);
  ctx->stats.fill_ms = ms;
  cudaEventElapsedTime(&ms, ctx->ev[1], ctx->ev[2]);
  ctx->stats.traceback_ms = ms;
  ctx->stats.compact_ms = 0.0f;  // compaction is fused into the traceback kernel (fields kept for ABI stability)
  ctx->stats.text_ms = 0.0f;
  if (dev_text) {
    cudaEventElapsedTime(&ms, ctx->ev[6], ctx->ev[7]);
    ctx->stats.text_ms = ms;
  }
  ctx->stats.dir_bytes = (int64_t)ctx->dir_used * 4;
  ctx->stats.cigar_runs = (int64_t)ctx->runs_used;
  ctx->stats.host_run_ms = (float)(now_ms() - t_run0);
  ctx->ran = true;
  return 0;
}

}  // extern "C"

namespace {

// Device text mode: results straight from the TextOut records and the pinned text / region arenas.
int fetch_device_text(ngmlr_b200_ctx* ctx, ngmlr_b200_align_result* results) {
  const int n = ctx->n;
  cudaStream_t st = ctx->stream;
  const int slot = std::max(0, std::min(ctx->text_slot, TEXT_SLOTS - 1));
  const double t_f0 = now_ms();
  CU(ctx->h_text[slot].reserve((size_t)ctx->text_used + 16));
  CU(ctx->h_peaks[slot].reserve((size_t)ctx->peaks_used + 4));
  if (ctx->nm_used) CU(ctx->h_nm[slot].reserve((size_t)ctx->nm_used + 4));
  CU(cudaMemcpyAsync(ctx->h_fill.p, ctx->d_fill.p, (size_t)n * sizeof(FillOut), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(ctx->h_trace.p, ctx->d_trace.p, (size_t)n * sizeof(TraceOut), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(ctx->h_textout.p, ctx->d_textout.p, (size_t)n * sizeof(TextOut), cudaMemcpyDeviceToHost, st));
  if (ctx->text_used)
    CU(cudaMemcpyAsync(ctx->h_text[slot].p, ctx->d_text.p, (size_t)ctx->text_used, cudaMemcpyDeviceToHost, st));
  if (ctx->peaks_used)
    CU(cudaMemcpyAsync(ctx->h_peaks[slot].p, ctx->d_peaks.p, (size_t)ctx->peaks_used * sizeof(int4),
                       cudaMemcpyDeviceToHost, st));
  if (ctx->nm_used)
    CU(cudaMemcpyAsync(ctx->h_nm[slot].p, ctx->d_nm.p, (size_t)ctx->nm_used * sizeof(int32_t),
                       cudaMemcpyDeviceToHost, st));
  CU(nb_stream_sync(ctx, st));
  const double t_f1 = now_ms();
  ctx->stats.d2h_bytes = (int64_t)((size_t)n * (sizeof(FillOut) + sizeof(TraceOut) + sizeof(TextOut)) +
                                   ctx->text_used + ctx->peaks_used * sizeof(int4) + ctx->nm_used * 4);
  const char* text = ctx->h_text[slot].p;
  const int4* peaks = ctx->h_peaks[slot].p;
  const int32_t* nmv = ctx->h_nm[slot].p;
  int64_t cells = 0, steps = 0;
  for (int i = 0; i < n; ++i) {
    const FillOut& f = ctx->h_fill.p[i];
    const TextOut& x = ctx->h_textout.p[i];
    ngmlr_b200_align_result& r = results[i];
    memset(&r, 0, sizeof(r));
    r.ret = -1;
    r.score = -1.0f;
    r.cigar = "";
    r.md = "";
    r.cells = (int64_t)f.cells;
    cells += (int64_t)f.cells;
    steps += ctx->h_trace.p[i].steps;
    if (x.status == TX_OVERFLOW || ctx->h_trace.p[i].status == ST_DIR_OVERFLOW)
      return ctx->fail("convex_fetch: internal arena overflow survived run()");
    if (ctx->h_trace.p[i].status == ST_THROW || x.status == TX_THROW) {
      r.threw = 1;
      continue;
    }
    if (x.status != TX_OK) continue;
    r.ret = x.ret;
    r.score = f.best_score;
    r.identity = x.identity;
    r.position_offset = ctx->h_trace.p[i].ref_position;
    r.qstart = x.qstart;
    r.qend = x.qend;
    r.nm = x.nm;
    r.alignment_length = x.alignment_length;
    r.cigar_op_count = x.cigar_op_count;
    r.sv_type = x.sv_type;
    r.first_ref = x.first_ref;
    r.first_read = x.first_read;
    r.last_ref = x.last_ref;
    r.last_read = x.last_read;
    r.nm_count = x.nm_count;
    r.cigar_len = x.cigar_len;
    r.md_len = x.md_len;
    r.cigar = text + x.text_off;
    r.md = text + x.text_off + x.cigar_len + 1;
    r.nm_positions = ctx->nm_used ? nmv + x.nm_off : nullptr;
    r.n_sv_regions = x.n_peaks;
    r.n_sv_regions_stored = x.n_peaks_stored;
    r.sv_regions = x.n_peaks_stored ? reinterpret_cast<const int32_t*>(peaks + x.peak_off) : nullptr;
  }
  ctx->stats.cells = cells;
  ctx->stats.path_steps = steps;
  ctx->stats.host_d2h_ms = (float)(t_f1 - t_f0);
  ctx->stats.host_text_ms = (float)(now_ms() - t_f1);
  ctx->stats.text_bytes = (int64_t)ctx->text_used;
  return 0;
}

}  // namespace

extern "C" {

int ngmlr_b200_convex_fetch(ngmlr_b200_ctx* ctx, ngmlr_b200_align_result* results) {
  if (!ctx) return -1;
  if (!ctx->ran) return ctx->fail("convex_fetch: call convex_run first");
  const int n = ctx->n;
  if (n == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  if (ctx->text_mode) return fetch_device_text(ctx, results);
  cudaStream_t st = ctx->stream;
  const double t_f0 = now_ms();
  CU(ctx->h_runs.reserve((size_t)ctx->runs_used + 16));
  CU(cudaMemcpyAsync(ctx->h_fill.p, ctx->d_fill.p, (size_t)n * sizeof(FillOut), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(ctx->h_trace.p, ctx->d_trace.p, (size_t)n * sizeof(TraceOut), cudaMemcpyDeviceToHost, st));
  if (ctx->runs_used)
    CU(cudaMemcpyAsync(ctx->h_runs.p, ctx->d_runs.p, (size_t)ctx->runs_used * sizeof(int32_t),
                       cudaMemcpyDeviceToHost, st));
  int64_t extra_d2h = 0;
  if (!ctx->ref_on_host) {
    // the text stage was switched to the host after an upload that left the sequences on the device
    CU(ctx->h_seq.reserve(ctx->seq_bytes + 64));
    CU(cudaMemcpyAsync(ctx->h_seq.p, ctx->d_seq.p, ctx->seq_bytes, cudaMemcpyDeviceToHost, st));
    extra_d2h = (int64_t)ctx->seq_bytes;
    ctx->ref_on_host = true;
  }
  CU(nb_stream_sync(ctx, st));
  const double t_f1 = now_ms();
  ctx->stats.d2h_bytes = (int64_t)((size_t)n * (sizeof(FillOut) + sizeof(TraceOut)) + ctx->runs_used * 4) +
                         ctx->upload_d2h_bytes + extra_d2h;
  if ((int)ctx->texts.size() < n) ctx->texts.resize(n);
  if ((int)ctx->host_peaks.size() < n) ctx->host_peaks.resize(n);
  for (int i = 0; i < n; ++i)
    if (ctx->h_trace.p[i].status == ST_DIR_OVERFLOW)
      return ctx->fail("convex_fetch: internal arena overflow survived run()");
  parallel_for(n, 8, [&](int i) {
    const AlnDesc& d = ctx->h_desc.p[i];
    const FillOut& f = ctx->h_fill.p[i];
    const TraceOut& t = ctx->h_trace.p[i];
    ngmlr_b200_align_result& r = results[i];
    memset(&r, 0, sizeof(r));
    r.ret = -1;
    r.score = -1.0f;  // align.Score = -1.0f on entry and on failure (:457, :537)
    r.cigar = "";
    r.md = "";
    r.cells = (int64_t)f.cells;
    if (t.status == ST_THROW) {
      r.threw = 1;
      return;
    }
    if (t.status != ST_OK) return;
    AlignText& tx = ctx->texts[i];
    const char* ref = reinterpret_cast<const char*>(ctx->h_seq.p + d.ref_off);
    if (!binary_cigar_to_text(ctx->h_runs.p + t.run_off, t.n_runs, ref, d.ref_len, t.ref_position,
                              ctx->ext_qs[i], ctx->ext_qe[i], tx)) {
      r.threw = 1;
      return;
    }
    r.ret = tx.ret;
    r.score = f.best_score;
    r.identity = tx.identity;
    r.position_offset = t.ref_position;
    r.qstart = tx.qstart;
    r.qend = tx.qend;
    r.nm = tx.nm;
    r.alignment_length = tx.alignment_length;
    r.cigar_op_count = tx.cigar_op_count;
    r.sv_type = tx.sv_type;
    r.first_ref = tx.first_ref;
    r.first_read = tx.first_read;
    r.last_ref = tx.last_ref;
    r.last_read = tx.last_read;
    r.nm_count = (int32_t)(tx.nm_positions.size() / 3);
    r.cigar_len = (int32_t)tx.cigar.size();
    r.md_len = (int32_t)tx.md.size();
    r.cigar = tx.cigar.c_str();
    r.md = tx.md.c_str();
    r.nm_positions = tx.nm_positions.data();
    std::vector<int32_t>& pk = ctx->host_peaks[i];
    r.n_sv_regions = scan_low_identity_regions(tx.nm_positions.data(), r.nm_count, tx.alignment_length, pk,
                                               TEXT_PEAK_CAP);
    r.n_sv_regions_stored = (int32_t)(pk.size() / 4);
    r.sv_regions = pk.empty() ? nullptr : pk.data();
  });
  int64_t cells = 0, steps = 0;
  for (int i = 0; i < n; ++i) {
    cells += (int64_t)ctx->h_fill.p[i].cells;
    steps += ctx->h_trace.p[i].steps;
  }
  ctx->stats.cells = cells;
  ctx->stats.path_steps = steps;
  ctx->stats.host_d2h_ms = (float)(t_f1 - t_f0);
  ctx->stats.host_text_ms = (float)(now_ms() - t_f1);
  return 0;
}

int ngmlr_b200_convex_align_batch(ngmlr_b200_ctx* ctx, int n, const char* const* refs,
                                  const int32_t* ref_lens, const char* const* qrys,
                                  const int32_t* qry_lens, const int32_t* corridor_offsets,
                                  const int32_t* corridor_lengths, const int64_t* row_start,
                                  const int32_t* ext_qstart, const int32_t* ext_qend,
                                  ngmlr_b200_align_result* results) {
  int rc = ngmlr_b200_convex_upload(ctx, n, refs, ref_lens, qrys, qry_lens, corridor_offsets,
                                    corridor_lengths, row_start, ext_qstart, ext_qend);
  if (rc) return rc;
  rc = ngmlr_b200_convex_run(ctx);
  if (rc) return rc;
  return ngmlr_b200_convex_fetch(ctx, results);
}

}  // extern "C"
