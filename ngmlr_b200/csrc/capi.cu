// ngmlr_b200/csrc/capi.cu -- host runtime + plain-C ABI (include/ngmlr_b200.h).
//
// Owns the device arenas (sequences, corridor rows, descriptors, direction arena, traceback
// strips), the pinned staging buffers and the stream; packs a batch of SingleAlign problems,
// launches fill -> traceback (which also compacts the binary CIGARs), and turns the binary CIGARs into the reference's `Align`
// fields. There is no CPU compute path: every entry point needs a CUDA device.
#include "runtime.h"

namespace nb {

int host_threads() {
  static int n = [] {
    const char* e = getenv("NGMLR_B200_HOST_THREADS");
    int v = e ? atoi(e) : 0;
    if (v <= 0) v = (int)std::min(32u, std::max(1u, std::thread::hardware_concurrency()));
    return v;
  }();
  return n;
}

}  // namespace nb

namespace {

using namespace nb;

std::string g_create_error;

}  // namespace

namespace nb {

// When may a batch take the scalar-rule kernel? The as-coded SSE fill (raw indelRun in the run tests) and the
// scalar rule differ only where a gap-open out of a cell that was itself reached through the *other* gap type ties
// with or beats the diagonal. Take an insertion opened below a deletion cell: with S = S(x-1, y-1),
//   U  = fl(fl(S + p) + open)   (p <= max(open, ext_min): the deletion's open or convex extension)
//   dg = fl(S + sub)            (sub >= min(match, mismatch))
// (the deletion opened right of an insertion cell is the same with the roles swapped). Exactly, U <= dg - margin with
//   margin = min(match, mismatch) - max(max(open, ext_min) + open)   (both gap kinds),
// and the three roundings move U - dg by at most 1.5 ulp(M), M a bound on the magnitude of S + max(p, 0) and dg.
// So U < dg, and the scalar rule equals the SSE fill, when open < 0 and margin > 1.5 ulp(M). The margin is an
// absolute number while ulp(M) grows with the scores: at (512,-64,-32.125,-32.125,-32.125,0.5) (margin 0.25, every
// option in ngmlr's CLI range) a 9 kb read scores ~4 M, where 1.5 ulp = 0.375, and the two rules do give different
// alignments (tests/test_scoring_oracle.py).
// The class test keeps its float form and 0.25 floor (what the oracle and the reference have been compared on); the
// magnitude test takes M from score_magnitude_bound() of the batch's largest problem. Default scoring
// (2,-5,-5,-5,-1,0.15), margin 1: scalar kernel until M reaches 2^23, i.e. reads and windows of about 2.9 M bases.
bool scoring_needs_raw(const Scoring& s, double magnitude) {
  const float sub_min = std::min(s.mat, s.mis);
  const bool in_class = s.open_read < 0.0f && s.open_ref < 0.0f &&
                        std::max(s.open_ref, s.ext_min) + s.open_read <= sub_min - 0.25f &&
                        std::max(s.open_read, s.ext_min) + s.open_ref <= sub_min - 0.25f;
  if (!in_class) return true;
  const double margin = (double)sub_min - std::max((double)std::max(s.open_ref, s.ext_min) + (double)s.open_read,
                                                   (double)std::max(s.open_read, s.ext_min) + (double)s.open_ref);
  int e = 0;
  std::frexp(magnitude, &e);  // magnitude in [2^(e-1), 2^e): float ulp 2^(e-24)
  const double ulp = magnitude > 0.0 ? std::ldexp(1.0, e - 24) : 0.0;
  return !(margin > 1.5 * ulp);
}

// Bound on the magnitude M above for one problem. A path to any cell takes at most min(qryLen, refLen) diagonal
// steps, each adding <= max(match, mismatch, 0), and at most qryLen + refLen gap steps, each adding <= max(open,
// ext_min, 0) (positive only through the C ABI); S is never below 0. Each of those <= qryLen + refLen float
// additions rounds by at most 2^-24 relative, which the last factor, exp(steps 2^-24) >= (1 + 2^-24)^steps, covers. Then S + max(p, 0) and |dg| add one gap
// and one substitution score.
double score_magnitude_bound(const Scoring& s, long long qry_len, long long ref_len) {
  const double gain = std::max({(double)s.mat, (double)s.mis, 0.0});
  const double gap = std::max({(double)s.open_read, (double)s.open_ref, (double)s.ext_min, 0.0});
  const double steps = (double)(qry_len + ref_len);
  const double smax = (gain * (double)std::min(qry_len, ref_len) + gap * steps) * std::exp(steps * 0x1p-24);
  return smax + gap + std::max(std::fabs((double)s.mat), std::fabs((double)s.mis));
}

}  // namespace nb

void nb_cs_release(ngmlr_b200_ctx* ctx);  // candidate-search state lives in a side table (below)

extern "C" {

int ngmlr_b200_abi_version(void) { return NGMLR_B200_ABI_VERSION; }

int ngmlr_b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

const char* ngmlr_b200_last_error(const ngmlr_b200_ctx* ctx) {
  return ctx ? ctx->error.c_str() : g_create_error.c_str();
}

int ngmlr_b200_create(int gpu_id, const ngmlr_b200_scoring* s, ngmlr_b200_ctx** out) {
  if (!out) return -1;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    g_create_error = std::string("ngmlr_b200: no CUDA device available (") + cudaGetErrorString(e) +
                     "); this library has no CPU fallback";
    return -1;
  }
  if (gpu_id < 0 || gpu_id >= count) {
    g_create_error = "ngmlr_b200: gpu_id out of range";
    return -1;
  }
  ngmlr_b200_ctx* ctx = new ngmlr_b200_ctx();
  ctx->device = gpu_id;
  if ((e = cudaSetDevice(gpu_id)) != cudaSuccess) {
    g_create_error = std::string("cudaSetDevice: ") + cudaGetErrorString(e);
    delete ctx;
    return -1;
  }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, gpu_id);
  ctx->num_sms = prop.multiProcessorCount;
  if (prop.major != 9 || prop.minor != 0) {  // only sm_90a SASS is embedded (no PTX for other architectures)
    g_create_error = "ngmlr_b200: kernels are built for sm_90a only; device is sm_" +
                     std::to_string(prop.major) + std::to_string(prop.minor);
    delete ctx;
    return -1;
  }
  ctx->sm_ids = fill_sm_id_bound();
  if (ctx->sm_ids <= 0) {
    g_create_error = "ngmlr_b200: could not read the SM id range of the device";
    delete ctx;
    return -1;
  }
  int prio_least = 0, prio_greatest = 0;
  cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
  // the context's stream (candidate search, traceback, text, copies) outranks its fill launches
  cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, prio_greatest);
  cudaStreamCreateWithPriority(&ctx->stream2, cudaStreamNonBlocking, prio_least);
  cudaStreamCreateWithPriority(&ctx->stream3, cudaStreamNonBlocking, prio_least);
  cudaStreamCreateWithPriority(&ctx->stream_fill, cudaStreamNonBlocking, prio_least);
  cudaEventCreateWithFlags(&ctx->ev_fill, cudaEventDisableTiming);
  if (const char* e = getenv("NGMLR_B200_FILL_PERSISTENT")) ctx->fill_persistent = atoi(e);
  if (const char* e = getenv("NGMLR_B200_SMALL_BATCH_BIG_TEAMS")) ctx->small_batch_big_teams = atoi(e);
  if (const char* e = getenv("NGMLR_B200_FILL_RESIDENT")) ctx->fill_resident = std::max(0, atoi(e));
  cudaEventCreateWithFlags(&ctx->ev_big, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ctx->ev_team, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ctx->ev_sync, cudaEventDisableTiming | cudaEventBlockingSync);
  if (const char* e = getenv("NGMLR_B200_SPIN_SYNC")) ctx->spin_sync = atoi(e) != 0;
  for (auto& ev : ctx->ev) cudaEventCreate(&ev);
  ngmlr_b200_scoring d = {2.0f, -5.0f, -5.0f, -5.0f, -1.0f, 0.15f};
  if (s) d = *s;
  ctx->sc.mat = d.match;
  ctx->sc.mis = d.mismatch;
  ctx->sc.open_read = d.gap_open;  // gap_open_read = gap_open_ref = gapOpen (:39-40)
  ctx->sc.open_ref = d.gap_open;
  ctx->sc.gap_ext = d.gap_extend;
  ctx->sc.ext_min = d.gap_extend_min;
  ctx->sc.decay = d.gap_decay;
  if (const char* e = getenv("NGMLR_B200_FILL_TEAM")) ctx->force_team = atoi(e);
  if (const char* e = getenv("NGMLR_B200_FILL_SCHEDULE")) {
    if (!strcmp(e, "ramped")) ctx->fill_schedule = 0;
    else if (!strcmp(e, "rampfree")) ctx->fill_schedule = 1;
    else if (!strcmp(e, "rampfree-all")) ctx->fill_schedule = 2;
    else {
      g_create_error = std::string("ngmlr_b200: NGMLR_B200_FILL_SCHEDULE=") + e + ": expected ramped, rampfree or rampfree-all";
      ngmlr_b200_destroy(ctx);
      return -1;
    }
  }
  if (const char* e = getenv("NGMLR_B200_FILL_ROWS_PER_LANE")) {
    if (!strcmp(e, "1")) ctx->rows_per_lane = 1;
    else if (!strcmp(e, "2")) ctx->rows_per_lane = 2;
    else {
      g_create_error = std::string("ngmlr_b200: NGMLR_B200_FILL_ROWS_PER_LANE=") + e + ": expected 1 or 2";
      ngmlr_b200_destroy(ctx);
      return -1;
    }
  }
  if (const char* e = getenv("NGMLR_B200_FILL_RF2_SKEW")) {
    if (!strcmp(e, "0")) ctx->rf2_skew = 0;
    else if (!strcmp(e, "1")) ctx->rf2_skew = 1;
    else {
      g_create_error = std::string("ngmlr_b200: NGMLR_B200_FILL_RF2_SKEW=") + e + ": expected 0 or 1";
      ngmlr_b200_destroy(ctx);
      return -1;
    }
  }
  if (const char* e = getenv("NGMLR_B200_RF_TEAM_CELLS")) ctx->rf_team_cells = strtoull(e, nullptr, 10);
  if (const char* e = getenv("NGMLR_B200_FILL_CTAS_PER_SM")) ctx->fill_ctas_cap = std::max(0, atoi(e));
  if (const char* e = getenv("NGMLR_B200_NO_CORRIDOR_PACKING")) ctx->no_corridor_packing = atoi(e);
  if (const char* e = getenv("NGMLR_B200_DEBUG_ARENA_CAP")) ctx->debug_arena_cap = std::max(-1LL, atoll(e));
  *out = ctx;
  return 0;
}

void ngmlr_b200_destroy(ngmlr_b200_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  nb_stream_sync(ctx, ctx->stream);
  nb_cs_release(ctx);
  ctx->h_seq.release(); ctx->h_coff.release(); ctx->h_clen.release(); ctx->h_order.release(); ctx->h_blkbase.release(); ctx->h_delta.release();
  ctx->h_desc.release(); ctx->h_fill.release(); ctx->h_trace.release(); ctx->h_runs.release();
  ctx->h_counters.release();
  ctx->d_seq.release(); ctx->d_coff.release(); ctx->d_clen.release(); ctx->d_order.release(); ctx->d_blkbase.release(); ctx->d_delta.release();
  ctx->d_desc.release(); ctx->d_blocks.release(); ctx->d_dir.release(); ctx->d_bnd.release();
  ctx->d_fill.release(); ctx->d_scratch.release(); ctx->d_trace.release(); ctx->d_runs.release();
  ctx->d_counters.release();
  ctx->h_sw_seq.release(); ctx->h_sw_off.release(); ctx->h_sw_len.release(); ctx->h_sw_out.release();
  ctx->d_sw_seq.release(); ctx->d_sw_off.release(); ctx->d_sw_len.release(); ctx->d_sw_out.release();
  ctx->d_sw_scratch.release();
  for (auto& ev : ctx->ev) cudaEventDestroy(ev);
  if (ctx->ev_big) cudaEventDestroy(ctx->ev_big);
  if (ctx->ev_team) cudaEventDestroy(ctx->ev_team);
  if (ctx->ev_sync) cudaEventDestroy(ctx->ev_sync);
  if (ctx->stream2) cudaStreamDestroy(ctx->stream2);
  if (ctx->stream3) cudaStreamDestroy(ctx->stream3);
  if (ctx->stream_fill) cudaStreamDestroy(ctx->stream_fill);
  if (ctx->ev_fill) cudaEventDestroy(ctx->ev_fill);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

int ngmlr_b200_set_stream(ngmlr_b200_ctx* ctx, void* s) {
  if (!ctx) return -1;
  cudaSetDevice(ctx->device);
  nb_stream_sync(ctx, ctx->stream);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  if (s) {
    ctx->stream = (cudaStream_t)s;
    ctx->own_stream = false;
  } else {
    int prio_least = 0, prio_greatest = 0;
    cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
    cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, prio_greatest);
    ctx->own_stream = true;
  }
  return 0;
}

void* ngmlr_b200_get_stream(ngmlr_b200_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

// Test hook: start convex_run with a direction arena of `words` 32-bit words (-1 = estimate).
int ngmlr_b200_debug_set_arena_words(ngmlr_b200_ctx* ctx, long long words) {
  if (!ctx) return -1;
  ctx->debug_arena_words = words;
  return 0;
}

// Test hooks: the device arenas of convex batches may hold at most `bytes` bytes (-1 = no cap; NGMLR_B200_DEBUG_ARENA_CAP
// sets it at creation), and what they hold now. A batch that needs more than the cap fails with "out of memory", as on
// a full device, deterministically and without touching the driver's limits.
int ngmlr_b200_debug_set_arena_cap(ngmlr_b200_ctx* ctx, long long bytes) {
  if (!ctx) return -1;
  ctx->debug_arena_cap = bytes < 0 ? -1 : bytes;
  return 0;
}

long long ngmlr_b200_debug_arena_bytes(ngmlr_b200_ctx* ctx) { return ctx ? (long long)ctx->arena_bytes : -1; }

int ngmlr_b200_release_arenas(ngmlr_b200_ctx* ctx) {
  if (!ctx) return -1;
  CU(cudaSetDevice(ctx->device));
  nb_stream_sync(ctx, ctx->stream);
  ctx->arena_release(ctx->d_seq); ctx->arena_release(ctx->d_coff); ctx->arena_release(ctx->d_clen);
  ctx->arena_release(ctx->d_order); ctx->arena_release(ctx->d_blkbase); ctx->arena_release(ctx->d_delta);
  ctx->arena_release(ctx->d_desc); ctx->arena_release(ctx->d_blocks); ctx->arena_release(ctx->d_dir);
  ctx->arena_release(ctx->d_bnd); ctx->arena_release(ctx->d_fill); ctx->arena_release(ctx->d_scratch);
  ctx->arena_release(ctx->d_trace); ctx->arena_release(ctx->d_runs); ctx->arena_release(ctx->d_counters);
  ctx->arena_release(ctx->d_aux); ctx->arena_release(ctx->d_sm_slots); ctx->arena_release(ctx->d_textout);
  ctx->arena_release(ctx->d_text); ctx->arena_release(ctx->d_peaks); ctx->arena_release(ctx->d_nm);
  ctx->sm_slots_zeroed = false;
  ctx->h_seq.release(); ctx->h_coff.release(); ctx->h_clen.release(); ctx->h_order.release(); ctx->h_blkbase.release();
  ctx->h_delta.release(); ctx->h_desc.release(); ctx->h_fill.release(); ctx->h_trace.release(); ctx->h_runs.release();
  ctx->h_counters.release(); ctx->h_aux.release(); ctx->h_textout.release();
  for (int s = 0; s < TEXT_SLOTS; ++s) {
    ctx->h_text[s].release();
    ctx->h_peaks[s].release();
    ctx->h_nm[s].release();
  }
  ctx->n = 0;
  ctx->ran = false;
  // a cudaMalloc that failed stays the thread's last error: the launch checks of the next batch must not see it
  cudaGetLastError();
  return 0;
}

// Cap the persistent fill grid at v CTAs per SM (0 = full occupancy, the default). With several
// contexts sharing a GPU a smaller grid per launch lets the launches of different contexts -- and
// their memory-bound candidate-search / traceback kernels -- reside on the SMs together.
// NGMLR_B200_FILL_CTAS_PER_SM sets the initial value. Tuning hook.
int ngmlr_b200_set_fill_ctas_per_sm(ngmlr_b200_ctx* ctx, int v) {
  if (!ctx) return -1;
  ctx->fill_ctas_cap = v > 0 ? v : 0;
  return 0;
}

int ngmlr_b200_set_small_batch_teams(ngmlr_b200_ctx* ctx, int on) {
  if (!ctx) return -1;
  ctx->small_batch_big_teams = on ? 1 : 0;
  return 0;
}

// Test hook (host only, no context): the CIGAR/MD/nmPerPosition text stage on a given binary CIGAR.
// Outputs: ints[0..11] = ret, qstart, qend, nm, alignment_length, cigar_op_count, sv_type, first_ref,
// first_read, last_ref, last_read, nm_count (triples); *identity; cigar/md NUL-terminated (truncated
// to the caps); nm_out receives min(3 * nm_count, nm_cap) ints. Returns 1, or 0 where the reference throws.
int ngmlr_b200_debug_cigar_text(const int32_t* runs, int n_runs, const char* ref, int ref_len, int ref_position,
                                int ext_qstart, int ext_qend, int32_t* ints, float* identity, char* cigar,
                                int cigar_cap, char* md, int md_cap, int32_t* nm_out, int nm_cap) {
  AlignText t;
  t.nm_positions.assign(7, -1);  // stale content of a reused buffer must not leak into the result
  const bool ok = binary_cigar_to_text(runs, n_runs, ref, ref_len, ref_position, ext_qstart, ext_qend, t);
  const int v[12] = {t.ret, t.qstart, t.qend, t.nm, t.alignment_length, t.cigar_op_count, t.sv_type, t.first_ref,
                     t.first_read, t.last_ref, t.last_read, (int)(t.nm_positions.size() / 3)};
  memcpy(ints, v, sizeof(v));
  *identity = t.identity;
  snprintf(cigar, (size_t)cigar_cap, "%s", t.cigar.c_str());
  snprintf(md, (size_t)md_cap, "%s", t.md.c_str());
  const size_t n = std::min(t.nm_positions.size(), (size_t)std::max(nm_cap, 0));
  if (n) memcpy(nm_out, t.nm_positions.data(), n * sizeof(int32_t));
  return ok ? 1 : 0;
}

// Test / tuning hook: which problems get FILL_BIG_TEAM-warp teams (cells and corridor width from which a
// matrix counts as huge; defaults 8 Mi cells, 768 columns).
int ngmlr_b200_debug_set_big_team(ngmlr_b200_ctx* ctx, long long cells, int width) {
  if (!ctx) return -1;
  ctx->big_cells = cells < 0 ? ~0ull : (unsigned long long)cells;
  ctx->big_width = width;
  return 0;
}

// Test hooks: problems filled by the ramp-free kernels since the context was created; of those, by the kernel with
// two rows per lane.
long long ngmlr_b200_debug_rampfree_problems(ngmlr_b200_ctx* ctx) { return ctx ? (long long)ctx->rf_problems : -1; }
long long ngmlr_b200_debug_rampfree2_problems(ngmlr_b200_ctx* ctx) { return ctx ? (long long)ctx->rf2_problems : -1; }
long long ngmlr_b200_debug_rampfree2_skew_problems(ngmlr_b200_ctx* ctx) {
  return ctx ? (long long)ctx->rf2_skew_problems : -1;
}

// Test hook: the fill's routing counters since the context was created, out[0..min(n, 9)) = problems filled by the
// 16-warp launch, by the ramp-free schedule's 4-warp team launch, by the ramp-free kernels, by the ramped one-warp
// kernel, by the ramped 4-warp team kernel (ordinary launch), by the RAW instantiation; fill launches, those with more
// than one of the three concurrent launches non-empty, and those with all three. Returns the number of entries written.
int ngmlr_b200_debug_fill_counts(ngmlr_b200_ctx* ctx, long long* out, int n) {
  if (!ctx || !out) return -1;
  const unsigned long long v[9] = {ctx->big_team_problems,    ctx->rf_team_problems,    ctx->rf_problems,
                                   ctx->ramped_warp_problems, ctx->ramped_team_problems, ctx->raw_problems,
                                   ctx->fill_launch_count,    ctx->multi_launch_count,  ctx->three_way_launch_count};
  const int k = std::max(0, std::min(n, 9));
  for (int i = 0; i < k; ++i) out[i] = (long long)v[i];
  return k;
}

// force_team: -1 auto, 0 one warp per problem, 1 four-warp teams. Test / tuning hook.
int ngmlr_b200_set_force_team(ngmlr_b200_ctx* ctx, int v) {
  if (!ctx) return -1;
  ctx->force_team = v;
  return 0;
}

// force_raw: -1 auto (by scoring), 0 scalar-rule kernel, 1 as-coded (RAW) kernel. Test hook.
int ngmlr_b200_set_force_raw(ngmlr_b200_ctx* ctx, int v) {
  if (!ctx) return -1;
  ctx->force_raw = v;
  return 0;
}

}  // extern "C"

extern "C" {

int ngmlr_b200_convex_stats(ngmlr_b200_ctx* ctx, ngmlr_b200_batch_stats* out) {
  if (!ctx || !out) return -1;
  *out = ctx->stats;
  return 0;
}

int ngmlr_b200_convex_debug_directions(ngmlr_b200_ctx* ctx, int i, uint8_t* dirs, size_t dirs_cap,
                                       float* best_score, int32_t* best_ref, int32_t* best_read) {
  if (!ctx) return -1;
  if (!ctx->ran || i < 0 || i >= ctx->n) return ctx->fail("debug_directions: bad state/index");
  CU(cudaSetDevice(ctx->device));
  const AlnDesc& d = ctx->h_desc.p[i];
  const int H = d.height;
  const size_t nblk = ((size_t)H + 31) / 32;
  std::vector<BlockRec> blocks(nblk);
  FillOut f;
  CU(cudaMemcpy(&f, ctx->d_fill.p + i, sizeof(f), cudaMemcpyDeviceToHost));
  if (nblk) CU(cudaMemcpy(blocks.data(), ctx->d_blocks.p + d.blk_off, nblk * sizeof(BlockRec), cudaMemcpyDeviceToHost));
  std::vector<int32_t> offs_v(H), lens_v(H);
  CorridorForm form = {d.ckind, d.c0, d.cstep, d.const_len, d.cd, d.ck, d.cright};
  for (int y = 0; y < H; ++y) {
    if (d.packed == 2) {
      offs_v[y] = corridor_form_offset(form, y);
      lens_v[y] = d.const_len;
    } else if (d.packed) {
      offs_v[y] = (y & 31) ? offs_v[y - 1] + ctx->h_delta.p[d.row_off + y] : ctx->h_blkbase.p[d.blk_off + (y >> 5)];
      lens_v[y] = d.const_len;
    } else {
      offs_v[y] = ctx->h_coff.p[d.row_off + y];
      lens_v[y] = ctx->h_clen.p[d.row_off + y];
    }
  }
  const int32_t* offs = offs_v.data();
  const int32_t* lens = lens_v.data();
  std::vector<char> ref_v((size_t)d.ref_len + 1), qry_v((size_t)H + 1);  // from the device: works for every input form
  if (d.ref_len) CU(cudaMemcpy(ref_v.data(), ctx->d_seq.p + d.ref_off, (size_t)d.ref_len, cudaMemcpyDeviceToHost));
  if (H) CU(cudaMemcpy(qry_v.data(), ctx->d_seq.p + d.qry_off, (size_t)H, cudaMemcpyDeviceToHost));
  const char* ref = ref_v.data();
  const char* qry = qry_v.data();
  size_t total = 0;
  for (int y = 0; y < H; ++y) total += (size_t)std::max(lens[y], 0);
  if (total > dirs_cap) return ctx->fail("debug_directions: buffer too small (%zu > %zu)", total, dirs_cap);
  memset(dirs, 0xFF, total);
  std::vector<uint32_t> words;
  size_t row_base = 0;
  for (size_t b = 0; b < nblk; ++b) {
    const BlockRec& br = blocks[b];
    const int sh = f.dir_shift == 2 ? 0 : f.dir_shift;  // step offset of row t: t >> sh (device_types.h BlockRec)
    const size_t stride = f.dir_shift ? 64 : 32, ng = (size_t)((br.nsteps + 15) / 16);
    const size_t nw = ng ? (ng - 1) * stride + 32 : 0;
    words.resize(nw);
    if (nw) CU(cudaMemcpy(words.data(), ctx->d_dir.p + br.word_off, nw * 4, cudaMemcpyDeviceToHost));
    for (int t = 0; t < 32; ++t) {
      const int y = (int)b * 32 + t;
      if (y >= H) break;
      const int lo = std::max(offs[y], 0);
      const int hi = (int)std::min<long long>((long long)offs[y] + lens[y], d.ref_len);
      for (int x = lo; x < hi; ++x) {
        const int s = x - br.base + (t >> sh);
        const uint32_t code = (words[(size_t)(s >> 4) * stride + t] >> ((s & 15) * 2)) & 3u;
        uint8_t v = OP_STOP;
        if (code == DIR_DIAG) v = qry[y] == ref[x] ? OP_EQ : OP_X;
        else if (code == DIR_I) v = OP_I;
        else if (code == DIR_D) v = OP_D;
        dirs[row_base + (size_t)(x - offs[y])] = v;
      }
      row_base += (size_t)std::max(lens[y], 0);
    }
  }
  if (best_score) *best_score = f.best_score;
  if (best_ref) *best_ref = f.best_x;
  if (best_read) *best_read = f.best_y;
  return 0;
}

int ngmlr_b200_sw_score_batch(ngmlr_b200_ctx* ctx, int n, const char* const* refs,
                              const char* const* qrys, float* results) {
  if (!ctx) return -1;
  if (n <= 0) return 0;
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  CU(ctx->h_sw_off.reserve((size_t)2 * n));
  CU(ctx->h_sw_len.reserve((size_t)2 * n));
  CU(ctx->h_sw_out.reserve(n));
  size_t bytes = 0;
  int max_ref = 0, max_qry = 0;
  for (int i = 0; i < n; ++i) {
    const size_t rl = strlen(refs[i]) + 1, ql = strlen(qrys[i]) + 1;  // NUL included (:130-131)
    ctx->h_sw_off.p[i] = bytes;
    ctx->h_sw_len.p[i] = (int32_t)std::min<size_t>(rl, 1u << 30);
    bytes += align_up(rl, 16);
    ctx->h_sw_off.p[n + i] = bytes;
    ctx->h_sw_len.p[n + i] = (int32_t)std::min<size_t>(ql, 1u << 30);
    bytes += align_up(ql, 16);
    if (rl < 100000 && ql < 100000) {
      max_ref = std::max(max_ref, (int)rl);
      max_qry = std::max(max_qry, (int)ql);
    }
  }
  CU(ctx->h_sw_seq.reserve(bytes + 16));
  for (int i = 0; i < n; ++i) {
    memcpy(ctx->h_sw_seq.p + ctx->h_sw_off.p[i], refs[i], (size_t)ctx->h_sw_len.p[i]);
    memcpy(ctx->h_sw_seq.p + ctx->h_sw_off.p[n + i], qrys[i], (size_t)ctx->h_sw_len.p[n + i]);
  }
  CU(ctx->d_sw_seq.reserve(bytes + 16));
  CU(ctx->d_sw_off.reserve((size_t)2 * n));
  CU(ctx->d_sw_len.reserve((size_t)2 * n));
  CU(ctx->d_sw_out.reserve(n));
  const int warps_per_cta = 4;
  const int grid = std::max(1, std::min(ctx->num_sms * 8, (n + warps_per_cta - 1) / warps_per_cta));
  const size_t stride = max_qry > 288 ? align_up((size_t)max_ref + 2, 4) : 4;
  CU(ctx->d_sw_scratch.reserve((size_t)grid * warps_per_cta * stride * 2));
  CU(cudaMemcpyAsync(ctx->d_sw_seq.p, ctx->h_sw_seq.p, bytes, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(ctx->d_sw_off.p, ctx->h_sw_off.p, (size_t)2 * n * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(ctx->d_sw_len.p, ctx->h_sw_len.p, (size_t)2 * n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  SwParams sp;
  memset(&sp, 0, sizeof(sp));
  sp.seq = ctx->d_sw_seq.p;
  sp.ref_off = ctx->d_sw_off.p;
  sp.qry_off = ctx->d_sw_off.p + n;
  sp.ref_len = ctx->d_sw_len.p;
  sp.qry_len = ctx->d_sw_len.p + n;
  sp.out = ctx->d_sw_out.p;
  sp.n = n;
  sp.scratch = ctx->d_sw_scratch.p;
  sp.scratch_stride = stride;
  CU(cudaEventRecord(ctx->ev[4], st));
  CU(launch_sw_score(sp, grid, max_qry, max_ref - 1, st));
  CU(cudaEventRecord(ctx->ev[5], st));
  CU(cudaMemcpyAsync(ctx->h_sw_out.p, ctx->d_sw_out.p, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, st));
  CU(nb_stream_sync(ctx, st));
  memcpy(results, ctx->h_sw_out.p, (size_t)n * sizeof(float));
  return n;
}

float ngmlr_b200_sw_last_kernel_ms(ngmlr_b200_ctx* ctx) {
  float ms = 0;
  if (ctx) cudaEventElapsedTime(&ms, ctx->ev[4], ctx->ev[5]);
  return ms;
}

}  // extern "C"

// ============================================================================================
// candidate search
// ============================================================================================
namespace {

std::vector<std::pair<ngmlr_b200_ctx*, CsState*>> g_cs_states;
std::mutex* g_cs_mutex = new std::mutex();

}  // namespace

namespace nb {
CsState* cs_state(ngmlr_b200_ctx* ctx, bool create) {
  std::lock_guard<std::mutex> lock(*g_cs_mutex);
  for (auto& kv : g_cs_states)
    if (kv.first == ctx) return kv.second;
  if (!create) return nullptr;
  g_cs_states.emplace_back(ctx, new CsState());
  return g_cs_states.back().second;
}
}  // namespace nb

void nb_cs_release(ngmlr_b200_ctx* ctx) {
  std::lock_guard<std::mutex> lock(*g_cs_mutex);
  for (size_t i = 0; i < g_cs_states.size(); ++i) {
    if (g_cs_states[i].first != ctx) continue;
    CsState* cs = g_cs_states[i].second;
    cs->d_packed.release(); cs->d_tab.release(); cs->d_pos.release(); cs->d_order.release(); cs->d_ref_starts.release();
    cs->d_used.release(); cs->d_seq.release(); cs->d_tables.release(); cs->d_off.release();
    cs->d_len.release(); cs->d_count.release(); cs->d_cap.release(); cs->d_hits.release();
    cs->d_max.release(); cs->d_out.release(); cs->d_enc.release(); cs->d_rev.release();
    cs->d_winpos.release(); cs->d_qoff.release(); cs->d_qlen.release(); cs->d_sw.release();
    cs->d_swscratch.release(); cs->d_a.release(); cs->d_b.release(); cs->d_c.release();
    cs->d_sa.release(); cs->d_sb.release(); cs->d_sc.release(); cs->d_cnt64.release();
    cs->d_cstart.release(); cs->d_cloc.release(); cs->d_scan_tmp.release(); cs->d_cscore.release();
    if (cs->ev0) cudaEventDestroy(cs->ev0);
    if (cs->ev1) cudaEventDestroy(cs->ev1);
    cs->p_seq.release(); cs->p_rev.release(); cs->p_score.release(); cs->p_sw.release(); cs->p_loc.release();
    delete cs;
    g_cs_states.erase(g_cs_states.begin() + i);
    return;
  }
}

extern "C" {

int ngmlr_b200_cs_set_index(ngmlr_b200_ctx* ctx, const void* packed_index, uint32_t index_len,
                            const uint32_t* positions, uint32_t n_positions, uint64_t unit_offset,
                            int k, int bin_shift) {
  if (!ctx) return -1;
  if (k < 1 || k > 16) return ctx->fail("cs_set_index: k must be in 1..16");
  if (index_len != (1u << (2 * k)) + 1u) return ctx->fail("cs_set_index: index_len must be 4^k + 1");
  CU(cudaSetDevice(ctx->device));
  CsState* cs = cs_state(ctx, true);
  cudaStream_t st = ctx->stream;
  CU(cs->d_packed.reserve((size_t)index_len * 5));
  CU(cs->d_tab.reserve((size_t)index_len + 1));
  CU(cs->d_used.reserve(((size_t)index_len + 255) / 256 * 8 + 8));  // one word per 32 prefixes, whole blocks
  CU(cs->d_pos.reserve((size_t)n_positions + 1));
  CU(cudaMemcpyAsync(cs->d_packed.p, packed_index, (size_t)index_len * 5, cudaMemcpyHostToDevice, st));
  if (n_positions)
    CU(cudaMemcpyAsync(cs->d_pos.p, positions, (size_t)n_positions * 4, cudaMemcpyHostToDevice, st));
  CU(launch_unpack_index(cs->d_packed.p, index_len, cs->d_tab.p, cs->d_used.p, st));
  {  // m_RevCompIndex, kept for cs_get_index
    std::vector<int8_t> rci(index_len);
    const uint8_t* src = static_cast<const uint8_t*>(packed_index);
    for (size_t i = 0; i < index_len; ++i) rci[i] = (int8_t)src[5 * i + 4];
    CU(cs->d_rci.reserve((size_t)index_len + 1));
    CU(cudaMemcpyAsync(cs->d_rci.p, rci.data(), index_len, cudaMemcpyHostToDevice, st));
    CU(nb_stream_sync(ctx, st));
  }
  CU(nb_stream_sync(ctx, st));
  cs->d_packed.release();
  cs->index_len = index_len;
  cs->n_pos = n_positions;
  cs->unit_offset = unit_offset;
  cs->k = k;
  cs->bin_shift = bin_shift;
  return 0;
}

// Several contexts on one GPU (one per host thread, as the reference has one aligner object per worker
// thread) need the same encoded reference and k-mer index: `ctx` uses the device arrays of `owner` instead of
// holding copies. `owner` must outlive `ctx` and must not replace its reference / index meanwhile.
int ngmlr_b200_cs_share_reference(ngmlr_b200_ctx* ctx, ngmlr_b200_ctx* owner) {
  if (!ctx || !owner) return -1;
  if (ctx == owner) return 0;
  if (ctx->device != owner->device) return ctx->fail("cs_share_reference: contexts live on different devices");
  CsState* from = cs_state(owner, false);
  if (!from || !from->enc_bytes) return ctx->fail("cs_share_reference: the owner has no reference");
  CsState* cs = cs_state(ctx, true);
  cs->d_enc.borrow(from->d_enc);
  cs->enc_bytes = from->enc_bytes;
  cs->concat_len = from->concat_len;
  cs->d_ref_starts.borrow(from->d_ref_starts);
  cs->ref_starts = from->ref_starts;
  if (from->index_len) {
    cs->d_tab.borrow(from->d_tab);
    cs->d_used.borrow(from->d_used);
    cs->d_rci.borrow(from->d_rci);
    cs->d_pos.borrow(from->d_pos);
    cs->index_len = from->index_len;
    cs->n_pos = from->n_pos;
    cs->unit_offset = from->unit_offset;
    cs->k = from->k;
    cs->bin_shift = from->bin_shift;
  }
  return 0;
}

// Builds the k-mer index of the encoded reference that is resident on the device (cs_set_reference) and
// installs it as the context's index: CompactPrefixTable::CreateTable on the GPU (cs_index_build.cu).
int ngmlr_b200_cs_build_index(ngmlr_b200_ctx* ctx, const uint64_t* contig_start, const uint64_t* contig_len,
                              int n_contigs, int k, int kmer_skip, int bin_shift, int max_prefix_freq,
                              uint32_t* n_positions) {
  if (!ctx) return -1;
  CsState* cs = cs_state(ctx, false);
  if (!cs || !cs->enc_bytes) return ctx->fail("cs_build_index: call cs_set_reference first");
  if (k < 1 || k > 15) return ctx->fail("cs_build_index: k must be in 1..15");
  if (n_contigs < 1 || kmer_skip < 0 || max_prefix_freq < 1) return ctx->fail("cs_build_index: bad arguments");
  if (cs->concat_len >= 0xffff0000ull) return ctx->fail("cs_build_index: one table unit holds < 4 G positions");
  if (!index_build_fits(cs->concat_len, n_contigs, kmer_skip))
    return ctx->fail("cs_build_index: %llu positions give more k-mer callbacks than the build sorts (2^31) at kmer_skip %d",
                     (unsigned long long)cs->concat_len, kmer_skip);
  for (int i = 0; i < n_contigs; ++i) {
    if (i && contig_start[i] < contig_start[i - 1] + contig_len[i - 1]) return ctx->fail("cs_build_index: contigs must be sorted and disjoint");
    if (contig_start[i] + contig_len[i] > cs->concat_len) return ctx->fail("cs_build_index: contig %d leaves the reference", i);
  }
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const unsigned long long cl = cs->concat_len;
  const uint32_t n_kmers = 1u << (2 * k);
  const unsigned long long cb_cap = cl / (unsigned long long)(kmer_skip + 1) + (unsigned long long)n_contigs * 64 + 1024;
  DevBuf<uint32_t> lastn, prefix, pos, key, key_out, pos_out, freq, alloc_cnt, used_cnt, alloc_start, used_start;
  DevBuf<uint8_t> flag, keep, cub_tmp;
  DevBuf<unsigned long long> d_contigs;
  CU(lastn.reserve(cl + 16));
  CU(flag.reserve(cl + 16));
  CU(prefix.reserve(cb_cap)); CU(pos.reserve(cb_cap)); CU(key.reserve(cb_cap)); CU(key_out.reserve(cb_cap)); CU(pos_out.reserve(cb_cap));
  CU(keep.reserve(cb_cap));
  CU(freq.reserve(n_kmers + 2)); CU(alloc_cnt.reserve(n_kmers + 2)); CU(used_cnt.reserve(n_kmers + 2));
  CU(alloc_start.reserve(n_kmers + 2)); CU(used_start.reserve(n_kmers + 2));
  const size_t cub_bytes = index_build_cub_bytes(cl, cb_cap, k);
  CU(cub_tmp.reserve(cub_bytes));
  CU(d_contigs.reserve((size_t)2 * n_contigs));
  std::vector<unsigned long long> hc((size_t)2 * n_contigs);
  for (int i = 0; i < n_contigs; ++i) {
    hc[i] = contig_start[i];
    hc[n_contigs + i] = contig_len[i];
  }
  CU(cudaMemcpyAsync(d_contigs.p, hc.data(), hc.size() * 8, cudaMemcpyHostToDevice, st));
  CU(cs->d_tab.reserve((size_t)n_kmers + 2));
  CU(cs->d_rci.reserve((size_t)n_kmers + 2));
  CU(cs->d_used.reserve(((size_t)n_kmers + 1 + 255) / 256 * 8 + 8));
  CU(cs->d_pos.reserve(cb_cap + 1));
  IndexBuildParams p;
  p.enc = cs->d_enc.p;
  p.concat_len = cl;
  p.contig_start = d_contigs.p;
  p.contig_len = d_contigs.p + n_contigs;
  p.n_contigs = n_contigs;
  p.k = k;
  p.skip = kmer_skip;
  p.bin_shift = bin_shift;
  p.max_freq = max_prefix_freq;
  p.unit_offset = 0;
  IndexBuildScratch s;
  memset(&s, 0, sizeof(s));
  s.lastn = lastn.p; s.slot = lastn.p; s.flag = flag.p;
  s.cb_capacity = cb_cap;
  s.prefix = prefix.p; s.pos = pos.p; s.key = key.p; s.key_out = key_out.p; s.pos_out = pos_out.p; s.keep = keep.p;
  s.freq = freq.p; s.alloc_cnt = alloc_cnt.p; s.used_cnt = used_cnt.p; s.alloc_start = alloc_start.p; s.used_start = used_start.p;
  s.tab = cs->d_tab.p; s.rci = cs->d_rci.p; s.used_bits = cs->d_used.p; s.out_pos = cs->d_pos.p;
  s.out_capacity = cs->d_pos.cap;
  s.cub_tmp = cub_tmp.p; s.cub_bytes = cub_bytes;
  CU(cudaEventRecord(ctx->ev[4], st));
  CU(build_kmer_index(p, s, st));
  CU(cudaEventRecord(ctx->ev[5], st));
  CU(nb_stream_sync(ctx, st));
  cs->index_len = n_kmers + 1;
  cs->n_pos = s.n_positions;
  cs->unit_offset = 0;
  cs->k = k;
  cs->bin_shift = bin_shift;
  cs->rn = 0;
  cs->reads_searched = false;
  if (n_positions) *n_positions = s.n_positions;
  return 0;
}

// The context's index in the reference's in-memory format (whatever installed it): packed_index receives
// index_len x 5 bytes (Index{uint m_TabIndex; char m_RevCompIndex}, #pragma pack(1)), positions n_positions
// uint32 (either may be NULL to query the sizes only).
int ngmlr_b200_cs_get_index(ngmlr_b200_ctx* ctx, uint32_t* index_len, uint32_t* n_positions, void* packed_index,
                            uint32_t* positions) {
  if (!ctx) return -1;
  CsState* cs = cs_state(ctx, false);
  if (!cs || !cs->index_len) return ctx->fail("cs_get_index: no index");
  if (index_len) *index_len = cs->index_len;
  if (n_positions) *n_positions = cs->n_pos;
  CU(cudaSetDevice(ctx->device));
  if (packed_index) {
    if (!cs->d_rci.p) return ctx->fail("cs_get_index: index was installed without m_RevCompIndex");
    std::vector<uint32_t> tab(cs->index_len);
    std::vector<int8_t> rci(cs->index_len);
    CU(cudaMemcpy(tab.data(), cs->d_tab.p, (size_t)cs->index_len * 4, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(rci.data(), cs->d_rci.p, (size_t)cs->index_len, cudaMemcpyDeviceToHost));
    uint8_t* out = static_cast<uint8_t*>(packed_index);
    for (size_t i = 0; i < cs->index_len; ++i) {
      memcpy(out + 5 * i, &tab[i], 4);
      out[5 * i + 4] = (uint8_t)rci[i];
    }
  }
  if (positions && cs->n_pos) CU(cudaMemcpy(positions, cs->d_pos.p, (size_t)cs->n_pos * 4, cudaMemcpyDeviceToHost));
  return 0;
}

float ngmlr_b200_cs_last_build_ms(ngmlr_b200_ctx* ctx) {
  float ms = 0;
  if (ctx) cudaEventElapsedTime(&ms, ctx->ev[4], ctx->ev[5]);
  return ms;
}

int ngmlr_b200_cs_search_batch(ngmlr_b200_ctx* ctx, int n, const char* const* seqs,
                               const int32_t* lens, float sensitivity, float min_kmer_hits,
                               int64_t* cand_start, const float** scores, const uint64_t** locs,
                               const uint8_t** reverse, float* max_hits) {
  if (!ctx) return -1;
  CsState* cs = cs_state(ctx, false);
  if (!cs || !cs->index_len) return ctx->fail("cs_search_batch: call cs_set_index first");
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  cs->scores.clear();
  cs->locs.clear();
  cs->reverse.clear();
  cand_start[0] = 0;
  if (n <= 0) return 0;
  // ---- reads -> device ----
  std::vector<uint64_t> seq_off(n);
  size_t bytes = 0;
  int max_len = 0;
  for (int i = 0; i < n; ++i) {
    seq_off[i] = bytes;
    bytes += align_up((size_t)std::max(lens[i], 0) + 1, 16);
    max_len = std::max(max_len, lens[i]);
  }
  cs->last_seq_off = seq_off;
  cs->rn = 0;              // d_seq / d_off / d_len are shared with the resident pipeline: invalidate it
  cs->reads_searched = false;
  cs->seq_base = nullptr;
  std::vector<uint8_t> hseq(bytes + 16, 0);
  parallel_for(n, 256, [&](int i) { memcpy(hseq.data() + seq_off[i], seqs[i], (size_t)std::max(lens[i], 0)); });
  CU(cs->d_seq.reserve(bytes + 16));
  CU(cs->d_off.reserve((size_t)4 * n));
  CU(cs->d_len.reserve(n));
  CU(cs->d_hits.reserve(n));
  CU(cs->d_cap.reserve(n));
  CU(cs->d_count.reserve(n));
  CU(cs->d_max.reserve(n));
  CU(cudaMemcpyAsync(cs->d_seq.p, hseq.data(), bytes, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(cs->d_off.p, seq_off.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(cs->d_len.p, lens, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  CsParams p;
  memset(&p, 0, sizeof(p));
  p.tab = cs->d_tab.p;
  p.used_bits = cs->d_used.p;
  p.pos = cs->d_pos.p;
  p.unit_offset = cs->unit_offset;
  p.k = cs->k;
  p.bin_shift = cs->bin_shift;
  p.sensitivity = sensitivity;
  p.min_kmer_hits = min_kmer_hits;
  p.seq = cs->d_seq.p;
  p.seq_off = cs->d_off.p;
  p.seq_len = cs->d_len.p;
  p.n = n;
  p.hits = cs->d_hits.p;
  // ---- pass 1: hits per read ----
  CU(cudaEventRecord(ctx->ev[4], st));
  CU(launch_cs_search(p, true, false, st));
  std::vector<unsigned long long> hits(n);
  CU(cudaMemcpyAsync(hits.data(), cs->d_hits.p, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  CU(nb_stream_sync(ctx, st));
  // ---- pass 2 in chunks bounded by a device-memory budget ----
  const size_t budget = (size_t)4 << 30;
  std::vector<uint64_t> toff(n), ooff(n), roff(n);
  std::vector<uint32_t> caps(n);
  std::vector<int32_t> counts(n);
  std::vector<CsCandidate> hout;
  int first = 0;
  while (first < n) {
    size_t tent = 0, oent = 0, rent = 0;
    int last = first;
    while (last < n) {
      unsigned long long cap64 = 16;
      while (cap64 < 2 * hits[last] + 2) cap64 <<= 1;
      if (cap64 > (1ull << 31))
        return ctx->fail("cs_search_batch: (sub-)read %d has %llu k-mer hits; split the read (ReadProvider::splitRead)",
                         last, hits[last]);
      const uint32_t cap = (uint32_t)cap64;
      const size_t arena_cap = cap > CS_SMEM_CAP ? cap : 0;  // small tables live in shared memory
      const size_t need = arena_cap * 16 + (size_t)hits[last] * 4 + (size_t)hits[last] * 2 * 16;
      if (last > first && (tent * 16 + oent * 4 + rent * 16 + need) > budget) break;
      caps[last] = cap;
      toff[last] = tent;
      ooff[last] = oent;
      roff[last] = rent;
      tent += arena_cap;
      oent += (size_t)hits[last];
      rent += (size_t)hits[last] * 2;
      ++last;
    }
    const int m = last - first;
    CU(cs->d_tables.reserve(tent * 16 + 16));
    CU(cs->d_order.reserve(oent + 4));
    CU(cs->d_out.reserve(rent + 4));
    CU(cudaMemsetAsync(cs->d_tables.p, 0, tent * 16, st));
    CU(cudaMemcpyAsync(cs->d_off.p + (size_t)n, toff.data() + first, (size_t)m * 8, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(cs->d_off.p + (size_t)2 * n, ooff.data() + first, (size_t)m * 8, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(cs->d_off.p + (size_t)3 * n, roff.data() + first, (size_t)m * 8, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(cs->d_cap.p, caps.data() + first, (size_t)m * 4, cudaMemcpyHostToDevice, st));
    CsParams q = p;
    q.seq_off = cs->d_off.p + first;
    q.seq_len = cs->d_len.p + first;
    q.n = m;
    q.tables = cs->d_tables.p;
    q.table_off = cs->d_off.p + (size_t)n;
    q.table_cap = cs->d_cap.p;
    q.order = cs->d_order.p;
    q.order_off = cs->d_off.p + (size_t)2 * n;
    q.out = cs->d_out.p;
    q.out_off = cs->d_off.p + (size_t)3 * n;
    q.out_count = cs->d_count.p;
    q.max_hits = cs->d_max.p;
    bool any_small = false;
    for (int i = first; i < last; ++i) any_small = any_small || caps[i] <= CS_SMEM_CAP;
    CU(launch_cs_search(q, false, any_small, st));
    hout.resize(rent + 1);
    CU(cudaMemcpyAsync(counts.data() + first, cs->d_count.p, (size_t)m * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(max_hits + first, cs->d_max.p, (size_t)m * 4, cudaMemcpyDeviceToHost, st));
    if (rent) CU(cudaMemcpyAsync(hout.data(), cs->d_out.p, rent * sizeof(CsCandidate), cudaMemcpyDeviceToHost, st));
    CU(nb_stream_sync(ctx, st));
    for (int i = first; i < last; ++i) {
      const CsCandidate* c = hout.data() + roff[i];
      for (int j = 0; j < counts[i]; ++j) {
        cs->scores.push_back(c[j].score);
        cs->locs.push_back(c[j].loc);
        cs->reverse.push_back((uint8_t)c[j].reverse);
      }
      cand_start[i + 1] = (int64_t)cs->scores.size();
    }
    first = last;
  }
  CU(cudaEventRecord(ctx->ev[5], st));
  CU(nb_stream_sync(ctx, st));
  *scores = cs->scores.data();
  *locs = cs->locs.data();
  *reverse = cs->reverse.data();
  return n;
}

}  // extern "C"

extern "C" {

int ngmlr_b200_cs_set_reference(ngmlr_b200_ctx* ctx, const uint8_t* bin_ref, uint64_t n_bytes,
                                uint64_t concat_len) {
  if (!ctx) return -1;
  if (concat_len > 2 * n_bytes) return ctx->fail("cs_set_reference: concat_len exceeds 2 * n_bytes");
  CU(cudaSetDevice(ctx->device));
  CsState* cs = cs_state(ctx, true);
  CU(cs->d_enc.reserve(n_bytes + 64));
  CU(cudaMemsetAsync(cs->d_enc.p, 0x44, n_bytes + 64, ctx->stream));  // 'N','N' past the end
  CU(cudaMemcpyAsync(cs->d_enc.p, bin_ref, n_bytes, cudaMemcpyHostToDevice, ctx->stream));
  CU(nb_stream_sync(ctx, ctx->stream));
  cs->enc_bytes = n_bytes;
  cs->concat_len = concat_len;
  cs->contig_names.clear();  // no longer the contigs of a load_reference
  return 0;
}

int ngmlr_b200_set_ref_starts(ngmlr_b200_ctx* ctx, const uint64_t* ref_start_pos, int n_entries) {
  if (!ctx) return -1;
  if (n_entries < 2 || !ref_start_pos) return ctx->fail("set_ref_starts: need the contig starts plus the end entry");
  for (int i = 1; i < n_entries; ++i)
    if (ref_start_pos[i] <= ref_start_pos[i - 1]) return ctx->fail("set_ref_starts: entries must increase");
  CU(cudaSetDevice(ctx->device));
  CsState* cs = cs_state(ctx, true);
  cs->ref_starts.assign(ref_start_pos, ref_start_pos + n_entries);
  CU(cs->d_ref_starts.reserve((size_t)n_entries));
  CU(cudaMemcpyAsync(cs->d_ref_starts.p, cs->ref_starts.data(), (size_t)n_entries * 8, cudaMemcpyHostToDevice,
                     ctx->stream));
  CU(nb_stream_sync(ctx, ctx->stream));
  return 0;
}

// The encoded genome built ON THE DEVICE from contig text: replaces the encoding loop of _SequenceProvider::Init
// (src/SequenceProvider.cpp:292-400) -- 1000-N spacers (500 bytes of 0x44) before, between and after the contigs,
// contigs of <= 10 characters skipped (minRefSeqLen), every contig starting on a byte boundary -- and installs the
// result as the context's reference together with refStartPos (ngmlr_b200_cs_set_reference + set_ref_starts).
int ngmlr_b200_cs_encode_reference(ngmlr_b200_ctx* ctx, int n_contigs, const char* const* seqs, const uint64_t* lens,
                                   int32_t* n_kept, uint64_t* kept_start, uint64_t* kept_len, uint64_t* n_bytes,
                                   uint64_t* concat_len) {
  if (!ctx) return -1;
  if (n_contigs < 0 || (n_contigs && (!seqs || !lens))) return ctx->fail("cs_encode_reference: bad arguments");
  CU(cudaSetDevice(ctx->device));
  CsState* cs = cs_state(ctx, true);
  std::vector<unsigned long long> starts, klens;
  std::vector<int> which;
  unsigned long long bytes = 500, longest = 0;
  for (int i = 0; i < n_contigs; ++i) {
    if (!(lens[i] > 10)) continue;
    starts.push_back(bytes * 2);
    klens.push_back(lens[i]);
    which.push_back(i);
    bytes += (lens[i] + 1) / 2 + 500;
    longest = std::max<unsigned long long>(longest, lens[i]);
  }
  CU(cs->d_enc.reserve(bytes + 64));
  CU(cudaMemsetAsync(cs->d_enc.p, 0x44, bytes + 64, ctx->stream));  // spacers, and 'N','N' past the end
  DevBuf<uint8_t> text;
  CU(text.reserve(longest + 16));
  for (size_t j = 0; j < which.size(); ++j) {
    const int i = which[j];
    CU(cudaMemcpyAsync(text.p, seqs[i], lens[i], cudaMemcpyHostToDevice, ctx->stream));
    CU(launch_encode_contig(text.p, lens[i], cs->d_enc.p + starts[j] / 2, ctx->stream));
  }
  CU(nb_stream_sync(ctx, ctx->stream));
  cs->enc_bytes = bytes;
  cs->concat_len = bytes * 2 - 1;
  cs->contig_names.clear();  // no longer the contigs of a load_reference
  if (n_kept) *n_kept = (int32_t)which.size();
  for (size_t j = 0; j < which.size(); ++j) {
    if (kept_start) kept_start[j] = starts[j];
    if (kept_len) kept_len[j] = klens[j];
  }
  if (n_bytes) *n_bytes = bytes;
  if (concat_len) *concat_len = cs->concat_len;
  if (!starts.empty()) {   // refStartPos: the starts plus the artificial last entry (src/SequenceProvider.cpp:416-424)
    std::vector<uint64_t> rs(starts.begin(), starts.end());
    rs.push_back(starts.back() + klens.back() + 1000);
    return ngmlr_b200_set_ref_starts(ctx, rs.data(), (int)rs.size());
  }
  return 0;
}

// The context's encoded genome back in host memory (for the -enc.2.ngm writer): *n_bytes always, the bytes where
// bin_ref is not NULL and cap suffices.
int ngmlr_b200_cs_get_reference(ngmlr_b200_ctx* ctx, uint8_t* bin_ref, uint64_t cap, uint64_t* n_bytes,
                                uint64_t* concat_len) {
  if (!ctx) return -1;
  CsState* cs = cs_state(ctx, false);
  if (!cs || !cs->enc_bytes) return ctx->fail("cs_get_reference: no reference");
  if (n_bytes) *n_bytes = cs->enc_bytes;
  if (concat_len) *concat_len = cs->concat_len;
  if (bin_ref) {
    if (cap < cs->enc_bytes) return ctx->fail("cs_get_reference: buffer too small");
    CU(cudaSetDevice(ctx->device));
    CU(cudaMemcpy(bin_ref, cs->d_enc.p, cs->enc_bytes, cudaMemcpyDeviceToHost));
  }
  return 0;
}

namespace {

// The contract of the window calls: the window starts inside a contig or inside the 1000-N spacer in
// front of one (where the reference itself is well defined).
int check_windows(ngmlr_b200_ctx* ctx, const CsState* cs, int n, const uint64_t* start, const char* who) {
  if (!cs || !cs->enc_bytes || cs->ref_starts.empty())
    return ctx->fail("%s: call cs_set_reference and set_ref_starts first", who);
  const auto& rs = cs->ref_starts;
  for (int i = 0; i < n; ++i) {
    const uint64_t p = start[i];
    if (p >= cs->concat_len || p >= rs.back() || p == 0)
      return ctx->fail("%s: window %d starts outside the reference", who, i);
    size_t u = std::upper_bound(rs.begin(), rs.end(), (unsigned long long)p) - rs.begin();
    if (rs[u] - p < 1000ull) ++u;
    if (u >= rs.size() || p > rs[u] - 1000ull)
      return ctx->fail("%s: window %d starts behind the end of a contig", who, i);
  }
  return 0;
}

}  // namespace

int ngmlr_b200_decode_windows(ngmlr_b200_ctx* ctx, int n, const uint64_t* start, const int32_t* seq_len,
                              char* out, const int64_t* out_off) {
  if (!ctx) return -1;
  if (n <= 0) return 0;
  CsState* cs = cs_state(ctx, false);
  if (check_windows(ctx, cs, n, start, "decode_windows")) return -1;
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  size_t total = 0;
  for (int i = 0; i < n; ++i) {
    if (seq_len[i] < 1) return ctx->fail("decode_windows: sequence length %d < 1", seq_len[i]);
    total += align_up((size_t)seq_len[i], 16);
  }
  CU(ctx->h_win.reserve((size_t)n * 3 + 2));
  CU(ctx->d_win.reserve((size_t)n * 3 + 2));
  CU(ctx->d_sw_seq.reserve(total + 64));
  CU(ctx->h_sw_seq.reserve(total + 64));
  unsigned long long* hw = ctx->h_win.p;
  int32_t* hl = reinterpret_cast<int32_t*>(hw + 2 * (size_t)n);
  size_t at = 0;
  for (int i = 0; i < n; ++i) {
    hw[i] = start[i];
    hw[n + i] = at;
    hl[i] = seq_len[i];
    hl[n + i] = seq_len[i];
    at += align_up((size_t)seq_len[i], 16);
  }
  CU(cudaMemcpyAsync(ctx->d_win.p, hw, (size_t)n * 24, cudaMemcpyHostToDevice, st));
  RefDecodeParams rp;
  rp.enc = cs->d_enc.p;
  rp.ref_starts = cs->d_ref_starts.p;
  rp.n_starts = (int)cs->ref_starts.size();
  rp.n = n;
  rp.win_start = ctx->d_win.p;
  rp.out_off = reinterpret_cast<const uint64_t*>(ctx->d_win.p + n);
  rp.win_len = reinterpret_cast<const int32_t*>(ctx->d_win.p + 2 * (size_t)n);
  rp.out_span = rp.win_len + n;
  rp.out = ctx->d_sw_seq.p;
  CU(launch_decode_windows(rp, st));
  CU(cudaMemcpyAsync(ctx->h_sw_seq.p, ctx->d_sw_seq.p, total, cudaMemcpyDeviceToHost, st));
  CU(nb_stream_sync(ctx, st));
  parallel_for(n, 64, [&](int i) { memcpy(out + out_off[i], ctx->h_sw_seq.p + hw[n + i], (size_t)seq_len[i]); });
  return n;
}

int ngmlr_b200_convex_upload_windows(ngmlr_b200_ctx* ctx, int n, const uint64_t* on_ref_start,
                                     const uint64_t* on_ref_stop, const char* const* qrys,
                                     const int32_t* qry_lens, const int32_t* corridor_offsets,
                                     const int32_t* corridor_lengths, const int64_t* row_start,
                                     const int32_t* ext_qstart, const int32_t* ext_qend) {
  if (!ctx) return -1;
  if (n < 0) return ctx->fail("convex_upload_windows: n < 0");
  CsState* cs = cs_state(ctx, false);
  if (n > 0 && check_windows(ctx, cs, n, on_ref_start, "convex_upload_windows")) return -1;
  std::vector<int32_t> ref_lens((size_t)std::max(n, 1));
  for (int i = 0; i < n; ++i) {
    // extractReferenceSequenceForAlignment: onRefStart >= onRefStop -> no sequence (src/AlignmentBuffer.cpp:204-207)
    if (on_ref_start[i] >= on_ref_stop[i] || on_ref_stop[i] - on_ref_start[i] > 0x7ffffff0ull)
      return ctx->fail("convex_upload_windows: window %d is empty or too long", i);
    ref_lens[i] = (int32_t)(on_ref_stop[i] - on_ref_start[i]);  // strlen of the decoded refSeqLength = stop-start+1 buffer
  }
  RefWindows w;
  w.d_enc = cs ? cs->d_enc.p : nullptr;
  w.d_ref_starts = cs ? cs->d_ref_starts.p : nullptr;
  w.n_starts = cs ? (int)cs->ref_starts.size() : 0;
  w.win_start = on_ref_start;
  UploadSpec sp;
  sp.n = n;
  sp.win = &w;
  sp.ref_lens = ref_lens.data();
  sp.qrys = qrys;
  sp.qry_lens = qry_lens;
  sp.corridor_offsets = corridor_offsets;
  sp.corridor_lengths = corridor_lengths;
  sp.row_start = row_start;
  sp.ext_qstart = ext_qstart;
  sp.ext_qend = ext_qend;
  if (n > 0 && !qrys) return ctx->fail("convex_upload_windows: qrys is NULL");
  return convex_upload_spec(ctx, sp);
}

int ngmlr_b200_cs_score_batch(ngmlr_b200_ctx* ctx, int n, const char* const* seqs,
                              const int32_t* lens, float sensitivity, float min_kmer_hits,
                              int corridor, int read_part_length, int64_t* cand_start,
                              const float** cs_scores, const uint64_t** locs, const uint8_t** reverse,
                              const float** sw_scores, float* max_hits) {
  if (!ctx) return -1;
  CsState* cs = cs_state(ctx, false);
  if (!cs || !cs->enc_bytes) return ctx->fail("cs_score_batch: call cs_set_reference first");
  int rc = ngmlr_b200_cs_search_batch(ctx, n, seqs, lens, sensitivity, min_kmer_hits, cand_start,
                                      cs_scores, locs, reverse, max_hits);
  if (rc < 0) return rc;
  cs->sw_scores.clear();
  *sw_scores = cs->sw_scores.data();
  if (n <= 0) return rc;
  const size_t m = (size_t)cand_start[n];
  if (m > 0x7fffffffull) return ctx->fail("cs_score_batch: %zu candidates in one batch; use smaller batches", m);
  cs->sw_scores.assign(m, -1.0f);
  *sw_scores = cs->sw_scores.data();
  if (!m) return rc;
  cudaStream_t st = ctx->stream;
  // per candidate: window position, strand, and the arena location of its read (already on device)
  std::vector<unsigned long long> win(m);
  std::vector<uint64_t> qoff(m);
  std::vector<int32_t> qlen(m);
  int max_q = 0;
  for (int i = 0; i < n; ++i) {
    for (int64_t j = cand_start[i]; j < cand_start[i + 1]; ++j) {
      win[j] = (unsigned long long)cs->locs[j] - (unsigned long long)(corridor >> 1);  // uloc arithmetic (:110)
      qoff[j] = cs->last_seq_off[i];
      qlen[j] = lens[i] + 1;  // strlen + 1
    }
    max_q = std::max(max_q, lens[i] + 1);
  }
  const int win_len = ((read_part_length + 10 + corridor) | 1) + 1;  // refMaxLen, src/ScoreBuffer.h:71-72
  CU(cs->d_winpos.reserve(m));
  CU(cs->d_qoff.reserve(m));
  CU(cs->d_qlen.reserve(m));
  CU(cs->d_rev.reserve(m));
  CU(cs->d_sw.reserve(m));
  CU(cudaMemcpyAsync(cs->d_winpos.p, win.data(), m * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(cs->d_qoff.p, qoff.data(), m * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(cs->d_qlen.p, qlen.data(), m * 4, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(cs->d_rev.p, cs->reverse.data(), m, cudaMemcpyHostToDevice, st));
  const int warps_per_cta = 4;
  const int grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->num_sms * 8, (m + warps_per_cta - 1) / warps_per_cta));
  const size_t stride = max_q > 288 ? align_up((size_t)win_len + 4, 4) : 4;
  CU(cs->d_swscratch.reserve((size_t)grid * warps_per_cta * stride * 2));
  SwParams sp;
  memset(&sp, 0, sizeof(sp));
  sp.seq = cs->d_seq.p;
  sp.ref_off = cs->d_qoff.p;  // unused in gather mode
  sp.qry_off = cs->d_qoff.p;
  sp.ref_len = cs->d_qlen.p;  // unused in gather mode
  sp.qry_len = cs->d_qlen.p;
  sp.out = cs->d_sw.p;
  sp.n = (int)m;
  sp.scratch = cs->d_swscratch.p;
  sp.scratch_stride = stride;
  sp.enc = cs->d_enc.p;
  sp.concat_len = cs->concat_len;
  sp.win_pos = cs->d_winpos.p;
  sp.rev = cs->d_rev.p;
  sp.win_len = win_len;
  CU(cs->d_sub_counts.reserve(2));
  CU(cudaMemsetAsync(cs->d_sub_counts.p, 0, 2 * sizeof(unsigned int), st));
  sp.general_pairs = cs->d_sub_counts.p;
  sp.wide_pairs = cs->d_sub_counts.p + 1;
  CU(launch_sw_score_gather(sp, grid, max_q, win_len, st));
  CU(cudaMemcpyAsync(cs->sw_scores.data(), cs->d_sw.p, m * 4, cudaMemcpyDeviceToHost, st));
  CU(nb_stream_sync(ctx, st));
  return rc;
}

}  // extern "C"

extern "C" {

int ngmlr_b200_cs_upload(ngmlr_b200_ctx* ctx, int n, const char* const* seqs, const int32_t* lens) {
  if (!ctx) return -1;
  if (n < 0) return ctx->fail("cs_upload: n < 0");
  CU(cudaSetDevice(ctx->device));
  CsState* cs = cs_state(ctx, true);
  cudaStream_t st = ctx->stream;
  std::vector<uint64_t> seq_off((size_t)n + 1);
  size_t bytes = 0;
  int max_len = 0;
  for (int i = 0; i < n; ++i) {
    seq_off[i] = bytes;
    bytes += align_up((size_t)std::max(lens[i], 0) + 1, 16);
    max_len = std::max(max_len, lens[i]);
  }
  CU(cs->p_seq.reserve(bytes + 16));
  uint8_t* hseq = cs->p_seq.p;
  parallel_for(n, 256, [&](int i) {
    const size_t L = (size_t)std::max(lens[i], 0);
    memcpy(hseq + seq_off[i], seqs[i], L);
    memset(hseq + seq_off[i] + L, 0, align_up(L + 1, 16) - L);
  });
  CU(cs->d_seq.reserve(bytes + 16));
  CU(cs->d_off.reserve((size_t)n + 1));
  CU(cs->d_len.reserve((size_t)n + 1));
  CU(cudaMemcpyAsync(cs->d_seq.p, hseq, bytes, cudaMemcpyHostToDevice, st));
  if (n) {
    CU(cudaMemcpyAsync(cs->d_off.p, seq_off.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(cs->d_len.p, lens, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  }
  CU(nb_stream_sync(ctx, st));
  cs->rn = n;
  cs->rmax = max_len;
  cs->rbytes = bytes;
  cs->seq_base = cs->d_seq.p;
  cs->n_cand = 0;
  cs->reads_searched = false;
  return 0;
}

int ngmlr_b200_cs_run(ngmlr_b200_ctx* ctx, float sensitivity, float min_kmer_hits, int corridor,
                      int read_part_length, int64_t* n_candidates, float* kernel_ms) {
  if (!ctx) return -1;
  CsState* cs = cs_state(ctx, false);
  if (!cs || !cs->index_len) return ctx->fail("cs_run: call cs_set_index first");
  if (!cs->enc_bytes) return ctx->fail("cs_run: call cs_set_reference first");
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int n = cs->rn;
  if (n_candidates) *n_candidates = 0;
  if (kernel_ms) *kernel_ms = 0.0f;
  if (n <= 0) return 0;
  if (!cs->seq_base) return ctx->fail("cs_run: the resident (sub-)reads were replaced by cs_search_batch; upload again");
  if (!cs->ev0) {
    CU(cudaEventCreate(&cs->ev0));
    CU(cudaEventCreate(&cs->ev1));
  }
  const size_t n1 = (size_t)n + 1;
  CU(cs->d_hits.reserve(n1));
  CU(cs->d_cap.reserve(n1));
  CU(cs->d_count.reserve(n1));
  CU(cs->d_max.reserve(n1));
  CU(cs->d_a.reserve(n1)); CU(cs->d_b.reserve(n1)); CU(cs->d_c.reserve(n1));
  CU(cs->d_sa.reserve(n1)); CU(cs->d_sb.reserve(n1)); CU(cs->d_sc.reserve(n1));
  CU(cs->d_cnt64.reserve(n1)); CU(cs->d_cstart.reserve(n1));
  size_t tmp_bytes = 0;
  CU(cs_exclusive_scan(nullptr, tmp_bytes, cs->d_a.p, cs->d_sa.p, (int)n1, st));
  CU(cs->d_scan_tmp.reserve(tmp_bytes + 256));
  CsParams p;
  memset(&p, 0, sizeof(p));
  p.tab = cs->d_tab.p;
  p.used_bits = cs->d_used.p;
  p.pos = cs->d_pos.p;
  p.unit_offset = cs->unit_offset;
  p.k = cs->k;
  p.bin_shift = cs->bin_shift;
  p.sensitivity = sensitivity;
  p.min_kmer_hits = min_kmer_hits;
  p.seq = cs->seq_base;
  p.seq_off = cs->d_off.p;
  p.seq_len = cs->d_len.p;
  p.n = n;
  p.hits = cs->d_hits.p;
  CU(cudaEventRecord(cs->ev0, st));
  CU(launch_cs_search(p, true, false, st));
  CU(cudaMemsetAsync(cs->d_hits.p + n, 0, 8, st));  // counter of small (shared-memory) tables
  CU(launch_cs_sizes(cs->d_hits.p, n, cs->d_cap.p, cs->d_a.p, cs->d_b.p, cs->d_c.p, st));
  size_t tb = cs->d_scan_tmp.cap;
  CU(cs_exclusive_scan(cs->d_scan_tmp.p, tb, cs->d_a.p, cs->d_sa.p, (int)n1, st));
  tb = cs->d_scan_tmp.cap;
  CU(cs_exclusive_scan(cs->d_scan_tmp.p, tb, cs->d_b.p, cs->d_sb.p, (int)n1, st));
  tb = cs->d_scan_tmp.cap;
  CU(cs_exclusive_scan(cs->d_scan_tmp.p, tb, cs->d_c.p, cs->d_sc.p, (int)n1, st));
  unsigned long long totals[3] = {0, 0, 0};
  unsigned long long n_small = 1;
  CU(cudaMemcpyAsync(&n_small, cs->d_hits.p + n, 8, cudaMemcpyDeviceToHost, st));  // cs_sizes_kernel's counter
  CU(cudaMemcpyAsync(&totals[0], cs->d_sa.p + n, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(&totals[1], cs->d_sb.p + n, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(&totals[2], cs->d_sc.p + n, 8, cudaMemcpyDeviceToHost, st));
  CU(nb_stream_sync(ctx, st));
  cs->n_small_tables = n_small;
  const size_t need = (size_t)totals[0] * 16 + (size_t)totals[1] * 4 + (size_t)totals[2] * 16;
  if (need > ((size_t)96 << 30))
    return ctx->fail("cs_run: %zu bytes of vote tables needed; use cs_score_batch (chunked) for this batch", need);
  CU(cs->d_tables.reserve((size_t)totals[0] * 16 + 16));
  CU(cs->d_order.reserve((size_t)totals[1] + 4));
  CU(cs->d_out.reserve((size_t)totals[2] + 4));
  CU(cudaMemsetAsync(cs->d_tables.p, 0, (size_t)totals[0] * 16, st));
  p.tables = cs->d_tables.p;
  p.table_off = reinterpret_cast<const uint64_t*>(cs->d_sa.p);
  p.table_cap = cs->d_cap.p;
  p.order = cs->d_order.p;
  p.order_off = reinterpret_cast<const uint64_t*>(cs->d_sb.p);
  p.out = cs->d_out.p;
  p.out_off = reinterpret_cast<const uint64_t*>(cs->d_sc.p);
  p.out_count = cs->d_count.p;
  p.max_hits = cs->d_max.p;
  // small tables take no arena space: the arena holds exactly sum(cap > CS_SMEM_CAP ? cap : 0) entries, and every big
  // table has at least 2 * CS_SMEM_CAP of them -- so "no small table" <=> arena >= 2 * CS_SMEM_CAP * n can only be
  // decided safely in one direction; the shared-memory variant is always correct, the other only without small tables
  const bool any_small = cs->n_small_tables != 0;
  CU(launch_cs_search(p, false, any_small, st));
  CU(launch_cs_count_to_u64(cs->d_count.p, n, cs->d_cnt64.p, st));
  tb = cs->d_scan_tmp.cap;
  CU(cs_exclusive_scan(cs->d_scan_tmp.p, tb, cs->d_cnt64.p, cs->d_cstart.p, (int)n1, st));
  unsigned long long m64 = 0;
  CU(cudaMemcpyAsync(&m64, cs->d_cstart.p + n, 8, cudaMemcpyDeviceToHost, st));
  CU(nb_stream_sync(ctx, st));
  const size_t m = (size_t)m64;
  if (m > 0x7fffffffull) return ctx->fail("cs_run: %zu candidates in one batch; use smaller batches", m);
  cs->n_cand = (long long)m;
  CU(cs->d_cloc.reserve(m + 1));
  CU(cs->d_cscore.reserve(m + 1));
  CU(cs->d_rev.reserve(m + 1));
  CU(cs->d_winpos.reserve(m + 1));
  CU(cs->d_qoff.reserve(m + 1));
  CU(cs->d_qlen.reserve(m + 1));
  CU(cs->d_sw.reserve(m + 1));
  CU(launch_cs_compact(cs->d_out.p, reinterpret_cast<const uint64_t*>(cs->d_sc.p), cs->d_count.p, cs->d_cstart.p,
                       cs->d_off.p, cs->d_len.p, n, corridor >> 1, cs->d_cloc.p, cs->d_cscore.p, cs->d_rev.p,
                       cs->d_winpos.p, cs->d_qoff.p, cs->d_qlen.p, st));
  CU(cs->d_sub_counts.reserve(2));
  CU(cudaMemsetAsync(cs->d_sub_counts.p, 0, 2 * sizeof(unsigned int), st));
  if (m) {
    const int win_len = ((read_part_length + 10 + corridor) | 1) + 1;  // refMaxLen, src/ScoreBuffer.h:71-72
    const int warps_per_cta = 4;
    const int grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->num_sms * 8, (m + warps_per_cta - 1) / warps_per_cta));
    const size_t stride = align_up((size_t)win_len + 4, 4);
    CU(cs->d_swscratch.reserve((size_t)grid * warps_per_cta * stride * 2));
    SwParams sp;
    memset(&sp, 0, sizeof(sp));
    sp.seq = cs->seq_base;
    sp.ref_off = cs->d_qoff.p;
    sp.qry_off = cs->d_qoff.p;
    sp.ref_len = cs->d_qlen.p;
    sp.qry_len = cs->d_qlen.p;
    sp.out = cs->d_sw.p;
    sp.n = (int)m;
    sp.scratch = cs->d_swscratch.p;
    sp.scratch_stride = stride;
    sp.enc = cs->d_enc.p;
    sp.concat_len = cs->concat_len;
    sp.win_pos = cs->d_winpos.p;
    sp.rev = cs->d_rev.p;
    sp.win_len = win_len;
    sp.general_pairs = cs->d_sub_counts.p;
    sp.wide_pairs = cs->d_sub_counts.p + 1;
    CU(launch_sw_score_gather(sp, grid, cs->rmax + 1, win_len, st));
  }
  CU(cudaEventRecord(cs->ev1, st));
  CU(nb_stream_sync(ctx, st));
  cs->reads_searched = cs->seq_base == ctx->d_reads.p;
  if (n_candidates) *n_candidates = (int64_t)m;
  if (kernel_ms) cudaEventElapsedTime(kernel_ms, cs->ev0, cs->ev1);
  return 0;
}

// Test-only counters of the last sub-read scoring launch (cs_run or cs_score_batch): pairs that took the general
// path, and pairs that took the ungapped path of the wide instantiation.
static unsigned int subread_count(ngmlr_b200_ctx* ctx, int which) {
  CsState* cs = ctx ? cs_state(ctx, false) : nullptr;
  unsigned int v[2] = {0u, 0u};
  if (!cs || !cs->d_sub_counts.p) return 0u;
  if (cudaSetDevice(ctx->device) != cudaSuccess || cudaStreamSynchronize(ctx->stream) != cudaSuccess ||
      cudaMemcpy(v, cs->d_sub_counts.p, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess)
    return 0u;
  return v[which];
}

unsigned int ngmlr_b200_debug_subread_general_pairs(ngmlr_b200_ctx* ctx) { return subread_count(ctx, 0); }

unsigned int ngmlr_b200_debug_subread_wide_pairs(ngmlr_b200_ctx* ctx) { return subread_count(ctx, 1); }

int ngmlr_b200_cs_fetch(ngmlr_b200_ctx* ctx, int64_t* cand_start, const float** cs_scores,
                        const uint64_t** locs, const uint8_t** reverse, const float** sw_scores,
                        float* max_hits) {
  if (!ctx) return -1;
  CsState* cs = cs_state(ctx, false);
  if (!cs) return ctx->fail("cs_fetch: nothing to fetch");
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int n = cs->rn;
  const size_t m = (size_t)cs->n_cand;
  CU(cs->p_score.reserve(m + 1));
  CU(cs->p_loc.reserve(m + 1));
  CU(cs->p_rev.reserve(m + 1));
  CU(cs->p_sw.reserve(m + 1));
  static_assert(sizeof(unsigned long long) == sizeof(int64_t), "");
  if (n) CU(cudaMemcpyAsync(cand_start, cs->d_cstart.p, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, st));
  else cand_start[0] = 0;
  if (n && max_hits) CU(cudaMemcpyAsync(max_hits, cs->d_max.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  if (m) {
    CU(cudaMemcpyAsync(cs->p_score.p, cs->d_cscore.p, m * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(cs->p_loc.p, cs->d_cloc.p, m * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(cs->p_rev.p, cs->d_rev.p, m, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(cs->p_sw.p, cs->d_sw.p, m * 4, cudaMemcpyDeviceToHost, st));
  }
  CU(nb_stream_sync(ctx, st));
  *cs_scores = cs->p_score.p;
  *locs = cs->p_loc.p;
  *reverse = cs->p_rev.p;
  *sw_scores = cs->p_sw.p;
  return n;
}

// Host glue after scoring: ScoreBuffer::topNSE + computeMQ (src/ScoreBuffer.cpp:170-192, 33-45).
// Candidates of one (sub-)read are ordered with std::sort and the reference's comparator
// (a.Score.f > b.Score.f, :25-27) -- the same libstdc++ routine, because the order of tied scores is
// part of the behaviour --, then those scoring above 0.75 x best are kept.
int ngmlr_b200_select_candidates(int n, const int64_t* cand_start, const float* sw_scores, int32_t* order,
                                 int32_t* kept, int32_t* mq) {
  if (n < 0 || (n > 0 && (!cand_start || !order || !kept || !mq))) return -1;
  struct Item {
    float score;
    int32_t idx;
  };
  parallel_for(n, 512, [&](int i) {
    const int64_t b = cand_start[i];
    const int m = (int)(cand_start[i + 1] - b);
    Item small[32];
    std::vector<Item> big;
    Item* it = small;
    if (m > 32) {
      big.resize((size_t)m);
      it = big.data();
    }
    for (int j = 0; j < m; ++j) {
      it[j].score = sw_scores[b + j];
      it[j].idx = (int32_t)(b + j);
    }
    std::sort(it, it + m, [](Item x, Item y) { return x.score > y.score; });
    int keep = m;
    if (m > 1) {
      const float min_score = it[0].score * 0.75f;
      int j = 1;
      while (j < m && it[j].score > min_score) ++j;
      keep = j;
    }
    int q = 60;  // MAX_MQ (src/ScoreBuffer.cpp:16)
    if (m > 1) q = (int)ceil(60.0f * (it[0].score - it[1].score) / it[0].score);
    for (int j = 0; j < m; ++j) order[b + j] = it[j].idx;
    kept[i] = keep;
    mq[i] = q;
  });
  return n;
}

}  // extern "C"
