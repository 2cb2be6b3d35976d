// ngmlr_b200/csrc/convex_traceback.cu -- traceback + binary-CIGAR emission for sm_90a.
//
// Replaces Convex::ConvexAlignFast::revBacktrack (src/ConvexAlignFast.cpp:335-432) with
// AlignmentMatrixFast::getDirection / validPath (src/AlignmentMatrixFast.cpp:185-195, 213-220).
//
// The walk is a pointer chase (each step depends on the previous direction), at most H + W steps
// against H x W cells of fill, so it is latency- not bandwidth-bound. One WARP per problem: for
// every 32-row block the lanes load, in a few coalesced requests, everything the path can touch
// there -- lane t keeps row 32b+t's corridor line, read byte and a 64-step window of its direction
// words around the expected diagonal; a 128-column window of reference bytes is kept likewise --
// and the walk itself then runs on registers + warp shuffles (uniform control flow, ~100 cycles
// per step instead of several dependent L2/HBM round trips). A path that drifts out of a window
// falls back to a direct load. Runs are emitted back-to-front into a per-problem strip exactly
// like the reference's binaryCigar (element = len << 4 | op, EQ and X separate ops); the same
// warp then copies them, coalesced, into a compact arena so the host needs a single D2H copy.
#include <cuda_runtime.h>

#include "device_types.h"
#include "kernels.h"

namespace nb {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int TB_WARPS_PER_CTA = 4;
constexpr int NW = 4;  // direction words (16 steps each) a lane keeps per block

struct RowWindow {
  int off, len;        // corridor line of row 32*blk + lane
  int min_c, max_c;    // validPath bounds of that row (exclusive)
  uint32_t q;          // read byte of that row
  int g0;              // first 16-step group held in w[]
  uint32_t w[NW];
};

__global__ void __launch_bounds__(TB_WARPS_PER_CTA * 32) convex_traceback_kernel(const TraceParams p) {
  const int slot = blockIdx.x * TB_WARPS_PER_CTA + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (slot >= p.n) return;
  const int i = p.order[slot];  // longest walks first: no straggler warps at the end of the launch
  const AlnDesc d = p.desc[i];
  const FillOut f = p.fill[i];
  TraceOut o;
  o.status = ST_INVALID;
  o.n_runs = 0;
  o.ref_position = 0;
  o.qstart = 0;
  o.qend = 0;
  o.steps = 0;
  o.run_off = 0;
  if (f.status != ST_OK) {
    o.status = f.status;
    if (lane == 0) p.out[i] = o;
    return;
  }
  const int H = d.height;
  const uint8_t* __restrict__ ref = p.seq + d.ref_off;
  const uint8_t* __restrict__ qry = p.seq + d.qry_off;
  CorridorView cv;

  cv.bind(p.c_off, p.c_len, p.c_blkbase, p.c_delta, d);
  const BlockRec* __restrict__ blocks = p.blocks + d.blk_off;
  int32_t* __restrict__ bc = p.scratch + d.tb_off;
  const int cap = d.tb_cap;        // our strip
  const int ref_cap = d.ref_cap;   // the reference's binaryCigar length (for its overflow throw)

  int x = f.best_x, y = f.best_y;
  const int qend = H - y - 1;  // (:1281)
  o.qend = qend;
  if (y <= 0) {  // (:338)
    if (lane == 0) p.out[i] = o;
    return;
  }
  int idx = cap - 1;       // next free slot, filled downwards
  int used = 0;            // slots the reference would have consumed
  int op = OP_S;
  int op_len = qend;
  int read_len = qend;
  int steps = 0;
  bool ok = true, threw = false;

  int cur_blk = -1;
  BlockRec br;
  br.word_off = 0; br.base = 0; br.nsteps = 0;
  int ngroups = 0;
  RowWindow rw;
  rw.off = 0; rw.len = 0; rw.q = 0; rw.g0 = 0; rw.min_c = 0; rw.max_c = 0;
#pragma unroll
  for (int j = 0; j < NW; ++j) rw.w[j] = 0;
  int xw0 = 1 << 30;       // reference byte window [xw0, xw0 + 128), 4 bytes per lane
  uint32_t refw = 0;

  // A diagonal run that ends inside its block ends at a cell the fast path has just rejected (same registers, same
  // tests): the next iteration goes straight to the single step instead of evaluating that rejection again.
  bool rejected = false;
  for (;;) {
    // ---- getDirection(x, y) ----
    if (y < 0 || x < 0) break;  // STOP (y > H-1 cannot happen: y only decreases from best_y)
    const int blk = y >> 5, t = y & 31;
    if (blk != cur_blk) {
      cur_blk = blk;
      br = blocks[blk];
      ngroups = (br.nsteps + 15) >> 4;
      const int yy = (blk << 5) + lane;
      rw.q = 0;
      load_corridor_rows(cv, blk, lane, H, rw.off, rw.len);
      if (yy < H) rw.q = qry[yy];
      {  // validPath(x, y) bounds: float math then truncation, as in the reference (:213-220)
        const float wf = (float)rw.len;
        rw.min_c = (int)__fadd_rn((float)rw.off, __fmul_rn(0.1f, wf));
        rw.max_c = (int)__fsub_rn((float)(rw.min_c + rw.len), __fmul_rn(0.1f, wf));
      }
      // expected step index of the path in row `lane`: two steps per row along the diagonal
      const int s_here = x - br.base + t;
      const int s_exp = s_here - 2 * (t - lane);
      int g0 = (s_exp >> 4) - (NW / 2 - 1) - 1;
      g0 = max(0, min(g0, ngroups - NW));
      rw.g0 = g0;
#pragma unroll
      for (int j = 0; j < NW; ++j) {
        const int g = g0 + j;
        rw.w[j] = (g < ngroups && lane <= t) ? p.dir[br.word_off + (unsigned long long)g * 32ull + (unsigned)lane] : 0u;
      }
    }
    // ---- fast path: a whole run of diagonal moves in one go ----
    // Lane L <= t examines the cell the path reaches in row L if it keeps moving diagonally,
    // (x - (t - L), 32*blk + L), entirely from its own registers: inside the corridor, direction
    // DIAG, validPath. The leading run of lanes t, t-1, ... that all agree is consumed at once
    // (on 15 %-error reads ~6 steps per iteration instead of 1).
    if (!rejected) {
      const int xx = x - (t - lane);
      bool okd = false;
      if (lane <= t && xx >= 0 && xx >= rw.off && (long long)xx < (long long)rw.off + (long long)rw.len) {
        const int s2 = xx - br.base + lane;
        const int j2 = (s2 >> 4) - rw.g0;
        if ((unsigned)j2 < (unsigned)NW) {
          const uint32_t w2 = j2 == 0 ? rw.w[0] : (j2 == 1 ? rw.w[1] : (j2 == 2 ? rw.w[2] : rw.w[3]));
          okd = ((w2 >> ((s2 & 15) * 2)) & 3u) == DIR_DIAG && xx > rw.min_c && xx < rw.max_c;
        }
      }
      const unsigned okm = __ballot_sync(FULL, okd) << (31 - t);
      const int n_diag = __clz(~okm);
      if (n_diag > 0) {
        if (x - 31 < xw0 || x >= xw0 + 128) {
          xw0 = max(0, x - 124) & ~3;
          refw = *reinterpret_cast<const uint32_t*>(ref + xw0 + 4 * lane);  // arena is padded
        }
        const int rx = min(max(xx - xw0, 0), 127);
        const uint32_t rword = __shfl_sync(FULL, refw, rx >> 2);
        const bool eqd = okd && rw.q == ((rword >> ((rx & 3) * 8)) & 0xffu);
        uint32_t e = __ballot_sync(FULL, eqd) << (31 - t);
        int rem = n_diag;
        while (rem > 0) {
          const bool iseq = (e >> 31) != 0u;
          int run = __clz(iseq ? ~e : e);
          run = run < rem ? run : rem;
          const int dir = iseq ? OP_EQ : OP_X;
          if (dir == op) {
            op_len += run;
          } else {
            if (lane == 0 && idx >= 0) bc[idx] = (op_len << 4) | op;
            --idx;
            ++used;
            op = dir;
            op_len = run;
            if (used >= ref_cap || idx < 0) {  // binaryCigarIndex < 0 -> throw 1 (:404-407)
              threw = true;
              break;
            }
          }
          if (run < 32) e <<= run;
          rem -= run;
        }
        if (threw) break;
        steps += n_diag;
        read_len += n_diag;
        x -= n_diag;
        y -= n_diag;
        rejected = n_diag <= t;  // still in this block: lane t - n_diag is the cell that ended the run
        continue;
      }
    }
    rejected = false;
    // ---- generic single step ----
    const int off = __shfl_sync(FULL, rw.off, t);
    const int len = __shfl_sync(FULL, rw.len, t);
    if (x < off || (long long)x >= (long long)off + (long long)len) break;  // STOP: outside the corridor
    const int s = x - br.base + t;
    const int g = s >> 4;
    const int j = g - __shfl_sync(FULL, rw.g0, t);
    uint32_t wd;
    if ((unsigned)j < (unsigned)NW) {
      const uint32_t mine = j == 0 ? rw.w[0] : (j == 1 ? rw.w[1] : (j == 2 ? rw.w[2] : rw.w[3]));
      wd = __shfl_sync(FULL, mine, t);
    } else {
      wd = p.dir[br.word_off + (unsigned long long)g * 32ull + (unsigned)t];  // drifted out of the window
    }
    const uint32_t code = (wd >> ((s & 15) * 2)) & 3u;
    if (code == DIR_STOP) break;
    // ---- validPath(x, y) ----
    {
      const int min_c = __shfl_sync(FULL, rw.min_c, t);
      const int max_c = __shfl_sync(FULL, rw.max_c, t);
      if (!(x > min_c && x < max_c)) {
        ok = false;
        break;
      }
    }
    int dir;
    if (code == DIR_DIAG) {
      if (x < xw0 || x >= xw0 + 128) {
        xw0 = max(0, x - 124) & ~3;
        refw = *reinterpret_cast<const uint32_t*>(ref + xw0 + 4 * lane);  // arena is padded
      }
      const int rx = x - xw0;
      const uint32_t rword = __shfl_sync(FULL, refw, rx >> 2);
      const uint32_t rc = (rword >> ((rx & 3) * 8)) & 0xffu;
      const uint32_t qc = __shfl_sync(FULL, rw.q, t);
      dir = (qc == rc) ? OP_EQ : OP_X;
    } else {
      dir = (code == DIR_I) ? OP_I : OP_D;
    }
    ++steps;
    if (dir == OP_EQ || dir == OP_X) {
      --y; --x; ++read_len;
    } else if (dir == OP_I) {
      --y; ++read_len;
    } else {
      --x;
    }
    if (dir == op) {
      ++op_len;
    } else {
      if (lane == 0 && idx >= 0) bc[idx] = (op_len << 4) | op;
      --idx;
      ++used;
      op = dir;
      op_len = 1;
    }
    if (used >= ref_cap || idx < 0) {  // binaryCigarIndex < 0 -> throw 1 (:404-407)
      threw = true;
      break;
    }
  }
  o.steps = steps;
  if (threw) {
    o.status = ST_THROW;
    if (lane == 0) p.out[i] = o;
    return;
  }
  if (!ok) {
    if (lane == 0) p.out[i] = o;
    return;
  }
  // last run + leading clip (:411-416); the reference writes both slots unchecked
  if (idx < 1 || used + 2 > ref_cap) {
    o.status = ST_THROW;
    if (lane == 0) p.out[i] = o;
    return;
  }
  if (lane == 0) {
    bc[idx] = (op_len << 4) | op;
    bc[idx - 1] = ((y + 1) << 4) | OP_S;
  }
  idx -= 2;
  read_len += y + 1;
  o.ref_position = x + 1;
  o.qstart = y + 1;
  const int n = cap - 1 - idx;
  o.n_runs = n;
  if (H != read_len) {  // (:424-428)
    if (lane == 0) p.out[i] = o;
    return;
  }
  unsigned long long at = 0;
  if (lane == 0) at = atomicAdd(p.runs_alloc, (unsigned long long)n);
  at = __shfl_sync(FULL, at, 0);
  o.run_off = at;
  o.status = (at + (unsigned long long)n <= p.runs_capacity) ? ST_OK : ST_DIR_OVERFLOW;
  __syncwarp();
  if (o.status == ST_OK) {
    // strip [cap-n, cap) -> compact arena, same order (leading clip, runs..., trailing clip)
    const int32_t* __restrict__ src = bc + (cap - n);
    int32_t* __restrict__ dst = p.runs + at;
    for (int k = lane; k < n; k += 32) dst[k] = src[k];
  }
  if (lane == 0) p.out[i] = o;
}

}  // namespace

cudaError_t launch_convex_traceback(const TraceParams& p, cudaStream_t stream) {
  if (p.n <= 0) return cudaSuccess;
  convex_traceback_kernel<<<(p.n + TB_WARPS_PER_CTA - 1) / TB_WARPS_PER_CTA, TB_WARPS_PER_CTA * 32, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace nb
