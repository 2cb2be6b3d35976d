// ngmlr_b200/csrc/convex_fill.cu -- convex-gap banded Smith-Waterman forward fill for sm_90a.
//
// Replaces Convex::ConvexAlignFast::fwdFillMatrixSSESimple (src/ConvexAlignFast.cpp:914-1287)
// over Convex::AlignmentMatrixFast (src/AlignmentMatrixFast.{h,cpp}).
//
// Mapping. One warp owns one alignment problem (a persistent grid pulls problems, largest
// first, from an atomic counter). The warp walks the DP matrix in blocks of 32 rows: lane t owns
// row y = 32*b + t and sweeps it left to right, staggered one step behind lane t-1, so that at
// step s lane t evaluates column x = base + s - t. That is an anti-diagonal wavefront:
//   up   (x,   y-1)  = what lane t-1 produced one step ago   -> __shfl_up
//   diag (x-1, y-1)  = what lane t-1 produced two steps ago  -> last step's "up", kept in a register
//   left (x-1, y)    = this lane's previous cell             -> registers
// The rolling rows of the reference (2 x W x 8 B, AlignmentMatrixFast.h:34-54) therefore never
// leave the register file. Row 32*b+31 is handed to lane 0 of the next block through a per-warp
// strip in global memory indexed by absolute column (it stays in L2; ~16 B/column/block), staged
// through shared memory in 64-step chunks: all 32 lanes copy a chunk of the strip (+ the reference
// bytes for those columns, merged into the same 16-byte records) into shared memory one chunk
// ahead, lane 0 then needs a single LDS.128 per step and lane 31 a single STS.128; finished
// chunks are flushed back coalesced. Because lane 31 always trails lane 0 by 31 columns the strip
// is updated in place for any corridor shape.
//
// Team mode (NW = 4). One warp per problem leaves a long tail behind the largest matrices (the
// reference sees 93 M-cell matrices). In team mode the 4 warps of a CTA share one problem: warp w
// takes the 32-row blocks b = w, w+4, w+8, ... and block b+1 consumes the strip records of block b
// as they are produced (16-step chunks, progress published through shared memory), so the four
// warps run as a software pipeline about 100 columns apart and a problem finishes ~4x sooner at
// the same total work.
//
// HBM traffic. The only per-cell output is the traceback direction: 2 bits per cell (EQ/X are
// re-derived by the traceback), 16 steps per 32-bit word, written as one fully coalesced 128-byte
// warp store every 16 steps (word index = group*32 + lane). The reference spends 1 byte per cell
// (AlignmentMatrixFast.h:261).
//
// Arithmetic is float32 exactly as the reference: every add/multiply is a separately rounded
// __fadd_rn/__fmul_rn (the reference binary has no FMA), comparisons are exact, and the
// direction priority is the reference's. `RAW` selects the as-coded SSE semantics in which the
// run tests use the neighbours' raw indelRun for all but the last <=12 cells of a row (executable
// spec: oracle/convex_oracle.c chain_cell, rule 2); RAW=false is the scalar rule, which is
// identical for every scoring in the "default class" up to the score magnitude where float rounding can erase the
// class's margin (see capi.cu scoring_needs_raw(), chosen per batch).
#include <cuda_runtime.h>
#include <limits.h>

#include <type_traits>

#include "device_types.h"
#include "kernels.h"

namespace nb {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int STRIP_PAD = 32;    // strip index = column + STRIP_PAD (columns >= -31 lockstep, >= -1 ramp-free)
constexpr unsigned X_BIAS = 1u << 20;
#ifndef FILL_TEAM_CHUNK
#define FILL_TEAM_CHUNK 16
#endif
#ifndef FILL_LANE0_LDS
#define FILL_LANE0_LDS 0  // 1: lane 0 loads its strip record itself instead of receiving it through lane 31's shuffle sources
#endif

__device__ __forceinline__ uint4 ld_strip(const uint4* p) { return __ldcg(p); }
__device__ __forceinline__ void st_strip(uint4* p, uint4 v) { __stcg(p, v); }

// CTA-scope fence ordering the strip records (st.cg / ld.cg) against the progress word in shared memory
// (fence.acq_rel.cta instead of the sequentially consistent fence measured no difference)
__device__ __forceinline__ void team_fence() { __threadfence_block(); }

// progress words live in shared memory; plain 32-bit shared addresses (computed once per kernel) instead of the
// generic-address sequence the compiler emits for a volatile shared array indexed at run time
__device__ __forceinline__ unsigned long long ld_prog(uint32_t saddr) {
  unsigned long long v;
  asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"(saddr) : "memory");
  return v;
}
__device__ __forceinline__ void st_prog(uint32_t saddr, unsigned long long v) {
  asm volatile("st.volatile.shared.u64 [%0], %1;" ::"r"(saddr), "l"(v) : "memory");
}

__device__ __forceinline__ unsigned long long prog_key(int blk, int x) {
  return ((unsigned long long)(unsigned)(blk + 1) << 32) | (unsigned long long)((unsigned)x + X_BIAS);
}

// Geometry of one 32-row block, identical for the warp that fills it and the warp that consumes it.
struct BlockGeom {
  int base, ngroups;
};

__device__ __forceinline__ void row_span(int off, int len, int ref_len, int& xlo, int& xhi, unsigned& rlen) {
  // columns of a row: [max(0,off), min(off+len, refLen))   (:943-950)
  xlo = off > 0 ? off : 0;
  const long long hi64 = (long long)off + (long long)len;
  xhi = hi64 < (long long)ref_len ? (int)hi64 : ref_len;
  rlen = xhi > xlo ? (unsigned)(xhi - xlo) : 0u;
}

__device__ __forceinline__ BlockGeom block_geom(int xlo, int xhi, unsigned rlen, int lane, int& nsteps) {
  // base = leftmost column of the block: lane t first becomes active at step >= t, i.e. after the
  // reference byte for its column has travelled down the shuffle chain from lane 0
  const int lo_key = rlen ? xlo : INT_MAX;
  const int hi_key = rlen ? xhi + lane : INT_MIN;
  int base = __reduce_min_sync(FULL, lo_key);
  const int send = __reduce_max_sync(FULL, hi_key);
  nsteps = 0;
  if (base != INT_MAX) nsteps = send - base; else base = 0;
  BlockGeom g;
  g.base = base;
  g.ngroups = (nsteps + 15) >> 4;
  return g;
}

struct TeamBest {
  float S;
  int x, y, firstX, firstY, status;
  unsigned long long cells;
};

// What one lane carries from step to step.
struct LaneState {
  // What this lane hands down / keeps for its right neighbour. EMPTY = {0, 0, STOP}.
  // oP: scalar kernel = the I-run length as a float (0 unless the cell is an insertion);
  //     RAW kernel    = indelRun (low 16 bits) | direction << 16.
  float oS, oU;
  uint32_t oP, oC;
  float dS;     // score of (x-1, y-1)
  float lL;     // left_cell contribution of (x-1, y)
  float lRunF;  // scalar kernel: D-run length of (x-1, y), 0 unless it is a deletion
  bool lIsD;
  int lRun;     // RAW kernel: raw indelRun / direction of (x-1, y)
  uint32_t lDir;
  float kS;     // best score of the current row so far (strictly above the lane's earlier best)
  int kStep;    // step at which it was reached, -1: none
  int rel;      // x - xlo of the current step; inside the corridor iff (unsigned)rel < rlen
};

// One cell (x, y) at step s. `st` is the row's state (LaneState or RowState: lL, lRunF / lIsD or lRun / lDir, kS /
// kStep, rel); dS = S of (x-1, y-1), {nU, nP} = U and run of (x, y-1), r = the column's reference byte, q = the row's
// read byte. Returns the direction code; {S, U, P} is what the cell below sees as its up neighbour.
// TRIM (the skewed two-row kernel, Row = RowState) trims the half-rate ALU work of a cell, with the same results:
//  - dg: pick the score, then add (both scores stay in registers) instead of a predicated second add, which the
//    compiler turns into a constant-bank load at the head of the cell's dependency chain; the same rounding either way;
//  - scalar rule: "the left cell is a deletion" is read as lRunF > 0 instead of a bool carried across steps (which
//    the compiler packed into a register with a SEL / LOP3 per cell);
//  - scalar rule: the factor [S != 0] of e below is a saturating multiply (FMA pipe) instead of an FSET (ALU pipe).
template <bool RAW, bool ALL_ACTIVE, bool TRIM = false, class Row>
__device__ __forceinline__ uint32_t cell_update(Row& st, const Scoring& sc, const float dS, const float nU,
                                                const uint32_t nP, const uint32_t r, const uint32_t q, const bool act,
                                                const int t0rel, const int s, float& S, float& U, uint32_t& P) {
  float dg;
  if (TRIM) {
    dg = __fadd_rn(dS, r == q ? sc.mat : sc.mis);
  } else {
    dg = __fadd_rn(dS, sc.mis);
    if (r == q) dg = __fadd_rn(dS, sc.mat);
  }
  // Outside the corridor the cell must degenerate to {0, 0, STOP}: a NaN maximum makes every
  // equality below false, and fmaxf(NaN, 0) = 0 gives the score.
  const float m0 = fmaxf(fmaxf(fmaxf(st.lL, 0.0f), dg), nU);
  const float m = (ALL_ACTIVE || act) ? m0 : __int_as_float(0x7fffffff);
  const bool eL = (m == st.lL), eU = (m == nU), eG = (m == dg);
  S = ALL_ACTIVE ? m : fmaxf(m, 0.0f);  // STOP implies m == 0
  uint32_t code;
  float L;
  if (RAW) {
    const int upRaw = (int)(short)(nP & 0xffffu);
    const uint32_t upDir = (nP >> 16) & 3u;
    const bool rawHere = st.rel < t0rel;
    const int upRun = (rawHere || upDir == DIR_I) ? upRaw : 0;
    const int leftRun = (rawHere || st.lDir == DIR_D) ? st.lRun : 0;
    // priority (:1232-1267): continue D, continue I, diagonal, open D, open I, STOP
    const bool dc = eL && (leftRun > 0);
    const bool ic = !dc && eU && (upRun > 0);
    const bool gg = !dc && !ic && eG;
    const bool resolved = dc || ic || gg;
    const bool isD = dc || (!resolved && eL);
    const bool isI = ic || (!resolved && !eL && eU);
    int run = dc ? leftRun : (ic ? upRun : 0);
    run = (isD || isI) ? run + 1 : 0;
    run = (int)(short)run;  // MatrixElement::indelRun is a short
    code = gg ? DIR_DIAG : (isI ? DIR_I : (isD ? DIR_D : DIR_STOP));
    // what the neighbours will see: S + min(ext_min, gap_ext + run*decay), 0 if S == 0 (:666-676)
    const float pen = fminf(sc.ext_min, __fadd_rn(sc.gap_ext, __fmul_rn((float)run, sc.decay)));
    float e = __fadd_rn(S, pen);
    if (S == 0.0f) e = 0.0f;
    U = isI ? e : __fadd_rn(S, sc.open_read);
    L = isD ? e : __fadd_rn(S, sc.open_ref);
    P = (code << 16) | ((uint32_t)run & 0xffffu);
    st.lRun = run;
    st.lDir = code;
  } else {
    // Same priority chain as a 3-input predicate network (verified exhaustively):
    //   D  <=>  eL && (lr || !((eU && ur) || eG))
    //   I  <=>  !D && eU && (ur || !eG)
    // with run lengths kept as floats (exact below 2^24; rows are < 32768 wide here).
    const float upRunF = __uint_as_float(nP);
    bool lr;  // the left cell's run is > 0 iff it is a deletion
    if constexpr (TRIM) lr = st.lRunF > 0.0f;
    else lr = st.lIsD;
    const bool ur = upRunF > 0.0f;
    const bool X = (eU & ur) | eG;  // bitwise on purpose: straight PLOP3s, no short-circuit
    const bool pD = eL & (lr | !X);
    const bool pI = (!pD) & eU & (ur | !eG);
    code = eG ? DIR_DIAG : DIR_STOP;
    if (pI) asm volatile("mad.lo.u32 %0, %1, 0, 1;" : "=r"(code) : "r"(code));
    if (pD) asm volatile("mad.lo.u32 %0, %1, 0, 2;" : "=r"(code) : "r"(code));
    // at most one of the two run counters is alive after this cell
    // "zero, then an addition under the predicate" instead of add + select: the selects, compares and
    // min/max of this loop all go through the half-rate ALU pipe, which is what binds the kernel; a
    // predicated FADD runs on the FMA pipe (same for dg above and U / L below)
    float newD = 0.0f, newI = 0.0f;
    if (pD) asm volatile("add.rn.f32 %0, %1, 0f3F800000;" : "=f"(newD) : "f"(st.lRunF));
    if (pI) asm volatile("add.rn.f32 %0, %1, 0f3F800000;" : "=f"(newI) : "f"(upRunF));
    const float runF = __fadd_rn(newD, newI);
    const float pen = fminf(sc.ext_min, __fadd_rn(sc.gap_ext, __fmul_rn(runF, sc.decay)));
    // e = (S == 0) ? 0 : S + pen  as one exact fused op: S + pen * [S != 0]
    float nz;
    if (TRIM)  // S * 2^127 saturates to 1 for every S >= 2^-127 (S >= 0). A nonzero S is a sum of scoring values and
               // so at least the smallest of their ulps: exact for every scoring whose nonzero values are >= 2^-103
      asm("mul.sat.f32 %0, %1, 0f7F000000;" : "=f"(nz) : "f"(S));
    else
      asm("set.ne.f32.f32 %0, %1, 0f00000000;" : "=f"(nz) : "f"(S));
    U = __fadd_rn(S, sc.open_read);
    L = __fadd_rn(S, sc.open_ref);
    if (pI) asm volatile("fma.rn.f32 %0, %1, %2, %3;" : "=f"(U) : "f"(pen), "f"(nz), "f"(S));
    if (pD) asm volatile("fma.rn.f32 %0, %1, %2, %3;" : "=f"(L) : "f"(pen), "f"(nz), "f"(S));
    P = __float_as_uint(newI);
    st.lRunF = newD;
    if constexpr (!TRIM) st.lIsD = pD;
  }
  st.lL = L;
  if (S > st.kS) {  // strict: first maximum in row-major order (:1165-1170)
    // S + 0 == S bit for bit (S >= +0); as predicated FMA-pipe instructions instead of two selects
    asm volatile("add.rn.f32 %0, %1, 0f00000000;" : "=f"(st.kS) : "f"(S));
    asm volatile("mad.lo.s32 %0, %1, 1, 0;" : "=r"(st.kStep) : "r"(s));
  }
  return code;
}

// 16 steps of one lane: cells (x, y) with x = the lane's column at step 16 g + k. `iop` and `dwp` address the
// chunk's staging records and the lane's direction word of group 0. ALL_ACTIVE: every lane of the warp stays
// inside its corridor row for all 16 steps (no masking at all: the common case away from a block's wavefront ends).
// SELF_REF (ramp-free kernel, masked groups): a lane outside its row takes the reference byte of its column
// (step - colbase) from ref (columns outside [0, ref_len) read the padding byte ref[ref_len]) instead of from the
// lane above.
template <bool RAW, bool ALL_ACTIVE, int GPC, bool SELF_REF = false>
__device__ __forceinline__ void fill_group(LaneState& st, const Scoring& sc, uint4* const io_s, uint32_t* const dwp,
                                           const int g, const unsigned rlen, const uint32_t q, const int t0rel,
                                           const bool is0, const bool is31, const int src_lane,
                                           const uint8_t* ref = nullptr, int colbase = 0, unsigned ref_len = 0) {
  uint4* iop = io_s + ((g % GPC) << 5);  // [0] lane 0's input of this step, [1] lane 31's output
  uint32_t dw = 0;
  {
#pragma unroll 2  // 2 keeps the per-step predicates in registers; 4 makes ptxas spill them to a bit mask
    for (int k = 0; k < 16; ++k) {
      const int s = (g << 4) + k;
      uint4 v;
#if FILL_LANE0_LDS
      // lanes 1..31 take their upper neighbour's cell from lane t-1, lane 0 from the staged strip record
      v.x = __float_as_uint(__shfl_up_sync(FULL, st.oS, 1));
      v.y = __float_as_uint(__shfl_up_sync(FULL, st.oU, 1));
      v.z = __shfl_up_sync(FULL, st.oP, 1);
      v.w = __shfl_up_sync(FULL, st.oC, 1);
      if (is0) v = iop[0];
#else
      v.x = __float_as_uint(__shfl_sync(FULL, st.oS, src_lane));
      v.y = __float_as_uint(__shfl_sync(FULL, st.oU, src_lane));
      v.z = __shfl_sync(FULL, st.oP, src_lane);
      v.w = __shfl_sync(FULL, st.oC, src_lane);
#endif
      const float nS = __uint_as_float(v.x), nU = __uint_as_float(v.y);
      const bool act = ALL_ACTIVE ? true : ((unsigned)st.rel < rlen);
      uint32_t r = v.w;
      if (SELF_REF && !act) r = __ldg(ref + min((unsigned)(s - colbase), ref_len));
      float S, U;
      uint32_t P;
      const uint32_t code = cell_update<RAW, ALL_ACTIVE>(st, sc, st.dS, nU, v.z, r, q, act, t0rel, s, S, U, P);
      st.dS = nS;
      st.oS = S;
      st.oU = U;
      st.oP = P;
      st.oC = r;
      dw = __funnelshift_r(dw, code, 2);
#if FILL_LANE0_LDS
      if (is31) iop[1] = make_uint4(__float_as_uint(st.oS), __float_as_uint(st.oU), st.oP, st.oC);
#else
      if (is31) {
        // the record is exactly the four shuffle sources (w is rewritten when the chunk is staged)
        iop[1] = make_uint4(__float_as_uint(st.oS), __float_as_uint(st.oU), st.oP, st.oC);
        const uint4 t = iop[2];
        st.oS = __uint_as_float(t.x);
        st.oU = __uint_as_float(t.y);
        st.oP = t.z;
        st.oC = t.w;
      }
#endif
      iop += 2;
      if (!ALL_ACTIVE || RAW) ++st.rel;  // the RAW kernel needs the column for its tail rule
    }
  }
  if (ALL_ACTIVE && !RAW) st.rel += 16;
  // a lane whose 16 steps all lie outside its row has nothing the traceback will ever read: the block's
  // leading and trailing wavefront stays out of HBM (whole 32-byte sectors, the idle lanes are neighbours)
  if (ALL_ACTIVE || (st.rel > 0 && st.rel - 16 < (int)rlen)) dwp[(size_t)g * 32] = dw;
}

// NW = warps that pipeline ONE problem (1: every warp of the CTA has its own problem; otherwise the whole
// CTA is the team: 4 warps for ordinary corridors, FILL_BIG_TEAM warps for the few huge matrices of a batch
// -- a 10^8-cell realignment matrix would otherwise keep one 4-warp team busy long after the rest of the
// grid has drained).
template <bool RAW, int NW, bool PERSIST>
__global__ void __launch_bounds__((NW == 1 ? FILL_WARPS_PER_CTA : NW) * 32,
                                  NW > FILL_WARPS_PER_CTA ? 1 : (NW == 1 ? FILL_CTAS_PER_SM : FILL_TEAM_CTAS_PER_SM))
convex_fill_kernel(const FillParams p) {
  constexpr int WARPS = NW == 1 ? FILL_WARPS_PER_CTA : NW;  // warps per CTA
  constexpr int CHUNK = NW == 1 ? 64 : FILL_TEAM_CHUNK;  // steps staged through shared memory at a time
  constexpr int GPC = CHUNK / 16;           // 16-step groups per chunk
  // staging records of a chunk, interleaved: s_io[w][2 * j] = what lane 0 consumes at step j of the chunk,
  // s_io[w][2 * j + 1] = what lane 31 produced at step j (one base register + immediates serve both)
  __shared__ uint4 s_io[WARPS][2 * (CHUNK + 1)];  // +1: lane 31 reads one record ahead
  __shared__ volatile unsigned long long s_prog[WARPS];
  __shared__ int s_work, s_slot;
  __shared__ TeamBest s_best[WARPS];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int tw = NW == 1 ? 0 : wib;  // warp index within the team
  // Boundary strips: a persistent launch (grid capped, every CTA loops over problems) owns strip blockIdx.x. A
  // launch of short-lived CTAs (one problem each, so that SM slots keep coming free for the other kernels of the
  // step) takes one of p.sm_slot_count strips of the SM it happens to run on and gives it back when it exits; a
  // CTA that finds them all taken (registers would let one more team in than the kernel runs best with: more
  // strips competing for L2) sleeps until one is returned.
  unsigned smid = 0, slot_bit = 0;
  if (!PERSIST) {
    if (threadIdx.x == 0) {
      asm("mov.u32 %0, %%smid;" : "=r"(smid));
      int got = -1;
      for (;;) {
        for (int b = 0; b < p.sm_slot_count && got < 0; ++b)
          if (!(atomicOr(p.sm_slots + smid, 1u << b) & (1u << b))) got = b;
        if (got >= 0) break;
        __nanosleep(2000);
      }
      slot_bit = 1u << got;
      s_slot = (int)smid * FILL_SM_SLOTS + got;
    }
    __syncthreads();
  }
  const int cta_slot = PERSIST ? (int)blockIdx.x : s_slot;
  const int team_global = NW == 1 ? cta_slot * WARPS + wib : cta_slot;
  uint4* const io_s = s_io[wib];
  // strip[x + STRIP_PAD] = {S, U, run, ref byte} of column x of the most recently finished bottom row
  uint4* const strip = reinterpret_cast<uint4*>(p.bnd) + (size_t)team_global * p.bnd_stride + STRIP_PAD;
  const Scoring sc = p.sc;
  const uint32_t empty_pack = RAW ? (DIR_STOP << 16) : 0u;  // scalar kernel: run 0.0f
  const uint4 EMPTY = make_uint4(0u, __float_as_uint(sc.open_read), empty_pack, 0u);
  const bool is0 = lane == 0, is31 = lane == 31;
  const int src_lane = (lane + 31) & 31;  // rotate: lane 0 receives what lane 31 staged for it
  const uint32_t my_prog = (uint32_t)__cvta_generic_to_shared(const_cast<unsigned long long*>(&s_prog[tw]));
  const uint32_t prev_prog =
      (uint32_t)__cvta_generic_to_shared(const_cast<unsigned long long*>(&s_prog[(tw + NW - 1) % NW]));

  // A short-lived CTA takes p.problems_per_cta (= 1) problems per warp / team. The bound is a kernel parameter on
  // purpose: with a literal 1 the compiler peels the loop away and allocates registers for straight-line code,
  // which runs slower than the loop form the kernel was tuned in.
  for (int taken = 0; PERSIST || taken < p.problems_per_cta; ++taken) {
    int w = 0;
    if (NW == 1) {
      if (is0) w = atomicAdd(p.work_counter, 1);
      w = __shfl_sync(FULL, w, 0);
    } else {
      __syncthreads();  // previous problem fully retired (strip, progress words, s_work)
      if (threadIdx.x == 0) s_work = atomicAdd(p.work_counter, 1);
      if (threadIdx.x < NW) s_prog[threadIdx.x] = 0ull;
      __syncthreads();
      w = s_work;
    }
    w += p.first;  // this launch works on order[first, last)
    if (w >= p.last) break;
    const int ai = p.order[w];
    const AlnDesc d = p.desc[ai];
    const uint8_t* __restrict__ ref = p.seq + d.ref_off;
    const uint8_t* __restrict__ qry = p.seq + d.qry_off;
    CorridorView cv;

    cv.bind(p.c_off, p.c_len, p.c_blkbase, p.c_delta, d);
    const int H = d.height, ref_len = d.ref_len;
    const int nblk = (H + 31) >> 5;

    // curr_max starts at -1 (:921), so the first visited cell is always recorded and only strictly
    // larger scores replace it: track improvements over 0 here and remember the first visited cell.
    float bestS = 0.0f;
    int bestX = 0, bestY = 0;
    int firstX = 0, firstY = -1;
    unsigned long long cells = 0;
    int status = ST_OK;

    // strip columns [wlo, whi) hold records of the row above the current block; everything else
    // reads as EMPTY. Nothing is written before block 0.
    int wlo = 0, whi = 0;

    // rows of this warp's next block are fetched one block ahead
    int n_off = 0, n_len = 0;
    uint32_t n_q = 0x100u;  // never equals a byte
    load_corridor_rows(cv, tw, lane, H, n_off, n_len);
    if ((tw << 5) + lane < H) n_q = qry[(tw << 5) + lane];

    for (int b = tw; b < nblk; b += NW) {
      const int y = (b << 5) + lane;
      const int off = n_off, len = n_len;
      const uint32_t q = n_q;
      {
        const int yn = y + 32 * NW;
        n_q = 0x100u;
        load_corridor_rows(cv, b + NW, lane, H, n_off, n_len);
        if (yn < H) n_q = qry[yn];
      }
      int xlo, xhi, nsteps;
      unsigned rlen;
      row_span(off, len, ref_len, xlo, xhi, rlen);
      const BlockGeom geo = block_geom(xlo, xhi, rlen, lane, nsteps);
      const int base = geo.base, ngroups = geo.ngroups;
      const int nchunks = (ngroups + GPC - 1) / GPC;
      cells += rlen;
      if (firstY < 0) {
        const unsigned any = __ballot_sync(FULL, rlen != 0);
        if (any) {
          const int l0 = __ffs(any) - 1;
          firstY = (b << 5) + l0;
          firstX = __shfl_sync(FULL, xlo, l0);
        }
      }
      if (NW > 1) {
        // what the warp filling block b-1 writes: recompute its geometry from its rows
        wlo = 0; whi = 0;
        if (b > 0) {
          int poff, plen, pxlo, pxhi, pn;
          unsigned prl;
          load_corridor_rows(cv, b - 1, lane, H, poff, plen);
          row_span(poff, plen, ref_len, pxlo, pxhi, prl);
          const BlockGeom pg = block_geom(pxlo, pxhi, prl, lane, pn);
          wlo = pg.base - 31;
          whi = wlo + (pg.ngroups << 4);
        }
      }
      // team mode: block until the producer of block b-1 has flushed strip columns < x_end
      auto wait_for = [&](int x_end) {
        if (NW > 1 && b > 0) {
          const int need = x_end < whi ? x_end : whi;
          if (need > wlo) {
            const unsigned long long key = prog_key(b - 1, need);
            if (is0) {
              while (ld_prog(prev_prog) < key) __nanosleep(64);
              team_fence();  // acquire on the polling lane, BEFORE the barrier that releases the others
            }
            __syncwarp();
          }
        }
      };
      auto strip_rec = [&](int x) -> uint4 { return (x >= wlo && x < whi) ? ld_strip(strip + x) : EMPTY; };

      unsigned long long word_off = 0;
      if (is0) {
        word_off = atomicAdd(p.dir_alloc, (unsigned long long)ngroups * 32ull);
        BlockRec br;
        br.word_off = word_off;
        br.base = base;
        br.nsteps = nsteps;
        p.blocks[d.blk_off + b] = br;
      }
      word_off = __shfl_sync(FULL, word_off, 0);
      if (word_off + (unsigned long long)ngroups * 32ull > p.dir_capacity) {
        status = ST_DIR_OVERFLOW;
        break;
      }
      uint32_t* __restrict__ dwp = p.dir + word_off + lane;

      const int t0rel = (int)rlen > 12 ? (int)rlen - 12 : 0;  // tail start max(x0, xMax-12) - xlo (:1179)

      LaneState st;
      st.rel = base - lane - xlo;  // x - xlo at step 0
      st.oS = 0.0f;
      st.oU = sc.open_read;
      st.oP = empty_pack;
      st.oC = 0u;
      st.dS = 0.0f;
      st.lL = sc.open_ref;
      st.lRunF = 0.0f;
      st.lIsD = false;
      st.lRun = 0;
      st.lDir = DIR_STOP;
      st.kS = bestS;
      st.kStep = -1;

      // stage chunk 0 (+ the diagonal neighbour of lane 0's first cell)
      wait_for(base + CHUNK);
      if (is0) st.dS = __uint_as_float(strip_rec(base - 1).x);
      uint4 pa = EMPTY, pb = EMPTY;
      uint32_t ra = 0, rb = 0;
      {
        const int x0 = base + lane;
        if (lane < CHUNK) {
          pa = strip_rec(x0);
          ra = __ldg(ref + x0);
        }
        if (CHUNK > 32) {
          pb = strip_rec(x0 + 32);
          rb = __ldg(ref + x0 + 32);
        }
      }

      for (int c = 0; c < nchunks; ++c) {
        pa.w = ra;  // the reference byte of the column rides in the record
        pb.w = rb;
        if (lane < CHUNK) io_s[2 * lane] = pa;
        if (CHUNK > 32) io_s[2 * (lane + 32)] = pb;
        __syncwarp();
#if !FILL_LANE0_LDS
        if (is31) {  // lane 31's shuffle sources carry the strip record lane 0 needs next
          const uint4 t = io_s[0];
          st.oS = __uint_as_float(t.x);
          st.oU = __uint_as_float(t.y);
          st.oP = t.z;
          st.oC = t.w;
        }
#endif
        if (c + 1 < nchunks) {  // fetch the next chunk while this one is computed
          const int x0 = base + (c + 1) * CHUNK + lane;
          wait_for(base + (c + 2) * CHUNK);
          if (lane < CHUNK) {
            pa = strip_rec(x0);
            ra = __ldg(ref + x0);
          }
          if (CHUNK > 32) {
            pb = strip_rec(x0 + 32);
            rb = __ldg(ref + x0 + 32);
          }
        }
        const int g_end = min(ngroups, (c + 1) * GPC);
        for (int g = c * GPC; g < g_end; ++g) {
          const bool all_active = __all_sync(FULL, st.rel >= 0 && st.rel + 15 < (int)rlen);
          if (all_active) fill_group<RAW, true, GPC>(st, sc, io_s, dwp, g, rlen, q, t0rel, is0, is31, src_lane);
          else fill_group<RAW, false, GPC>(st, sc, io_s, dwp, g, rlen, q, t0rel, is0, is31, src_lane);
        }
        __syncwarp();
        // flush lane 31's records of this chunk: columns [base - 31 + CHUNK*c, ...)
        {
          const int done = (g_end - c * GPC) << 4;  // steps executed in this chunk
          const int xo = base - 31 + c * CHUNK;
          if (lane < done) st_strip(strip + xo + lane, io_s[2 * lane + 1]);
          if (CHUNK > 32 && lane + 32 < done) st_strip(strip + xo + lane + 32, io_s[2 * (lane + 32) + 1]);
          if (NW > 1) {
            team_fence();
            __syncwarp();
            if (is0) st_prog(my_prog, prog_key(b, xo + done));
          }
        }
        __syncwarp();
      }

      if (st.kStep >= 0) {
        bestS = st.kS;
        bestY = y;
        bestX = base + st.kStep - lane;
      }
      if (NW == 1) {
        wlo = base - 31;
        whi = base - 31 + (ngroups << 4);
      } else if (is0) {
        st_prog(my_prog, prog_key(b, (1 << 30)));  // block complete
      }
      __syncwarp();
    }
    if (NW > 1) {
      if (is0) st_prog(my_prog, ~0ull);  // also after an arena overflow: never leave a consumer waiting
    }

    // first maximum in row-major order across lanes: larger score, then smaller y, then smaller x
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float s2 = __shfl_xor_sync(FULL, bestS, o);
      const int y2 = __shfl_xor_sync(FULL, bestY, o);
      const int x2 = __shfl_xor_sync(FULL, bestX, o);
      const unsigned long long c2 = __shfl_xor_sync(FULL, cells, o);
      const bool take = (s2 > bestS) || (s2 == bestS && (y2 < bestY || (y2 == bestY && x2 < bestX)));
      if (take) {
        bestS = s2;
        bestY = y2;
        bestX = x2;
      }
      cells += c2;
    }
    if (NW > 1) {
      if (is0) {
        TeamBest tb;
        tb.S = bestS; tb.x = bestX; tb.y = bestY; tb.firstX = firstX; tb.firstY = firstY;
        tb.status = status; tb.cells = cells;
        s_best[tw] = tb;
      }
      __syncthreads();
      if (wib == 0) {
        for (int t = 1; t < NW; ++t) {
          const TeamBest tb = s_best[t];
          const bool take = (tb.S > bestS) || (tb.S == bestS && (tb.y < bestY || (tb.y == bestY && tb.x < bestX)));
          if (take) { bestS = tb.S; bestY = tb.y; bestX = tb.x; }
          cells += tb.cells;
          if (tb.status != ST_OK) status = tb.status;
          if (tb.firstY >= 0 && (firstY < 0 || tb.firstY < firstY)) { firstY = tb.firstY; firstX = tb.firstX; }
        }
      }
    }
    if (bestS == 0.0f) {  // no positive score anywhere: the first visited cell stands (or nothing was visited)
      bestS = firstY >= 0 ? 0.0f : -1.0f;
      bestX = firstY >= 0 ? firstX : 0;
      bestY = firstY >= 0 ? firstY : 0;
    }
    if (is0 && (NW == 1 || wib == 0)) {
      FillOut o;
      o.best_score = bestS;
      o.best_x = bestX;
      o.best_y = bestY;
      o.status = status;
      o.cells = cells;
      o.dir_shift = 0;
      p.out[ai] = o;
    }
  }
  if (!PERSIST) {
    __syncthreads();
    if (threadIdx.x == 0) atomicAnd(p.sm_slots + smid, ~slot_bit);
  }
}

// ---- ramp-free schedule -------------------------------------------------------------------------------------------
// The kernel above runs a block's 32 rows in lockstep from the block's first column to its last: lane t of a block
// whose corridor advances ~1 column per row idles ~2t steps before its row starts and ~2(31-t) steps after it ends,
// W + ~62 steps for W useful ones. Here every lane moves on to its row of the warp's next block as soon as its own
// part of the current one is done, so a warp step evaluates ~32 cells wherever the block boundary is. One warp per
// problem: teams of this schedule wait on each other's strip hand-off (a team of NW warps needs corridors wider than
// NW * (32 * (1 + slope) + hand-off latency) to run without stalls) and measured slower than one warp per problem.
//
// Within a block nothing changes: lane t evaluates column x of row 32b+t at warp step O_b + t + x, so every shuffle
// dependency is the lockstep one. Lane t sweeps the columns [A, E) of block b, A = min(xlo_t, xlo_t+1) - 1,
// E = max(xhi_t, xhi_t+1): that covers its row, the up / diagonal neighbours lane t+1 reads from it, and one
// out-of-corridor step first, which resets its left neighbour state. Lane 31's range reaches the block's rightmost
// column (the strip window of the next block). A lane enters block b at a 16-step group boundary (the switch costs
// nothing inside a group, and a direction word holds one row), the last such boundary at or before step O_b + t + A.
// O_b is the least origin that satisfies, for every lane:
//   - its entry comes after the end of its previous range (no overlap within a lane);
//   - its entry comes at least one chunk after the chunk in which the last lane entered the previous block: the
//     warp keeps two blocks' descriptions (shared memory) and places the next one at a chunk boundary;
//   - O_b >= O_{b-1} + RING: lane 31's record of column x, flushed at the end of its chunk, must be in the strip when
//     lane 0 of the next block stages x two chunks ahead (31 + 2 chunks).
// The reference byte of a column travels down the lanes with the cell values. A lane outside its row no longer gets a
// valid one from above (the lane two rows up may have moved on), so there it loads the byte itself: every lane that
// is inside its row then receives it from a lane that is in the same block.
// Direction words: the warp's 16-step groups are numbered from its first step, and each block's BlockRec maps its
// cells into them (base = 16 * first group - O_b): readers see the lockstep layout.
constexpr int RF_NONE = INT_MIN;  // no entry: the lane has no columns in that block

struct RfFrame {
  int blk;        // -1: none
  int O;          // lane t evaluates column x of row 32 * blk + t at warp step O + t + x
  int wlo, whi;   // strip columns lane 31 of block blk-1 wrote (what lane 0 reads; everything else is EMPTY)
  int a31, e31;   // lane 31's columns [a31, e31)
  int sw0, sw31;  // entry steps of lanes 0 and 31 (RF_NONE: none)
  int swmax;      // entry step of the last lane (no entries: the earliest allowed one - 1)
};

struct RfWarp {
  unsigned long long word_off;  // the warp's direction words: group g of its steps at word_off + 32 g
  int G;                        // groups of 16 steps the warp runs for its problem
  int next_b, R, O_last;        // the block to place next, its earliest entry, the last placed origin
  int firstX, firstY;           // first visited cell
};

// Lane t's columns [A, E) of a block (A = INT_MAX: none), from its row and the row below.
__device__ __forceinline__ void rf_cols(int xlo, int xhi, unsigned rlen, int lane, int& A, int& E) {
  const int a = rlen ? xlo : INT_MAX;
  const int e = rlen ? xhi : INT_MIN;
  int a1 = __shfl_down_sync(FULL, a, 1), e1 = __shfl_down_sync(FULL, e, 1);
  const int emax = __reduce_max_sync(FULL, e);
  if (lane == 31) {
    a1 = INT_MAX;
    e1 = emax;
  }
  const int amin = min(a, a1);
  A = amin == INT_MAX ? INT_MAX : amin - 1;
  E = max(e, e1);
}

// Origin and entry step of a block from the lane's columns [A, ...). lag: the lane's stagger (it evaluates column x
// at step O + lag + x); L: end of the lane's previous range (RF_NONE: none); R: earliest entry; O_min: the hand-off
// bound.
__device__ __forceinline__ void rf_origin(int lag, int A, int L, int R, int O_min, int& O, int& sw) {
  const int from = max(L, R);
  const int need = A == INT_MAX ? INT_MIN : ((from + 15) & ~15) - lag - A;
  O = max(O_min, __reduce_max_sync(FULL, need));
  sw = A == INT_MAX ? RF_NONE : ((O + lag + A) & ~15);
}

// Origin and entry steps of block b (see rf_origin).
__device__ __forceinline__ void rf_place(const CorridorView& cv, int b, int lane, int H, int ref_len, int L, int R,
                                         int O_min, int& xlo, unsigned& rlen, int& A, int& E, int& O, int& sw) {
  int off, len, xhi;
  load_corridor_rows(cv, b, lane, H, off, len);
  row_span(off, len, ref_len, xlo, xhi, rlen);
  rf_cols(xlo, xhi, rlen, lane, A, E);
  rf_origin(lane, A, L, R, O_min, O, sw);
}

constexpr int RF_CHUNK = 64;                  // steps staged through shared memory at a time
constexpr int RF_RING = 32 + 2 * RF_CHUNK;    // hand-off spacing of consecutive origins

// the earliest entry into the block after one whose last lane enters at step swmax
__device__ __forceinline__ int rf_next_entry(int swmax) { return ((swmax + RF_CHUNK) / RF_CHUNK + 1) * RF_CHUNK; }

// A strip slot of the SM the calling CTA runs on (short-lived CTAs, see convex_fill_kernel): SM * FILL_SM_SLOTS + slot.
__device__ __forceinline__ int take_sm_slot(const FillParams& p) {
  unsigned smid;
  asm("mov.u32 %0, %%smid;" : "=r"(smid));
  int got = -1;
  for (;;) {
    for (int b = 0; b < p.sm_slot_count && got < 0; ++b)
      if (!(atomicOr(p.sm_slots + smid, 1u << b) & (1u << b))) got = b;
    if (got >= 0) break;
    __nanosleep(2000);
  }
  return (int)smid * FILL_SM_SLOTS + got;
}

template <bool RAW, bool PERSIST>
__global__ void __launch_bounds__(FILL_WARPS_PER_CTA * 32, FILL_CTAS_PER_SM)
convex_fill_rf_kernel(const FillParams p) {
  constexpr int WARPS = FILL_WARPS_PER_CTA;
  constexpr int CHUNK = RF_CHUNK;
  constexpr int GPC = CHUNK / 16;
  __shared__ uint4 s_io[WARPS][2 * (CHUNK + 1)];
  __shared__ int s_slot;
  __shared__ RfFrame s_f0[WARPS], s_f31[WARPS], s_nx[WARPS];  // the blocks lanes 0 / 31 are in, the next block
  __shared__ int4 s_nrow[WARPS][32];     // the lane's row of the next block: {rel at entry, rlen, q}
  __shared__ int4 s_cur[WARPS][32];      // {O, y} of the lane's current row, L = end of its last range, its cells
  __shared__ float4 s_bestl[WARPS][32];  // the lane's best cell of its finished rows {S, x, y}
  __shared__ RfWarp s_w[WARPS];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  if (!PERSIST) {  // as in convex_fill_kernel; the slot is given back from s_slot (no registers held meanwhile)
    if (threadIdx.x == 0) s_slot = take_sm_slot(p);
    __syncthreads();
  }
  const int cta_slot = PERSIST ? (int)blockIdx.x : s_slot;
  uint4* const io_s = s_io[wib];
  uint4* const strip = reinterpret_cast<uint4*>(p.bnd) + (size_t)(cta_slot * WARPS + wib) * p.bnd_stride + STRIP_PAD;
  const Scoring sc = p.sc;
  const uint32_t empty_pack = RAW ? (DIR_STOP << 16) : 0u;
  const uint4 EMPTY = make_uint4(0u, __float_as_uint(sc.open_read), empty_pack, 0u);
  const bool is0 = lane == 0, is31 = lane == 31;
  const int src_lane = (lane + 31) & 31;
  RfWarp& ws = s_w[wib];

  for (int taken = 0; PERSIST || taken < p.problems_per_cta; ++taken) {
    int w = 0;
    if (is0) w = atomicAdd(p.work_counter, 1);
    w = __shfl_sync(FULL, w, 0) + p.first;
    if (w >= p.last) break;
    const int ai = p.order[w];
    // The descriptor and the corridor view are re-read where they are needed (block boundaries) instead of being
    // kept in registers across the cell loop; likewise the warp's bookkeeping lives in shared memory.
    auto corridor = [&]() {
      CorridorView cv;
      cv.bind(p.c_off, p.c_len, p.c_blkbase, p.c_delta, p.desc[ai]);
      return cv;
    };
    const uint8_t* __restrict__ ref = p.seq + p.desc[ai].ref_off;
    const unsigned ref_len = (unsigned)p.desc[ai].ref_len;
    int status = ST_OK;

    // Pass 1: the warp's schedule (the same placements as pass 2 makes) -> its number of steps.
    {
      const CorridorView cv = corridor();
      const int H = p.desc[ai].height, nblk = (H + 31) >> 5;
      int L = RF_NONE, R = 0, O_last = RF_NONE;
      for (int b = 0; b < nblk; ++b) {
        int xlo, A, E, O, sw;
        unsigned rlen;
        rf_place(cv, b, lane, H, (int)ref_len, L, R, O_last == RF_NONE ? INT_MIN : O_last + RF_RING, xlo, rlen, A, E,
                 O, sw);
        if (__any_sync(FULL, sw != RF_NONE)) O_last = O;
        if (sw != RF_NONE) L = O + lane + E;
        R = rf_next_entry(__reduce_max_sync(FULL, sw != RF_NONE ? sw : R - 1));
      }
      const int T = max(0, __reduce_max_sync(FULL, L));
      const int G = (T + 15) >> 4;
      unsigned long long wo = 0;
      if (is0) wo = atomicAdd(p.dir_alloc, (unsigned long long)G * 32ull);
      wo = __shfl_sync(FULL, wo, 0);
      if (wo + (unsigned long long)G * 32ull > p.dir_capacity) status = ST_DIR_OVERFLOW;
      if (is0) {
        ws.word_off = wo;
        ws.G = G;
        ws.next_b = 0;
        ws.R = 0;
        ws.O_last = RF_NONE;
        ws.firstX = 0;
        ws.firstY = -1;
        RfFrame none;
        none.blk = -1;
        none.O = none.wlo = none.whi = none.a31 = none.e31 = 0;
        none.sw0 = none.sw31 = RF_NONE;
        none.swmax = 0;
        s_f0[wib] = none;
        s_f31[wib] = none;
        s_nx[wib] = none;
      }
      s_cur[wib][lane] = make_int4(0, 0, RF_NONE, 0);
      s_bestl[wib][lane] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      __syncwarp();
    }
    uint32_t* __restrict__ dwp = p.dir + ws.word_off + lane;

    // Pass 2.
    LaneState st;
    st.rel = 0;
    st.oS = 0.0f;
    st.oU = sc.open_read;
    st.oP = empty_pack;
    st.oC = 0u;
    st.dS = 0.0f;
    st.lL = sc.open_ref;
    st.lRunF = 0.0f;
    st.lIsD = false;
    st.lRun = 0;
    st.lDir = DIR_STOP;
    st.kS = 0.0f;
    st.kStep = -1;
    unsigned rlen = 0;  // before its first row a lane is outside every corridor
    uint32_t q = 0x100u;
    int t0rel = 0;
    int sw = RF_NONE;   // step at which this lane enters the next block

    // next block -> s_nx / s_nrow / sw, its BlockRec, the lane's cells and the warp's first visited cell
    auto place = [&]() {
      const CorridorView cv = corridor();
      const AlnDesc* dp = p.desc + ai;
      const int H = dp->height;
      const int b = ws.next_b, R = ws.R, O_last = ws.O_last;
      int4 me = s_cur[wib][lane];
      int nxlo, A, E, O, swl;
      unsigned rl;
      rf_place(cv, b, lane, H, (int)ref_len, me.z, R, O_last == RF_NONE ? INT_MIN : O_last + RF_RING, nxlo, rl, A, E,
               O, swl);
      const bool any = __any_sync(FULL, swl != RF_NONE);
      if (swl != RF_NONE) me.z = O + lane + E;
      me.w += (int)rl;  // cells of this lane's rows (< 2^32 for every problem the ordinary launches get)
      const int swmax = __reduce_max_sync(FULL, swl != RF_NONE ? swl : R - 1);
      const int y = (b << 5) + lane;
      const int4 nrow = make_int4(swl - (O + lane + nxlo), (int)rl, y < H ? (int)p.seq[dp->qry_off + y] : 0x100, 0);
      const unsigned hit = __ballot_sync(FULL, rl != 0);
      const int fx = hit ? __shfl_sync(FULL, nxlo, __ffs(hit) - 1) : 0;
      // lane 31's columns of block b-1: what lane 0 of block b reads from the strip
      int wlo = 0, whi = 0;
      if (b > 0) {
        int pxlo, pxhi, poff, plen, pA, pE;
        unsigned prl;
        load_corridor_rows(cv, b - 1, lane, H, poff, plen);
        row_span(poff, plen, (int)ref_len, pxlo, pxhi, prl);
        rf_cols(pxlo, pxhi, prl, lane, pA, pE);
        pA = __shfl_sync(FULL, pA, 31);
        pE = __shfl_sync(FULL, pE, 31);
        if (pA != INT_MAX) {
          wlo = pA;
          whi = pE;
        }
      }
      const int g0 = __reduce_min_sync(FULL, swl != RF_NONE ? swl : INT_MAX);
      const int end = __reduce_max_sync(FULL, swl != RF_NONE ? O + lane + E : INT_MIN);
      const int a31 = __shfl_sync(FULL, A, 31), e31 = __shfl_sync(FULL, E, 31);
      const int sw0 = __shfl_sync(FULL, swl, 0), sw31 = __shfl_sync(FULL, swl, 31);
      s_cur[wib][lane] = me;
      s_nrow[wib][lane] = nrow;
      sw = swl;
      __syncwarp();
      if (is0) {
        BlockRec br;
        br.word_off = ws.word_off + (any ? (unsigned long long)(g0 >> 4) * 32ull : 0ull);
        br.base = any ? g0 - O : 0;
        br.nsteps = any ? end - g0 : 0;
        p.blocks[dp->blk_off + b] = br;
        RfFrame f;
        f.blk = b;
        f.O = O;
        f.wlo = wlo;
        f.whi = whi;
        f.a31 = a31;
        f.e31 = e31;
        f.sw0 = sw0;
        f.sw31 = sw31;
        f.swmax = swmax;
        s_nx[wib] = f;
        ws.next_b = b + 1;
        ws.R = rf_next_entry(swmax);
        if (any) ws.O_last = O;
        if (hit && ws.firstY < 0) {
          ws.firstY = (b << 5) + __ffs(hit) - 1;
          ws.firstX = fx;
        }
      }
      __syncwarp();
    };
    // the strip records and reference bytes lane 0 consumes at steps [kk * CHUNK, (kk + 1) * CHUNK): record j is
    // the record of lane 0's column at step kk * CHUNK + j in the block lane 0 is in at that step
    uint4 pa = EMPTY, pb = EMPTY;
    auto stage = [&](int kk) {
      const RfFrame* n = &s_nx[wib];
      const RfFrame* f = &s_f0[wib];
      const int nblk_ = n->blk, nsw0 = n->sw0, fblk = f->blk;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int sigma = kk * CHUNK + lane + 32 * h;
        const bool in_n = nblk_ >= 0 && nsw0 != RF_NONE && sigma >= nsw0;
        const RfFrame* fr = in_n ? n : f;
        const int col = sigma - fr->O;
        uint4 rec = EMPTY;
        if (in_n || fblk >= 0) {
          if (col >= fr->wlo && col < fr->whi) rec = ld_strip(strip + col);
          rec.w = (unsigned)col < ref_len ? __ldg(ref + col) : 0u;  // the column's reference byte
        }
        if (h == 0) pa = rec;
        else pb = rec;
      }
    };

    const int nchunks = status == ST_OK ? (ws.G + GPC - 1) / GPC : 0;
    if (nchunks > 0) {
      place();
      stage(0);
    }
    for (int c = 0; c < nchunks; ++c) {
      // every lane has entered the next block: it becomes the current one, and the one after it is placed
      for (;;) {
        const RfFrame n = s_nx[wib];
        if (n.blk < 0 || n.swmax >= c * CHUNK) break;
        __syncwarp();
        if (is0) {
          if (n.sw0 != RF_NONE) s_f0[wib] = n;
          if (n.sw31 != RF_NONE) s_f31[wib] = n;
          s_nx[wib].blk = -1;
        }
        __syncwarp();
        if (ws.next_b < ((p.desc[ai].height + 31) >> 5)) place();
        else sw = RF_NONE;
      }
      io_s[2 * lane] = pa;
      io_s[2 * (lane + 32)] = pb;
      __syncwarp();
#if !FILL_LANE0_LDS
      if (is31) {
        const uint4 t = io_s[0];
        st.oS = __uint_as_float(t.x);
        st.oU = __uint_as_float(t.y);
        st.oP = t.z;
        st.oC = t.w;
      }
#endif
      if (c + 1 < nchunks) stage(c + 1);
      const int g_end = min(ws.G, (c + 1) * GPC);
      for (int g = c * GPC; g < g_end; ++g) {
        if ((g << 4) == sw) {  // this lane enters its row of the next block
          int4 me = s_cur[wib][lane];
          if (st.kStep >= 0) {
            s_bestl[wib][lane] = make_float4(st.kS, __int_as_float(st.kStep - me.x - lane), __int_as_float(me.y), 0.0f);
            st.kStep = -1;
          }
          const int4 nr = s_nrow[wib][lane];
          st.rel = nr.x;
          rlen = (unsigned)nr.y;
          q = (uint32_t)nr.z;
          t0rel = nr.y > 12 ? nr.y - 12 : 0;
          me.x = s_nx[wib].O;
          me.y = (s_nx[wib].blk << 5) + lane;
          s_cur[wib][lane] = me;
          sw = RF_NONE;
        }
        const bool all_active = __all_sync(FULL, st.rel >= 0 && st.rel + 15 < (int)rlen);
        if (all_active) {
          fill_group<RAW, true, GPC>(st, sc, io_s, dwp, g, rlen, q, t0rel, is0, is31, src_lane);
        } else {
          // column of the lane at step s: s - (O + lane), O of the row it is in
          fill_group<RAW, false, GPC, true>(st, sc, io_s, dwp, g, rlen, q, t0rel, is0, is31, src_lane, ref,
                                             s_cur[wib][lane].x + lane, ref_len);
        }
      }
      __syncwarp();
      // flush lane 31's records of this chunk that lie in its columns of the block it was in
      {
        const RfFrame* n = &s_nx[wib];
        const RfFrame* f = &s_f31[wib];
        const int done = (g_end - c * GPC) << 4;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int j = lane + 32 * h;
          const int sigma = c * CHUNK + j;
          const bool in_n = n->blk >= 0 && n->sw31 != RF_NONE && sigma >= n->sw31;
          const RfFrame* fr = in_n ? n : f;
          const int x = sigma - fr->O - 31;
          if (j < done && (in_n || f->blk >= 0) && x >= fr->a31 && x < fr->e31) st_strip(strip + x, io_s[2 * j + 1]);
        }
      }
      __syncwarp();
    }
    const int4 me = s_cur[wib][lane];
    const float4 bl = s_bestl[wib][lane];
    float bestS = bl.x;
    int bestX = __float_as_int(bl.y), bestY = __float_as_int(bl.z);
    if (st.kStep >= 0) {
      bestS = st.kS;
      bestX = st.kStep - me.x - lane;
      bestY = me.y;
    }
    unsigned long long cells = (unsigned)me.w;
    // blocks the schedule never reached have no cells
    if (is0 && status == ST_OK)
      for (int b = ws.next_b; b < ((p.desc[ai].height + 31) >> 5); ++b) {
        BlockRec br;
        br.word_off = ws.word_off;
        br.base = 0;
        br.nsteps = 0;
        p.blocks[p.desc[ai].blk_off + b] = br;
      }

    // first maximum in row-major order across lanes: larger score, then smaller y, then smaller x
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float s2 = __shfl_xor_sync(FULL, bestS, o);
      const int y2 = __shfl_xor_sync(FULL, bestY, o);
      const int x2 = __shfl_xor_sync(FULL, bestX, o);
      const unsigned long long c2 = __shfl_xor_sync(FULL, cells, o);
      const bool take = (s2 > bestS) || (s2 == bestS && (y2 < bestY || (y2 == bestY && x2 < bestX)));
      if (take) {
        bestS = s2;
        bestY = y2;
        bestX = x2;
      }
      cells += c2;
    }
    if (bestS == 0.0f) {  // no positive score anywhere: the first visited cell stands (or nothing was visited)
      const bool any = ws.firstY >= 0;
      bestS = any ? 0.0f : -1.0f;
      bestX = any ? ws.firstX : 0;
      bestY = any ? ws.firstY : 0;
    }
    if (is0) {
      FillOut o;
      o.best_score = bestS;
      o.best_x = bestX;
      o.best_y = bestY;
      o.status = status;
      o.cells = cells;
      o.dir_shift = 0;
      p.out[ai] = o;
    }
    __syncwarp();
  }
  if (!PERSIST) {
    __syncthreads();
    if (threadIdx.x == 0) atomicAnd(p.sm_slots + s_slot / FILL_SM_SLOTS, ~(1u << (s_slot % FILL_SM_SLOTS)));
  }
}

// ---- ramp-free schedule, two rows per lane -------------------------------------------------------------------------
// The schedule above with 64-row blocks: lane t owns rows 64b + 2t (its first row) and 64b + 2t + 1 (its second) and
// evaluates column x of both at warp step O_b + t + x, the first row before the second. The first row takes its up and
// diagonal neighbours from lane t-1's second row through the shuffle, as before; the second row takes them from the
// first row's fresh cell and from its cell of the step before, in registers, and both rows use the same reference
// byte. Every shuffle, strip hand-off, loop step and reference byte therefore serves two cells, and the per-block work
// (placement, masked groups at the block switch) is spread over 64 rows.
// Lane t's columns [A, E) of a block cover its two rows and the row below (lane t+1's first row), one
// out-of-corridor step first; lane 31's reach the block's rightmost column. The placement rules are those above.
// Where the first row is outside its corridor lane t-1 may have left the block, so the lane loads the reference byte
// itself there (its second row may still be inside).
// Direction words: group g of the warp's steps is a line of 64 words, lane t's two rows at 64 g + 2t and 64 g + 2t + 1
// (one 8-byte store per lane). The two 32-row halves of a block keep a BlockRec each: half h at word_off + 32 h with
// base - 16 h, so that cell (x, 32 (2b + h) + j) lies at step x - base + (j >> 1) (FillOut::dir_shift = 1).

// What one row of a lane carries from step to step (the fields of LaneState that belong to a row).
struct RowState {
  float lL;
  float lRunF;
  bool lIsD;
  int lRun;
  uint32_t lDir;
  float kS;
  int kStep;
  int rel;
};

struct Lane2State {
  float oS, oU;  // the second row's cell: what lane t+1 (or lane 0 of the next block) reads, as in LaneState
  uint32_t oP, oC;
  float dS;      // S of (x-1, first row - 1)
  float dS2;     // S of (x-1, first row); SKEW: of (x-2, first row)
  // SKEW only: the first row's cell of the step before {S, U, run} (column x-1: the second row's up neighbour) and
  // the reference byte of column x-1 (the second row's)
  float pS, pU;
  uint32_t pP, r1;
  RowState a, b; // first and second row
};

struct RowGeom {
  unsigned rlen;
  uint32_t q;
  int t0rel;
};

__device__ __forceinline__ void row_init(RowState& r, const Scoring& sc) {
  r.lL = sc.open_ref;
  r.lRunF = 0.0f;
  r.lIsD = false;
  r.lRun = 0;
  r.lDir = DIR_STOP;
  r.kS = 0.0f;
  r.kStep = -1;
  r.rel = 0;
}

// fill_group for two rows per lane; `dwp` addresses the lane's pair of direction words of group 0. At step s the
// first row is at column x = s - colbase; the second row is at x too, or at x - 1 with SKEW.
template <bool RAW, bool SKEW, bool ALL_ACTIVE, int GPC, bool SELF_REF = false>
__device__ __forceinline__ void fill_group2(Lane2State& st, const Scoring& sc, uint4* const io_s, uint2* const dwp,
                                            const int g, const RowGeom& ga, const RowGeom& gb, const bool is31,
                                            const int src_lane, const uint8_t* ref = nullptr, int colbase = 0,
                                            unsigned ref_len = 0) {
  uint4* iop = io_s + ((g % GPC) << 5);
  uint32_t dwa = 0, dwb = 0;
  uint32_t qa = 0, qb = 0;  // SKEW: the codes of the current 4 steps, step j at bits 2j
  {
#pragma unroll(SKEW ? 4 : 2)
    for (int k = 0; k < 16; ++k) {
      const int s = (g << 4) + k;
      uint4 v;
      v.x = __float_as_uint(__shfl_sync(FULL, st.oS, src_lane));
      v.y = __float_as_uint(__shfl_sync(FULL, st.oU, src_lane));
      v.z = __shfl_sync(FULL, st.oP, src_lane);
      v.w = __shfl_sync(FULL, st.oC, src_lane);
      const float nS = __uint_as_float(v.x), nU = __uint_as_float(v.y);
      const bool actA = ALL_ACTIVE ? true : ((unsigned)st.a.rel < ga.rlen);
      const bool actB = ALL_ACTIVE ? true : ((unsigned)st.b.rel < gb.rlen);
      uint32_t r = v.w;
      float SA, UA, SB, UB;
      uint32_t PA, PB, ca, cb;
      if (SKEW) {
        // the two cells share no data: the second row's neighbours are all from earlier steps
        const uint32_t rb = st.r1;
        // outside its corridor the first row's cell does not depend on r, so the byte the lane loads there is only
        // kept for the second row (next step): the load stays off this step's dependency chain
        uint32_t rk = r;
        if (SELF_REF && !actA) rk = __ldg(ref + min((unsigned)(s - colbase), ref_len));
        ca = cell_update<RAW, ALL_ACTIVE, true>(st.a, sc, st.dS, nU, v.z, r, ga.q, actA, ga.t0rel, s, SA, UA, PA);
        cb = cell_update<RAW, ALL_ACTIVE, true>(st.b, sc, st.dS2, st.pU, st.pP, rb, gb.q, actB, gb.t0rel, s, SB, UB,
                                                PB);
        st.dS = nS;
        st.dS2 = st.pS;
        st.pS = SA;
        st.pU = UA;
        st.pP = PA;
        st.r1 = rk;
        r = rb;  // what lane t+1 receives with the second row's cell
      } else {
        if (SELF_REF && !actA) r = __ldg(ref + min((unsigned)(s - colbase), ref_len));
        ca = cell_update<RAW, ALL_ACTIVE>(st.a, sc, st.dS, nU, v.z, r, ga.q, actA, ga.t0rel, s, SA, UA, PA);
        st.dS = nS;
        cb = cell_update<RAW, ALL_ACTIVE>(st.b, sc, st.dS2, UA, PA, r, gb.q, actB, gb.t0rel, s, SB, UB, PB);
        st.dS2 = SA;
      }
      st.oS = SB;
      st.oU = UB;
      st.oP = PB;
      st.oC = r;
      if (SKEW) {
        // four steps' codes gathered by multiply-adds (FMA pipe), then one funnel shift per row (ALU pipe)
        const uint32_t m = 1u << (2 * (k & 3));
        asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(qa) : "r"(ca), "r"(m), "r"(qa));
        asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(qb) : "r"(cb), "r"(m), "r"(qb));
        if ((k & 3) == 3) {
          dwa = __funnelshift_r(dwa, qa, 8);
          dwb = __funnelshift_r(dwb, qb, 8);
          qa = qb = 0;
        }
      } else {
        dwa = __funnelshift_r(dwa, ca, 2);
        dwb = __funnelshift_r(dwb, cb, 2);
      }
      if (is31) {
        iop[1] = make_uint4(__float_as_uint(st.oS), __float_as_uint(st.oU), st.oP, st.oC);
        const uint4 t = iop[2];
        st.oS = __uint_as_float(t.x);
        st.oU = __uint_as_float(t.y);
        st.oP = t.z;
        st.oC = t.w;
      }
      iop += 2;
      if (!ALL_ACTIVE || RAW) {
        ++st.a.rel;
        ++st.b.rel;
      }
    }
  }
  if (ALL_ACTIVE && !RAW) {
    st.a.rel += 16;
    st.b.rel += 16;
  }
  if (ALL_ACTIVE || (st.a.rel > 0 && st.a.rel - 16 < (int)ga.rlen) || (st.b.rel > 0 && st.b.rel - 16 < (int)gb.rlen))
    dwp[(size_t)g * 32] = make_uint2(dwa, dwb);
}

// Corridor rows 64b + 2 lane and 64b + 2 lane + 1 of the whole warp; rows >= H read as {0, 0}.
__device__ __forceinline__ void load_row_pair(const CorridorView& cv, int b, int lane, int H, int& offA, int& lenA,
                                              int& offB, int& lenB) {
  int o0, l0, o1, l1;
  load_corridor_rows(cv, 2 * b, lane, H, o0, l0);
  load_corridor_rows(cv, 2 * b + 1, lane, H, o1, l1);
  const int sa = (2 * lane) & 31, sb = sa + 1;
  const bool hi = lane >= 16;
  const int oa0 = __shfl_sync(FULL, o0, sa), oa1 = __shfl_sync(FULL, o1, sa);
  const int la0 = __shfl_sync(FULL, l0, sa), la1 = __shfl_sync(FULL, l1, sa);
  const int ob0 = __shfl_sync(FULL, o0, sb), ob1 = __shfl_sync(FULL, o1, sb);
  const int lb0 = __shfl_sync(FULL, l0, sb), lb1 = __shfl_sync(FULL, l1, sb);
  offA = hi ? oa1 : oa0;
  lenA = hi ? la1 : la0;
  offB = hi ? ob1 : ob0;
  lenB = hi ? lb1 : lb0;
}

// Lane t's columns [A, E) of a 64-row block (A = INT_MAX: none), from its two rows and the row below.
__device__ __forceinline__ void rf2_cols(int xloA, int xhiA, unsigned rlenA, int xloB, int xhiB, unsigned rlenB,
                                         int lane, int& A, int& E) {
  const int aA = rlenA ? xloA : INT_MAX, eA = rlenA ? xhiA : INT_MIN;
  const int aB = rlenB ? xloB : INT_MAX, eB = rlenB ? xhiB : INT_MIN;
  const int e = max(eA, eB);
  int a1 = __shfl_down_sync(FULL, aA, 1), e1 = __shfl_down_sync(FULL, eA, 1);
  const int emax = __reduce_max_sync(FULL, e);
  if (lane == 31) {
    a1 = INT_MAX;
    e1 = emax;
  }
  const int amin = min(min(aA, aB), a1);
  A = amin == INT_MAX ? INT_MAX : amin - 1;
  E = max(e, e1);
}

// rf_place for 64-row block b; lag: the lane's stagger (lane, or 2 lane with SKEW).
__device__ __forceinline__ void rf2_place(const CorridorView& cv, int b, int lane, int lag, int H, int ref_len, int L,
                                          int R, int O_min, int& xloA, unsigned& rlenA, int& xloB, unsigned& rlenB,
                                          int& A, int& E, int& O, int& sw) {
  int offA, lenA, offB, lenB, xhiA, xhiB;
  load_row_pair(cv, b, lane, H, offA, lenA, offB, lenB);
  row_span(offA, lenA, ref_len, xloA, xhiA, rlenA);
  row_span(offB, lenB, ref_len, xloB, xhiB, rlenB);
  rf2_cols(xloA, xhiA, rlenA, xloB, xhiB, rlenB, lane, A, E);
  rf_origin(lag, A, L, R, O_min, O, sw);
}

// Skewed variant (SKEW = true, the default; NGMLR_B200_FILL_RF2_SKEW=0 selects the schedule above). Lane t evaluates
// column x of its first row at warp step O_b + 2t + x and column x - 1 of its second row in the same step, so the two
// cell updates of a step share no data and each step's dependency chain is one cell long instead of two:
//   first row:  up (x, 2t-1) and diagonal (x-1, 2t-1) are lane t-1's second-row cells of the step before and the one
//               before that (the shuffle and dS, as above);
//   second row: up (x-1, 2t) and diagonal (x-2, 2t) are the first row's cells of the step before and the one before
//               that, left (x-2, 2t+1) is its own cell of the step before; the reference byte of x-1 is the one the
//               first row had the step before (kept in a register, never reloaded).
// Lane t+1's first row reaches column x one step after lane t's second row (O_b + 2t + 2 + x against O_b + 2t + 1 + x):
// the same shuffle distances as above.
// Both rows sweep the columns [A, E) of rf2_cols, so in first-row columns the lane runs [A, E + 1): its range ends
// at step O_b + 2t + E + 1 (pass 1's step count and the next block's entry bound L use that end).
// Hand-off: lane 31 trails lane 0 by 63 steps (62 of lane stagger + 1 of row skew), so its record of warp step sigma
// is its second row's column sigma - O - 63 (the flush window). The record of column x, produced at step
// O_{b-1} + 63 + x, is flushed at the end of its chunk; lane 0 of block b stages column x at the start of the chunk two
// before the one holding step O_b + x. Since floor((a + 2 CHUNK) / CHUNK) = floor(a / CHUNK) + 2,
// O_b >= O_{b-1} + 63 + 2 CHUNK is enough: RF2S_RING = 64 + 2 CHUNK.
// Strip columns: lane 31 writes and lane 0 reads lane 31's [A, E) of rf2_cols, within [-1, refLen] as in the other
// schedules; the stagger changes when a column passes through the strip, not which, so STRIP_PAD = 32 (>= 1) and the
// host's STRIP_SLACK still cover it.
// Direction words (FillOut::dir_shift = 2): the layout above (a 64-word line per group, one 8-byte store per lane) with
// half h's BlockRec at word_off + 32 h and base = 16 * first group - O_b - 32 h, so that cell (x, 32 (2b + h) + j) lies
// at step x - base + j (lane 16 h + (j >> 1), row j & 1: warp step O_b + 2 (16 h + (j >> 1)) + (j & 1) + x).
// Step count: a block still advances the warp's steps by at most its column span plus the hand-off and placement
// slack (RF2S_RING + 2 chunks + a group < 400), so the host's int guard holds unchanged.
constexpr int RF2S_RING = 64 + 2 * RF_CHUNK;

template <bool RAW, bool PERSIST, bool SKEW>
__global__ void __launch_bounds__(FILL_WARPS_PER_CTA * 32, FILL_RF2_CTAS_PER_SM)
convex_fill_rf2_kernel(const FillParams p) {
  constexpr int WARPS = FILL_WARPS_PER_CTA;
  constexpr int CHUNK = RF_CHUNK;
  constexpr int GPC = CHUNK / 16;
  constexpr int RING = SKEW ? RF2S_RING : RF_RING;
  constexpr int TAIL = SKEW ? 1 : 0;          // steps the second row runs behind the first
  constexpr int LAG31 = SKEW ? 63 : 31;       // steps lane 31's second row trails lane 0's first row
  __shared__ uint4 s_io[WARPS][2 * (CHUNK + 1)];
  __shared__ int s_slot;
  __shared__ RfFrame s_f0[WARPS], s_f31[WARPS], s_nx[WARPS];  // as in convex_fill_rf_kernel, blk counts 64-row blocks
  __shared__ int4 s_nrow[WARPS][2][32];  // the lane's two rows of the next block: {rel at entry, rlen, q}
  __shared__ int4 s_cur[WARPS][32];      // {O, y of the first row} of the lane's current rows, L, its cells
  __shared__ float4 s_bestl[WARPS][32];  // the lane's best cell of its finished rows {S, x, y}
  __shared__ RfWarp s_w[WARPS];          // word_off: group g of the warp's steps at word_off + 64 g
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  if (!PERSIST) {
    if (threadIdx.x == 0) s_slot = take_sm_slot(p);
    __syncthreads();
  }
  const int cta_slot = PERSIST ? (int)blockIdx.x : s_slot;
  uint4* const io_s = s_io[wib];
  uint4* const strip = reinterpret_cast<uint4*>(p.bnd) + (size_t)(cta_slot * WARPS + wib) * p.bnd_stride + STRIP_PAD;
  const Scoring sc = p.sc;
  const uint32_t empty_pack = RAW ? (DIR_STOP << 16) : 0u;
  const uint4 EMPTY = make_uint4(0u, __float_as_uint(sc.open_read), empty_pack, 0u);
  const bool is0 = lane == 0, is31 = lane == 31;
  const int src_lane = (lane + 31) & 31;
  const int lag = SKEW ? 2 * lane : lane;  // lane t's first row is at column x at step O_b + lag + x
  RfWarp& ws = s_w[wib];

  for (int taken = 0; PERSIST || taken < p.problems_per_cta; ++taken) {
    int w = 0;
    if (is0) w = atomicAdd(p.work_counter, 1);
    w = __shfl_sync(FULL, w, 0) + p.first;
    if (w >= p.last) break;
    const int ai = p.order[w];
    auto corridor = [&]() {
      CorridorView cv;
      cv.bind(p.c_off, p.c_len, p.c_blkbase, p.c_delta, p.desc[ai]);
      return cv;
    };
    const uint8_t* __restrict__ ref = p.seq + p.desc[ai].ref_off;
    const unsigned ref_len = (unsigned)p.desc[ai].ref_len;
    int status = ST_OK;

    // Pass 1: the warp's schedule (the same placements as pass 2 makes) -> its number of steps.
    {
      const CorridorView cv = corridor();
      const int H = p.desc[ai].height, nblk = (H + 63) >> 6;
      int L = RF_NONE, R = 0, O_last = RF_NONE;
      for (int b = 0; b < nblk; ++b) {
        int xloA, xloB, A, E, O, sw;
        unsigned rlA, rlB;
        rf2_place(cv, b, lane, lag, H, (int)ref_len, L, R, O_last == RF_NONE ? INT_MIN : O_last + RING, xloA, rlA,
                  xloB, rlB, A, E, O, sw);
        if (__any_sync(FULL, sw != RF_NONE)) O_last = O;
        if (sw != RF_NONE) L = O + lag + E + TAIL;
        R = rf_next_entry(__reduce_max_sync(FULL, sw != RF_NONE ? sw : R - 1));
      }
      const int T = max(0, __reduce_max_sync(FULL, L));
      const int G = (T + 15) >> 4;
      unsigned long long wo = 0;
      if (is0) wo = atomicAdd(p.dir_alloc, (unsigned long long)G * 64ull);
      wo = __shfl_sync(FULL, wo, 0);
      if (wo + (unsigned long long)G * 64ull > p.dir_capacity) status = ST_DIR_OVERFLOW;
      if (is0) {
        ws.word_off = wo;
        ws.G = G;
        ws.next_b = 0;
        ws.R = 0;
        ws.O_last = RF_NONE;
        ws.firstX = 0;
        ws.firstY = -1;
        RfFrame none;
        none.blk = -1;
        none.O = none.wlo = none.whi = none.a31 = none.e31 = 0;
        none.sw0 = none.sw31 = RF_NONE;
        none.swmax = 0;
        s_f0[wib] = none;
        s_f31[wib] = none;
        s_nx[wib] = none;
      }
      s_cur[wib][lane] = make_int4(0, 0, RF_NONE, 0);
      s_bestl[wib][lane] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      __syncwarp();
    }
    // every allocation of the arena is a multiple of 32 words: the pair is 8-byte aligned
    uint2* __restrict__ dwp = reinterpret_cast<uint2*>(p.dir + ws.word_off) + lane;

    // Pass 2.
    Lane2State st;
    st.oS = 0.0f;
    st.oU = sc.open_read;
    st.oP = empty_pack;
    st.oC = 0u;
    st.dS = 0.0f;
    st.dS2 = 0.0f;
    st.pS = 0.0f;
    st.pU = sc.open_read;
    st.pP = empty_pack;
    st.r1 = 0u;
    row_init(st.a, sc);
    row_init(st.b, sc);
    RowGeom ga, gb;  // before its first rows a lane is outside every corridor
    ga.rlen = gb.rlen = 0;
    ga.q = gb.q = 0x100u;
    ga.t0rel = gb.t0rel = 0;
    int sw = RF_NONE;

    // the lane's best cell so far into s_bestl: the later row wins only with a larger score (row-major order); both
    // trackers go on from it
    auto take_best = [&](const int4& me) {
      const bool second = st.b.kS > st.a.kS;
      const int ks = second ? st.b.kStep : st.a.kStep;
      const float kS = second ? st.b.kS : st.a.kS;
      if (ks >= 0)
        s_bestl[wib][lane] = make_float4(kS, __int_as_float(ks - me.x - lag - (second ? TAIL : 0)),
                                         __int_as_float(me.y + (second ? 1 : 0)), 0.0f);
      st.a.kS = st.b.kS = kS;
      st.a.kStep = st.b.kStep = -1;
    };

    auto place = [&]() {
      const CorridorView cv = corridor();
      const AlnDesc* dp = p.desc + ai;
      const int H = dp->height;
      const int b = ws.next_b, R = ws.R, O_last = ws.O_last;
      int4 me = s_cur[wib][lane];
      int xloA, xloB, A, E, O, swl;
      unsigned rlA, rlB;
      rf2_place(cv, b, lane, lag, H, (int)ref_len, me.z, R, O_last == RF_NONE ? INT_MIN : O_last + RING, xloA, rlA,
                xloB, rlB, A, E, O, swl);
      const bool any = __any_sync(FULL, swl != RF_NONE);
      if (swl != RF_NONE) me.z = O + lag + E + TAIL;
      me.w += (int)(rlA + rlB);
      const int swmax = __reduce_max_sync(FULL, swl != RF_NONE ? swl : R - 1);
      const int y = (b << 6) + 2 * lane;
      const int4 na = make_int4(swl - (O + lag + xloA), (int)rlA, y < H ? (int)p.seq[dp->qry_off + y] : 0x100, 0);
      const int4 nb2 = make_int4(swl - (O + lag + xloB) - TAIL, (int)rlB,
                                 y + 1 < H ? (int)p.seq[dp->qry_off + y + 1] : 0x100, 0);
      // the first row of the block with a cell (rows 2t, 2t + 1 of lane t in row-major order)
      const int key = rlA ? 2 * lane : (rlB ? 2 * lane + 1 : INT_MAX);
      const int kmin = __reduce_min_sync(FULL, key);
      const int fx = __shfl_sync(FULL, rlA ? xloA : xloB, (kmin >> 1) & 31);
      // lane 31's columns of block b-1: what lane 0 of block b reads from the strip
      int wlo = 0, whi = 0;
      if (b > 0) {
        int poA, plA, poB, plB, pxloA, pxhiA, pxloB, pxhiB, pA, pE;
        unsigned prlA, prlB;
        load_row_pair(cv, b - 1, lane, H, poA, plA, poB, plB);
        row_span(poA, plA, (int)ref_len, pxloA, pxhiA, prlA);
        row_span(poB, plB, (int)ref_len, pxloB, pxhiB, prlB);
        rf2_cols(pxloA, pxhiA, prlA, pxloB, pxhiB, prlB, lane, pA, pE);
        pA = __shfl_sync(FULL, pA, 31);
        pE = __shfl_sync(FULL, pE, 31);
        if (pA != INT_MAX) {
          wlo = pA;
          whi = pE;
        }
      }
      const int g0 = __reduce_min_sync(FULL, swl != RF_NONE ? swl : INT_MAX);
      const int end = __reduce_max_sync(FULL, swl != RF_NONE ? O + lag + E + TAIL : INT_MIN);
      const int a31 = __shfl_sync(FULL, A, 31), e31 = __shfl_sync(FULL, E, 31);
      const int sw0 = __shfl_sync(FULL, swl, 0), sw31 = __shfl_sync(FULL, swl, 31);
      s_cur[wib][lane] = me;
      s_nrow[wib][0][lane] = na;
      s_nrow[wib][1][lane] = nb2;
      sw = swl;
      __syncwarp();
      if (is0) {
        const int nblk32 = (H + 31) >> 5;
        for (int h = 0; h < 2 && 2 * b + h < nblk32; ++h) {
          BlockRec br;
          br.word_off = ws.word_off + (any ? (unsigned long long)(g0 >> 4) * 64ull : 0ull) + 32ull * h;
          br.base = any ? g0 - O - (SKEW ? 32 : 16) * h : 0;
          br.nsteps = any ? end - g0 : 0;
          p.blocks[dp->blk_off + 2 * b + h] = br;
        }
        RfFrame f;
        f.blk = b;
        f.O = O;
        f.wlo = wlo;
        f.whi = whi;
        f.a31 = a31;
        f.e31 = e31;
        f.sw0 = sw0;
        f.sw31 = sw31;
        f.swmax = swmax;
        s_nx[wib] = f;
        ws.next_b = b + 1;
        ws.R = rf_next_entry(swmax);
        if (any) ws.O_last = O;
        if (kmin != INT_MAX && ws.firstY < 0) {
          ws.firstY = (b << 6) + kmin;
          ws.firstX = fx;
        }
      }
      __syncwarp();
    };
    // as in convex_fill_rf_kernel
    uint4 pa = EMPTY, pb = EMPTY;
    auto stage = [&](int kk) {
      const RfFrame* n = &s_nx[wib];
      const RfFrame* f = &s_f0[wib];
      const int nblk_ = n->blk, nsw0 = n->sw0, fblk = f->blk;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int sigma = kk * CHUNK + lane + 32 * h;
        const bool in_n = nblk_ >= 0 && nsw0 != RF_NONE && sigma >= nsw0;
        const RfFrame* fr = in_n ? n : f;
        const int col = sigma - fr->O;
        uint4 rec = EMPTY;
        if (in_n || fblk >= 0) {
          if (col >= fr->wlo && col < fr->whi) rec = ld_strip(strip + col);
          rec.w = (unsigned)col < ref_len ? __ldg(ref + col) : 0u;
        }
        if (h == 0) pa = rec;
        else pb = rec;
      }
    };

    const int nchunks = status == ST_OK ? (ws.G + GPC - 1) / GPC : 0;
    if (nchunks > 0) {
      place();
      stage(0);
    }
    for (int c = 0; c < nchunks; ++c) {
      for (;;) {
        const RfFrame n = s_nx[wib];
        if (n.blk < 0 || n.swmax >= c * CHUNK) break;
        __syncwarp();
        if (is0) {
          if (n.sw0 != RF_NONE) s_f0[wib] = n;
          if (n.sw31 != RF_NONE) s_f31[wib] = n;
          s_nx[wib].blk = -1;
        }
        __syncwarp();
        if (ws.next_b < ((p.desc[ai].height + 63) >> 6)) place();
        else sw = RF_NONE;
      }
      io_s[2 * lane] = pa;
      io_s[2 * (lane + 32)] = pb;
      __syncwarp();
      if (is31) {
        const uint4 t = io_s[0];
        st.oS = __uint_as_float(t.x);
        st.oU = __uint_as_float(t.y);
        st.oP = t.z;
        st.oC = t.w;
      }
      if (c + 1 < nchunks) stage(c + 1);
      const int g_end = min(ws.G, (c + 1) * GPC);
      for (int g = c * GPC; g < g_end; ++g) {
        if ((g << 4) == sw) {  // this lane enters its rows of the next block
          int4 me = s_cur[wib][lane];
          take_best(me);
          const int4 na = s_nrow[wib][0][lane], nb2 = s_nrow[wib][1][lane];
          st.a.rel = na.x;
          ga.rlen = (unsigned)na.y;
          ga.q = (uint32_t)na.z;
          ga.t0rel = na.y > 12 ? na.y - 12 : 0;
          st.b.rel = nb2.x;
          gb.rlen = (unsigned)nb2.y;
          gb.q = (uint32_t)nb2.z;
          gb.t0rel = nb2.y > 12 ? nb2.y - 12 : 0;
          me.x = s_nx[wib].O;
          me.y = (s_nx[wib].blk << 6) + 2 * lane;
          s_cur[wib][lane] = me;
          sw = RF_NONE;
        }
        const bool all_active = __all_sync(FULL, st.a.rel >= 0 && st.a.rel + 15 < (int)ga.rlen && st.b.rel >= 0 &&
                                                     st.b.rel + 15 < (int)gb.rlen);
        if (all_active) {
          fill_group2<RAW, SKEW, true, GPC>(st, sc, io_s, dwp, g, ga, gb, is31, src_lane);
        } else {
          fill_group2<RAW, SKEW, false, GPC, true>(st, sc, io_s, dwp, g, ga, gb, is31, src_lane, ref,
                                                    s_cur[wib][lane].x + lag, ref_len);
        }
      }
      __syncwarp();
      // flush lane 31's records of this chunk that lie in its columns of the block it was in
      {
        const RfFrame* n = &s_nx[wib];
        const RfFrame* f = &s_f31[wib];
        const int done = (g_end - c * GPC) << 4;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int j = lane + 32 * h;
          const int sigma = c * CHUNK + j;
          const bool in_n = n->blk >= 0 && n->sw31 != RF_NONE && sigma >= n->sw31;
          const RfFrame* fr = in_n ? n : f;
          const int x = sigma - fr->O - LAG31;
          if (j < done && (in_n || f->blk >= 0) && x >= fr->a31 && x < fr->e31) st_strip(strip + x, io_s[2 * j + 1]);
        }
      }
      __syncwarp();
    }
    const int4 me = s_cur[wib][lane];
    take_best(me);
    const float4 bl = s_bestl[wib][lane];
    float bestS = bl.x;
    int bestX = __float_as_int(bl.y), bestY = __float_as_int(bl.z);
    unsigned long long cells = (unsigned)me.w;
    // blocks the schedule never reached have no cells
    if (is0 && status == ST_OK)
      for (int b = 2 * ws.next_b; b < ((p.desc[ai].height + 31) >> 5); ++b) {
        BlockRec br;
        br.word_off = ws.word_off;
        br.base = 0;
        br.nsteps = 0;
        p.blocks[p.desc[ai].blk_off + b] = br;
      }

    // first maximum in row-major order across lanes: larger score, then smaller y, then smaller x
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float s2 = __shfl_xor_sync(FULL, bestS, o);
      const int y2 = __shfl_xor_sync(FULL, bestY, o);
      const int x2 = __shfl_xor_sync(FULL, bestX, o);
      const unsigned long long c2 = __shfl_xor_sync(FULL, cells, o);
      const bool take = (s2 > bestS) || (s2 == bestS && (y2 < bestY || (y2 == bestY && x2 < bestX)));
      if (take) {
        bestS = s2;
        bestY = y2;
        bestX = x2;
      }
      cells += c2;
    }
    if (bestS == 0.0f) {  // no positive score anywhere: the first visited cell stands (or nothing was visited)
      const bool any = ws.firstY >= 0;
      bestS = any ? 0.0f : -1.0f;
      bestX = any ? ws.firstX : 0;
      bestY = any ? ws.firstY : 0;
    }
    if (is0) {
      FillOut o;
      o.best_score = bestS;
      o.best_x = bestX;
      o.best_y = bestY;
      o.status = status;
      o.cells = cells;
      o.dir_shift = SKEW ? 2 : 1;
      p.out[ai] = o;
    }
    __syncwarp();
  }
  if (!PERSIST) {
    __syncthreads();
    if (threadIdx.x == 0) atomicAnd(p.sm_slots + s_slot / FILL_SM_SLOTS, ~(1u << (s_slot % FILL_SM_SLOTS)));
  }
}

}  // namespace

namespace {
template <bool RAW>
void launch_fill_rf(const FillParams& p, int grid, cudaStream_t stream) {
  const int threads = FILL_WARPS_PER_CTA * 32;
  if (p.sm_slots) convex_fill_rf_kernel<RAW, false><<<grid, threads, 0, stream>>>(p);
  else convex_fill_rf_kernel<RAW, true><<<grid, threads, 0, stream>>>(p);
}

template <bool RAW, bool SKEW>
void launch_fill_rf2(const FillParams& p, int grid, cudaStream_t stream) {
  const int threads = FILL_WARPS_PER_CTA * 32;
  if (p.sm_slots) convex_fill_rf2_kernel<RAW, false, SKEW><<<grid, threads, 0, stream>>>(p);
  else convex_fill_rf2_kernel<RAW, true, SKEW><<<grid, threads, 0, stream>>>(p);
}

template <bool RAW, int NW>
void launch_fill(const FillParams& p, int grid, cudaStream_t stream) {
  const int threads = (NW == 1 ? FILL_WARPS_PER_CTA : NW) * 32;
  if (p.sm_slots) convex_fill_kernel<RAW, NW, false><<<grid, threads, 0, stream>>>(p);
  else convex_fill_kernel<RAW, NW, true><<<grid, threads, 0, stream>>>(p);
}
}  // namespace

// p.sm_slots != nullptr selects the short-lived-CTA instantiation (one problem per warp / team, strips by SM slot)
cudaError_t launch_convex_fill(const FillParams& p, bool raw, bool team, int rampfree, int grid, cudaStream_t stream) {
  if (rampfree == 3) {
    if (raw) launch_fill_rf2<true, true>(p, grid, stream);
    else launch_fill_rf2<false, true>(p, grid, stream);
  } else if (rampfree == 2) {
    if (raw) launch_fill_rf2<true, false>(p, grid, stream);
    else launch_fill_rf2<false, false>(p, grid, stream);
  } else if (rampfree) {
    if (raw) launch_fill_rf<true>(p, grid, stream);
    else launch_fill_rf<false>(p, grid, stream);
  } else if (raw) {
    if (team) launch_fill<true, FILL_WARPS_PER_CTA>(p, grid, stream);
    else launch_fill<true, 1>(p, grid, stream);
  } else {
    if (team) launch_fill<false, FILL_WARPS_PER_CTA>(p, grid, stream);
    else launch_fill<false, 1>(p, grid, stream);
  }
  return cudaGetLastError();
}

cudaError_t launch_convex_fill_big(const FillParams& p, bool raw, int grid, cudaStream_t stream) {
  const int threads = FILL_BIG_TEAM * 32;
  if (raw) convex_fill_kernel<true, FILL_BIG_TEAM, true><<<grid, threads, 0, stream>>>(p);
  else convex_fill_kernel<false, FILL_BIG_TEAM, true><<<grid, threads, 0, stream>>>(p);
  return cudaGetLastError();
}

int fill_max_ctas_per_sm(bool raw, bool team, int rampfree) {
  int n = 0;
  const int threads = FILL_WARPS_PER_CTA * 32;
  auto occ = [&](auto kernel) { cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, 0); };
  if (rampfree == 3) {
    raw ? occ(convex_fill_rf2_kernel<true, true, true>) : occ(convex_fill_rf2_kernel<false, true, true>);
  } else if (rampfree == 2) {
    raw ? occ(convex_fill_rf2_kernel<true, true, false>) : occ(convex_fill_rf2_kernel<false, true, false>);
  } else if (rampfree) {
    raw ? occ(convex_fill_rf_kernel<true, true>) : occ(convex_fill_rf_kernel<false, true>);
  } else if (raw) {
    team ? occ(convex_fill_kernel<true, FILL_WARPS_PER_CTA, true>) : occ(convex_fill_kernel<true, 1, true>);
  } else {
    team ? occ(convex_fill_kernel<false, FILL_WARPS_PER_CTA, true>) : occ(convex_fill_kernel<false, 1, true>);
  }
  return n;
}

namespace {
__global__ void nsmid_kernel(unsigned* out) {
  unsigned v;
  asm("mov.u32 %0, %%nsmid;" : "=r"(v));
  *out = v;
}
}  // namespace

int fill_sm_id_bound() {
  unsigned* d = nullptr;
  unsigned h = 0;
  if (cudaMalloc(&d, sizeof(unsigned)) != cudaSuccess) return -1;
  nsmid_kernel<<<1, 1>>>(d);
  const bool ok = cudaMemcpy(&h, d, sizeof(unsigned), cudaMemcpyDeviceToHost) == cudaSuccess;
  cudaFree(d);
  return ok ? (int)h : -1;
}

}  // namespace nb
