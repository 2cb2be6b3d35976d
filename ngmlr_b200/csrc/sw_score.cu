// ngmlr_b200/csrc/sw_score.cu -- score-only local alignment of sub-read x candidate pairs (sm_90a).
//
// Replaces StrippedSW::BatchScore / SingleScore (src/StrippedSW.cpp:118-202) and the part of the
// vendored SSW library they reach: ssw_init -> qP_word, ssw_align(flag=0) -> sw_sse2_word
// (lib/Complete-Striped-Smith-Waterman-Library/src/ssw.c:964-989, 342-364, 997-1054, 366-538).
//
// Semantics kept bit-for-bit (SURVEY.md appendix A.3):
//   * both sequences are scored INCLUDING their terminating NUL (lengths are strlen+1); the NUL
//     and every non-ACGT byte map to code 4, which scores 0 against everything;
//   * +1 match / -1 mismatch; gap open = gap extend = 255 (int32 -1 narrowed to uint8_t);
//   * H = max(diag + s, E, F) with signed-saturating 16-bit adds; E/F updates use unsigned
//     saturating subtraction (clamp at 0); result = max H as uint16 -> float.
//
// Mapping: one warp per pair; the warp sweeps the reference columns as a wavefront (lane t is one
// column behind lane t-1). The hot case (256-bp sub-read against a ~306-bp window) is provably
// ungapped and runs in sw_ungapped() below: packed 16-bit rows, substitution scores by PRMT table
// lookup, ~2 instructions per cell. Everything else takes the general affine path: lane t owns
// SW_ROWS consecutive query rows and passes the H and F of its last row down with __shfl_up;
// queries longer than 32*SW_ROWS rows are processed in several passes, the bottom row of a pass is
// carried to the next through a per-warp strip in global memory; 32-bit integer lanes emulate the
// int16 saturation (values never exceed 32767).
#include <cuda_runtime.h>

#include "device_types.h"
#include "kernels.h"

namespace nb {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int SW_ROWS = 9;  // 32 * 9 = 288 >= 257 = 256-bp sub-read + NUL: one pass for the hot case
constexpr int SW_GAP = 255;
constexpr int SW_COLS = 384;  // widest window of the ungapped hot path (ScoreBuffer windows: 307)
// widest window of the short-read scorer's instantiation: scoreShortRead's windows have
// len + (int)(len * 0.3 + 256) <= 588 characters for reads of <= 256 bases
constexpr int SW_COLS_SHORT = 640;
constexpr int SW_WARPS_PER_CTA = 4;

__device__ __forceinline__ int nt_code(uint32_t c) {
  // nt_table, src/StrippedSW.cpp:111-116 (A/a 0, C/c 1, G/g 2, T/t 3, everything else 4), branch-free:
  // (c >> 1) & 3 orders the four letters A C T G; k ^ (k >> 1) swaps the last two
  const uint32_t u = (c & 0xdfu) - 0x41u;  // A 0, C 2, G 6, T 19
  const uint32_t k = (c >> 1) & 3u;
  const bool acgt = u < 20u && ((0x80045u >> u) & 1u);
  return acgt ? (int)(k ^ (k >> 1)) : 4;
}

// nt_code(cpl(c)) with cpl() of src/MappedRead.cpp:35-46: only the UPPER-case letters are complemented
__device__ __forceinline__ int nt_code_cpl(uint32_t c) {
  const int code = nt_code(c);
  return (code < 4 && !(c & 0x20u)) ? 3 - code : code;
}

// DecodeRefSequence(sequence, 0, position, bufferLength) as a random-access function
// (src/SequenceProvider.cpp:567-625): character i of the window, as an nt_table code.
struct GenomeWindow {
  const uint8_t* enc;
  unsigned long long pos, concat_len;
  int odd;        // position & 1: one extra leading base
  int pairs2;     // 2 * ceil(len / 2) characters decoded pairwise
  int x_at;       // index (after the odd base) that is overwritten by 'x' when len is odd, else pairs2 (none: the
                  // odd leading base has index -1)
  int str_len;    // strlen of the decoded window
  bool invalid;   // position >= concat_len: the caller fills the buffer with 'N'
  __device__ void init(const uint8_t* e, unsigned long long p, unsigned long long cl, int buffer_len) {
    enc = e; pos = p; concat_len = cl;
    invalid = p >= cl;
    unsigned long long len = (unsigned long long)(buffer_len - 2), end = 0;
    if (!invalid && p + len > cl) { end = p + len - cl; len -= end; }
    odd = (int)(p & 1ull);
    pairs2 = (int)(((len + 1) / 2) * 2);
    x_at = (len & 1ull) ? pairs2 - 1 : pairs2;
    str_len = invalid ? buffer_len : odd + pairs2 + (int)end;
  }
  __device__ __forceinline__ int code(int i) const {
    if (invalid) return 4;                   // memset(buf, 'N', refMaxLen), src/ScoreBuffer.cpp:114
    if (i >= str_len) return 4;              // the terminating NUL (scored as N)
    const int k = i - odd;
    if (k >= pairs2 || k == x_at) return 4;  // 'x' padding
    const unsigned long long b = pos + (unsigned long long)i;  // base index in the concatenated genome
    const uint32_t byte = enc[b >> 1];
    const uint32_t c4 = (b & 1ull) ? (byte & 0xFu) : (byte >> 4);
    // enc4 A0 T1 G2 C3 N4 -> nt_table A0 C1 G2 T3 N4
    return (int)((0x41230u >> (4u * min(c4, 4u))) & 0xfu);
  }
};

__device__ __forceinline__ uint32_t cpl(uint32_t c) {  // src/MappedRead.cpp:35-46
  return c == 'A' ? 'T' : (c == 'T' ? 'A' : (c == 'C' ? 'G' : (c == 'G' ? 'C' : c)));
}

// Ungapped hot path. One warp per pair; lane t owns 2*PAIRS consecutive query rows, two rows per
// register in 16-bit halves: register k holds rows (r0 + k, r0 + k + PAIRS), so the H values of
// "the row above, one column back" of register k are simply the old register k-1 (no per-register
// shuffling of halves); only register 0 needs the neighbour lane's last row (one SHFL per step).
// The warp sweeps the columns as a wavefront (lane t one column behind lane t-1).
//
// Substitution scores by table lookup: for column base r the word A_r has byte q = 0x01 if q == r
// else 0xff (q = 0..3), and is 0 for N / padding columns. PRMT with a per-register selector built
// once from the two query codes (nibbles: q_lo, q_lo|8, q_hi, q_hi|8 -- |8 replicates the sign of
// the selected byte) turns A_r into the packed (+1 | -1 | 0, +1 | -1 | 0) pair; query code 4 (N,
// NUL, rows beyond the query) selects a zero byte. The A words of the window are decoded once per
// pair into shared memory with 32 zero words of padding either side, so that lanes which have not
// started or are already finished compute on zeros (H = relu(H + 0) never raises the maximum) and the
// step loop needs no activity test. The terminating NULs (last query row, last column) score 0
// against everything and are not evaluated. Per step and lane: 1 SHFL, 1 LDS, PAIRS x (PRMT,
// VIADDMNMX.S16x2.RELU, VIMNMX.S16x2) + 3.
template <int PAIRS, bool GATHER>
__device__ __forceinline__ float sw_ungapped(const GenomeWindow& gw, const uint8_t* __restrict__ ref,
                                             const uint8_t* __restrict__ qry, int qrows, int cols, bool q_rev,
                                             uint32_t* tab, int lane, uint32_t zero) {
  __syncwarp();
  for (int i = lane; i < cols + 64; i += 32) {
    const int c = i - 32;
    uint32_t a = 0u;
    if (c >= 0 && c < cols) {
      const int rc = GATHER ? gw.code(c) : nt_code(ref[c]);
      if (rc != 4) a = 0xffffffffu ^ (0xfeu << (8 * rc));
    }
    tab[i] = a;
  }
  const int row0 = lane * 2 * PAIRS;
  uint32_t sel[PAIRS], H[PAIRS];
#pragma unroll
  for (int k = 0; k < PAIRS; ++k) {
    uint32_t codes[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + k + h * PAIRS;
      int cq = 4;
      if (row < qrows) cq = q_rev ? nt_code_cpl(qry[qrows - 1 - row]) : nt_code(qry[row]);
      codes[h] = (uint32_t)cq;
    }
    sel[k] = codes[0] | ((codes[0] | 8u) << 4) | (codes[1] << 8) | ((codes[1] | 8u) << 12);
    H[k] = 0u;
  }
  __syncwarp();
  uint32_t best2 = 0u, diag_top = 0u;
  const uint32_t not_lane0 = lane ? 0xffffffffu : 0u;
  const uint32_t* tp = tab + 32 - lane;
  const int nsteps = cols + 31;
#pragma unroll 4
  for (int s = 0; s < nsteps; ++s) {
    const uint32_t up = __shfl_up_sync(FULL, H[PAIRS - 1], 1) & not_lane0;
    const uint32_t a = tp[s];
    // (row r0-1 from the lane above, row r0+PAIRS-1 = low half of the last register), column c-1
    const uint32_t d0 = __byte_perm(diag_top, H[PAIRS - 1], 0x5432);
#pragma unroll
    for (int k = PAIRS - 1; k >= 0; --k) {
      uint32_t sub;
      asm("prmt.b32 %0, %1, %2, %3;" : "=r"(sub) : "r"(a), "r"(0u), "r"(sel[k]));
      const uint32_t h = __viaddmax_s16x2_relu(k ? H[k - 1] : d0, sub, zero);
      H[k] = h;
      best2 = __vmaxs2(best2, h);
    }
    diag_top = up;
  }
  int best = max((int)(best2 & 0xffffu), (int)(best2 >> 16));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(FULL, best, o));
  return (float)(best & 0xffff);
}

// COLS: widest window of the ungapped path (shared table size); PAIR_WIN: window lengths per pair (p.win_lens)
template <bool GATHER, int COLS, bool PAIR_WIN>
__global__ void __launch_bounds__(SW_WARPS_PER_CTA * 32) sw_score_kernel(const SwParams p) {
  const int lane = threadIdx.x & 31;
  const int warp_global = blockIdx.x * SW_WARPS_PER_CTA + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * SW_WARPS_PER_CTA;
  int2* strip = reinterpret_cast<int2*>(p.scratch) + (size_t)warp_global * p.scratch_stride;
  __shared__ uint32_t s_tab[SW_WARPS_PER_CTA][COLS + 64];
  // 0 the compiler cannot see through: keeps the RELU floor of the packed ops in one register
  // (a literal 0 is re-materialised with a PRMT per use)
  const uint32_t zero = (uint32_t)p.n >> 31;

  for (int pair = warp_global; pair < p.n; pair += nwarps) {
    GenomeWindow gw;
    int rlen_g = 0;
    if (GATHER) {
      gw.init(p.enc, p.win_pos[pair], p.concat_len, PAIR_WIN ? p.win_lens[pair] : p.win_len);
      rlen_g = gw.str_len + 1;  // strlen + 1: the NUL is scored
    }
    const bool q_rev = GATHER && p.rev[pair];
    const int qlen = p.qry_len[pair], rlen = GATHER ? rlen_g : p.ref_len[pair];
    if (qlen >= 100000 || rlen >= 100000) {  // maxSeqLen, src/StrippedSW.h:88
      if (lane == 0) p.out[pair] = -1.0f;
      continue;
    }
    const uint8_t* __restrict__ ref = GATHER ? p.seq : p.seq + p.ref_off[pair];
    const uint8_t* __restrict__ qry = p.seq + p.qry_off[pair];
    int best = 0;
    // ---- hot case: at most 320 query characters (256-bp sub-read + NUL), window of <= COLS columns ----
    // A gap costs 255 per base, so a gapped path beats its best ungapped piece only if it gains
    // more than 255 before AND after the gap: impossible with fewer than 512 query characters.
    // Then E and F never influence the maximum and the recurrence is H = max(0, diag + s).
    if (qlen - 1 <= 64 * 5 && rlen - 1 <= COLS) {
      const float r = (qlen - 1 <= 64 * 4)
                          ? sw_ungapped<4, GATHER>(gw, ref, qry, qlen - 1, rlen - 1, q_rev, s_tab[threadIdx.x >> 5], lane, zero)
                          : sw_ungapped<5, GATHER>(gw, ref, qry, qlen - 1, rlen - 1, q_rev, s_tab[threadIdx.x >> 5], lane, zero);
      if (lane == 0) p.out[pair] = r;
      continue;
    }
    if (PAIR_WIN && p.general_pairs && lane == 0) atomicAdd(p.general_pairs, 1u);
    const int rows_per_pass = 32 * SW_ROWS;
    for (int row_base = 0; row_base < qlen; row_base += rows_per_pass) {
      const bool first_pass = row_base == 0;
      const bool last_pass = row_base + rows_per_pass >= qlen;
      const int row0 = row_base + lane * SW_ROWS;
      int qc[SW_ROWS], H[SW_ROWS], E[SW_ROWS];
#pragma unroll
      for (int r = 0; r < SW_ROWS; ++r) {
        const int row = row0 + r;
        // the NUL at qlen-1 is part of the query and maps to 4; rows >= qlen do not exist (-1)
        if (q_rev) {  // RevSeq[j] = cpl(Seq[len - 1 - j]), then the NUL
          const int L = qlen - 1;
          qc[r] = row < L ? nt_code_cpl(qry[L - 1 - row]) : (row < qlen ? 4 : -1);
        } else {
          // the terminator is code 4 by position, not by content: a sub-read may be a view into a longer read
          qc[r] = row < qlen - 1 ? nt_code(qry[row]) : (row < qlen ? 4 : -1);
        }
        H[r] = 0;
        E[r] = 0;
      }
      int outH = 0, outF = 0, diagTop = 0;
      const int nsteps = rlen + 31;
      for (int s = 0; s < nsteps; ++s) {
        const int c = s - lane;
        int upH = __shfl_up_sync(FULL, outH, 1);
        int upF = __shfl_up_sync(FULL, outF, 1);
        const bool in = c >= 0 && c < rlen;
        if (lane == 0) {
          upH = 0;
          upF = 0;
          if (!first_pass && in) {
            const int2 v = __ldcg(strip + c);
            upH = v.x;
            upF = v.y;
          }
        }
        if (in) {
          const int rc = GATHER ? gw.code(c) : nt_code(ref[c]);
          int diag = diagTop;
          diagTop = upH;
          int F = upF;
#pragma unroll
          for (int r = 0; r < SW_ROWS; ++r) {
            const int hOld = H[r];
            const int sub = ((rc | qc[r]) & 4) ? 0 : (rc == qc[r] ? 1 : -1);
            int h = min(diag + sub, 32767);      // _mm_adds_epi16
            h = max(h, E[r]);
            h = max(h, F);
            if (qc[r] < 0) h = 0;                // row beyond the query
            best = max(best, h);
            H[r] = h;
            const int hg = max(h - SW_GAP, 0);   // _mm_subs_epu16
            E[r] = max(max(E[r] - SW_GAP, 0), hg);
            F = max(max(F - SW_GAP, 0), hg);
            diag = hOld;
          }
          outH = H[SW_ROWS - 1];
          outF = F;
          if (lane == 31 && !last_pass) __stcg(strip + c, make_int2(outH, outF));
        }
      }
      __syncwarp();
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(FULL, best, o));
    if (lane == 0) p.out[pair] = (float)(best & 0xffff);
  }
}

}  // namespace

cudaError_t launch_sw_score(const SwParams& p, int grid, cudaStream_t stream) {
  if (p.n <= 0) return cudaSuccess;
  sw_score_kernel<false, SW_COLS, false><<<grid, SW_WARPS_PER_CTA * 32, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_sw_score_gather(const SwParams& p, int grid, cudaStream_t stream) {
  if (p.n <= 0) return cudaSuccess;
  sw_score_kernel<true, SW_COLS, false><<<grid, SW_WARPS_PER_CTA * 32, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_sw_score_gather_short(const SwParams& p, int grid, cudaStream_t stream) {
  if (p.n <= 0) return cudaSuccess;
  sw_score_kernel<true, SW_COLS_SHORT, true><<<grid, SW_WARPS_PER_CTA * 32, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace nb
