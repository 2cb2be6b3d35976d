// ngmlr_b200/csrc/convex_text.cu -- CIGAR / MD / NM text and the inversion-peak scan on the device (sm_90a).
//
// Replaces, for a whole batch, the text half of Convex::ConvexAlignFast::SingleAlign:
//   convertCigar   (src/ConvexAlignFast.cpp:112-333, addPosition :76-99)  binary CIGAR -> CIGAR and
//                  MD strings, NM, identity, QStart/QEnd, first/lastPosition, nmPerPosition
//   the 'X' probe  (src/ConvexAlignFast.cpp:494-529)                     -> svType
// and the part of its only consumer that reads every alignment column:
//   AlignmentBuffer::detectMisalignment's peak scan (src/AlignmentBuffer.cpp:1319-1388): columns
//   whose 32-event error count nm has 0 < (32 - nm) / 32 < 0.75 are merged into low-identity
//   regions (columns at most 20 apart), each closed region {startInv, stopInv, startInvRead,
//   stopInvRead} is what the reference hands to checkForSV.
// Only strings, a 96-byte record and the (few) regions per alignment cross PCIe; the 12 bytes per
// alignment column of nmPerPosition never exist unless a caller asks for them (plugin / tests).
//
// Mapping: one warp per alignment. The compact binary CIGAR of the traceback kernel is consumed 32
// runs at a time (lane = run): warp scans give every run its reference / read position, its event
// index and its text offsets; merged M operations and the MD match counter are segmented scans
// with a carry between chunks. Pass 1 sizes the strings and bump-allocates the text arena, pass 2
// writes them and walks the alignment columns 32 events at a time (lane = event): the reference's
// 32-bit shift register of error events becomes two ballots (this tile, the 32 events before it)
// and a popcount per lane; the "level" the reference records after the first base of an indel
// (previous level + 1, not a recount) is resolved with one more ballot and a shuffle.
//
// The reference's scan reads align->alignmentLength entries of nmPerPosition although convertCigar
// wrote fewer (insertions and the first 17 columns are not recorded); the entries in between come
// from an uninitialised `new PositionNM[]`. They are taken as zero here (fresh pages; nm = 0 is
// "no error", i.e. they only count down the merge distance), documented in DESIGN.md.
#include <cuda_runtime.h>

#include "device_types.h"
#include "kernels.h"

namespace nb {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int TEXT_WARPS_PER_CTA = 4;

__device__ __forceinline__ unsigned lowmask(int n) { return n >= 32 ? 0xffffffffu : ((1u << n) - 1u); }

__device__ __forceinline__ int ndigits(unsigned v) {
  int n = 1;
  if (v >= 100000000u) { n += 8; v /= 100000000u; }
  if (v >= 10000u) { n += 4; v /= 10000u; }
  if (v >= 100u) { n += 2; v /= 100u; }
  if (v >= 10u) n += 1;
  return n;
}

__device__ __forceinline__ void write_uint(char* p, unsigned v, int nd) {
  for (int i = nd - 1; i >= 0; --i) {
    p[i] = (char)('0' + v % 10u);
    v /= 10u;
  }
}

__device__ __forceinline__ int incl_scan(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(FULL, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// Inclusive segmented sum: lanes with `head` start a new segment (their own value included).
// On return v = sum over [latest head at or before this lane, this lane]; open = no head at or
// before this lane (the segment began in an earlier chunk: the caller adds its carry).
__device__ __forceinline__ void seg_scan(int& v, bool head, bool& open, int lane) {
  int f = head ? 1 : 0;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int tv = __shfl_up_sync(FULL, v, o);
    const int tf = __shfl_up_sync(FULL, f, o);
    if (lane >= o && !f) {
      v += tv;
      f = tf;
    }
  }
  open = f == 0;
}

struct PeakState {
  bool open;
  int gap, sR, eR, sQ, eQ, n, stored;
};

__global__ void __launch_bounds__(TEXT_WARPS_PER_CTA * 32) convex_text_kernel(const TextParams p) {
  __shared__ int4 s_peaks[TEXT_WARPS_PER_CTA][TEXT_PEAK_CAP];
  const int wib = threadIdx.x >> 5;
  const int slot = blockIdx.x * TEXT_WARPS_PER_CTA + wib;
  const int lane = threadIdx.x & 31;
  if (slot >= p.n) return;
  const int i = p.order[slot];
  const AlnDesc d = p.desc[i];
  const TraceOut t = p.trace[i];
  TextOut o;
  o.status = TX_SKIP;
  o.ret = -1;
  o.qstart = o.qend = o.nm = o.alignment_length = o.cigar_op_count = o.sv_type = 0;
  o.first_ref = o.first_read = o.last_ref = o.last_read = 0;
  o.nm_count = o.cigar_len = o.md_len = o.n_peaks = 0;
  o.identity = 0.0f;
  o.n_peaks_stored = 0;
  o.text_off = o.peak_off = o.nm_off = 0;
  if (t.status != ST_OK) {  // invalid / thrown / overflowed alignments carry no text
    if (lane == 0) p.out[i] = o;
    return;
  }
  const int n_runs = t.n_runs;
  if (n_runs < 2) {
    o.status = TX_THROW;
    if (lane == 0) p.out[i] = o;
    return;
  }
  const int32_t* __restrict__ runs = p.runs + t.run_off;
  const uint8_t* __restrict__ ref = p.seq + d.ref_off;
  const uint8_t* __restrict__ aref = ref + t.ref_position;  // convertCigar receives refSeq + ref_position (:489)
  const int lead = runs[0] >> 4, trail = runs[n_runs - 1] >> 4;
  const int qstart = lead + d.ext_qstart, qend = trail + d.ext_qend;
  const int n_inner = n_runs - 2;
  const int nchunks = (n_inner + 31) >> 5;

  char* cig = nullptr;
  char* md = nullptr;
  int32_t* nm_out = nullptr;
  int total_ref = 0, total_read = 0, matches = 0, columns = 0, ops = 0, nm_count = 0;
  int cigar_len = 0, md_len = 0;
  bool bad = false;

  for (int pass = 0; pass < 2; ++pass) {
    const bool emit = pass == 1;
    int pending_m = 0, md_run = 0, pos_ref = 0, pos_read = lead;
    int cig_off = 0, md_off = 0, noted_total = 0;
    ops = 0;
    matches = 0;
    columns = 0;
    if (qstart > 0) {
      const int nd = ndigits((unsigned)qstart);
      if (emit && lane == 0) {
        write_uint(cig, (unsigned)qstart, nd);
        cig[nd] = 'S';
      }
      cig_off = nd + 1;
      ops = 1;
    }
    // column walk state (pass 2)
    unsigned prev32 = 0u;
    int level_carry = 0;
    PeakState pk;
    pk.open = false;
    pk.gap = pk.sR = pk.eR = pk.sQ = pk.eQ = pk.n = pk.stored = 0;

    for (int c = 0; c < nchunks; ++c) {
      const int idx = 1 + (c << 5) + lane;
      const bool valid = idx < n_runs - 1;
      const int w = valid ? runs[idx] : 0;
      const int wn = (idx + 1 < n_runs - 1) ? runs[idx + 1] : 0;
      const int op = w & 15, len = valid ? (w >> 4) : 0;
      const bool isEQ = valid && op == OP_EQ, isX = valid && op == OP_X, isD = valid && op == OP_D,
                 isI = valid && op == OP_I;
      const bool isM = isEQ || isX;
      const int opn = wn & 15;
      const bool next_isM = (idx + 1 < n_runs - 1) && (opn == OP_EQ || opn == OP_X);
      if (__any_sync(FULL, valid && !(isM || isD || isI))) {  // "Invalid cigar string" -> throw 1 (:272-274)
        bad = true;
        break;
      }
      const int refadv = (isM || isD) ? len : 0, readadv = (isM || isI) ? len : 0;
      const int ref_inc = incl_scan(refadv, lane), read_inc = incl_scan(readadv, lane);
      const int ev_inc = incl_scan(len, lane);
      const int pr0 = pos_ref + ref_inc - refadv;    // posInRef at the first column of the run
      const int pq0 = pos_read + read_inc - readadv;  // posInRead at the first column of the run
      // columns of this run recorded by addPosition (posInRead > 16 && posInRef > 16): a suffix of the run
      int cnt = 0;
      if (isM) cnt = max(0, len - max(0, max(17 - pr0, 17 - pq0)));
      if (isD) cnt = pq0 > 16 ? max(0, len - max(0, 17 - pr0)) : 0;
      const int cnt_inc = incl_scan(cnt, lane);

      // ---- CIGAR: consecutive EQ/X runs are one M; the last run of a group emits it ----
      int grp = isM ? len : 0;
      bool openM;
      seg_scan(grp, !isM, openM, lane);
      if (isM && openM) grp += pending_m;
      const bool emitM = isM && !next_isM;
      const bool has_tok = emitM || isD || isI;
      const int tokval = emitM ? grp : len;
      const int tok_nd = has_tok ? ndigits((unsigned)tokval) : 0;
      const int toklen = has_tok ? tok_nd + 1 : 0;
      const int tok_inc = incl_scan(toklen, lane);
      if (emit && has_tok) {
        char* q = cig + cig_off + tok_inc - toklen;
        write_uint(q, (unsigned)tokval, tok_nd);
        q[tok_nd] = emitM ? 'M' : (isD ? 'D' : 'I');
      }
      ops += __popc(__ballot_sync(FULL, has_tok));
      cig_off += __shfl_sync(FULL, tok_inc, 31);
      pending_m = __shfl_sync(FULL, (isM && next_isM) ? grp : 0, 31);

      // ---- MD: matches since the last mismatch / deletion (insertions do not reset the counter) ----
      int eqs = isEQ ? len : 0;
      bool openE;
      seg_scan(eqs, isX || isD, openE, lane);
      int s_prev = __shfl_up_sync(FULL, eqs, 1);
      int open_prev = __shfl_up_sync(FULL, openE ? 1 : 0, 1);
      if (lane == 0) {
        s_prev = 0;
        open_prev = 1;
      }
      const int md_before = s_prev + (open_prev ? md_run : 0);
      const int md_nd = (isX || isD) ? ndigits((unsigned)md_before) : 0;
      const int mdl = isX ? md_nd + 1 + 2 * (len - 1) : (isD ? md_nd + 1 + len : 0);
      const int md_inc = incl_scan(mdl, lane);
      const int md_at = md_off + md_inc - mdl;
      const bool long_d = isD && len >= 64;
      if (emit) {
        if (isX) {
          char* q = md + md_at;
          write_uint(q, (unsigned)md_before, md_nd);
          q += md_nd;
          *q++ = (char)aref[pr0];
          for (int k = 1; k < len; ++k) {
            *q++ = '0';
            *q++ = (char)aref[pr0 + k];
          }
        } else if (isD) {
          char* q = md + md_at;
          write_uint(q, (unsigned)md_before, md_nd);
          q[md_nd] = '^';
          if (!long_d)
            for (int k = 0; k < len; ++k) q[md_nd + 1 + k] = (char)aref[pr0 + k];
        }
        unsigned lm = __ballot_sync(FULL, long_d);  // long deletions: the warp copies the bases together
        while (lm) {
          const int src = __ffs(lm) - 1;
          lm &= lm - 1u;
          const int dst0 = __shfl_sync(FULL, md_at + md_nd + 1, src);
          const int s0 = __shfl_sync(FULL, pr0, src);
          const int nn = __shfl_sync(FULL, len, src);
          for (int k = lane; k < nn; k += 32) md[dst0 + k] = (char)aref[s0 + k];
        }
      }
      md_off += __shfl_sync(FULL, md_inc, 31);
      md_run = __shfl_sync(FULL, eqs + (openE ? md_run : 0), 31);
      matches += __shfl_sync(FULL, incl_scan(isEQ ? len : 0, lane), 31);

      // ---- pass 2: alignment columns, 32 events at a time ----
      if (emit) {
        const int T = __shfl_sync(FULL, ev_inc, 31);
        const int E0 = ev_inc - len;               // event index of the run's first base within the chunk
        const int nm0 = noted_total + cnt_inc - cnt;  // index of the run's first recorded column
        for (int tb = 0; tb < T; tb += 32) {
          const int e = tb + lane;
          const bool ev = e < T;
          const unsigned heads = __reduce_or_sync(FULL, (len > 0 && E0 > tb && E0 < tb + 32) ? (1u << (E0 - tb)) : 0u);
          const int frun = __popc(__ballot_sync(FULL, len > 0 && E0 <= tb)) - 1;
          const int jr = frun + __popc(heads & lowmask(lane + 1));
          const int rw = __shfl_sync(FULL, w, jr);
          const int rE = __shfl_sync(FULL, E0, jr);
          const int rpr = __shfl_sync(FULL, pr0, jr);
          const int rpq = __shfl_sync(FULL, pq0, jr);
          const int rcnt = __shfl_sync(FULL, cnt, jr);
          const int rnm0 = __shfl_sync(FULL, nm0, jr);
          const int rop = rw & 15, rlen = rw >> 4;
          const int k = e - rE;
          const bool gap_ev = ev && (rop == OP_D || rop == OP_I);
          const bool eqx_ev = ev && !gap_ev;
          const bool gfirst = gap_ev && k == 0;   // only the first base of an indel counts (maxIndelLength = 1)
          const unsigned cur = __ballot_sync(FULL, (ev && rop == OP_X) || gfirst);
          const unsigned eqx_mask = __ballot_sync(FULL, eqx_ev);
          const unsigned gf_mask = __ballot_sync(FULL, gfirst);
          // errors among the last 32 events: this tile up to the lane, the rest from the events before it
          const int ones = __popc(cur & lowmask(lane + 1)) + (lane < 31 ? __popc(prev32 >> (lane + 1)) : 0);
          // level = what the reference records: the recount after a match / mismatch; "previous + 1"
          // after the first base of an indel, unchanged on its further bases
          const unsigned below = eqx_mask & lowmask(lane);
          const int pl = below ? 31 - __clz(below) : 0;
          const int base_lvl = __shfl_sync(FULL, ones, pl);
          int level;
          if (eqx_ev) level = ones;
          else if (below) level = base_lvl + __popc(gf_mask & lowmask(lane + 1) & ~lowmask(pl + 1));
          else level = level_carry + __popc(gf_mask & lowmask(lane + 1));
          const int m = min(32, T - tb);
          level_carry = __shfl_sync(FULL, level, m - 1);
          prev32 = m == 32 ? cur : ((prev32 >> m) | (cur << (32 - m)));
          // addPosition: recorded column?
          const int pr = rpr + k;
          const int pq = rop == OP_D ? rpq : rpq + k;
          const bool noted = ev && rop != OP_I && pr > 16 && pq > 16;
          if (nm_out && noted) {
            int32_t* q = nm_out + 3 * (size_t)(rnm0 + k - (rlen - rcnt));
            q[0] = pr - 16;
            q[1] = pq - 16;
            q[2] = level;
          }
          // detectMisalignment: isInversion((32 - nm) / 32.0f)  <=>  8 < nm < 32
          const bool inv = noted && level > 8 && level < 32;
          const unsigned cm = __ballot_sync(FULL, noted);
          unsigned im = __ballot_sync(FULL, inv);
          int lastpos = -1;
          while (im) {
            const int b = __ffs(im) - 1;
            im &= im - 1u;
            const int between = __popc(cm & lowmask(b) & ~lowmask(lastpos + 1));
            if (pk.open) {
              pk.gap += between;
              if (pk.gap > 20) {  // the 21st column without a peak closes the region
                if (pk.stored < TEXT_PEAK_CAP) {
                  if (lane == 0) s_peaks[wib][pk.stored] = make_int4(pk.sR, pk.eR, pk.sQ, pk.eQ);
                  ++pk.stored;
                }
                ++pk.n;
                pk.open = false;
              }
            }
            const int R = __shfl_sync(FULL, pr - 16, b), Q = __shfl_sync(FULL, pq - 16, b);
            if (!pk.open) {
              pk.open = true;
              pk.sR = R;
              pk.sQ = Q;
            }
            pk.eR = R;
            pk.eQ = Q;
            pk.gap = 0;
            lastpos = b;
          }
          if (pk.open) {
            pk.gap += __popc(cm & ~lowmask(lastpos + 1));
            if (pk.gap > 20) {
              if (pk.stored < TEXT_PEAK_CAP) {
                if (lane == 0) s_peaks[wib][pk.stored] = make_int4(pk.sR, pk.eR, pk.sQ, pk.eQ);
                ++pk.stored;
              }
              ++pk.n;
              pk.open = false;
            }
          }
        }
      }
      noted_total += __shfl_sync(FULL, cnt_inc, 31);
      columns += __shfl_sync(FULL, ev_inc, 31);
      pos_ref += __shfl_sync(FULL, ref_inc, 31);
      pos_read += __shfl_sync(FULL, read_inc, 31);
    }
    if (bad) break;
    // final match count, trailing clip
    const int md_nd = ndigits((unsigned)md_run);
    if (emit && lane == 0) write_uint(md + md_off, (unsigned)md_run, md_nd);
    md_off += md_nd;
    if (qend > 0) {
      const int nd = ndigits((unsigned)qend);
      if (emit && lane == 0) {
        write_uint(cig + cig_off, (unsigned)qend, nd);
        cig[cig_off + nd] = 'S';
      }
      cig_off += nd + 1;
      ++ops;
    }
    if (!emit) {
      cigar_len = cig_off;
      md_len = md_off;
      total_ref = pos_ref;
      total_read = pos_read;
      nm_count = noted_total;
      unsigned long long at = 0, nat = 0;
      const unsigned long long need = (unsigned long long)cigar_len + (unsigned long long)md_len + 2ull;
      if (lane == 0) {
        at = atomicAdd(p.text_alloc, need);
        if (p.nm) nat = atomicAdd(p.nm_alloc, (unsigned long long)nm_count * 3ull);
      }
      at = __shfl_sync(FULL, at, 0);
      nat = __shfl_sync(FULL, nat, 0);
      o.text_off = at;
      o.nm_off = nat;
      if (at + need > p.text_capacity || (p.nm && nat + (unsigned long long)nm_count * 3ull > p.nm_capacity)) {
        o.status = TX_OVERFLOW;
        if (lane == 0) p.out[i] = o;
        return;
      }
      cig = p.text + at;
      md = cig + cigar_len + 1;
      nm_out = p.nm ? p.nm + nat : nullptr;
    } else {
      if (lane == 0) {
        cig[cigar_len] = '\0';
        md[md_len] = '\0';
      }
      // the columns the reference's scan reads beyond what convertCigar wrote (see the header)
      if (pk.open) {
        pk.gap += columns - nm_count;
        if (pk.gap > 20) {
          if (pk.stored < TEXT_PEAK_CAP) {
            if (lane == 0) s_peaks[wib][pk.stored] = make_int4(pk.sR, pk.eR, pk.sQ, pk.eQ);
            ++pk.stored;
          }
          ++pk.n;
        }
      }
      o.n_peaks = pk.n;
      o.n_peaks_stored = pk.stored;
      if (pk.stored > 0) {
        unsigned long long pat = 0;
        if (lane == 0) pat = atomicAdd(p.peaks_alloc, (unsigned long long)pk.stored);
        pat = __shfl_sync(FULL, pat, 0);
        o.peak_off = pat;
        __syncwarp();
        if (pat + (unsigned long long)pk.stored > p.peaks_capacity) {
          o.status = TX_OVERFLOW;
          if (lane == 0) p.out[i] = o;
          return;
        }
        if (lane < pk.stored) p.peaks[pat + lane] = s_peaks[wib][lane];
      }
    }
  }
  if (bad) {
    o.status = TX_THROW;
    if (lane == 0) p.out[i] = o;
    return;
  }
  // ---- scalars (:276-333) ----
  o.status = TX_OK;
  o.qstart = qstart;
  o.qend = qend;
  o.first_ref = 0;
  o.first_read = lead;
  o.last_ref = total_ref;
  o.last_read = total_read;
  o.identity = __fdiv_rn(__fmul_rn((float)matches, 1.0f), (float)columns);
  o.nm = columns - matches;
  o.alignment_length = columns;
  o.cigar_op_count = ops;
  o.nm_count = nm_count;
  o.cigar_len = cigar_len;
  o.md_len = md_len;
  o.ret = (qstart > 0 ? qstart : 0) + (total_read - lead) + qend;
  // Was the clipping caused by N in the reference? (:494-529): probes for 'X', which the reference's
  // own decoder never emits -- kept for equality.
  {
    const int rp = t.ref_position;
    const int lo = rp - 100 > 0 ? rp - 100 : 0;
    int cnt = 0;
    for (int k = rp - lane; k > lo; k -= 32) cnt += ref[k] == 'X';
    cnt = __reduce_add_sync(FULL, cnt);
    int probes = rp - lo;
    int sv = 0;
    if ((float)cnt > __fmul_rn((float)probes, 0.8f)) sv |= 1;
    const int rest = d.ref_len - rp;
    const int hi = total_ref + 100 < rest ? total_ref + 100 : rest;
    cnt = 0;
    for (int k = total_ref + lane; k < hi; k += 32) cnt += ref[rp + k] == 'X';
    cnt = __reduce_add_sync(FULL, cnt);
    probes = hi > total_ref ? hi - total_ref : 0;
    if ((float)cnt > __fmul_rn((float)probes, 0.8f)) sv |= 1;
    o.sv_type = sv;
  }
  if (lane == 0) p.out[i] = o;
}

}  // namespace

cudaError_t launch_convex_text(const TextParams& p, cudaStream_t stream) {
  if (p.n <= 0) return cudaSuccess;
  convex_text_kernel<<<(p.n + TEXT_WARPS_PER_CTA - 1) / TEXT_WARPS_PER_CTA, TEXT_WARPS_PER_CTA * 32, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace nb
