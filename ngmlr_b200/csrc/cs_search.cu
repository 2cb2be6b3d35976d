// ngmlr_b200/csrc/cs_search.cu -- k-mer candidate search (stage 0) for sm_90a.
//
// Replaces, per (sub-)read, CS::RunRead's search (src/CS.cpp:324-398): CS::PrefixIteration
// (src/CSstatic.cpp:23-73) -> CS::PrefixSearch (src/CS.cpp:57-96) ->
// CompactPrefixTable::GetRefEntry (src/PrefixTable.cpp:476-532, revComp :70-88) ->
// CS::AddLocationStd (src/CS.cpp:98-149) -> CS::CollectResultsStd (src/CS.cpp:217-269).
//
// The vote is order dependent (the acceptance threshold 0.8 x max-so-far runs along with the
// hits, and candidates are emitted in the order in which their bin first crossed it), so each
// (sub-)read is processed by ONE thread that replays the reference's sequence of hits exactly;
// parallelism comes from the hundreds of thousands of independent sub-reads of a batch (a 2048-
// thread SM keeps 2048 of these latency-bound walks in flight). The index (5-byte Index records
// unpacked to tab/used arrays + uint32 position lists) and the open-addressing vote tables live in
// HBM (the used() flags as an L2-resident bitmap); a first pass counts each read's hits so that its table can be sized (the reference instead
// restarts with a larger table on overflow -- results do not depend on the table size).
//
// Assumes, like the reference's 1000-N leading spacer guarantees, position >= offset-in-read.
#include <cuda_runtime.h>

#include "device_types.h"
#include "kernels.h"

namespace nb {

namespace {

__device__ __forceinline__ uint32_t rev_comp(uint32_t prefix, int k, uint32_t mask) {
  // complement = xor 10b per base (A0 C1 T2 G3), then reverse the 2-bit groups
  uint32_t c = (prefix ^ 0xAAAAAAAAu) & mask;
  c = __brev(c);                                            // bit reversal also swaps bits in a pair
  c = ((c >> 1) & 0x55555555u) | ((c & 0x55555555u) << 1);  // swap them back
  return c >> (32 - 2 * k);
}

struct alignas(16) VoteEntry {
  uint32_t key;    // bin = (loc - correction) >> bin_shift   (CSTableEntry::m_Location is a uint)
  uint32_t state;  // bit 0: used, bit 1: already listed
  float f, r;
};

constexpr unsigned FULL = 0xffffffffu;
constexpr int CS_WARPS = 4;

__device__ __forceinline__ unsigned lowmask(int n) { return n >= 32 ? 0xffffffffu : ((1u << n) - 1u); }

// One WARP per (sub-)read. The reference's vote is order dependent (the acceptance threshold 0.8 x
// max-so-far runs along with the hits, candidates are emitted in the order in which their bin first
// crossed it), but only through three quantities that have closed forms over the canonical hit sequence:
//   score of hit j          = 1 + number of earlier hits with the same (bin, strand)
//   max-so-far at hit j     = prefix maximum of the scores
//   bin b is listed at      = its first hit (either strand) whose score >= 0.8 x max-so-far
// So the warp replays the hits 32 AT A TIME in canonical order (lane = hit): equal bins of a batch are
// grouped with __match_any_sync (the group's leader finds / inserts the table entry, everybody derives its
// own score from the entry's old counts and its rank within the group), the running maximum is a warp
// max-scan, listing is a ballot. 32 k-mer lookups, 32 position reads and up to 32 table probes are in
// flight per warp instead of one dependent chain per sub-read -- the kernel was bound by exactly that
// latency (one thread per sub-read: issue slots 17 %, 5.3 ms per 299 k sub-reads; 7 300 hits per sub-read
// on a human-sized index). Small vote tables (<= CS_SMEM_CAP entries) live in shared memory.
// SMEM_TAB = false: no table of the batch is small (human-sized index: thousands of hits per sub-read), the
// 32 KB of shared memory per CTA are not reserved and more warps are resident.
template <bool COUNT_ONLY, bool SMEM_TAB>
__global__ void __launch_bounds__(CS_WARPS * 32) cs_search_kernel(const CsParams p) {
  constexpr bool HAS_SMEM = !COUNT_ONLY && SMEM_TAB;
  __shared__ VoteEntry s_tab[HAS_SMEM ? CS_WARPS : 1][HAS_SMEM ? CS_SMEM_CAP : 1];  // 32 KB per CTA
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int i = blockIdx.x * CS_WARPS + wib;
  if (i >= p.n) return;
  const uint8_t* __restrict__ seq = p.seq + p.seq_off[i];
  const int len = p.seq_len[i];
  const int k = p.k;
  const uint32_t mask = (k == 16) ? 0xffffffffu : ((1u << (2 * k)) - 1u);

  VoteEntry* tab = nullptr;
  uint32_t cap_mask = 0;
  uint32_t* order = nullptr;
  int n_order = 0;
  float max_hits = 0.0f, thresh = 0.0f;
  unsigned long long hits = 0;
  if (!COUNT_ONLY) {
    const uint32_t cap = p.table_cap[i];
    cap_mask = cap - 1u;
    if (HAS_SMEM && cap <= CS_SMEM_CAP) {
      tab = s_tab[wib];
      uint4* z = reinterpret_cast<uint4*>(tab);
      for (uint32_t j = lane; j < cap; j += 32) z[j] = make_uint4(0u, 0u, 0u, 0u);
      __syncwarp();
    } else {
      tab = reinterpret_cast<VoteEntry*>(p.tables) + p.table_off[i];
    }
    order = p.order + p.order_off[i];
  }

  // CS::PrefixIteration with prefixskip = 0 (src/CSstatic.cpp:23-73): a callback for every N-free window of
  // k characters, in order; the walk ends early when an N-run (reached through the N-skipping branch: it
  // starts the sequence or is at least two long) leaves no more than k characters (:38-41) -- which drops
  // exactly one window, the last one, when it starts right behind such a run.
  const int n_win = len - k + 1;
  // the two position lists CompactPrefixTable::GetRefEntry returns for a k-mer: forward list, then the list of the
  // reverse-complement k-mer
  auto lists = [&](uint32_t prefix, uint32_t& fs, uint32_t& fn, uint32_t& rs, uint32_t& rn) {
    if ((p.used_bits[prefix >> 5] >> (prefix & 31u)) & 1u) {
      fs = p.tab[prefix] - 1u;
      fn = p.tab[prefix + 1] - 1u - fs;
    }
    const uint32_t rc = rev_comp(prefix, k, mask);
    if ((p.used_bits[rc >> 5] >> (rc & 31u)) & 1u) {
      rs = p.tab[rc] - 1u;
      rn = p.tab[rc + 1] - 1u - rs;
    }
  };
  // the window that ends the read is dropped when it starts right behind an N-run that is two long or starts the sequence
  auto dropped_last = [&](int pos) {
    if (!(pos + k == len && pos >= 1 && seq[pos - 1] == 'N')) return false;
    int q = pos - 1;
    while (q > 0 && seq[q - 1] == 'N') --q;
    return q == 0 || pos - q >= 2;
  };
  // two consecutive windows (pos, pos + 1): k + 1 characters are read once, the second k-mer is the first one shifted
  auto window_pair = [&](int pos, uint32_t& fs0, uint32_t& fn0, uint32_t& rs0, uint32_t& rn0, uint32_t& fs1, uint32_t& fn1,
                         uint32_t& rs1, uint32_t& rn1) {
    fs0 = fn0 = rs0 = rn0 = fs1 = fn1 = rs1 = rn1 = 0;
    if (pos >= n_win) return;
    uint32_t prefix = 0, nmask = 0;
    for (int j = 0; j < k; ++j) {
      const uint32_t ch = seq[pos + j];
      nmask |= (ch == 'N' ? 1u : 0u) << j;
      prefix = (prefix << 2) | ((ch >> 1) & 3u);
    }
    if (nmask == 0 && !dropped_last(pos)) lists(prefix & mask, fs0, fn0, rs0, rn0);
    if (pos + 1 < n_win) {
      const uint32_t ch = seq[pos + k];
      nmask = (nmask >> 1) | ((ch == 'N' ? 1u : 0u) << (k - 1));
      prefix = (prefix << 2) | ((ch >> 1) & 3u);
      if (nmask == 0 && !dropped_last(pos + 1)) lists(prefix & mask, fs1, fn1, rs1, rn1);
    }
  };
  // 64 windows per round, two consecutive ones per lane: on a 50 Mb index a window has ~0.5 hits, so that rounds of 32
  // windows left the 32-hit batches below half empty
  for (int c0 = 0; c0 < n_win; c0 += 64) {
    uint32_t fs0, fn0, rs0, rn0, fs1, fn1, rs1, rn1;
    window_pair(c0 + 2 * lane, fs0, fn0, rs0, rn0, fs1, fn1, rs1, rn1);
    if (COUNT_ONLY) {
      hits += fn0 + rn0 + fn1 + rn1;
      continue;
    }
    // canonical hit order of the round: window by window, forward list before reverse list
    const uint32_t mine_n = fn0 + rn0 + fn1 + rn1;
    uint32_t incl = mine_n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(FULL, incl, o);
      if (lane >= o) incl += t;
    }
    const uint32_t T = __shfl_sync(FULL, incl, 31);
    for (uint32_t hb = 0; hb < T; hb += 32) {
      const uint32_t h = hb + (uint32_t)lane;
      const bool act = h < T;
      // owner = first lane whose inclusive count exceeds h
      int lo = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1) {
        const uint32_t v = __shfl_sync(FULL, incl, lo + step - 1);
        if (v <= h) lo += step;
      }
      const int owner = lo > 31 ? 31 : lo;
      const uint32_t o_incl = __shfl_sync(FULL, incl, owner), o_n = __shfl_sync(FULL, mine_n, owner);
      const uint32_t o_fn0 = __shfl_sync(FULL, fn0, owner), o_rn0 = __shfl_sync(FULL, rn0, owner);
      const uint32_t o_fn1 = __shfl_sync(FULL, fn1, owner);
      const uint32_t o_fs0 = __shfl_sync(FULL, fs0, owner), o_rs0 = __shfl_sync(FULL, rs0, owner);
      const uint32_t o_fs1 = __shfl_sync(FULL, fs1, owner), o_rs1 = __shfl_sync(FULL, rs1, owner);
      uint32_t off = h - (o_incl - o_n);  // index within the owner's four lists
      int second = 0;                      // which of the owner's two windows
      if (off >= o_fn0 + o_rn0) {
        off -= o_fn0 + o_rn0;
        second = 1;
      }
      const uint32_t w_fn = second ? o_fn1 : o_fn0;
      const bool rev = off >= w_fn;
      uint32_t bin = 0;
      if (act) {
        const uint32_t idx = rev ? (second ? o_rs1 : o_rs0) + (off - w_fn) : (second ? o_fs1 : o_fs0) + off;
        const unsigned long long loc = (unsigned long long)p.pos[idx] + p.unit_offset;
        const int kpos = c0 + 2 * owner + second;
        const unsigned long long corr = rev ? (unsigned long long)(len - (kpos + k)) : (unsigned long long)kpos;
        bin = (uint32_t)((loc - corr) >> p.bin_shift);
      }
    // ---- CS::AddLocationStd for 32 hits at once ----
      const unsigned long long mkey = act ? (unsigned long long)bin : (0x100000000ull | (unsigned long long)lane);
      const unsigned peers = __match_any_sync(FULL, mkey);
      const int leader = __ffs(peers) - 1;
      // The group leaders find or insert their entries (open addressing). No atomics: only this warp touches
      // the table, and leaders that reach the same empty slot in the same round settle it with a match --
      // the lowest lane takes the slot, the others probe on.
      uint32_t slot = ((bin * 2654435761u) >> 7) & cap_mask;
      VoteEntry e;
      e.key = 0; e.state = 0; e.f = 0.0f; e.r = 0.0f;
      bool pending = act && lane == leader;
      while (__any_sync(FULL, pending)) {
        bool empty = false;
        if (pending) {
          e = tab[slot];
          if (e.state & 1u) {
            if (e.key == bin) pending = false;               // found
            else slot = (slot + 1u) & cap_mask;              // occupied by another bin
          } else {
            empty = true;
          }
        }
        const unsigned claim = __match_any_sync(FULL, empty ? (unsigned long long)slot : (0x100000000ull | (unsigned long long)lane));
        if (empty) {
          if (lane == __ffs(claim) - 1) {
            e.key = bin; e.state = 1u; e.f = 0.0f; e.r = 0.0f;
            tab[slot] = e;                                   // inserted
            pending = false;
          } else {
            slot = (slot + 1u) & cap_mask;                   // lost the slot to a lower lane
          }
        }
        __syncwarp();
      }
      slot = __shfl_sync(FULL, slot, leader);
      const float f_old = __shfl_sync(FULL, e.f, leader), r_old = __shfl_sync(FULL, e.r, leader);
      const uint32_t st_old = __shfl_sync(FULL, e.state, leader);
      const unsigned rev_mask = __ballot_sync(FULL, act && rev);
      const unsigned same = peers & (rev ? rev_mask : ~rev_mask);
      const float score = (rev ? r_old : f_old) + (float)(__popc(same & lowmask(lane)) + 1);
      // running maximum in canonical order (:136-141)
      float m = act ? score : 0.0f;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(FULL, m, o);
        if (lane >= o) m = fmaxf(m, t);
      }
      m = fmaxf(m, max_hits);
      const float th = m > max_hits ? __fmul_rn(m, p.sensitivity) : thresh;
      // listing (:143-147): the first hit of a bin that is not listed yet and reaches the threshold
      const bool cond = act && score >= th;
      const unsigned cm = __ballot_sync(FULL, cond);
      const unsigned mine = peers & cm;
      const bool lister = cond && !(st_old & 2u) && lane == (__ffs(mine) - 1);
      const unsigned lm = __ballot_sync(FULL, lister);
      if (lister) order[n_order + __popc(lm & lowmask(lane))] = slot;
      n_order += __popc(lm);
      if (act && lane == leader) {
        e.f = f_old + (float)__popc(peers & ~rev_mask);
        e.r = r_old + (float)__popc(peers & rev_mask);
        e.state = st_old | 1u | ((mine && !(st_old & 2u)) ? 2u : 0u);
        e.key = bin;
        tab[slot] = e;
      }
      const float m_all = __shfl_sync(FULL, m, 31);
      if (m_all > max_hits) {
        max_hits = m_all;
        thresh = __fmul_rn(max_hits, p.sensitivity);
      }
      __syncwarp();
    }
  }

  if (COUNT_ONLY) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) hits += __shfl_xor_sync(FULL, hits, o);
    if (lane == 0) p.hits[i] = hits;
    return;
  }
  // ---- CS::CollectResultsStd: listed bins in listing order, forward before reverse ----
  const float thr = fmaxf(p.min_kmer_hits, thresh);
  CsCandidate* out = p.out + p.out_off[i];
  int n = 0;
  const unsigned long long half = p.bin_shift > 0 ? (1ull << (p.bin_shift - 1)) : 0ull;
  for (int j0 = 0; j0 < n_order; j0 += 32) {
    const int j = j0 + lane;
    VoteEntry e;
    e.key = 0; e.state = 0; e.f = -1.0f; e.r = -1.0f;
    if (j < n_order) e = tab[order[j]];
    const bool ef = j < n_order && e.f >= thr, er = j < n_order && e.r >= thr;
    int cnt = (ef ? 1 : 0) + (er ? 1 : 0);
    int inc = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(FULL, inc, o);
      if (lane >= o) inc += t;
    }
    int at = n + inc - cnt;
    const unsigned long long loc = ((unsigned long long)e.key << p.bin_shift) + half;  // ResolveBin
    if (ef) {
      out[at].loc = loc;
      out[at].score = e.f;
      out[at].reverse = 0;
      ++at;
    }
    if (er) {
      out[at].loc = loc;
      out[at].score = e.r;
      out[at].reverse = 1;
    }
    n += __shfl_sync(FULL, inc, 31);
  }
  if (lane == 0) {
    p.out_count[i] = n;
    p.max_hits[i] = max_hits;
  }
}

// Unpack the reference's 5-byte Index records {uint m_TabIndex; char m_RevCompIndex}
// (#pragma pack(1), src/PrefixTable.h:17-35) into an aligned uint32 array plus a bitmap of
// Index::used() (m_RevCompIndex != 0). The bitmap of a 13-mer index is 8 MB and stays in L2, so the
// ~75 % of lookups that hit an unused prefix never go to HBM.
__global__ void unpack_index_kernel(const uint8_t* __restrict__ packed, uint32_t n, uint32_t* __restrict__ tab,
                                    uint32_t* __restrict__ used_bits) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;  // blockDim is a multiple of 32
  bool used = false;
  if (i < n) {
    const uint8_t* r = packed + (size_t)i * 5;
    tab[i] = (uint32_t)r[0] | ((uint32_t)r[1] << 8) | ((uint32_t)r[2] << 16) | ((uint32_t)r[3] << 24);
    used = r[4] != 0;
  }
  const uint32_t word = __ballot_sync(0xffffffffu, used);
  if ((threadIdx.x & 31) == 0) used_bits[i >> 5] = word;
}

}  // namespace

cudaError_t launch_cs_search(const CsParams& p, bool count_only, bool small_tables, cudaStream_t stream) {
  if (p.n <= 0) return cudaSuccess;
  const int grid = (p.n + CS_WARPS - 1) / CS_WARPS;
  if (count_only)
    cs_search_kernel<true, false><<<grid, CS_WARPS * 32, 0, stream>>>(p);
  else if (small_tables)
    cs_search_kernel<false, true><<<grid, CS_WARPS * 32, 0, stream>>>(p);
  else
    cs_search_kernel<false, false><<<grid, CS_WARPS * 32, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_unpack_index(const uint8_t* packed, uint32_t n, uint32_t* tab, uint32_t* used_bits,
                                cudaStream_t stream) {
  if (!n) return cudaSuccess;
  unpack_index_kernel<<<(n + 255) / 256, 256, 0, stream>>>(packed, n, tab, used_bits);
  return cudaGetLastError();
}

}  // namespace nb
