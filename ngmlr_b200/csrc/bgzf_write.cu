// ngmlr_b200/csrc/bgzf_write.cu -- BGZF output with the deflate on the device (ngmlr_b200_bgzf_*).
//
// The byte stream is cut into blocks of 0xff00 input bytes (htslib's BGZF_BLOCK_SIZE); only flush and close end a
// block early. A batch of whole blocks (the page-locked staging, double-buffered) is compressed on the handle's own
// stream while the caller fills the other staging buffer and the host writes the previous batch to the file:
//   1. k_keys: every position's 4-byte value, and its offset in its block.
//   2. one stable segmented radix sort (a segment per block) on the 4-byte value: the positions before a position in
//      its run of equal values are its prior occurrences, nearest first.
//   3. k_match: each position checks up to MAX_CAND of them within 32 KiB, by words, and keeps the longest (the
//      nearest on a tie): length | distance << 9, or 0.
//   4. k_deflate, one CTA per block: DT threads each parse a DT-th of the block greedily (a match is cut at the end of
//      the thread's slice), count symbols into shared histograms, build length-limited Huffman codes (15 bits, 7 for
//      the code-length code), pick the smallest of dynamic, fixed and stored by exact bit count, size their slices,
//      scan, and pack their tokens' bits into the block's 64 KiB slot. The BGZF header, the CRC32 (a slice per thread,
//      combined with inflate_core.cuh's GF(2) arithmetic) and ISIZE complete the member.
//   5. an exclusive scan of the member sizes, and k_gather packs the members back to back for the copy back.
// Nothing depends on timing or on the order of atomics: histograms are counts, the sort is stable, ties go to the
// nearer position, and every bit has one writer. So the file depends only on the bytes and the flush points.
#include <cub/cub.cuh>
#include <fcntl.h>
#include <unistd.h>

#include <cerrno>
#include <cstring>
#include <string>

#include "inflate_core.cuh"
#include "runtime.h"

namespace nb {
namespace {

constexpr uint32_t BLOCK = 0xff00;   // input bytes per member
constexpr uint32_t SLOT = 65536;     // device bytes per member before packing
constexpr uint32_t HDR = 18;         // BGZF member header
constexpr uint32_t MEMBER_OVERHEAD = HDR + 5 + 8;  // header, stored-block header, CRC32 + ISIZE
constexpr int DT = 64;               // threads of k_deflate, and parse slices per block
constexpr int MAX_CAND = 4;          // prior occurrences checked per position
constexpr uint32_t MAX_DIST = 32768;
constexpr int64_t DEFAULT_CHUNK = 64ll << 20;
constexpr int64_t MAX_CHUNK = 1ll << 30;

const uint8_t kEof[28] = {0x1f, 0x8b, 0x08, 0x04, 0, 0, 0, 0, 0, 0xff, 0x06, 0, 0x42, 0x43, 0x02, 0, 0x1b, 0, 0x03,
                          0, 0, 0, 0, 0, 0, 0, 0, 0};

// 4 bytes at byte offset i of word-aligned memory (reads the word after too)
__device__ __forceinline__ uint32_t ld32(const uint32_t* w, size_t i) {
  return __funnelshift_r(w[i >> 2], w[(i >> 2) + 1], (uint32_t)(i & 3) * 8);
}

__global__ void k_keys(const uint32_t* in, uint32_t n, uint32_t* keys, uint16_t* pos, int* seg, uint32_t n_blocks) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) {
    if (i < n) {
      keys[i] = ld32(in, i);
      pos[i] = (uint16_t)(i % BLOCK);
    }
    if (i <= n_blocks) seg[i] = (int)min(i * BLOCK, n);
  }
}

__global__ void k_match(const uint32_t* in, uint32_t n, const uint32_t* keys, const uint16_t* pos, uint32_t* match) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t s = i / BLOCK * BLOCK, len = min(BLOCK, n - s), p = pos[i];
    uint32_t best = 0;
    if (p + 4 <= len) {
      const uint32_t key = keys[i], maxl = min(258u, len - p);
      uint32_t bl = 0, bd = 0;
      for (int c = 1; c <= MAX_CAND && i >= s + c; ++c) {
        if (keys[i - c] != key) break;
        const uint32_t q = pos[i - c], d = p - q;
        if (d > MAX_DIST) break;
        uint32_t k = 4;  // equal keys: the first 4 bytes match
        while (k < maxl) {
          const uint32_t x = ld32(in, s + q + k) ^ ld32(in, s + p + k);
          if (x) {
            k += (__ffs(x) - 1) >> 3;
            break;
          }
          k += 4;
        }
        k = min(k, maxl);
        if (k > bl) {
          bl = k;
          bd = d;
          if (k == maxl) break;
        }
      }
      best = bl | bd << 9;
    }
    match[s + p] = best;
  }
}

struct Tables {
  uint32_t lit_hist[286], dist_hist[30], cl_hist[19];
  uint16_t lit_code[288], dist_code[30], cl_code[19];  // 288: the fixed code's canonical order counts 286 and 287
  uint8_t lit_len[288], dist_len[30], cl_len[19];
  uint8_t len_sym[259];   // match length -> length symbol - 257
  uint8_t dist_sym[512];  // d - 1 < 256 ? [d - 1] : [256 + ((d - 1) >> 7)]
  uint32_t crc_tab[256];
  uint16_t sorted[288];   // used symbols by (frequency, symbol)
  uint32_t work[288];
  uint16_t cl_seq[320];   // a dynamic header's code-length symbols: symbol | extra value << 5
  uint32_t num[33], next_code[16];
  uint8_t all_len[316];
  uint32_t crc_part[DT / 32];
  int n_cl_seq, nlit, ndist, ncl, mode;  // mode: 0 stored, 1 fixed, 2 dynamic
  uint32_t hdr_bits;
};

// Minimum-redundancy code lengths of the ascending weights A[0..m), in place (Moffat and Katajainen, 1995).
__device__ void mk_lengths(uint32_t* A, int m) {
  A[0] += A[1];
  int root = 0, leaf = 2;
  for (int next = 1; next < m - 1; ++next) {
    if (leaf >= m || A[root] < A[leaf]) {
      A[next] = A[root];
      A[root++] = next;
    } else {
      A[next] = A[leaf++];
    }
    if (leaf >= m || (root < next && A[root] < A[leaf])) {
      A[next] += A[root];
      A[root++] = next;
    } else {
      A[next] += A[leaf++];
    }
  }
  A[m - 2] = 0;
  for (int next = m - 3; next >= 0; --next) A[next] = A[A[next]] + 1;
  int avail = 1, used = 0, depth = 0, root2 = m - 2, next = m - 1;
  while (avail > 0) {
    while (root2 >= 0 && (int)A[root2] == depth) {
      ++used;
      --root2;
    }
    while (avail > used) {
      A[next--] = depth;
      --avail;
    }
    avail = 2 * used;
    ++depth;
    used = 0;
  }
}

// Code lengths of freq[0..n) of at most `limit` bits, by the whole CTA. The used symbols are ranked by (frequency,
// symbol); over-long lengths are folded to `limit` and shorter codes lengthened until Kraft's sum is exact. A single
// used symbol gets a partner so that every code is complete.
__device__ void huff_lengths(const uint32_t* freq, int n, int limit, uint8_t* len, Tables& t) {
  for (int s = threadIdx.x; s < n; s += DT) {
    len[s] = 0;
    const uint32_t f = freq[s];
    if (!f) continue;
    int r = 0;
    for (int u = 0; u < n; ++u) {
      const uint32_t g = freq[u];
      r += g && (g < f || (g == f && u < s));
    }
    t.sorted[r] = (uint16_t)s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int m = 0;
    for (int s = 0; s < n; ++s) m += freq[s] != 0;
    if (m == 1) {
      len[t.sorted[0]] = 1;
      len[t.sorted[0] == 0 ? 1 : 0] = 1;
    } else if (m > 1) {
      for (int i = 0; i < m; ++i) t.work[i] = freq[t.sorted[i]];
      mk_lengths(t.work, m);
      for (int d = 0; d <= 32; ++d) t.num[d] = 0;
      for (int i = 0; i < m; ++i) ++t.num[min(t.work[i], 32u)];
      for (int d = limit + 1; d <= 32; ++d) {
        t.num[limit] += t.num[d];
        t.num[d] = 0;
      }
      uint32_t total = 0;
      for (int d = 1; d <= limit; ++d) total += t.num[d] << (limit - d);
      while (total > (1u << limit)) {
        --t.num[limit];
        for (int d = limit - 1; d > 0; --d)
          if (t.num[d]) {
            --t.num[d];
            t.num[d + 1] += 2;
            break;
          }
        --total;
      }
      int k = 0;  // the rarest symbols get the longest codes
      for (int d = limit; d >= 1; --d)
        for (uint32_t c = 0; c < t.num[d]; ++c) len[t.sorted[k++]] = (uint8_t)d;
    }
  }
  __syncthreads();
}

// canonical codes of len[0..n), bit-reversed for the LSB-first stream (one thread)
__device__ void canonical(const uint8_t* len, int n, uint16_t* code, uint32_t* num, uint32_t* next) {
  for (int b = 0; b < 16; ++b) num[b] = 0;
  for (int s = 0; s < n; ++s) ++num[len[s]];
  num[0] = 0;
  uint32_t c = 0;
  next[0] = 0;
  for (int b = 1; b < 16; ++b) {
    c = (c + num[b - 1]) << 1;
    next[b] = c;
  }
  for (int s = 0; s < n; ++s)
    if (len[s]) code[s] = (uint16_t)(__brev(next[len[s]]++) >> (32 - len[s]));
}

// LSB-first bit writer into a zeroed slot. Words it fills alone are stored; the first and last, which it may share
// with a neighbour, are ORed in.
struct BitWriter {
  uint32_t* w;
  uint32_t wi;
  uint64_t acc;
  int n;
  bool first;
  __device__ void init(uint32_t* base, uint32_t bit) {
    w = base;
    wi = bit >> 5;
    n = (int)(bit & 31);
    acc = 0;
    first = true;
  }
  __device__ __forceinline__ void put(uint32_t v, int nb) {
    acc |= (uint64_t)v << n;
    n += nb;
    if (n >= 32) {
      if (first) atomicOr(w + wi, (uint32_t)acc);
      else w[wi] = (uint32_t)acc;
      first = false;
      ++wi;
      acc >>= 32;
      n -= 32;
    }
  }
  __device__ void done() {
    if (n) atomicOr(w + wi, (uint32_t)acc);
  }
};

enum { HIST = 0, COUNT = 1, EMIT = 2 };

__device__ __forceinline__ int dsym_index(uint32_t d) { return d <= 256 ? (int)d - 1 : 256 + (int)((d - 1) >> 7); }

// the greedy parse of in[a, b) of the block: histogram, bit count or bits
template <int MODE>
__device__ uint32_t walk(const uint8_t* in, const uint32_t* match, uint32_t a, uint32_t b, Tables& t, BitWriter& bw) {
  uint32_t bits = 0;
  for (uint32_t p = a; p < b;) {
    const uint32_t m = match[p];
    const uint32_t L = min(m & 511, b - p);
    if (L >= 3) {
      const uint32_t d = m >> 9;
      const int ls = t.len_sym[L], ds = t.dist_sym[dsym_index(d)];
      if (MODE == HIST) {
        atomicAdd(&t.lit_hist[257 + ls], 1u);
        atomicAdd(&t.dist_hist[ds], 1u);
      } else if (MODE == COUNT) {
        bits += t.lit_len[257 + ls] + kLenExtra[ls] + t.dist_len[ds] + kDistExtra[ds];
      } else {
        bw.put(t.lit_code[257 + ls] | (L - kLenBase[ls]) << t.lit_len[257 + ls], t.lit_len[257 + ls] + kLenExtra[ls]);
        bw.put(t.dist_code[ds] | (d - kDistBase[ds]) << t.dist_len[ds], t.dist_len[ds] + kDistExtra[ds]);
      }
      p += L;
    } else {
      const int c = in[p];
      if (MODE == HIST) atomicAdd(&t.lit_hist[c], 1u);
      else if (MODE == COUNT) bits += t.lit_len[c];
      else bw.put(t.lit_code[c], t.lit_len[c]);
      ++p;
    }
  }
  return bits;
}

// run-length code of the dynamic header's code lengths (one thread)
__device__ void header_rle(Tables& t) {
  uint8_t* lens = t.all_len;
  int n = 0;
  for (int s = 0; s < t.nlit; ++s) lens[n++] = t.lit_len[s];
  for (int s = 0; s < t.ndist; ++s) lens[n++] = t.dist_len[s];
  int k = 0;
  for (int i = 0; i < n;) {
    const uint8_t v = lens[i];
    int r = 1;
    while (i + r < n && lens[i + r] == v) ++r;
    i += r;
    if (v == 0) {
      while (r >= 11) {
        const int c = min(r, 138);
        t.cl_seq[k++] = (uint16_t)(18 | (c - 11) << 5);
        r -= c;
      }
      if (r >= 3) {
        t.cl_seq[k++] = (uint16_t)(17 | (r - 3) << 5);
        r = 0;
      }
    } else {
      t.cl_seq[k++] = v;
      --r;
      while (r >= 3) {
        const int c = min(r, 6);
        t.cl_seq[k++] = (uint16_t)(16 | (c - 3) << 5);
        r -= c;
      }
    }
    while (r-- > 0) t.cl_seq[k++] = v;
  }
  t.n_cl_seq = k;
}

__device__ __forceinline__ int cl_extra_bits(int sym) { return sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0; }

__global__ void __launch_bounds__(DT) k_deflate(const uint8_t* __restrict__ in, uint32_t n,
                                                const uint32_t* __restrict__ match, uint8_t* slots, uint32_t* sizes,
                                                unsigned int* stored) {
  __shared__ Tables t;
  const int tid = threadIdx.x;
  const uint32_t s = blockIdx.x * BLOCK, len = min(BLOCK, n - s);
  in += s;
  match += s;
  uint8_t* slot = slots + (size_t)blockIdx.x * SLOT;
  uint32_t* slot_w = reinterpret_cast<uint32_t*>(slot);
  for (int i = tid; i < (int)(SLOT / 16); i += DT) reinterpret_cast<uint4*>(slot)[i] = make_uint4(0, 0, 0, 0);
  for (int i = tid; i < 256; i += DT) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
    t.crc_tab[i] = c;
  }
  for (int i = tid; i < 286; i += DT) t.lit_hist[i] = 0;
  if (tid < 30) t.dist_hist[tid] = 0;
  if (tid < 19) t.cl_hist[tid] = 0;
  for (int L = 3 + tid; L <= 258; L += DT) {
    int i = 28;
    while (kLenBase[i] > L) --i;
    t.len_sym[L] = (uint8_t)i;
  }
  for (int e = tid; e < 512; e += DT) {
    const uint32_t d = e < 256 ? e + 1 : ((uint32_t)(e - 256) << 7) + 1;
    int i = 29;
    while (kDistBase[i] > d) --i;
    t.dist_sym[e] = (uint8_t)i;
  }
  __syncthreads();

  const uint32_t seg = (len + DT - 1) / DT, a = min(len, tid * seg), b = min(len, a + seg);
  BitWriter bw;
  walk<HIST>(in, match, a, b, t, bw);
  // raw CRC of this thread's slice, shifted past the bytes after it
  uint32_t r = 0;
  for (uint32_t i = a; i < b; ++i) r = t.crc_tab[(r ^ in[i]) & 0xff] ^ (r >> 8);
  r = gf2_mul(r, x_pow_8n(len - b));
  for (int k = 16; k; k >>= 1) r ^= __shfl_xor_sync(FULL, r, k);
  if ((tid & 31) == 0) t.crc_part[tid / 32] = r;
  if (tid == 0) t.lit_hist[256] = 1;
  __syncthreads();

  huff_lengths(t.lit_hist, 286, 15, t.lit_len, t);
  huff_lengths(t.dist_hist, 30, 15, t.dist_len, t);
  if (tid == 0) {
    t.nlit = 286;
    while (t.nlit > 257 && !t.lit_len[t.nlit - 1]) --t.nlit;
    t.ndist = 30;
    while (t.ndist > 1 && !t.dist_len[t.ndist - 1]) --t.ndist;
    header_rle(t);
    for (int i = 0; i < t.n_cl_seq; ++i) ++t.cl_hist[t.cl_seq[i] & 31];
  }
  __syncthreads();
  huff_lengths(t.cl_hist, 19, 7, t.cl_len, t);
  if (tid == 0) {
    t.ncl = 19;
    while (t.ncl > 4 && !t.cl_len[kClOrder[t.ncl - 1]]) --t.ncl;
    uint32_t hdr = 5 + 5 + 4 + 3 * t.ncl;
    for (int i = 0; i < t.n_cl_seq; ++i) {
      const int sym = t.cl_seq[i] & 31;
      hdr += t.cl_len[sym] + cl_extra_bits(sym);
    }
    uint32_t extra = 0, dyn = 0, fix = 0;
    for (int i = 0; i < 29; ++i) extra += t.lit_hist[257 + i] * kLenExtra[i];
    for (int i = 0; i < 30; ++i) {
      extra += t.dist_hist[i] * kDistExtra[i];
      dyn += t.dist_hist[i] * t.dist_len[i];
      fix += t.dist_hist[i] * 5;
    }
    for (int i = 0; i < 286; ++i) {
      dyn += t.lit_hist[i] * t.lit_len[i];
      fix += t.lit_hist[i] * (i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8);
    }
    dyn += 3 + hdr + extra;
    fix += 3 + extra;
    const uint32_t sto = 8 * (5 + len);
    t.mode = sto <= min(fix, dyn) ? 0 : fix <= dyn ? 1 : 2;
    // RFC 1951's fixed literal / length code is canonical over all 288 symbols (286 and 287 have length 8); the
    // dynamic code never uses them
    if (t.mode == 1) {
      for (int i = 0; i < 288; ++i) t.lit_len[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
      for (int i = 0; i < 30; ++i) t.dist_len[i] = 5;
      t.hdr_bits = 3;
    } else {
      t.lit_len[286] = t.lit_len[287] = 0;
      t.hdr_bits = 3 + hdr;
      canonical(t.cl_len, 19, t.cl_code, t.num, t.next_code);
    }
    canonical(t.lit_len, 288, t.lit_code, t.num, t.next_code);
    canonical(t.dist_len, 30, t.dist_code, t.num, t.next_code);
  }
  __syncthreads();

  const int mode = t.mode;
  uint32_t dlen;  // deflate bytes
  if (mode == 0) {
    dlen = 5 + len;
    for (uint32_t i = tid; i < len; i += DT) slot[HDR + 5 + i] = in[i];
    if (tid == 0) {
      slot[HDR] = 1;
      slot[HDR + 1] = (uint8_t)len;
      slot[HDR + 2] = (uint8_t)(len >> 8);
      slot[HDR + 3] = (uint8_t)~len;
      slot[HDR + 4] = (uint8_t)(~len >> 8);
    }
  } else {
    uint32_t mine = walk<COUNT>(in, match, a, b, t, bw);
    if (tid == DT - 1) mine += t.lit_len[256];
    typedef cub::BlockScan<uint32_t, DT> Scan;
    __shared__ typename Scan::TempStorage scan_tmp;
    uint32_t off, total;
    Scan(scan_tmp).ExclusiveSum(mine, off, total);
    const uint32_t base = HDR * 8 + t.hdr_bits;
    bw.init(slot_w, base + off);
    walk<EMIT>(in, match, a, b, t, bw);
    if (tid == DT - 1) bw.put(t.lit_code[256], t.lit_len[256]);
    bw.done();
    if (tid == 0) {
      BitWriter hw;
      hw.init(slot_w, HDR * 8);
      hw.put(1 | mode << 1, 3);
      if (mode == 2) {
        hw.put(t.nlit - 257, 5);
        hw.put(t.ndist - 1, 5);
        hw.put(t.ncl - 4, 4);
        for (int i = 0; i < t.ncl; ++i) hw.put(t.cl_len[kClOrder[i]], 3);
        for (int i = 0; i < t.n_cl_seq; ++i) {
          const int sym = t.cl_seq[i] & 31;
          hw.put(t.cl_code[sym], t.cl_len[sym]);
          if (sym >= 16) hw.put(t.cl_seq[i] >> 5, cl_extra_bits(sym));
        }
      }
      hw.done();
    }
    dlen = (t.hdr_bits + total + 7) / 8;
  }
  __syncthreads();
  if (tid == 0) {
    uint32_t crc = 0;
    for (int k = 0; k < DT / 32; ++k) crc ^= t.crc_part[k];
    crc = crc ^ gf2_mul(0xffffffffu, x_pow_8n(len)) ^ 0xffffffffu;
    const uint32_t size = HDR + dlen + 8, bsize = size - 1;
    const uint8_t h[HDR] = {0x1f, 0x8b, 0x08, 0x04, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0,
                            (uint8_t)bsize, (uint8_t)(bsize >> 8)};
    for (uint32_t i = 0; i < HDR; ++i) slot[i] = h[i];
    uint8_t* tr = slot + HDR + dlen;
    for (int i = 0; i < 4; ++i) {
      tr[i] = (uint8_t)(crc >> (8 * i));
      tr[4 + i] = (uint8_t)(len >> (8 * i));
    }
    sizes[blockIdx.x] = size;
    if (mode == 0) atomicAdd(stored, 1u);
  }
}

__global__ void k_gather(const uint8_t* slots, const uint32_t* sizes, const uint32_t* off, uint8_t* out) {
  const uint8_t* src = slots + (size_t)blockIdx.x * SLOT;
  uint8_t* dst = out + off[blockIdx.x];
  for (uint32_t i = threadIdx.x; i < sizes[blockIdx.x]; i += blockDim.x) dst[i] = src[i];
}

template <class T>
void dfree(T*& p) {
  if (p) cudaFree(p);
  p = nullptr;
}

}  // namespace
}  // namespace nb

using namespace nb;

struct ngmlr_b200_bgzf_writer {
  int device = -1;
  int fd = -1;
  cudaStream_t st = nullptr;
  std::string error;
  bool failed = false;
  size_t cap = 0, fill = 0;  // staging bytes per batch (whole blocks), bytes staged in h_in[cur]
  int cur = 0;
  uint8_t* h_in[2] = {nullptr, nullptr};
  uint8_t* h_out[2] = {nullptr, nullptr};
  uint32_t* h_meta = nullptr;  // per buffer: packed bytes, stored blocks
  bool pending[2] = {false, false};
  cudaEvent_t ev_done[2] = {nullptr, nullptr}, ev_a[2] = {nullptr, nullptr}, ev_b[2] = {nullptr, nullptr};
  uint8_t* d_in = nullptr;
  uint32_t* d_keys[2] = {nullptr, nullptr};
  uint16_t* d_pos[2] = {nullptr, nullptr};
  int* d_seg = nullptr;
  uint32_t* d_match = nullptr;
  uint8_t* d_slots = nullptr;
  uint8_t* d_out = nullptr;
  uint32_t* d_sizes = nullptr;  // n_blocks + 1 (the last 0), then the scan into d_off
  uint32_t* d_off = nullptr;
  uint32_t* d_stored = nullptr;
  void* d_temp = nullptr;
  size_t temp_bytes = 0, device_bytes = 0;
  int64_t bytes_in = 0, bytes_out = 0, blocks = 0, stored = 0;
  double device_ms = 0;

  int fail(const std::string& msg) {
    if (!failed) error = msg;
    failed = true;
    return -1;
  }
  int cuda_fail(cudaError_t e, const char* what) {
    return fail(std::string("bgzf: ") + what + " failed: " + cudaGetErrorString(e));
  }
  int write_all(const uint8_t* p, size_t n) {
    while (n) {
      const ssize_t k = ::write(fd, p, n);
      if (k < 0) {
        if (errno == EINTR) continue;
        return fail(std::string("bgzf: write failed: ") + strerror(errno));
      }
      p += k;
      n -= (size_t)k;
    }
    return 0;
  }
};

namespace nb {
namespace {

#define WCU(call)                                          \
  do {                                                     \
    const cudaError_t e__ = (call);                        \
    if (e__ != cudaSuccess) return w->cuda_fail(e__, #call); \
  } while (0)

// wait for the batch of buffer b and append its members to the file
int finish(ngmlr_b200_bgzf_writer* w, int b) {
  if (!w->pending[b]) return 0;
  w->pending[b] = false;
  WCU(cudaEventSynchronize(w->ev_done[b]));
  float ms = 0;
  WCU(cudaEventElapsedTime(&ms, w->ev_a[b], w->ev_b[b]));
  w->device_ms += ms;
  w->stored += w->h_meta[2 * b + 1];
  w->bytes_out += w->h_meta[2 * b];
  return w->write_all(w->h_out[b], w->h_meta[2 * b]);
}

// compress the staged bytes of h_in[cur] on the handle's stream, then write the previous batch
int submit(ngmlr_b200_bgzf_writer* w) {
  const int b = w->cur;
  const uint32_t n = (uint32_t)w->fill;
  const uint32_t nb = (n + BLOCK - 1) / BLOCK;
  cudaStream_t st = w->st;
  WCU(cudaSetDevice(w->device));
  WCU(cudaMemcpyAsync(w->d_in, w->h_in[b], n, cudaMemcpyHostToDevice, st));
  WCU(cudaEventRecord(w->ev_a[b], st));
  WCU(cudaMemsetAsync(w->d_in + n, 0, 8, st));
  WCU(cudaMemsetAsync(w->d_sizes, 0, (nb + 1) * sizeof(uint32_t), st));
  WCU(cudaMemsetAsync(w->d_stored, 0, sizeof(uint32_t), st));
  const int grid = (int)std::min<uint32_t>((n + 255) / 256, 132u * 16);
  k_keys<<<grid, 256, 0, st>>>(reinterpret_cast<const uint32_t*>(w->d_in), n, w->d_keys[0], w->d_pos[0], w->d_seg, nb);
  cub::DoubleBuffer<uint32_t> keys(w->d_keys[0], w->d_keys[1]);
  cub::DoubleBuffer<uint16_t> vals(w->d_pos[0], w->d_pos[1]);
  size_t tb = w->temp_bytes;
  WCU(cub::DeviceSegmentedRadixSort::SortPairs(w->d_temp, tb, keys, vals, (int)n, (int)nb, w->d_seg, w->d_seg + 1, 0,
                                               32, st));
  k_match<<<grid, 256, 0, st>>>(reinterpret_cast<const uint32_t*>(w->d_in), n, keys.Current(), vals.Current(),
                                w->d_match);
  k_deflate<<<nb, DT, 0, st>>>(w->d_in, n, w->d_match, w->d_slots, w->d_sizes, w->d_stored);
  tb = w->temp_bytes;
  WCU(cub::DeviceScan::ExclusiveSum(w->d_temp, tb, w->d_sizes, w->d_off, (int)nb + 1, st));
  k_gather<<<nb, 256, 0, st>>>(w->d_slots, w->d_sizes, w->d_off, w->d_out);
  WCU(cudaGetLastError());
  WCU(cudaEventRecord(w->ev_b[b], st));
  WCU(cudaMemcpyAsync(w->h_out[b], w->d_out, (size_t)n + (size_t)nb * MEMBER_OVERHEAD, cudaMemcpyDeviceToHost, st));
  WCU(cudaMemcpyAsync(w->h_meta + 2 * b, w->d_off + nb, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  WCU(cudaMemcpyAsync(w->h_meta + 2 * b + 1, w->d_stored, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  WCU(cudaEventRecord(w->ev_done[b], st));
  w->pending[b] = true;
  w->bytes_in += n;
  w->blocks += nb;
  w->fill = 0;
  w->cur = 1 - b;
  return finish(w, 1 - b);
}

void release(ngmlr_b200_bgzf_writer* w) {
  if (w->device >= 0) cudaSetDevice(w->device);
  if (w->st) cudaStreamSynchronize(w->st);
  for (int b = 0; b < 2; ++b) {
    if (w->h_in[b]) cudaFreeHost(w->h_in[b]);
    if (w->h_out[b]) cudaFreeHost(w->h_out[b]);
    if (w->ev_done[b]) cudaEventDestroy(w->ev_done[b]);
    if (w->ev_a[b]) cudaEventDestroy(w->ev_a[b]);
    if (w->ev_b[b]) cudaEventDestroy(w->ev_b[b]);
    dfree(w->d_keys[b]);
    dfree(w->d_pos[b]);
  }
  if (w->h_meta) cudaFreeHost(w->h_meta);
  dfree(w->d_in);
  dfree(w->d_seg);
  dfree(w->d_match);
  dfree(w->d_slots);
  dfree(w->d_out);
  dfree(w->d_sizes);
  dfree(w->d_off);
  dfree(w->d_stored);
  dfree(w->d_temp);
  if (w->st) cudaStreamDestroy(w->st);
  if (w->fd >= 0) ::close(w->fd);
  delete w;
}

template <class T>
int dalloc(ngmlr_b200_bgzf_writer* w, T*& p, size_t count) {
  const size_t bytes = count * sizeof(T);
  WCU(cudaMalloc(&p, bytes));
  w->device_bytes += bytes;
  return 0;
}

int setup(ngmlr_b200_bgzf_writer* w) {
  const size_t cap = w->cap, nb = cap / BLOCK;
  WCU(cudaSetDevice(w->device));
  WCU(cudaStreamCreateWithFlags(&w->st, cudaStreamNonBlocking));
  for (int b = 0; b < 2; ++b) {
    WCU(cudaHostAlloc(&w->h_in[b], cap, cudaHostAllocDefault));
    WCU(cudaHostAlloc(&w->h_out[b], cap + nb * MEMBER_OVERHEAD, cudaHostAllocDefault));
    WCU(cudaEventCreateWithFlags(&w->ev_done[b], cudaEventBlockingSync));
    WCU(cudaEventCreate(&w->ev_a[b]));
    WCU(cudaEventCreate(&w->ev_b[b]));
    if (dalloc(w, w->d_keys[b], cap) || dalloc(w, w->d_pos[b], cap)) return -1;
  }
  WCU(cudaHostAlloc(&w->h_meta, 4 * sizeof(uint32_t), cudaHostAllocDefault));
  if (dalloc(w, w->d_in, cap + 8) || dalloc(w, w->d_seg, nb + 1) || dalloc(w, w->d_match, cap) ||
      dalloc(w, w->d_slots, nb * SLOT) || dalloc(w, w->d_out, cap + nb * MEMBER_OVERHEAD) ||
      dalloc(w, w->d_sizes, nb + 1) || dalloc(w, w->d_off, nb + 1) || dalloc(w, w->d_stored, 1))
    return -1;
  cub::DoubleBuffer<uint32_t> keys(w->d_keys[0], w->d_keys[1]);
  cub::DoubleBuffer<uint16_t> vals(w->d_pos[0], w->d_pos[1]);
  size_t sort_tmp = 0, scan_tmp = 0;
  WCU(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, sort_tmp, keys, vals, (int)cap, (int)nb, w->d_seg,
                                               w->d_seg + 1, 0, 32, w->st));
  WCU(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, w->d_sizes, w->d_off, (int)nb + 1, w->st));
  w->temp_bytes = std::max(sort_tmp, scan_tmp);
  return dalloc(w, reinterpret_cast<uint8_t*&>(w->d_temp), w->temp_bytes);
}

}  // namespace
}  // namespace nb

extern "C" {

int ngmlr_b200_bgzf_open(ngmlr_b200_ctx* ctx, const char* path, const ngmlr_b200_bgzf_options* opts,
                         ngmlr_b200_bgzf_writer** out) {
  if (!ctx || !path || !out) {
    set_error_without_context("bgzf_open: ctx, path and out must not be NULL");
    return -1;
  }
  *out = nullptr;
  const int64_t chunk = opts && opts->chunk_bytes > 0 ? opts->chunk_bytes : DEFAULT_CHUNK;
  if (chunk > MAX_CHUNK) {
    set_error_without_context("bgzf_open: chunk_bytes above 1 GiB");
    return -1;
  }
  const int fd = ::open(path, O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0666);
  if (fd < 0) {
    set_error_without_context(std::string("bgzf_open: cannot open ") + path + ": " + strerror(errno));
    return -1;
  }
  ngmlr_b200_bgzf_writer* w = new ngmlr_b200_bgzf_writer();
  w->fd = fd;
  w->device = ctx->device;
  w->cap = std::max<size_t>(1, (size_t)chunk / BLOCK) * BLOCK;
  if (setup(w)) {
    set_error_without_context(w->error);
    release(w);
    return -1;
  }
  *out = w;
  return 0;
}

int ngmlr_b200_bgzf_write(ngmlr_b200_bgzf_writer* w, const void* buf, size_t n) {
  if (!w || (n && !buf)) return -1;
  if (w->failed) return -1;
  const uint8_t* p = static_cast<const uint8_t*>(buf);
  while (n) {
    const size_t k = std::min(n, w->cap - w->fill);
    memcpy(w->h_in[w->cur] + w->fill, p, k);
    w->fill += k;
    p += k;
    n -= k;
    if (w->fill == w->cap && submit(w)) return -1;
  }
  return 0;
}

int ngmlr_b200_bgzf_flush(ngmlr_b200_bgzf_writer* w) {
  if (!w) return -1;
  if (w->failed) return -1;
  if (w->fill && submit(w)) return -1;
  if (finish(w, 0) || finish(w, 1)) return -1;
  return 0;
}

int ngmlr_b200_bgzf_close(ngmlr_b200_bgzf_writer* w) {
  if (!w) return -1;
  int rc = ngmlr_b200_bgzf_flush(w);
  if (!rc) rc = w->write_all(kEof, sizeof kEof);
  if (!rc) {
    const int fd = w->fd;
    w->fd = -1;
    if (::close(fd) != 0) rc = w->fail(std::string("bgzf: close failed: ") + strerror(errno));
  }
  if (rc) set_error_without_context(w->error);
  release(w);
  return rc;
}

const char* ngmlr_b200_bgzf_last_error(const ngmlr_b200_bgzf_writer* w) { return w ? w->error.c_str() : ""; }

int ngmlr_b200_bgzf_stats(const ngmlr_b200_bgzf_writer* w, int64_t* bytes_in, int64_t* bytes_out, int64_t* blocks,
                          int64_t* stored_blocks, float* device_ms, int64_t* device_bytes) {
  if (!w) return -1;
  if (bytes_in) *bytes_in = w->bytes_in;
  if (bytes_out) *bytes_out = w->bytes_out;
  if (blocks) *blocks = w->blocks;
  if (stored_blocks) *stored_blocks = w->stored;
  if (device_ms) *device_ms = (float)w->device_ms;
  if (device_bytes) *device_bytes = (int64_t)w->device_bytes;
  return 0;
}

}  // extern "C"
