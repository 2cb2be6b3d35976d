// ngmlr_b200/csrc/inflate.cu -- BGZF members inflated on the device (the stream layer of fasta.cpp launches it).
//
// One warp per member. Every lane runs the same bit reader and Huffman decode (shared-memory table reads broadcast),
// so control flow stays uniform; the warp splits what is parallel: table construction (ballots / match_any over 32
// symbols at a time), match and stored-block copies (one byte per lane), and the member's CRC32 (a slice per lane,
// combined with GF(2) shifts). The output goes straight to its offset in the round's output buffer.
//
// A member is accepted only when zlib's inflate would accept it with the same output: every case zlib rejects
// (block type 3, stored LEN / NLEN mismatch, HLIT > 286 or HDIST > 30, over-subscribed codes, incomplete codes other
// than a single code of length 1, a bad repeat code, no end-of-block code, literal / length symbols 286 / 287,
// distance symbols 30 / 31, a distance before the member's first byte) sets a nonzero status, as does a deflate
// stream that does not end exactly at the trailer, an output length other than ISIZE or a CRC32 other than the
// trailer's. The host then hands the member to zlib.
#include <cstdint>

#include "fasta.h"

namespace nb {

namespace {

constexpr int WARPS = 4;       // members per block
constexpr int LIT_FAST = 10;   // index bits of the literal / length lookup table
constexpr int DIST_FAST = 8;   // ... of the distance table (and of the code-length code, which it holds first)
constexpr unsigned FULL = 0xffffffffu;

enum : int32_t {
  ST_OK = 0,
  ST_BLOCK_TYPE = 1,
  ST_STORED_LEN = 2,
  ST_COUNTS = 3,
  ST_CODES = 4,
  ST_REPEAT = 5,
  ST_NO_EOB = 6,
  ST_SYMBOL = 7,
  ST_DISTANCE = 8,
  ST_OUTPUT = 9,
  ST_INPUT = 10,
  ST_END = 11,
  ST_ISIZE = 12,
  ST_CRC = 13,
};

__constant__ uint16_t kLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                      31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t kDistBase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                       193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct WarpTables {
  uint16_t lit_fast[1 << LIT_FAST];  // (code length << 9) | symbol for codes of at most LIT_FAST bits, else 0
  uint16_t dist_fast[1 << DIST_FAST];
  uint16_t lit_sym[288];             // symbols by code length, then by value (canonical order)
  uint16_t dist_sym[32];
  uint16_t lit_count[16], dist_count[16], next[16];
  uint8_t lens[320];
};

// LSB-first bit reader over aligned 32-bit words; every lane holds the same state.
struct Bits {
  const uint32_t* w;
  uint64_t wi;  // next word
  uint64_t bb;
  int nb;
  __device__ __forceinline__ void seek(const uint8_t* base, uint64_t byte) {
    w = reinterpret_cast<const uint32_t*>(base);
    wi = byte >> 2;
    const int skip = (int)(byte & 3) * 8;
    bb = __ldg(w + wi++) >> skip;
    nb = 32 - skip;
    refill();
  }
  // at least 32 bits buffered afterwards
  __device__ __forceinline__ void refill() {
    if (nb <= 32) {
      bb |= (uint64_t)__ldg(w + wi++) << nb;
      nb += 32;
    }
  }
  __device__ __forceinline__ uint32_t take(int n) {
    const uint32_t v = (uint32_t)(bb & ((1ull << n) - 1));
    bb >>= n;
    nb -= n;
    return v;
  }
  __device__ __forceinline__ uint64_t bit_pos() const { return wi * 32 - (uint64_t)nb; }  // from the buffer start
};

// Canonical Huffman tables of lens[0..n) (zlib's inflate_table rules): count, symbols in canonical order, the fast
// table. Returns false for a set zlib refuses: over-subscribed; incomplete, except a single code of length 1 for
// literal / length and distance codes; for distance codes an empty set is accepted (any use of it is an error).
// The code-length code is refused when empty too (zlib then reads only zero lengths and fails on the missing
// end-of-block code).
__device__ __forceinline__ bool build(const uint8_t* lens, int n, uint16_t* count, uint16_t* next, uint16_t* sym, uint16_t* fast,
                      int fast_bits, bool cl_code, int lane) {
  if (lane < 16) count[lane] = 0;
  __syncwarp();
  for (int b = 0; b < n; b += 32) {
    const int s = b + lane;
    const int L = s < n ? lens[s] : 0;
    const unsigned m = __match_any_sync(FULL, L);
    if (L && lane == __ffs(m) - 1) count[L] += __popc(m);
    __syncwarp();
  }
  int left = 1, max = 0;
  for (int L = 1; L <= 15; ++L) {
    left = (left << 1) - count[L];
    if (left < 0) return false;
    if (count[L]) max = L;
  }
  if (max == 0 ? cl_code : (left > 0 && (cl_code || max != 1))) return false;
  if (lane == 0) {
    int o = 0;
    for (int L = 1; L <= 15; ++L) {
      next[L] = (uint16_t)o;
      o += count[L];
    }
  }
  __syncwarp();
  for (int b = 0; b < n; b += 32) {
    const int s = b + lane;
    const int L = s < n ? lens[s] : 0;
    const unsigned m = __match_any_sync(FULL, L);
    if (L) sym[next[L] + __popc(m & ((1u << lane) - 1))] = (uint16_t)s;
    __syncwarp();
    if (L && lane == __ffs(m) - 1) next[L] += __popc(m);
    __syncwarp();
  }
  for (int e = lane; e < (1 << fast_bits); e += 32) {
    int code = 0, first = 0, index = 0;
    uint16_t v = 0;
    for (int L = 1; L <= fast_bits; ++L) {
      code |= (e >> (L - 1)) & 1;
      const int c = count[L];
      if (code - c < first) {
        v = (uint16_t)((L << 9) | sym[index + code - first]);
        break;
      }
      index += c;
      first = (first + c) << 1;
      code <<= 1;
    }
    fast[e] = v;
  }
  __syncwarp();
  return true;
}

// the next symbol, or -1 for a bit pattern no code has; needs 15 bits buffered
__device__ __forceinline__ int decode(Bits& br, const uint16_t* fast, int fast_bits, const uint16_t* count,
                                      const uint16_t* sym) {
  const uint16_t v = fast[br.bb & ((1u << fast_bits) - 1)];
  if (v) {
    br.take(v >> 9);
    return v & 511;
  }
  int code = 0, first = 0, index = 0;
  for (int L = 1; L <= 15; ++L) {
    code |= (int)(br.bb >> (L - 1)) & 1;
    const int c = count[L];
    if (code - c < first) {
      br.take(L);
      return sym[index + code - first];
    }
    index += c;
    first = (first + c) << 1;
    code <<= 1;
  }
  return -1;
}

// a * b modulo the CRC-32 polynomial, bit-reflected (bit 31 is x^0)
__device__ __forceinline__ uint32_t gf2_mul(uint32_t a, uint32_t b) {
  uint32_t p = 0;
  for (int i = 0; i < 32; ++i) {
    if (a & (0x80000000u >> i)) p ^= b;
    b = (b & 1) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
  }
  return p;
}

// x^(8n): the effect on a CRC register of n zero bytes
__device__ __forceinline__ uint32_t x_pow_8n(uint32_t n) {
  uint32_t p = 0x80000000u, sq = 0x00800000u;
  for (; n; n >>= 1) {
    if (n & 1) p = gf2_mul(p, sq);
    sq = gf2_mul(sq, sq);
  }
  return p;
}

__device__ __forceinline__ int32_t inflate_member(const uint8_t* __restrict__ in, const InflateMember& m, uint8_t* out, WarpTables& t,
                                  int lane) {
  const uint64_t start_bit = m.in_off * 8, end_bit = (m.in_off + m.in_len) * 8;
  Bits br;
  br.seek(in, m.in_off);
  uint32_t pos = 0;
  for (bool last = false; !last;) {
    if (br.bit_pos() - start_bit + 3 > end_bit - start_bit) return ST_INPUT;
    last = br.take(1);
    const uint32_t type = br.take(2);
    if (type == 0) {
      br.take(br.nb & 7);  // to the byte boundary (nb counts whole bytes from a word edge plus the partial byte)
      br.refill();
      const uint32_t len = br.take(16), nlen = br.take(16);
      if (len != (~nlen & 0xffffu)) return ST_STORED_LEN;
      const uint64_t byte = br.bit_pos() / 8;
      if ((byte + len) * 8 > end_bit) return ST_INPUT;
      if (pos + len > m.isize) return ST_OUTPUT;
      for (uint32_t i = lane; i < len; i += 32) out[pos + i] = in[byte + i];
      pos += len;
      br.seek(in, byte + len);
      continue;
    }
    if (type == 3) return ST_BLOCK_TYPE;
    int nlit, ndist;
    if (type == 1) {
      nlit = 288;
      ndist = 32;
      for (int s = lane; s < 320; s += 32) t.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
      __syncwarp();
    } else {
      br.refill();
      nlit = (int)br.take(5) + 257;
      ndist = (int)br.take(5) + 1;
      const int ncl = (int)br.take(4) + 4;
      if (nlit > 286 || ndist > 30) return ST_COUNTS;
      br.refill();
      if (lane < 19) t.lens[lane] = 0;
      __syncwarp();
      for (int i = 0; i < ncl; ++i) {
        const uint32_t v = br.take(3);
        if (lane == 0) t.lens[kClOrder[i]] = (uint8_t)v;
        if (i == 9) br.refill();
      }
      __syncwarp();
      // the code-length code lives in the distance arrays until the lengths are read; the lengths then overwrite
      // lens[] from 0 (lane 0 writes single lengths, the warp writes repeats; every lane tracks have / prev)
      if (!build(t.lens, 19, t.dist_count, t.next, t.dist_sym, t.dist_fast, DIST_FAST, true, lane)) return ST_CODES;
      int have = 0, prev = 0;
      while (have < nlit + ndist) {
        if (br.bit_pos() > end_bit + 64) return ST_INPUT;
        br.refill();
        const int s = decode(br, t.dist_fast, DIST_FAST, t.dist_count, t.dist_sym);
        if (s < 0) return ST_CODES;
        if (s < 16) {
          __syncwarp();
          if (lane == 0) t.lens[have] = (uint8_t)s;
          prev = s;
          ++have;
          continue;
        }
        int rep, val;
        if (s == 16) {
          if (have == 0) return ST_REPEAT;
          rep = 3 + (int)br.take(2);
          val = prev;
        } else if (s == 17) {
          rep = 3 + (int)br.take(3);
          val = 0;
        } else {
          rep = 11 + (int)br.take(7);
          val = 0;
        }
        if (have + rep > nlit + ndist) return ST_REPEAT;
        __syncwarp();
        if (lane < rep) t.lens[have + lane] = (uint8_t)val;
        if (lane + 32 < rep) t.lens[have + lane + 32] = (uint8_t)val;
        if (lane + 64 < rep) t.lens[have + lane + 64] = (uint8_t)val;
        if (lane + 96 < rep) t.lens[have + lane + 96] = (uint8_t)val;
        if (lane + 128 < rep) t.lens[have + lane + 128] = (uint8_t)val;
        have += rep;
        prev = val;
      }
      __syncwarp();
      if (t.lens[256] == 0) return ST_NO_EOB;
    }
    if (!build(t.lens, nlit, t.lit_count, t.next, t.lit_sym, t.lit_fast, LIT_FAST, false, lane)) return ST_CODES;
    if (!build(t.lens + nlit, ndist, t.dist_count, t.next, t.dist_sym, t.dist_fast, DIST_FAST, false, lane))
      return ST_CODES;
    for (;;) {
      if (br.bit_pos() > end_bit + 64) return ST_INPUT;
      br.refill();
      const int s = decode(br, t.lit_fast, LIT_FAST, t.lit_count, t.lit_sym);
      if (s < 0) return ST_SYMBOL;
      if (s < 256) {
        if (pos >= m.isize) return ST_OUTPUT;
        if (lane == 0) out[pos] = (uint8_t)s;
        ++pos;
        continue;
      }
      if (s == 256) break;
      if (s >= 286) return ST_SYMBOL;
      const uint32_t len = kLenBase[s - 257] + br.take(kLenExtra[s - 257]);
      br.refill();
      const int d = decode(br, t.dist_fast, DIST_FAST, t.dist_count, t.dist_sym);
      if (d < 0 || d >= 30) return ST_SYMBOL;
      const uint32_t dist = kDistBase[d] + br.take(kDistExtra[d]);
      if (dist > pos) return ST_DISTANCE;
      if (pos + len > m.isize) return ST_OUTPUT;
      __syncwarp();  // the bytes this copy reads (literals of lane 0, earlier copies of every lane) are written
      for (uint32_t i = lane; i < len; i += 32) out[pos + i] = out[pos - dist + (i < dist ? i : i % dist)];
      pos += len;
    }
  }
  // the deflate stream ends in the byte before the trailer
  if ((br.bit_pos() - start_bit + 7) / 8 != m.in_len) return ST_END;
  if (pos != m.isize) return ST_ISIZE;
  return ST_OK;
}

__global__ void __launch_bounds__(WARPS * 32, 4) k_inflate(const uint8_t* __restrict__ in, const InflateMember* members,
                                                        int n, uint8_t* out, int32_t* status) {
  __shared__ uint32_t crc_tab[256];
  __shared__ WarpTables tables[WARPS];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
    crc_tab[i] = c;
  }
  __syncthreads();
  const int warp = threadIdx.x / 32, lane = threadIdx.x & 31;
  const int mi = blockIdx.x * WARPS + warp;
  if (mi >= n) return;
  const InflateMember m = members[mi];
  uint8_t* o = out + m.out_off;
  int32_t st = inflate_member(in, m, o, tables[warp], lane);
  if (st == ST_OK) {
    __syncwarp();
    // raw CRC (register starting at 0) of this lane's slice, shifted past the bytes after it; then the standard CRC
    const uint32_t seg = (m.isize + 31) / 32, b = min(m.isize, lane * seg), e = min(m.isize, b + seg);
    uint32_t r = 0;
    for (uint32_t i = b; i < e; ++i) r = crc_tab[(r ^ o[i]) & 0xff] ^ (r >> 8);
    r = gf2_mul(r, x_pow_8n(m.isize - e));
    for (int k = 16; k; k >>= 1) r ^= __shfl_xor_sync(FULL, r, k);
    const uint32_t crc = r ^ gf2_mul(0xffffffffu, x_pow_8n(m.isize)) ^ 0xffffffffu;
    if (crc != m.crc) st = ST_CRC;
  }
  if (lane == 0) status[mi] = st;
}

}  // namespace

cudaError_t launch_inflate(const uint8_t* d_in, const InflateMember* d_members, int n, uint8_t* d_out,
                           int32_t* d_status, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  k_inflate<<<(n + WARPS - 1) / WARPS, WARPS * 32, 0, st>>>(d_in, d_members, n, d_out, d_status);
  return cudaGetLastError();
}

}  // namespace nb
