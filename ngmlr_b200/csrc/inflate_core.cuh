// ngmlr_b200/csrc/inflate_core.cuh -- the deflate decoder core shared by the BGZF member kernel (inflate.cu) and
// the plain gzip kernels (gzip_inflate.cu): status codes, length / distance tables, the bit reader, zlib's canonical
// Huffman table rules, symbol decode, a dynamic block header and the GF(2) arithmetic that combines CRC32s.
//
// Every function is warp-uniform: the lanes hold the same bit reader state and take the same branches, and the warp
// splits table construction.
#pragma once
#include <cstdint>

#include "inflate.h"  // the status codes

namespace nb {
namespace {

using namespace inflate_status;

constexpr int LIT_FAST = 10;   // index bits of the literal / length lookup table
constexpr int DIST_FAST = 8;   // ... of the distance table (and of the code-length code, which it holds first)
constexpr unsigned FULL = 0xffffffffu;


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

// A dynamic block's code lengths, after its 3 header bits: HLIT / HDIST / HCLEN, the code-length code, the lengths
// into t.lens (literal / length then distance), and the end-of-block code. ST_OK or the status zlib's rule gives.
// end_bit bounds the reader (ST_INPUT once it is more than 64 bits past it).
__device__ __forceinline__ int32_t dynamic_lengths(Bits& br, WarpTables& t, uint64_t end_bit, int& nlit, int& ndist,
                                                   int lane) {
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
  return ST_OK;
}

// the fixed code's lengths into t.lens (nlit = 288, ndist = 32)
__device__ __forceinline__ void fixed_lengths(WarpTables& t, int lane) {
  for (int s = lane; s < 320; s += 32) t.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
  __syncwarp();
}

// the literal / length and distance tables of t.lens
__device__ __forceinline__ bool build_codes(WarpTables& t, int nlit, int ndist, int lane) {
  if (!build(t.lens, nlit, t.lit_count, t.next, t.lit_sym, t.lit_fast, LIT_FAST, false, lane)) return false;
  return build(t.lens + nlit, ndist, t.dist_count, t.next, t.dist_sym, t.dist_fast, DIST_FAST, false, lane);
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

}  // namespace
}  // namespace nb
