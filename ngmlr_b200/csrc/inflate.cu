// ngmlr_b200/csrc/inflate.cu -- BGZF members inflated on the device (the stream layer of stream.cpp launches it).
//
// One warp per member. Every lane runs the same bit reader and Huffman decode (shared-memory table reads broadcast),
// so control flow stays uniform; the warp splits what is parallel: table construction (ballots / match_any over 32
// symbols at a time), match and stored-block copies (one byte per lane), and the member's CRC32 (a slice per lane,
// combined with GF(2) shifts). The output goes straight to its offset in the round's output buffer.
//
// The decoder core (bit reader, Huffman tables, block headers, CRC arithmetic) is inflate_core.cuh, shared with the
// plain gzip kernels of gzip_inflate.cu.
//
// A member is accepted only when zlib's inflate would accept it with the same output: every case zlib rejects
// (block type 3, stored LEN / NLEN mismatch, HLIT > 286 or HDIST > 30, over-subscribed codes, incomplete codes other
// than a single code of length 1, a bad repeat code, no end-of-block code, literal / length symbols 286 / 287,
// distance symbols 30 / 31, a distance before the member's first byte) sets a nonzero status, as does a deflate
// stream that does not end exactly at the trailer, an output length other than ISIZE or a CRC32 other than the
// trailer's. The host then hands the member to zlib.
#include <cstdint>

#include "inflate.h"
#include "inflate_core.cuh"

namespace nb {

namespace {

constexpr int WARPS = 4;  // members per block

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
      fixed_lengths(t, lane);
    } else {
      const int32_t st = dynamic_lengths(br, t, end_bit, nlit, ndist, lane);
      if (st != ST_OK) return st;
    }
    if (!build_codes(t, nlit, ndist, lane)) return ST_CODES;
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
