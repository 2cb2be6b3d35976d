// ngmlr_b200/csrc/gzip_inflate.cu -- plain gzip streams inflated on the device in rounds (the stream layer of
// stream.cpp drives them; the decoder core is inflate_core.cuh, shared with the BGZF kernel).
//
// A gzip member is one deflate stream whose block boundaries are recorded nowhere, and a back-reference reaches up
// to 32 KiB into output that precedes it. A round covers a span of compressed bytes that starts at a boundary known
// to lie on the true decode chain; the span is cut into chunks of fixed compressed size and:
//   1. k_gz_find: one warp per chunk finds the first bit offset at or after the chunk's nominal start that is a
//      plausible boundary -- a dynamic block header accepted by exactly the rules the decoder applies, a stored block
//      header (zero padding, LEN == ~NLEN), or a gzip member header at a byte offset. Lanes test 32 offsets at a time
//      cheaply; the warp checks each survivor fully.
//   2. k_gz_decode<false> (pass A) decodes each chunk from its start up to the first boundary at or past its stop
//      (the next chunk's start), counting output, recording member headers / trailers and how far back the chunk's
//      references reach before its own output. The host confirms the chain (stream.cpp) and places the chunks.
//   3. k_gz_decode<true> (pass B) writes 16-bit symbols: a back-reference before the chunk's own output becomes the
//      marker 256 + index into the 32 KiB window before the chunk.
//   4. k_gz_window: one CTA walks the placed chunks in order and resolves the markers of each chunk's last 32 KiB.
//   5. k_gz_final: one CTA per chunk resolves every other marker, narrows to bytes and computes the CRC32 of each
//      piece of the chunk between member ends (the host combines them per member and checks each trailer).
// Decoding crosses member ends: after a final block the trailer is read, and a member header that follows starts a
// new member (its references may not reach before its first byte).
#include <cstdint>

#include "inflate.h"
#include "inflate_core.cuh"

namespace nb {

namespace {

constexpr int FIND_WARPS = 4;
constexpr int DEC_WARPS = 4;

// Bits from an arbitrary bit offset (the reader seeks bytes).
__device__ __forceinline__ void seek_bit(Bits& br, const uint8_t* in, uint64_t bit) {
  br.seek(in, bit >> 3);
  br.take((int)(bit & 7));
  br.refill();
}

__device__ __forceinline__ uint32_t le32_dev(const uint8_t* p) {
  return p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24;
}

__device__ __forceinline__ uint32_t crc32_bytes(const uint8_t* p, uint32_t n) {
  uint32_t c = 0xffffffffu;
  for (uint32_t i = 0; i < n; ++i) {
    c ^= p[i];
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
  }
  return c ^ 0xffffffffu;
}

// A gzip member header at byte b as zlib's inflate reads it (1f 8b, method 8, no reserved flag, FEXTRA / FNAME /
// FCOMMENT skipped, FHCRC checked). Returns the byte after it, 0 when the bytes are no valid header, or -1 when the
// header runs past n bytes.
__device__ int64_t member_header(const uint8_t* in, uint64_t b, uint64_t n) {
  if (b + 10 > n) return b + 2 <= n && (in[b] != 0x1f || in[b + 1] != 0x8b) ? 0 : -1;
  if (in[b] != 0x1f || in[b + 1] != 0x8b || in[b + 2] != 8) return 0;
  const uint8_t flg = in[b + 3];
  if (flg & 0xe0) return 0;
  uint64_t q = b + 10;
  if (flg & 4) {
    if (q + 2 > n) return -1;
    q += 2 + (in[q] | in[q + 1] << 8);
    if (q > n) return -1;
  }
  for (int f = 8; f <= 16; f <<= 1) {
    if (!(flg & f)) continue;
    while (q < n && in[q]) ++q;
    if (q >= n) return -1;
    ++q;
  }
  if (flg & 2) {
    if (q + 2 > n) return -1;
    if ((crc32_bytes(in + b, (uint32_t)(q - b)) & 0xffff) != (uint32_t)(in[q] | in[q + 1] << 8)) return 0;
    q += 2;
  }
  return (int64_t)q;
}

// cheap per-lane test of bit offset p (p + 200 bits are readable)
__device__ __forceinline__ bool plausible(const uint8_t* in, uint64_t p, uint64_t span_bytes, bool& member) {
  member = false;
  if ((p & 7) == 0) {
    const uint64_t b = p >> 3;
    if (b + 4 <= span_bytes && in[b] == 0x1f && in[b + 1] == 0x8b && in[b + 2] == 8 && !(in[b + 3] & 0xe0)) {
      member = true;
      return true;
    }
  }
  Bits br;
  seek_bit(br, in, p);
  br.take(1);
  const uint32_t type = br.take(2);
  if (type == 0) {
    const int pad = (int)((8 - ((p + 3) & 7)) & 7);
    if (br.take(pad)) return false;
    br.refill();
    const uint32_t len = br.take(16), nlen = br.take(16);
    return len == (~nlen & 0xffffu);
  }
  if (type != 2) return false;
  const uint32_t hlit = br.take(5), hdist = br.take(5), ncl = br.take(4) + 4;
  if (hlit > 29 || hdist > 29) return false;
  br.refill();
  uint32_t kraft = 0;  // the code-length code must be complete: sum of 2^(7 - L) over its lengths == 128
  for (uint32_t i = 0; i < ncl; ++i) {
    const uint32_t v = br.take(3);
    if (v) kraft += 128u >> v;
    if (i == 9) br.refill();
  }
  return kraft == 128;
}

__global__ void __launch_bounds__(FIND_WARPS * 32) k_gz_find(const uint8_t* __restrict__ in, uint64_t span_bytes,
                                                            uint32_t chunk_bytes, int n_chunks, GzChunk* chunks) {
  __shared__ WarpTables tables[FIND_WARPS];
  const int warp = threadIdx.x / 32, lane = threadIdx.x & 31;
  const int j = 1 + blockIdx.x * FIND_WARPS + warp;  // chunk 0 starts at the round's confirmed boundary
  if (j >= n_chunks) return;
  WarpTables& t = tables[warp];
  const uint64_t lo = (uint64_t)j * chunk_bytes * 8, hi = min((uint64_t)(j + 1) * chunk_bytes, span_bytes) * 8;
  uint64_t found = GZ_NONE;
  bool found_member = false;
  for (uint64_t base = lo; base < hi && found == GZ_NONE; base += 32) {
    const uint64_t p = base + lane;
    bool member = false;
    const bool ok = p < hi && plausible(in, p, span_bytes, member);
    unsigned m = __ballot_sync(FULL, ok);
    const unsigned mm = __ballot_sync(FULL, member);
    while (m) {
      const int l = __ffs(m) - 1;
      m &= m - 1;
      const uint64_t q = base + l;
      bool good = (mm >> l) & 1;
      if (!good) {
        Bits br;
        seek_bit(br, in, q);
        br.take(1);
        if (br.take(2) == 0) {
          good = true;  // the stored test is complete
        } else {
          int nlit, ndist;
          good = dynamic_lengths(br, t, span_bytes * 8, nlit, ndist, lane) == ST_OK && build_codes(t, nlit, ndist, lane);
        }
      }
      if (good) {
        found = q;
        found_member = (mm >> l) & 1;
        break;
      }
    }
  }
  if (lane == 0) {
    chunks[j].start = found;
    chunks[j].start_member = found_member;
  }
}

// One chunk: from c.start (a member header when c.start_member) to the first boundary at or past c.stop, or past
// soft_cap output symbols, or with GZ_EVENTS - 2 events recorded. WRITE: the symbols go to out + c.out_off.
template <bool WRITE>
__device__ void gz_chunk(const uint8_t* __restrict__ in, uint64_t span_bytes, bool final_span, GzChunk& c, GzEvent* ev,
                         uint16_t* out, uint32_t soft_cap, uint32_t hard_cap, WarpTables& t, int lane) {
  const uint64_t span_bits = span_bytes * 8;
  uint64_t p = c.start;
  bool member = c.start_member;
  uint32_t pos = 0, reach = 0, mstart = 0, nev = 0;
  bool started = false;  // a member started in this chunk (at output mstart)
  int32_t st = ST_OK;
  uint16_t* o = WRITE ? out + c.out_off : nullptr;
  for (;;) {
    // at a boundary
    if (p != c.start && (p >= c.stop || pos >= soft_cap || nev + 2 > GZ_EVENTS)) break;
    if (member) {
      const uint64_t b = p >> 3;
      if (b == span_bytes) {
        st = final_span ? GZ_END : GZ_SPAN;
        break;
      }
      const int64_t q = member_header(in, b, span_bytes);
      if (q <= 0) {
        st = q < 0 && !final_span ? GZ_SPAN : GZ_MEMBER;
        break;
      }
      if (lane == 0) ev[nev] = GzEvent{p, pos, 0, 0, 0};
      ++nev;
      started = true;
      mstart = pos;
      p = (uint64_t)q * 8;
      member = false;
      continue;
    }
    Bits br;
    seek_bit(br, in, p);
    const bool last = br.take(1);
    const uint32_t type = br.take(2);
    if (type == 0) {
      br.take(br.nb & 7);
      br.refill();
      const uint32_t len = br.take(16), nlen = br.take(16);
      if (len != (~nlen & 0xffffu)) {
        st = ST_STORED_LEN;
        break;
      }
      const uint64_t data = br.bit_pos() / 8;
      if ((data + len) * 8 > span_bits) {
        st = ST_INPUT;
        break;
      }
      if (pos + len > hard_cap) {
        st = GZ_OVER;
        break;
      }
      if (WRITE)
        for (uint32_t i = lane; i < len; i += 32) o[pos + i] = in[data + i];
      pos += len;
      p = (data + len) * 8;
    } else if (type == 3) {
      st = ST_BLOCK_TYPE;
      break;
    } else {
      int nlit, ndist;
      if (type == 1) {
        nlit = 288;
        ndist = 32;
        fixed_lengths(t, lane);
      } else if ((st = dynamic_lengths(br, t, span_bits, nlit, ndist, lane)) != ST_OK) {
        break;
      }
      if (!build_codes(t, nlit, ndist, lane)) {
        st = ST_CODES;
        break;
      }
      for (;;) {
        if (br.bit_pos() > span_bits) {
          st = ST_INPUT;
          break;
        }
        br.refill();
        const int s = decode(br, t.lit_fast, LIT_FAST, t.lit_count, t.lit_sym);
        if (s < 0) {
          st = ST_SYMBOL;
          break;
        }
        if (s < 256) {
          if (pos >= hard_cap) {
            st = GZ_OVER;
            break;
          }
          if (WRITE && lane == 0) o[pos] = (uint16_t)s;
          ++pos;
          continue;
        }
        if (s == 256) break;
        if (s >= 286) {
          st = ST_SYMBOL;
          break;
        }
        const uint32_t len = kLenBase[s - 257] + br.take(kLenExtra[s - 257]);
        br.refill();
        const int d = decode(br, t.dist_fast, DIST_FAST, t.dist_count, t.dist_sym);
        if (d < 0 || d >= 30) {
          st = ST_SYMBOL;
          break;
        }
        const uint32_t dist = kDistBase[d] + br.take(kDistExtra[d]);
        if (started) {
          if (dist > pos - mstart) {
            st = ST_DISTANCE;
            break;
          }
        } else if (dist > pos) {
          reach = max(reach, dist - pos);
        }
        if (pos + len > hard_cap) {
          st = GZ_OVER;
          break;
        }
        if (WRITE) {
          __syncwarp();
          for (uint32_t i = lane; i < len; i += 32) {
            const int64_t src = (int64_t)pos - dist + (i < dist ? i : i % dist);
            o[pos + i] = src >= 0 ? o[src] : (uint16_t)(256 + 32768 + src);
          }
        }
        pos += len;
      }
      if (st != ST_OK) break;
      if (br.bit_pos() > span_bits) {
        st = ST_INPUT;
        break;
      }
      p = br.bit_pos();
    }
    if (last) {  // the trailer: CRC32, ISIZE at the next byte
      const uint64_t b = (p + 7) >> 3;
      if (b + 8 > span_bytes) {
        st = ST_INPUT;
        break;
      }
      if (lane == 0)
        ev[nev] = GzEvent{(b + 8) * 8, pos, le32_dev(in + b), le32_dev(in + b + 4), 1};
      ++nev;
      started = false;
      p = (b + 8) * 8;
      member = true;
    }
    if (WRITE) __syncwarp();
  }
  if (lane == 0) {
    c.end = p;
    c.end_member = member;
    c.out_len = pos;
    c.status = st;
    c.reach = reach;
    c.n_ev = nev;
  }
}

template <bool WRITE>
__global__ void __launch_bounds__(DEC_WARPS * 32) k_gz_decode(const uint8_t* __restrict__ in, uint64_t span_bytes,
                                                             int final_span, GzChunk* chunks, GzEvent* events, int n,
                                                             uint16_t* out, uint32_t soft_cap, uint32_t hard_cap) {
  __shared__ WarpTables tables[DEC_WARPS];
  const int warp = threadIdx.x / 32, lane = threadIdx.x & 31;
  const int j = blockIdx.x * DEC_WARPS + warp;
  if (j >= n || chunks[j].start == GZ_NONE) return;
  GzChunk c = chunks[j];
  gz_chunk<WRITE>(in, span_bytes, final_span != 0, c, events + (size_t)j * GZ_EVENTS, out, soft_cap, hard_cap,
                  tables[warp], lane);
  if (lane == 0 && !WRITE) chunks[j] = c;
}

// chunks in order: the last 32 KiB of each resolved against the 32 KiB before it (already resolved)
__global__ void __launch_bounds__(1024) k_gz_window(const GzChunk* chunks, int n, uint16_t* out) {
  for (int k = 0; k < n; ++k) {
    const uint64_t g = chunks[k].out_off, e = g + chunks[k].out_len;
    for (uint64_t i = max(g, e > 32768 ? e - 32768 : 0) + threadIdx.x; i < e; i += blockDim.x) {
      const uint16_t v = out[i];
      if (v >= 256) out[i] = out[g - 32768 + (v - 256)];
    }
    __syncthreads();
  }
}

// one CTA per chunk: bytes to out8 (whose offset 0 is out16's 32768) and the CRC32 of each piece between member ends
__global__ void __launch_bounds__(256) k_gz_final(const GzChunk* chunks, const GzEvent* events, const uint16_t* out,
                                                 uint8_t* out8, uint32_t* piece_crc) {
  __shared__ uint32_t crc_tab[256];
  __shared__ uint32_t part[8];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
    crc_tab[i] = c;
  }
  const GzChunk c = chunks[blockIdx.x];
  const uint64_t g = c.out_off;
  uint8_t* o = out8 + (g - 32768);
  for (uint32_t i = threadIdx.x; i < c.out_len; i += blockDim.x) {
    uint16_t v = out[g + i];
    if (v >= 256) v = out[g - 32768 + (v - 256)];
    o[i] = (uint8_t)v;
  }
  __syncthreads();
  const GzEvent* ev = events + (size_t)blockIdx.x * GZ_EVENTS;
  uint32_t pb = 0;
  int piece = 0;
  for (uint32_t k = 0; k <= c.n_ev; ++k) {
    if (k < c.n_ev && ev[k].kind != 1) continue;
    const uint32_t pe = k < c.n_ev ? ev[k].out : c.out_len, len = pe - pb;
    // raw CRC (register starting at 0) of this thread's slice, shifted past the bytes after it
    const uint32_t seg = (len + blockDim.x - 1) / blockDim.x, b = min(len, threadIdx.x * seg), e = min(len, b + seg);
    uint32_t r = 0;
    for (uint32_t i = b; i < e; ++i) r = crc_tab[(r ^ o[pb + i]) & 0xff] ^ (r >> 8);
    if (e > b) r = gf2_mul(r, x_pow_8n(len - e));
    for (int s = 16; s; s >>= 1) r ^= __shfl_xor_sync(FULL, r, s);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x / 32] = r;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t x = 0;
      for (int w = 0; w < (int)(blockDim.x / 32); ++w) x ^= part[w];
      piece_crc[(size_t)blockIdx.x * (GZ_EVENTS + 1) + piece] = x ^ gf2_mul(0xffffffffu, x_pow_8n(len)) ^ 0xffffffffu;
    }
    __syncthreads();
    pb = pe;
    ++piece;
  }
}

}  // namespace

cudaError_t launch_gz_find(const uint8_t* d_in, uint64_t span_bytes, uint32_t chunk_bytes, int n_chunks,
                           GzChunk* d_chunks, cudaStream_t st) {
  if (n_chunks <= 1) return cudaSuccess;
  k_gz_find<<<(n_chunks - 1 + FIND_WARPS - 1) / FIND_WARPS, FIND_WARPS * 32, 0, st>>>(d_in, span_bytes, chunk_bytes,
                                                                                    n_chunks, d_chunks);
  return cudaGetLastError();
}

cudaError_t launch_gz_decode(bool write, const uint8_t* d_in, uint64_t span_bytes, bool final_span, GzChunk* d_chunks,
                             GzEvent* d_events, int n, uint16_t* d_out, uint32_t soft_cap, uint32_t hard_cap,
                             cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  const int grid = (n + DEC_WARPS - 1) / DEC_WARPS;
  if (write)
    k_gz_decode<true><<<grid, DEC_WARPS * 32, 0, st>>>(d_in, span_bytes, final_span, d_chunks, d_events, n, d_out,
                                                       soft_cap, hard_cap);
  else
    k_gz_decode<false><<<grid, DEC_WARPS * 32, 0, st>>>(d_in, span_bytes, final_span, d_chunks, d_events, n, d_out,
                                                        soft_cap, hard_cap);
  return cudaGetLastError();
}

cudaError_t launch_gz_resolve(const GzChunk* d_chunks, const GzEvent* d_events, int n, uint16_t* d_out, uint8_t* d_out8,
                              uint32_t* d_piece_crc, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  k_gz_window<<<1, 1024, 0, st>>>(d_chunks, n, d_out);
  k_gz_final<<<n, 256, 0, st>>>(d_chunks, d_events, d_out, d_out8, d_piece_crc);
  return cudaGetLastError();
}

}  // namespace nb
