// ngmlr_b200/csrc/inflate.h -- the launch interfaces of the inflate kernels (inflate.cu: BGZF members;
// gzip_inflate.cu: plain gzip rounds), which the stream layer (stream.cpp) drives.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace nb {

// One member of a device inflate round: its deflate data [in_off, in_off + in_len) in the round's compressed
// buffer (which has at least 64 readable bytes after its end), its output at out_off, ISIZE and CRC32 from the
// trailer.
struct InflateMember {
  uint64_t in_off, out_off;
  uint32_t in_len, isize, crc, pad;
};
// status[i] = 0 when member i inflated to exactly what zlib's inflate gives, else nonzero (inflate.cu)
cudaError_t launch_inflate(const uint8_t* d_in, const InflateMember* d_members, int n, uint8_t* d_out,
                           int32_t* d_status, cudaStream_t st);

// Status of a member (inflate.cu) or a chunk (gzip_inflate.cu): 0, or the case zlib rejects or the decode stopped at.
namespace inflate_status {
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
}  // namespace inflate_status

// Plain gzip rounds (gzip_inflate.cu; stream.cpp drives them). Bit offsets count from the round's compressed span.
constexpr uint64_t GZ_NONE = ~0ull;  // a chunk without a plausible boundary
constexpr int GZ_EVENTS = 32;        // member headers / trailers one chunk records at most
// chunk status beyond the decoder's: the stream ends at a member boundary; the span ends there (more to read); the
// bytes at a member boundary are no member header zlib would read; output past the chunk's cap
enum : int32_t { GZ_END = 20, GZ_SPAN = 21, GZ_MEMBER = 22, GZ_OVER = 23 };
struct GzChunk {
  uint64_t start, stop;    // decode from start to the first boundary at or past stop
  uint64_t end, out_off;   // where it stopped; pass B: its symbols' offset in the round's 16-bit output
  uint32_t out_len, reach; // symbols; farthest reference before its own output (before a member starts in it)
  uint32_t n_ev;
  int32_t status;
  uint8_t start_member, end_member, pad[6];  // start / end is a member header (else a block header)
};
struct GzEvent {
  uint64_t bit;                   // kind 0: the member header's offset; kind 1: the offset after the trailer
  uint32_t out, crc, isize, kind;  // output offset in the chunk; kind 1: the trailer's CRC32 and ISIZE
};
// first plausible boundary of chunks 1 .. n_chunks - 1 into their start / start_member
cudaError_t launch_gz_find(const uint8_t* d_in, uint64_t span_bytes, uint32_t chunk_bytes, int n_chunks,
                           GzChunk* d_chunks, cudaStream_t st);
// pass A (write = false: counts, records end / events) or pass B (write: symbols at d_out + out_off)
cudaError_t launch_gz_decode(bool write, const uint8_t* d_in, uint64_t span_bytes, bool final_span, GzChunk* d_chunks,
                             GzEvent* d_events, int n, uint16_t* d_out, uint32_t soft_cap, uint32_t hard_cap,
                             cudaStream_t st);
// markers resolved, bytes to d_out8, CRC32 of each piece between member ends (GZ_EVENTS + 1 per chunk)
cudaError_t launch_gz_resolve(const GzChunk* d_chunks, const GzEvent* d_events, int n, uint16_t* d_out, uint8_t* d_out8,
                              uint32_t* d_piece_crc, cudaStream_t st);

}  // namespace nb
