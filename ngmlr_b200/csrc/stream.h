// ngmlr_b200/csrc/stream.h -- the byte stream ngmlr's readers see through gzopen / gzread, for the read loader
// (read_load.cu) and the reference reader (fasta.cpp).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <string>

namespace nb {

// What a stream's inflate did so far.
struct StreamCounters {
  int64_t compressed_bytes = 0;  // bytes read from the file
  int64_t device_members = 0;    // BGZF members inflated on the device
  int64_t host_bytes = 0;        // bytes returned by the host continuation (zlib, or the file as it is)
  float inflate_ms = 0;          // device inflate kernel time (CUDA events)
  // plain gzip on the device: bytes it returned, chunks placed, chunks decoded again after a chain mismatch (a false
  // block start), kernel milliseconds
  int64_t gzip_bytes = 0, gzip_chunks = 0, gzip_redecoded = 0;
  float gzip_ms = 0;
};

// The byte stream ngmlr's readers see through gzopen / gzread: a plain file as it is, a gzip file inflated.
// open_stream returns NULL when the file cannot be opened. read_stream reads up to n bytes (fewer only at the end of
// the stream) and returns the count, or -1 on a read error or a corrupt gzip stream. stream_truncated tells, once
// read_stream has returned 0, whether the gzip stream stopped before its end (zlib's gzread reports that as an end).
//
// The file is read with read(). One whose first member header is BGZF's (1f 8b 08, FLG 0x04, a BC extra subfield of
// length 2) is walked member by member: a read_stream call inflates the whole members that cover it in one round (on
// the bound device, else with zlib's raw inflate on the host) and keeps the bytes past the request. Any other file
// goes to the host continuation, which reproduces gzread (zlib's gz_read on the same buffer sizes) from the file's
// first byte; so does the stream from the first member a round cannot vouch for (see stream.cpp).
struct StreamFile;
StreamFile* open_stream(const char* path);
void close_stream(StreamFile* f);
int64_t read_stream(StreamFile* f, void* buf, size_t n);
bool stream_truncated(StreamFile* f);
//
// A regular file whose first member is gzip but not BGZF, bound to a device before the first read_stream, is
// inflated on the device in rounds instead (stream.cpp, "Plain gzip on the device"), and zlib continues from the
// first member the device cannot vouch for, with gzread's bytes, -1 and truncation flag. A stream read in rounds too
// small for the device (min_round and requests below 256 MiB), or whose first round inflates at a ratio where gzread
// is faster (incompressible data, long runs), goes to zlib whole.
// BGZF and plain gzip rounds run on this device and stream from now on, each inflating at least min_round output
// bytes (bytes past the request are kept). Returns false with the message in stream_error when buffers cannot be set
// up. NGMLR_B200_DEBUG_GZIP_CHUNK (a test hook) sets the compressed chunk size of plain gzip rounds at binding.
bool bind_stream_device(StreamFile* f, int device, cudaStream_t stream, int64_t min_round);
// compressed bytes per chunk of plain gzip rounds (>= 64; default 32 KiB); a stream given one stays on the device
// path whatever its compression ratio
void set_gzip_chunk(StreamFile* f, int64_t chunk_bytes);
StreamCounters stream_counters(const StreamFile* f);
size_t stream_device_bytes(const StreamFile* f);
// a device failure behind read_stream's -1 (empty for a read error or a corrupt stream)
const std::string& stream_error(const StreamFile* f);

}  // namespace nb
