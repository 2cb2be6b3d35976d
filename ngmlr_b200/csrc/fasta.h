// ngmlr_b200/csrc/fasta.h -- the reference FASTA/FASTQ reader of ngmlr_b200_load_reference.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

namespace nb {

struct FastaRecord {
  std::string name;  // up to the first whitespace of the header line, uncut
  uint64_t offset;   // of its sequence in FastaText::text
  uint64_t len;
};

// Every record of a FASTA / FASTQ file (plain or gzip), sequences back to back in one host buffer (page-locked when
// asked for, so that the contig copies to the device run at full speed).
struct FastaText {
  std::vector<FastaRecord> recs;
  char* text = nullptr;
  uint64_t size = 0, cap = 0;
  bool pinned = false;
  // binRefSize of _SequenceProvider::Init: ((getSize() / 2) | 1) + 1 with getSize() = 1000 + sum((len | 1) + 1 + 1000)
  // over every record, kept or not (src/SequenceProvider.cpp:274-290, 318)
  uint64_t alloc_bytes() const;
  void release_text();  // the records stay
  FastaText() = default;
  FastaText(const FastaText&) = delete;
  FastaText& operator=(const FastaText&) = delete;
  ~FastaText();
};

// What a stream's inflate did so far.
struct StreamCounters {
  int64_t compressed_bytes = 0;  // bytes read from the file
  int64_t device_members = 0;    // BGZF members inflated on the device
  int64_t host_bytes = 0;        // bytes inflated by the host continuation (zlib, from a member the device refused)
  float inflate_ms = 0;          // device inflate kernel time (CUDA events)
  // plain gzip on the device: bytes it returned, chunks placed, chunks decoded again after a chain mismatch (a false
  // block start), kernel milliseconds
  int64_t gzip_bytes = 0, gzip_chunks = 0, gzip_redecoded = 0;
  float gzip_ms = 0;
};

// Reads the records ngmlr's `while (kseq_read(seq) >= 0)` loop over gzopen(path) sees (see fasta.cpp). Stops with an
// error once the concatenated genome of the records of more than 10 bases would exceed max_concat_len positions.
// BGZF input is inflated on `device` / `stream` when device >= 0 (on the host without one). counters, when not NULL,
// receive the stream's counters. Returns 0, or < 0 with a message in err.
int read_fasta(const char* path, bool pinned, uint64_t max_concat_len, FastaText& out, std::string& err,
               int device = -1, cudaStream_t stream = nullptr, StreamCounters* counters = nullptr);

// The byte stream ngmlr's readers see through gzopen / gzread: a plain file as it is, a gzip file inflated.
// open_stream returns NULL when the file cannot be opened. read_stream reads up to n bytes (fewer only at the end of
// the stream) and returns the count, or -1 on a read error or a corrupt gzip stream. stream_truncated tells, once
// read_stream has returned 0, whether the gzip stream stopped before its end (zlib's gzread reports that as an end).
//
// A file whose first member header is BGZF's (1f 8b 08, FLG 0x04, a BC extra subfield of length 2) is read with
// read() and walked member by member instead: a read_stream call inflates the whole members that cover it in one
// round (on the bound device, else with zlib's raw inflate on the host) and keeps the bytes past the request. From
// the first member that round cannot vouch for (see fasta.cpp), a host continuation that reproduces gzread takes
// over for the rest of the stream. force_gzread skips the sniff (a reference for tests).
struct StreamFile;
StreamFile* open_stream(const char* path, bool force_gzread = false);
void close_stream(StreamFile* f);
int64_t read_stream(StreamFile* f, void* buf, size_t n);
bool stream_truncated(StreamFile* f);
//
// A gzip file whose first member is not BGZF goes to gzread, unless it is a regular file and a device is bound before
// the first read_stream:
// then it is read with read() and inflated on the device in rounds (fasta.cpp, "Plain gzip on the device"), and zlib
// continues from the first member the device cannot vouch for, with gzread's bytes, -1 and truncation flag. A stream
// read in rounds too small for the device (min_round and requests below 256 MiB), or whose first round inflates at a
// ratio where gzread is faster (incompressible data, long runs), goes to zlib whole.
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

// Plain gzip rounds (gzip_inflate.cu; fasta.cpp drives them). Bit offsets count from the round's compressed span.
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

// Length of the concatenated genome _SequenceProvider::Init builds from records of these lengths (1000-N spacers
// before, between and after the contigs of more than 10 bases, each contig starting on a byte boundary).
uint64_t concat_len_of(const std::vector<uint64_t>& lens);

}  // namespace nb
