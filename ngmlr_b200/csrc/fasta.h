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
// BGZF rounds run on this device and stream from now on, each inflating at least min_round output bytes (bytes
// past the request are kept). Returns false with the message in stream_error when buffers cannot be set up.
bool bind_stream_device(StreamFile* f, int device, cudaStream_t stream, int64_t min_round);
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

// Length of the concatenated genome _SequenceProvider::Init builds from records of these lengths (1000-N spacers
// before, between and after the contigs of more than 10 bases, each contig starting on a byte boundary).
uint64_t concat_len_of(const std::vector<uint64_t>& lens);

}  // namespace nb
