// ngmlr_b200/csrc/fasta.h -- the reference FASTA/FASTQ reader of ngmlr_b200_load_reference.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "stream.h"

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

// Reads the records ngmlr's `while (kseq_read(seq) >= 0)` loop over gzopen(path) sees (see fasta.cpp). Stops with an
// error once the concatenated genome of the records of more than 10 bases would exceed max_concat_len positions.
// BGZF input is inflated on `device` / `stream` when device >= 0 (on the host without one). counters, when not NULL,
// receive the stream's counters. Returns 0, or < 0 with a message in err.
int read_fasta(const char* path, bool pinned, uint64_t max_concat_len, FastaText& out, std::string& err,
               int device = -1, cudaStream_t stream = nullptr, StreamCounters* counters = nullptr);

// Length of the concatenated genome _SequenceProvider::Init builds from records of these lengths (1000-N spacers
// before, between and after the contigs of more than 10 bases, each contig starting on a byte boundary).
uint64_t concat_len_of(const std::vector<uint64_t>& lens);

}  // namespace nb
