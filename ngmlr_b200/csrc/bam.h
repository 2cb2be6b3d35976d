// ngmlr_b200/csrc/bam.h -- BAM input of the read loader (read_load.cu): the header and the record chain walked on the
// host over the page-locked chunk, the per-base decode on the device (bam_load.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

namespace nb {

// One whole record of a chunk. Offsets are into the chunk; qual / rev / skip come from the record's first quality byte
// (0xFF: no qualities) and its flag (0x10; 0x100 | 0x800).
struct BamRec {
  int64_t name, seq;
  int32_t l_seq;
  uint8_t l_name, qual, rev, skip;
};

// The host side of a BAM stream: where its header stands, the records of the current chunk, and the counters.
struct BamState {
  int phase = 0;          // header: 0 magic + l_text, 1 n_ref, 2 reference entries, 3 done
  int64_t skip = 0;       // header bytes still to pass over
  int64_t refs_left = 0;
  std::vector<BamRec> recs;
  int64_t header_bytes = 0, records = 0, skipped = 0, reversed = 0, no_quality = 0;
  bool header_done() const { return phase == 3; }
};

// Consumes the header from c[*p, n) as far as it is there (a text or a reference name of any size streams past).
// Returns 1 once it is whole, 0 when it needs the bytes after c[n), -1 with a message in err (base = stream offset
// of c[0]).
int bam_header(BamState& s, const uint8_t* c, int64_t n, int64_t* p, int64_t base, std::string& err);

// Walks the block_size chain from c[p]: every record that is whole in c[p, n) is validated and goes to s.recs (which
// is cleared first); *end = the first byte after the last of them. Returns 0, or -1 with a message in err.
int bam_walk(BamState& s, const uint8_t* c, int64_t n, int64_t p, int64_t base, int64_t* end, std::string& err);

// One read of a batch as the decode kernels see it: its packed sequence in the device chunk, where its qualities go
// in the quality arena (-1: none), its first segment (items[n].seg = segments of the batch), its length and strand.
struct BamItem {
  int64_t seq, qual, seg;
  int32_t len, rev;
};
constexpr int BAM_SEG_BASES = 1024;  // bases per segment: one warp each

// The batch's bases into the read arena at read_off (already zeroed: NUL padding), its qualities + 33 into qual_out
// (already zeroed: NUL terminators), its sub-read table; *bad_qual = the lowest read index with a quality value above
// 93 (left alone when there is none). Launches only.
void bam_decode(const uint8_t* chunk, const BamItem* items, int n, int64_t n_segs, const uint64_t* read_off,
                const uint64_t* sub_start, int read_part_length, uint8_t* reads, uint8_t* qual_out, int32_t* bad_qual,
                uint64_t* sub_off, int32_t* sub_len, cudaStream_t st);

}  // namespace nb
