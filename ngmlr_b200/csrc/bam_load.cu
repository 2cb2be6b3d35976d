// ngmlr_b200/csrc/bam_load.cu -- BAM records for the read loader (read_load.cu): the header and the block_size chain
// on the host, the bases, qualities and sub-read table of a batch on the device.
//
// The reads are those the unmodified ReadProvider makes from `samtools fastq -n` of the file: records flagged 0x100 /
// 0x800 are skipped; the name is read_name cut at kseq's first whitespace byte, then to 249 characters; the bases are
// seq through "=ACMGRSVTWYHKDBN" with everything but A / C / G / T as N, reverse-complemented back under 0x10; the
// qualities are qual + 33, reversed under 0x10, "*" when the first quality byte is 0xFF. The chain walk is one 4-byte
// read per record and stays on the host (DESIGN.md §4.9, "BAM input").
#include <cstring>

#include "bam.h"

namespace nb {

namespace {

inline int32_t rd32(const uint8_t* p) {
  int32_t v;
  memcpy(&v, p, 4);
  return v;
}

inline uint16_t rd16(const uint8_t* p) {
  uint16_t v;
  memcpy(&v, p, 2);
  return v;
}

std::string at_offset(int64_t off, const char* what) {
  char buf[160];
  snprintf(buf, sizeof(buf), "BAM %s at stream offset %lld", what, (long long)off);
  return buf;
}

}  // namespace

int bam_header(BamState& s, const uint8_t* c, int64_t n, int64_t* p, int64_t base, std::string& err) {
  int64_t q = *p;
  for (;;) {
    if (s.skip) {
      const int64_t take = std::min(s.skip, n - q);
      q += take;
      s.skip -= take;
      s.header_bytes += take;
      if (s.skip) break;
      continue;
    }
    if (s.phase == 3) break;
    const int64_t need = s.phase == 0 ? 8 : 4;
    if (s.phase == 2 && s.refs_left == 0) {
      s.phase = 3;
      break;
    }
    if (n - q < need) break;
    const int32_t v = rd32(c + q + need - 4);
    if (v < 0) {
      *p = q;
      err = at_offset(base + q, s.phase == 0 ? "header with l_text < 0" : s.phase == 1 ? "header with n_ref < 0"
                                                                                       : "reference entry with l_name < 0");
      return -1;
    }
    q += need;
    s.header_bytes += need;
    if (s.phase == 0) {
      s.skip = v;
      s.phase = 1;
    } else if (s.phase == 1) {
      s.refs_left = v;
      s.phase = 2;
    } else {
      s.skip = (int64_t)v + 4;  // the name and l_ref
      --s.refs_left;
    }
  }
  *p = q;
  return s.phase == 3 ? 1 : 0;
}

int bam_walk(BamState& s, const uint8_t* c, int64_t n, int64_t p, int64_t base, int64_t* end, std::string& err) {
  s.recs.clear();
  while (n - p >= 4) {
    const uint8_t* r = c + p;
    const int32_t bs = rd32(r);
    if (bs < 32) {
      err = at_offset(base + p, "record with block_size < 32");
      return -1;
    }
    if (n - p - 4 < bs) break;
    const int l_name = r[12];
    const int n_cigar = rd16(r + 16);
    const int flag = rd16(r + 18);
    const int32_t l_seq = rd32(r + 20);
    if (l_seq < 0) {
      err = at_offset(base + p, "record with l_seq < 0");
      return -1;
    }
    if (l_name == 0) {
      err = at_offset(base + p, "record with l_read_name = 0");
      return -1;
    }
    if (32 + l_name + 4ll * n_cigar + (l_seq + 1ll) / 2 + l_seq > bs) {
      err = at_offset(base + p, "record whose fixed fields do not fit its block_size");
      return -1;
    }
    if (r[36 + l_name - 1] != 0) {
      err = at_offset(base + p, "record whose read_name lacks its NUL");
      return -1;
    }
    BamRec o;
    o.name = p + 36;
    o.seq = o.name + l_name + 4ll * n_cigar;
    o.l_seq = l_seq;
    o.l_name = (uint8_t)l_name;
    o.qual = l_seq > 0 && c[o.seq + (l_seq + 1) / 2] != 0xff;
    o.rev = (flag & 0x10) != 0;
    o.skip = (flag & 0x900) != 0;
    ++s.records;
    if (o.skip) {
      ++s.skipped;
    } else {
      s.reversed += o.rev;
      s.no_quality += l_seq > 0 && !o.qual;
    }
    s.recs.push_back(o);
    p += 4 + (int64_t)bs;
  }
  *end = p;
  return 0;
}

namespace {

// seq's 4-bit codes "=ACMGRSVTWYHKDBN" after ngmlr's normalisation (A / C / G / T kept, everything else N), and their
// complements, as bytes of two 64-bit words per table
constexpr uint64_t pack8(const char* s) {
  uint64_t v = 0;
  for (int i = 7; i >= 0; --i) v = v << 8 | (uint8_t)s[i];
  return v;
}
constexpr uint64_t FWD_LO = pack8("NACNGNNN"), FWD_HI = pack8("TNNNNNNN");
constexpr uint64_t REV_LO = pack8("NTGNCNNN"), REV_HI = pack8("ANNNNNNN");

__device__ __forceinline__ uint8_t base_of(uint32_t code, uint64_t lo, uint64_t hi) {
  return (uint8_t)((code < 8 ? lo : hi) >> (8 * (code & 7)));
}

// the item whose segments hold segment w: the last of items[0 .. n) with seg <= w
__device__ __forceinline__ int item_of(const BamItem* items, int n, int64_t w) {
  int a = 0, b = n;
  while (a < b) {
    const int mid = (a + b) >> 1;
    if (items[mid].seg <= w) a = mid + 1;
    else b = mid;
  }
  return a - 1;
}

// one warp per segment of BAM_SEG_BASES bases; each lane unpacks two bases per packed byte
__global__ void k_bam_seq(const uint8_t* __restrict__ chunk, const BamItem* __restrict__ items, int n, int64_t n_segs,
                          const uint64_t* __restrict__ read_off, uint8_t* __restrict__ dst) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  if (w >= n_segs) return;
  const int i = item_of(items, n, w);
  const BamItem it = items[i];
  const int64_t b0 = (w - it.seg) * (BAM_SEG_BASES / 2);
  const int64_t b1 = min((int64_t)(it.len + 1) / 2, b0 + BAM_SEG_BASES / 2);
  const uint8_t* src = chunk + it.seq;
  uint8_t* d = dst + read_off[i];
  const int64_t L = it.len;
  if (!it.rev) {
    for (int64_t b = b0 + lane; b < b1; b += 32) {
      const uint32_t x = src[b];
      d[2 * b] = base_of(x >> 4, FWD_LO, FWD_HI);
      if (2 * b + 1 < L) d[2 * b + 1] = base_of(x & 15, FWD_LO, FWD_HI);
    }
  } else {
    for (int64_t b = b0 + lane; b < b1; b += 32) {
      const uint32_t x = src[b];
      d[L - 1 - 2 * b] = base_of(x >> 4, REV_LO, REV_HI);
      if (2 * b + 1 < L) d[L - 2 - 2 * b] = base_of(x & 15, REV_LO, REV_HI);
    }
  }
}

// the same segments: qual + 33, reversed under 0x10; a value above 93 marks the read
__global__ void k_bam_qual(const uint8_t* __restrict__ chunk, const BamItem* __restrict__ items, int n, int64_t n_segs,
                           uint8_t* __restrict__ dst, int32_t* bad) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  if (w >= n_segs) return;
  const int i = item_of(items, n, w);
  const BamItem it = items[i];
  if (it.qual < 0) return;
  const int64_t j0 = (w - it.seg) * BAM_SEG_BASES;
  const int64_t j1 = min((int64_t)it.len, j0 + BAM_SEG_BASES);
  const uint8_t* src = chunk + it.seq + (it.len + 1) / 2;
  uint8_t* d = dst + it.qual;
  const int64_t L = it.len;
  bool over = false;
  for (int64_t j = j0 + lane; j < j1; j += 32) {
    const uint32_t q = src[j];
    over |= q > 93;
    d[it.rev ? L - 1 - j : j] = (uint8_t)(q + 33);
  }
  if (__any_sync(0xffffffffu, over) && lane == 0) atomicMin(bad, i);
}

// ReadProvider::splitRead's sub-reads of each read, as reads_upload lays them out
__global__ void k_bam_subreads(const BamItem* items, int n, const uint64_t* read_off, const uint64_t* sub_start,
                               int read_part_length, uint64_t* soff, int32_t* slen) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int len = items[i].len;
  const int parts = len / read_part_length;
  const uint64_t s = sub_start[i];
  if (parts == 0) {
    soff[s] = read_off[i];
    slen[s] = len;
  } else {
    for (int p = 0; p < parts; ++p) {
      soff[s + p] = read_off[i] + (uint64_t)p * (uint64_t)read_part_length;
      slen[s + p] = read_part_length;
    }
  }
}

inline int blocks(int64_t n, int t) { return (int)std::max<int64_t>(1, (n + t - 1) / t); }

}  // namespace

void bam_decode(const uint8_t* chunk, const BamItem* items, int n, int64_t n_segs, const uint64_t* read_off,
                const uint64_t* sub_start, int read_part_length, uint8_t* reads, uint8_t* qual_out, int32_t* bad_qual,
                uint64_t* sub_off, int32_t* sub_len, cudaStream_t st) {
  if (n <= 0) return;
  if (n_segs > 0) {
    k_bam_seq<<<blocks(n_segs * 32, 256), 256, 0, st>>>(chunk, items, n, n_segs, read_off, reads);
    k_bam_qual<<<blocks(n_segs * 32, 256), 256, 0, st>>>(chunk, items, n, n_segs, qual_out, bad_qual);
  }
  k_bam_subreads<<<blocks(n, 128), 128, 0, st>>>(items, n, read_off, sub_start, read_part_length, sub_off, sub_len);
}

}  // namespace nb
