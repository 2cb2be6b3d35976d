// ngmlr_b200/csrc/sam_text.cpp -- SAM records of a batch of reads, formatted by host threads (SURVEY 8(f)4).
//
// Replaces SAMWriter::DoWriteProlog (src/SAMWriter.cpp:22-85), DoWriteRead -> DoWriteReadGeneric (:87-224),
// DoWriteUnmappedRead -> DoWriteUnmappedReadGeneric (:301-363) and the loop of GenericReadWriter::WriteRead
// (src/GenericReadWriter.h:78-108). The reference appends every field with vsprintf into one 100 MB buffer
// under the output mutex' eventual flush; here a record is emitted by one routine into a "sink" that either
// counts or copies, so a batch is sized (pass 1, parallel over reads), given offsets (one prefix sum) and
// written in place (pass 2, parallel) -- records come out in read order whatever the thread count. The same
// decisions (read_records: which alignments get a record, flags, quality strand, long CIGAR) feed a BAM sink too
// (ngmlr_b200_bam_format: what samtools makes of the text, SAMv1 section 4.2; no reference counterpart).
//
// As-coded details that are kept (the tests compare bytes with the unmodified writer):
//   * positions: `m_Location + 1` is a 64-bit value printed with %u (POS) and %d (SA:Z) -> low 32 bits;
//   * AS / XE are (int) of the float score, XS is the constant 0, XI is round(identity * 1e4) / 1e4 with %g,
//     CV is (length - clipped) * 100.0f / length with %f;
//   * a reverse-strand record reverses the read's quality string IN PLACE (:104-108), so a later reverse
//     record of the same read finds it forward again (opts->fix_quality_orientation = 1 turns that off);
//   * --bam-fix: >= 0x10000 CIGAR operations -> "<length>S" in the CIGAR column and the operations as
//     CG:B:I,(len << 4 | op) printed with %d (:123-130, :199-218);
//   * the unmapped record ends with the quality column (no trailing tab) and ORs 0x4 into the flags.
// Deliberate difference: a "*" quality (FASTA input) is never reversed; the reference reverses `length`
// bytes of a 2-byte buffer there (undefined behaviour, SURVEY 8(f)4 "FASTA reverse-strand overflow").
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/ngmlr_b200.h"

namespace nb {
int host_threads();  // capi.cu
void set_error_without_context(const std::string& msg);  // capi.cu
}

namespace {

struct CountSink {
  size_t n = 0;
  void put(const char*, size_t len) { n += len; }
  void ch(char) { ++n; }
  // sequence columns: only the length matters
  void seq_fwd(const char*, size_t len) { n += len; }
  void seq_revcomp(const char*, size_t len) { n += len; }
  void reversed(const char*, size_t len) { n += len; }
};

struct WriteSink {
  char* p;
  void put(const char* s, size_t len) {
    memcpy(p, s, len);
    p += len;
  }
  void ch(char c) { *p++ = c; }
  void seq_fwd(const char* s, size_t len) { put(s, len); }
  // MappedRead::computeReverseSeq (src/MappedRead.cpp:37-69): A<->T, C<->G, anything else unchanged
  void seq_revcomp(const char* s, size_t len) {
    static const struct Table {
      unsigned char t[256];
      Table() {
        for (int i = 0; i < 256; ++i) t[i] = (unsigned char)i;
        t['A'] = 'T'; t['T'] = 'A'; t['C'] = 'G'; t['G'] = 'C';
      }
    } tab;
    const unsigned char* src = (const unsigned char*)s + len;
    for (size_t i = 0; i < len; ++i) p[i] = (char)tab.t[*--src];
    p += len;
  }
  void reversed(const char* s, size_t len) {
    std::reverse_copy(s, s + len, p);
    p += len;
  }
};

template <class Sink>
inline void put_str(Sink& o, const char* s) { o.put(s, strlen(s)); }

template <class Sink>
inline void put_lit(Sink& o, const char* s, size_t n) { o.put(s, n); }
#define LIT(o, s) put_lit(o, s, sizeof(s) - 1)

template <class Sink>
inline void put_u64(Sink& o, uint64_t v) {
  char b[24];
  int n = 0;
  do { b[n++] = (char)('0' + v % 10); v /= 10; } while (v);
  char r[24];
  for (int i = 0; i < n; ++i) r[i] = b[n - 1 - i];
  o.put(r, (size_t)n);
}

template <class Sink>
inline void put_i32(Sink& o, int32_t v) {  // %d
  if (v < 0) {
    o.ch('-');
    put_u64(o, (uint64_t)(-(int64_t)v));
  } else {
    put_u64(o, (uint64_t)v);
  }
}

template <class Sink>
inline void put_u32(Sink& o, uint32_t v) { put_u64(o, v); }  // %u

// length of the prefix of s that "%.*s" with precision n prints
inline size_t prefix_len(const char* s, size_t n) {
  const void* z = memchr(s, 0, n);
  return z ? (size_t)((const char*)z - s) : n;
}

struct Ctx {
  const ngmlr_b200_sam_options* opts;
  const ngmlr_b200_sam_aln* alns;
  const char* const* ref_names;
  const int32_t* ref_name_lens;
  int n_refs;
};

template <class Sink>
inline void put_ref_name(Sink& o, const Ctx& c, int id) {
  if (id >= 0 && id < c.n_refs) o.put(c.ref_names[id], (size_t)c.ref_name_lens[id]);
}

// DoWriteUnmappedReadGeneric(read, -1, '*', -1, -1, 0, 0, flags | 0x4)   (:301-363)
template <class Sink>
void unmapped_record(Sink& o, const Ctx& c, const ngmlr_b200_sam_read& r) {
  put_str(o, r.name);
  LIT(o, "\t4\t*\t0\t0\t*\t*\t0\t0\t");
  o.seq_fwd(r.seq, prefix_len(r.seq, (size_t)r.length));
  o.ch('\t');
  if (r.qual) o.put(r.qual, prefix_len(r.qual, (size_t)r.length));
  else o.ch('*');
  if (c.opts->rg_id) {
    LIT(o, "\tRG:Z:");
    put_str(o, c.opts->rg_id);
  }
  o.ch('\n');
}

// What one record of a read is, decided once for the SAM and the BAM sink (GenericReadWriter::WriteRead,
// DoWriteReadGeneric). i < 0: the unmapped record.
struct Rec {
  int i;
  int flags;
  bool qual_reversed;  // state of the read's quality string when the record is printed
  bool long_cigar;     // --bam-fix: "<length>S" in the CIGAR column and the operations as CG:B:I
};

// whether record i gets an SA:Z tag: another alignment of the read is not skipped
inline bool has_sa(const Ctx& c, const ngmlr_b200_sam_read& r, int i) {
  for (int j = 0; j < r.n_aln; ++j)
    if (j != i && !c.alns[r.first_aln + j].skip) return true;
  return false;
}

// SA:Z's value for record i: every other non-skipped alignment as "rname,pos,strand,CIGAR,mapq,NM;"
template <class Sink>
void sa_value(Sink& o, const Ctx& c, const ngmlr_b200_sam_read& r, int i) {
  const ngmlr_b200_sam_aln* al = c.alns + r.first_aln;
  for (int j = 0; j < r.n_aln; ++j) {
    if (j == i || al[j].skip) continue;
    put_ref_name(o, c, al[j].ref_id);
    o.ch(',');
    put_i32(o, (int32_t)(al[j].ref_pos + 1));
    o.ch(',');
    o.ch(al[j].reverse ? '-' : '+');
    o.ch(',');
    put_str(o, al[j].cigar);
    o.ch(',');
    put_i32(o, al[j].mq);
    o.ch(',');
    put_i32(o, al[j].nm);
    o.ch(';');
  }
}

// CIGAR operation code of a text operation (the reference's --bam-fix switch maps anything unknown to M)
inline int cigar_op_code(char ch) {
  switch (ch) {
    case 'M': return 0;
    case 'I': return 1;
    case 'D': return 2;
    case 'N': return 3;
    case 'S': return 4;
    case 'H': return 5;
    case '=': return 7;
    case 'X': return 8;
    default: return 0;
  }
}

// XI:f's and CV:f's printed text (%g of the rounded identity, %f of the covered share)
inline int xi_text(char* b, size_t cap, const ngmlr_b200_sam_aln& a) {
  // the reference's unqualified round() is ::round(double): double quotient, narrowed by the assignment
  const float identity = (float)(::round((double)(a.identity * 10000.0f)) / (double)10000.0f);
  return snprintf(b, cap, "%g", identity);
}
inline int cv_text(char* b, size_t cap, const ngmlr_b200_sam_read& r, const ngmlr_b200_sam_aln& a) {
  const int clipped = a.qstart + a.qend;
  const float covered = (r.length - clipped) * 100.0f / r.length;
  return snprintf(b, cap, "%f", covered);
}

// DoWriteReadGeneric(read, i, "*", -1, 0, mappingQlty, 0)   (:92-224)
template <class Sink>
void mapped_record(Sink& o, const Ctx& c, const ngmlr_b200_sam_read& r, const Rec& rec) {
  const int i = rec.i;
  const ngmlr_b200_sam_aln& a = c.alns[r.first_aln + i];
  const bool qual_reversed = rec.qual_reversed;
  const size_t len = (size_t)r.length;
  put_str(o, r.name);
  o.ch('\t');
  put_i32(o, rec.flags);
  o.ch('\t');
  put_ref_name(o, c, a.ref_id);
  o.ch('\t');
  put_u32(o, (uint32_t)(a.ref_pos + 1));
  o.ch('\t');
  put_i32(o, a.mq);
  o.ch('\t');
  const bool long_cigar = rec.long_cigar;
  if (long_cigar) {
    put_i32(o, r.length);
    o.ch('S');
  } else {
    put_str(o, a.cigar);
  }
  LIT(o, "\t*\t0\t0\t");  // mate name "*", mate position -1 + 1 as %u, template length 0
  if (a.reverse) o.seq_revcomp(r.seq, len);  // RevSeq is zero-filled behind `length`: no embedded NUL possible
  else o.seq_fwd(r.seq, prefix_len(r.seq, len));
  o.ch('\t');
  if (r.qual) {
    const size_t ql = prefix_len(r.qual, len);
    if (qual_reversed && ql == len) o.reversed(r.qual, len);
    else o.put(r.qual, ql);
    o.ch('\t');
  } else {
    LIT(o, "*\t");
  }
  if (c.opts->rg_id) {
    LIT(o, "RG:Z:");
    put_str(o, c.opts->rg_id);
    o.ch('\t');
  }
  LIT(o, "AS:i:");
  put_i32(o, (int)a.score);
  LIT(o, "\tNM:i:");
  put_i32(o, a.nm);
  {
    char b[48];
    const int n = xi_text(b, sizeof b, a);
    LIT(o, "\tXI:f:");
    o.put(b, (size_t)n);
    LIT(o, "\tXS:i:0\tXE:i:");
  }
  put_i32(o, (int)a.score);
  LIT(o, "\tXR:i:");
  put_i32(o, r.length - a.qstart - a.qend);
  LIT(o, "\tMD:Z:");
  put_str(o, a.md);
  o.ch('\t');
  if (a.sv_type > -1) {
    LIT(o, "SV:i:");
    put_i32(o, a.sv_type);
    o.ch('\t');
  }
  if (r.n_aln > 1 && has_sa(c, r, i)) {
    LIT(o, "SA:Z:");
    sa_value(o, c, r, i);
    o.ch('\t');
  }
  LIT(o, "QS:i:");
  put_i32(o, a.qstart);
  LIT(o, "\tQE:i:");
  put_i32(o, r.length - a.qend);
  {
    char b[64];
    const int n = cv_text(b, sizeof b, r, a);
    LIT(o, "\tCV:f:");
    o.put(b, (size_t)n);
  }
  if (long_cigar) {
    LIT(o, "\tCG:B:I");
    char* p = const_cast<char*>(a.cigar);
    for (int k = 0; k < a.cigar_ops; ++k) {
      const long l = strtol(p, &p, 10);
      const int op = cigar_op_code(*p);
      ++p;
      o.ch(',');
      put_i32(o, (int32_t)((unsigned int)l << 4 | (unsigned int)op));
    }
  }
  o.ch('\n');
}

// GenericReadWriter::WriteRead(read, mapped): emit(rec) for each record of the read, in order
template <class Emit>
void read_records(const Ctx& c, const ngmlr_b200_sam_read& r, Emit&& emit) {
  bool mapped_once = false;
  bool qual_reversed = false;
  if (r.mapped) {
    for (int i = 0; i < r.n_aln; ++i) {
      const ngmlr_b200_sam_aln& a = c.alns[r.first_aln + i];
      if (a.skip) continue;
      mapped_once = true;
      if (a.reverse) qual_reversed = c.opts->fix_quality_orientation ? true : !qual_reversed;
      else if (c.opts->fix_quality_orientation) qual_reversed = false;
      const int flags = (a.primary ? 0 : 0x800) | (a.reverse ? 0x10 : 0);
      emit(Rec{i, flags, qual_reversed, c.opts->bam_cigar_fix && a.cigar_ops >= 0x10000});
    }
  }
  if (!mapped_once && !r.empty && c.opts->write_unmapped) emit(Rec{-1, 4, false, false});
}

template <class Sink>
void sam_records(Sink& o, const Ctx& c, const ngmlr_b200_sam_read& r) {
  read_records(c, r, [&](const Rec& rec) {
    if (rec.i < 0) unmapped_record(o, c, r);
    else mapped_record(o, c, r, rec);
  });
}


// ---- BAM (SAMv1 section 4.2): the encoding samtools gives the SAM text of the same records ----

enum BamError { BAM_OK = 0, BAM_POS, BAM_RNAME, BAM_MAPQ, BAM_NAME, BAM_CIGAR, BAM_QUAL };

const char* bam_error_text(int e) {
  switch (e) {
    case BAM_POS: return "POS above 2^31 does not fit BAM";
    case BAM_RNAME: return "RNAME is not a reference of the header";
    case BAM_MAPQ: return "MAPQ outside 0..255";
    case BAM_NAME: return "read name longer than 254 bytes";
    case BAM_CIGAR: return "malformed CIGAR";
    case BAM_QUAL: return "QUAL and SEQ differ in length";
    default: return "";
  }
}

struct BamCtx {
  Ctx c;
  const int32_t* target_of;  // header index of each ref_id's name, -1 when the header has none
};

// SAMv1 section 5.3
inline int reg2bin(int64_t beg, int64_t end) {
  --end;
  if (beg >> 14 == end >> 14) return (int)(((1 << 15) - 1) / 7 + (beg >> 14));
  if (beg >> 17 == end >> 17) return (int)(((1 << 12) - 1) / 7 + (beg >> 17));
  if (beg >> 20 == end >> 20) return (int)(((1 << 9) - 1) / 7 + (beg >> 20));
  if (beg >> 23 == end >> 23) return (int)(((1 << 6) - 1) / 7 + (beg >> 23));
  if (beg >> 26 == end >> 26) return (int)(((1 << 3) - 1) / 7 + (beg >> 26));
  return 0;
}

template <class Sink>
inline void le(Sink& o, uint64_t v, int bytes) {
  char b[8];
  for (int k = 0; k < bytes; ++k) b[k] = (char)(v >> (8 * k));
  o.put(b, (size_t)bytes);
}

// bytes put so far (a pointer's value for WriteSink: only differences count), and a 32-bit value written `back`
// bytes behind the sink's position
inline size_t o_size(const CountSink& o) { return o.n; }
inline size_t o_size(const WriteSink& o) { return (size_t)o.p; }
inline void patch_le32(CountSink&, size_t, uint32_t) {}
inline void patch_le32(WriteSink& o, size_t back, uint32_t v) {
  char* at = o.p - back;
  for (int k = 0; k < 4; ++k) at[k] = (char)(v >> (8 * k));
}

// "=ACMGRSVTWYHKDBN" code of a SEQ character (lower case as upper case, anything else N)
inline int nt16(unsigned char ch) {
  static const struct Table {
    uint8_t t[256];
    Table() {
      const char* s = "=ACMGRSVTWYHKDBN";
      for (int i = 0; i < 256; ++i) t[i] = 15;
      for (int k = 0; k < 16; ++k) {
        t[(unsigned char)s[k]] = (uint8_t)k;
        t[(unsigned char)tolower(s[k])] = (uint8_t)k;
      }
    }
  } tab;
  return tab.t[ch];
}

inline void bam_seq(CountSink& o, const char*, size_t len, bool) { o.n += (len + 1) / 2; }
inline void bam_seq(WriteSink& o, const char* s, size_t len, bool revcomp) {
  auto base = [&](size_t k) -> unsigned char {
    if (!revcomp) return (unsigned char)s[k];
    const unsigned char ch = (unsigned char)s[len - 1 - k];  // MappedRead::computeReverseSeq
    return ch == 'A' ? 'T' : ch == 'T' ? 'A' : ch == 'C' ? 'G' : ch == 'G' ? 'C' : ch;
  };
  for (size_t k = 0; k < len; k += 2) {
    const int hi = nt16(base(k)), lo = k + 1 < len ? nt16(base(k + 1)) : 0;
    *o.p++ = (char)(hi << 4 | lo);
  }
}

inline void bam_qual(CountSink& o, const char*, size_t len, bool) { o.n += len; }
inline void bam_qual(WriteSink& o, const char* q, size_t len, bool reversed) {
  if (!q) {
    memset(o.p, 0xff, len);
  } else {
    for (size_t k = 0; k < len; ++k) o.p[k] = (char)((unsigned char)q[reversed ? len - 1 - k : k] - 33);
  }
  o.p += len;
}

// an integer tag in htslib's smallest type
template <class Sink>
void tag_i(Sink& o, const char* key, int64_t v) {
  o.put(key, 2);
  if (v < 0) {
    if (v >= INT8_MIN) { o.ch('c'); le(o, (uint64_t)v, 1); }
    else if (v >= INT16_MIN) { o.ch('s'); le(o, (uint64_t)v, 2); }
    else { o.ch('i'); le(o, (uint64_t)v, 4); }
  } else {
    if (v <= UINT8_MAX) { o.ch('C'); le(o, (uint64_t)v, 1); }
    else if (v <= UINT16_MAX) { o.ch('S'); le(o, (uint64_t)v, 2); }
    else { o.ch('I'); le(o, (uint64_t)v, 4); }
  }
}

template <class Sink>
void tag_f(Sink& o, const char* key, const char* text) {
  o.put(key, 2);
  o.ch('f');
  const float f = (float)strtod(text, nullptr);
  uint32_t u;
  memcpy(&u, &f, 4);
  le(o, u, 4);
}

template <class Sink>
void tag_z_begin(Sink& o, const char* key) {
  o.put(key, 2);
  o.ch('Z');
}

// Walks a CIGAR text: op(len, code) per operation. Returns the number of operations, or -1 when malformed.
template <class Op>
int64_t parse_cigar(const char* s, Op&& op) {
  if (s[0] == '*' && s[1] == 0) return 0;
  int64_t n = 0;
  while (*s) {
    if (*s < '0' || *s > '9') return -1;
    uint64_t l = 0;
    while (*s >= '0' && *s <= '9') {
      l = l * 10 + (uint64_t)(*s++ - '0');
      if (l > 0x0fffffff) return -1;
    }
    const char* ops = "MIDNSHP=X";
    const char* hit = *s ? strchr(ops, *s) : nullptr;
    if (!hit) return -1;
    op((uint32_t)l, (int)(hit - ops));
    ++s;
    ++n;
  }
  return n;
}

inline bool consumes_ref(int code) { return code == 0 || code == 2 || code == 3 || code == 7 || code == 8; }

// the fixed part of a record (after block_size) up to l_seq, with next_refID / next_pos = -1 and tlen 0
template <class Sink>
void bam_fixed(Sink& o, int32_t ref, int32_t pos, size_t l_name, int mapq, int bin, uint32_t n_cigar, int flag,
               uint32_t l_seq) {
  le(o, (uint32_t)ref, 4);
  le(o, (uint32_t)pos, 4);
  le(o, l_name, 1);
  le(o, (uint64_t)mapq, 1);
  le(o, (uint64_t)bin, 2);
  le(o, n_cigar, 2);
  le(o, (uint64_t)flag, 2);
  le(o, l_seq, 4);
  le(o, 0xffffffffu, 4);
  le(o, 0xffffffffu, 4);
  le(o, 0, 4);
}

template <class Sink>
int bam_unmapped(Sink& o, const BamCtx& b, const ngmlr_b200_sam_read& r) {
  const size_t l_name = strlen(r.name) + 1;
  if (l_name > 255) return BAM_NAME;
  size_t l_seq = prefix_len(r.seq, (size_t)r.length);
  if (l_seq == 1 && r.seq[0] == '*') l_seq = 0;  // SEQ "*": no bases, as in bam_mapped
  const size_t ql = r.qual ? prefix_len(r.qual, (size_t)r.length) : 0;
  const bool no_qual = !r.qual || (ql == 1 && r.qual[0] == '*');
  if (!no_qual && ql != l_seq) return BAM_QUAL;
  bam_fixed(o, -1, -1, l_name, 0, 4680, 0, 4, (uint32_t)l_seq);
  o.put(r.name, l_name);
  bam_seq(o, r.seq, l_seq, false);
  bam_qual(o, no_qual ? nullptr : r.qual, l_seq, false);
  if (b.c.opts->rg_id) {
    tag_z_begin(o, "RG");
    o.put(b.c.opts->rg_id, strlen(b.c.opts->rg_id) + 1);
  }
  return BAM_OK;
}

template <class Sink>
int bam_mapped(Sink& o, const BamCtx& b, const ngmlr_b200_sam_read& r, const Rec& rec) {
  const Ctx& c = b.c;
  const ngmlr_b200_sam_aln& a = c.alns[r.first_aln + rec.i];
  const size_t len = (size_t)r.length;
  const size_t l_name = strlen(r.name) + 1;
  if (l_name > 255) return BAM_NAME;
  const int32_t ref = a.ref_id >= 0 && a.ref_id < c.n_refs ? b.target_of[a.ref_id] : -1;
  if (ref < 0) return BAM_RNAME;
  const uint32_t printed_pos = (uint32_t)(a.ref_pos + 1);
  if (printed_pos > (1u << 31)) return BAM_POS;
  const int32_t pos = (int32_t)(printed_pos - 1);
  if (a.mq < 0 || a.mq > 255) return BAM_MAPQ;
  // the CIGAR column: the alignment's text, or "<length>S" under --bam-fix
  char fix_text[16];
  const char* cigar = a.cigar;
  if (rec.long_cigar) {
    snprintf(fix_text, sizeof fix_text, "%dS", r.length);
    cigar = fix_text;
  }
  int64_t rlen = 0;
  const int64_t n_ops = parse_cigar(cigar, [&](uint32_t l, int code) {
    if (consumes_ref(code)) rlen += l;
  });
  if (n_ops < 0) return BAM_CIGAR;
  // SEQ / QUAL as printed
  const bool rev = a.reverse != 0;
  size_t l_seq = rev ? len : prefix_len(r.seq, len);
  if (!rev && l_seq == 1 && r.seq[0] == '*') l_seq = 0;
  const size_t ql = r.qual ? prefix_len(r.qual, len) : 0;
  const bool no_qual = !r.qual || (ql == 1 && r.qual[0] == '*');
  if (!no_qual && ql != l_seq) return BAM_QUAL;
  const bool qual_rev = rec.qual_reversed && ql == len;
  const bool placeholder = n_ops > 0xffff;  // SAMv1 4.2.2: <l_seq>S<rlen>N, the CIGAR itself in CG:B:I
  const int bin = reg2bin(pos, pos + std::max<int64_t>(rlen, 1));
  bam_fixed(o, ref, pos, l_name, a.mq, bin, placeholder ? 2u : (uint32_t)n_ops, rec.flags, (uint32_t)l_seq);
  o.put(r.name, l_name);
  if (placeholder) {
    le(o, (uint32_t)l_seq << 4 | 4, 4);
    le(o, (uint32_t)rlen << 4 | 3, 4);
  } else {
    parse_cigar(cigar, [&](uint32_t l, int code) { le(o, l << 4 | (uint32_t)code, 4); });
  }
  bam_seq(o, r.seq, l_seq, rev);
  bam_qual(o, no_qual ? nullptr : r.qual, l_seq, qual_rev);
  if (c.opts->rg_id) {
    tag_z_begin(o, "RG");
    o.put(c.opts->rg_id, strlen(c.opts->rg_id) + 1);
  }
  tag_i(o, "AS", (int)a.score);
  tag_i(o, "NM", a.nm);
  char text[64];
  xi_text(text, sizeof text, a);
  tag_f(o, "XI", text);
  tag_i(o, "XS", 0);
  tag_i(o, "XE", (int)a.score);
  tag_i(o, "XR", (int64_t)r.length - a.qstart - a.qend);
  tag_z_begin(o, "MD");
  o.put(a.md, strlen(a.md) + 1);
  if (a.sv_type > -1) tag_i(o, "SV", a.sv_type);
  if (r.n_aln > 1 && has_sa(c, r, rec.i)) {
    tag_z_begin(o, "SA");
    sa_value(o, c, r, rec.i);
    o.ch(0);
  }
  tag_i(o, "QS", a.qstart);
  tag_i(o, "QE", (int64_t)r.length - a.qend);
  cv_text(text, sizeof text, r, a);
  tag_f(o, "CV", text);
  if (rec.long_cigar || placeholder) {
    LIT(o, "CGBI");
    if (rec.long_cigar) {  // the text's CG:B:I values (printed with %d)
      le(o, (uint32_t)a.cigar_ops, 4);
      char* p = const_cast<char*>(a.cigar);
      for (int k = 0; k < a.cigar_ops; ++k) {
        const long l = strtol(p, &p, 10);
        const int op = cigar_op_code(*p);
        ++p;
        le(o, (uint32_t)((unsigned int)l << 4 | (unsigned int)op), 4);
      }
    } else {
      le(o, (uint64_t)n_ops, 4);
      parse_cigar(cigar, [&](uint32_t l, int code) { le(o, l << 4 | (uint32_t)code, 4); });
    }
  }
  return BAM_OK;
}

template <class Sink>
int bam_records(Sink& o, const BamCtx& b, const ngmlr_b200_sam_read& r) {
  int err = BAM_OK;
  read_records(b.c, r, [&](const Rec& rec) {
    if (err) return;
    const size_t at = o_size(o);
    le(o, 0, 4);  // block_size
    err = rec.i < 0 ? bam_unmapped(o, b, r) : bam_mapped(o, b, r, rec);
    patch_le32(o, o_size(o) - at, (uint32_t)(o_size(o) - at - 4));
  });
  return err;
}

template <typename F>
void run_parallel(int64_t n, int threads, F fn) {
  const int64_t chunk = 16;
  const int64_t pieces = (n + chunk - 1) / chunk;
  threads = (int)std::min<int64_t>(threads, pieces);
  std::atomic<int64_t> next(0);
  auto work = [&]() {
    for (;;) {
      const int64_t b = next.fetch_add(chunk);
      if (b >= n) break;
      const int64_t e = std::min(n, b + chunk);
      for (int64_t i = b; i < e; ++i) fn(i);
    }
  };
  if (threads <= 1) {
    work();
    return;
  }
  std::vector<std::thread> pool;
  pool.reserve((size_t)threads - 1);
  for (int t = 1; t < threads; ++t) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
}

}  // namespace

extern "C" {

size_t ngmlr_b200_sam_header(int n_refs, const char* const* ref_names, const uint64_t* ref_lens,
                             const char* version, const char* command_line, const ngmlr_b200_sam_options* opts,
                             const char* const* rg_fields, char* out, size_t cap) {
  auto emit = [&](auto& o) {
    LIT(o, "@HD\tVN:1.0\tSO:unsorted\n");
    for (int i = 0; i < n_refs; ++i) {
      LIT(o, "@SQ\tSN:");
      put_str(o, ref_names[i]);
      LIT(o, "\tLN:");
      put_u64(o, ref_lens[i]);
      o.ch('\n');
    }
    LIT(o, "@PG\tID:ngmlr\tPN:nextgenmap-lr\tVN:");
    put_str(o, version ? version : "");
    LIT(o, "\tCL:");
    put_str(o, command_line ? command_line : "(null)");  // vsprintf("%s", 0) prints "(null)"
    o.ch('\n');
    if (opts && opts->rg_id) {
      static const char* const keys[11] = {"SM", "LB", "PL", "DS", "DT", "PU", "PI", "PG", "CN", "FO", "KS"};
      LIT(o, "@RG\tID:");
      put_str(o, opts->rg_id);
      for (int k = 0; k < 11; ++k) {
        if (!rg_fields || !rg_fields[k]) continue;
        o.ch('\t');
        o.put(keys[k], 2);
        o.ch(':');
        put_str(o, rg_fields[k]);
      }
      o.ch('\n');
    }
  };
  CountSink cs;
  emit(cs);
  if (out && cs.n <= cap) {
    WriteSink ws{out};
    emit(ws);
  }
  return cs.n;
}

int ngmlr_b200_sam_format(const ngmlr_b200_sam_options* opts, int64_t n_reads, const ngmlr_b200_sam_read* reads,
                          const ngmlr_b200_sam_aln* alns, int n_refs, const char* const* ref_names,
                          const int32_t* ref_name_lens, char* out, size_t cap, size_t* written) {
  if (!opts || n_reads < 0 || (n_reads && !reads) || !written) return -1;
  for (int64_t i = 0; i < n_reads; ++i) {
    const ngmlr_b200_sam_read& r = reads[i];
    if (!r.name || !r.seq || r.length < 0 || (r.n_aln > 0 && !alns)) return -1;
  }
  const Ctx c{opts, alns, ref_names, ref_name_lens, n_refs};
  const int threads = opts->threads > 0 ? opts->threads : nb::host_threads();
  std::vector<size_t> off((size_t)n_reads + 1, 0);
  run_parallel(n_reads, threads, [&](int64_t i) {
    CountSink cs;
    sam_records(cs, c, reads[i]);
    off[(size_t)i + 1] = cs.n;
  });
  for (int64_t i = 0; i < n_reads; ++i) off[(size_t)i + 1] += off[(size_t)i];
  *written = off[(size_t)n_reads];
  if (*written > cap || (!out && *written)) return -2;
  run_parallel(n_reads, threads, [&](int64_t i) {
    WriteSink ws{out + off[(size_t)i]};
    sam_records(ws, c, reads[i]);
  });
  return 0;
}

int ngmlr_b200_bam_header(int n_refs, const char* const* ref_names, const uint64_t* ref_lens, const char* version,
                          const char* command_line, const ngmlr_b200_sam_options* opts,
                          const char* const* rg_fields, char* out, size_t cap, size_t* written) {
  if (n_refs < 0 || (n_refs && (!ref_names || !ref_lens)) || !written) {
    nb::set_error_without_context("bam_header: invalid arguments");
    return -1;
  }
  for (int i = 0; i < n_refs; ++i) {
    if (!ref_names[i]) {
      nb::set_error_without_context("bam_header: invalid arguments");
      return -1;
    }
    if (ref_lens[i] > (uint64_t)INT32_MAX) {
      nb::set_error_without_context(std::string("bam_header: reference ") + ref_names[i] + " has LN " +
                                    std::to_string(ref_lens[i]) + ", above BAM's 2^31 - 1");
      return -1;
    }
  }
  const size_t l_text = ngmlr_b200_sam_header(n_refs, ref_names, ref_lens, version, command_line, opts, rg_fields,
                                              nullptr, 0);
  size_t need = 4 + 4 + l_text + 4;
  for (int i = 0; i < n_refs; ++i) need += 4 + strlen(ref_names[i]) + 1 + 4;
  *written = need;
  if (!out || need > cap) return -2;
  WriteSink o{out};
  LIT(o, "BAM\1");
  le(o, l_text, 4);
  ngmlr_b200_sam_header(n_refs, ref_names, ref_lens, version, command_line, opts, rg_fields, o.p, l_text);
  o.p += l_text;
  le(o, (uint64_t)n_refs, 4);
  for (int i = 0; i < n_refs; ++i) {
    const size_t l = strlen(ref_names[i]) + 1;
    le(o, l, 4);
    o.put(ref_names[i], l);
    le(o, ref_lens[i], 4);
  }
  return 0;
}

int ngmlr_b200_bam_format(const ngmlr_b200_sam_options* opts, int64_t n_reads, const ngmlr_b200_sam_read* reads,
                          const ngmlr_b200_sam_aln* alns, int n_refs, const char* const* ref_names,
                          const int32_t* ref_name_lens, int n_targets, const char* const* target_names, char* out,
                          size_t cap, size_t* written) {
  bool ok = opts && n_reads >= 0 && (!n_reads || reads) && written && n_refs >= 0 && n_targets >= 0 &&
            (!n_refs || (ref_names && ref_name_lens)) && (!n_targets || target_names);
  for (int64_t i = 0; ok && i < n_reads; ++i) {
    const ngmlr_b200_sam_read& r = reads[i];
    ok = r.name && r.seq && r.length >= 0 && (r.n_aln <= 0 || alns);
  }
  if (!ok) {
    nb::set_error_without_context("bam_format: invalid arguments");
    return -1;
  }
  // refID of each ref_id: its printed name ("%.*s") looked up among the header's names (the first of equal names)
  std::unordered_map<std::string, int32_t> by_name;
  for (int t = n_targets - 1; t >= 0; --t) by_name[target_names[t] ? target_names[t] : ""] = t;
  std::vector<int32_t> target_of((size_t)std::max(n_refs, 1), -1);
  for (int id = 0; id < n_refs; ++id) {
    if (!ref_names[id]) continue;
    const auto it = by_name.find(std::string(ref_names[id], prefix_len(ref_names[id], (size_t)ref_name_lens[id])));
    if (it != by_name.end()) target_of[(size_t)id] = it->second;
  }
  const BamCtx b{Ctx{opts, alns, ref_names, ref_name_lens, n_refs}, target_of.data()};
  const int threads = opts->threads > 0 ? opts->threads : nb::host_threads();
  std::vector<size_t> off((size_t)n_reads + 1, 0);
  std::vector<int8_t> err((size_t)n_reads, 0);
  run_parallel(n_reads, threads, [&](int64_t i) {
    CountSink cs;
    err[(size_t)i] = (int8_t)bam_records(cs, b, reads[i]);
    off[(size_t)i + 1] = cs.n;
  });
  for (int64_t i = 0; i < n_reads; ++i) {
    if (err[(size_t)i]) {
      nb::set_error_without_context(std::string("bam_format: read ") + reads[i].name + ": " +
                                    bam_error_text(err[(size_t)i]));
      return -1;
    }
  }
  for (int64_t i = 0; i < n_reads; ++i) off[(size_t)i + 1] += off[(size_t)i];
  *written = off[(size_t)n_reads];
  if (*written > cap || (!out && *written)) return -2;
  run_parallel(n_reads, threads, [&](int64_t i) {
    WriteSink ws{out + off[(size_t)i]};
    bam_records(ws, b, reads[i]);
  });
  return 0;
}

}  // extern "C"
