// oracle/ref_cs_shim.cpp -- TEST INFRASTRUCTURE ONLY.
//
// extern "C" driver around the UNMODIFIED reference's candidate search, compiled together with all
// of /root/reference/src (except main.cpp) into oracle/_ref/libngmlr_full.so by oracle/Makefile.
// It runs the reference's own code for:
//   reference encoding      _SequenceProvider::Init / DecodeRefSequence   src/SequenceProvider.cpp:292-473, 567-625
//   k-mer index             CompactPrefixTable (build + GetRefEntry)        src/PrefixTable.cpp:233-532
//   k-mer iteration         CS::PrefixIteration                            src/CSstatic.cpp:23-73
//   vote + collect          CS::PrefixSearch / AddLocationStd / CollectResultsStd   src/CS.cpp:57-149, 217-269
// through a CS subclass that repeats only the control flow of CS::RunRead (src/CS.cpp:324-398)
// without handing the read to ScoreBuffer.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define private public
#define protected public
#include "AlignmentBuffer.h"  // (pulls in ConvexAlignFast.h, whose closing brace sits outside its include guard)
#include "CS.h"
#include "IConfig.h"
#include "Log.h"
#include "NGM.h"
#include "PrefixTable.h"
#include "SequenceProvider.h"
#include "ScoreBuffer.h"
#include "StrippedSW.h"
#undef private
#undef protected

ILog const* _log = 0;
IConfig* _config = 0;

// main.cpp (not linked) also owns this helper (src/main.cpp:135-155); same contract, via stat().
#include <sys/stat.h>
uloc const FileSize(char const* const filename) {
  struct stat st;
  if (stat(filename, &st) != 0) return 0;
  return (uloc)st.st_size;
}

namespace {

CompactPrefixTable* g_table = 0;

class CSProbe : public CS {
 public:
  explicit CSProbe(int bits = 24) : CS(false) {
    int len = (int)pow(2, bits);  // x_SrchTableBitLen = 24 in the reference, src/CS.cpp:27, 422-432
    rTable = new CSTableEntry[len];
    rList = new int[len];
    for (int i = 0; i < len; ++i) {
      rTable[i].m_Location = (uint)9223372036854775808ull;
      rTable[i].state = -1;
      rList[i] = -1;
    }
    m_CsSensitivity = Config.getSensitivity();
    m_RefProvider = g_table;
    m_entryCount = m_RefProvider->GetRefEntryChainLength();
    m_entry = new RefEntry[m_entryCount];
  }

  // CS::RunRead minus SendToBuffer. Returns candidate count or -1 if every table size overflowed.
  int search(MappedRead* read, int table_bits) {
    SetSearchTableBitLen(table_bits);
    currentState++;
    rListLength = 0;
    maxHitNumber = 0.0f;
    currentThresh = 0.0f;
    extern int kCount;
    m_CurrentReadLength = read->length;
    bool fallback = false;
    int n = -1;
    try {
      hpoc = c_SrchTableLen * 0.333f;
      PrefixIteration(read->Seq, read->length, &CS::PrefixSearch, 0, 0, this, m_PrefixBaseSkip);
      n = CollectResultsStd(read);
    } catch (int) {
      fallback = true;
    }
    if (fallback) {
      int backup = c_SrchTableBitLen, x = 2;
      while (fallback && (backup + x) <= 20) {
        fallback = false;
        try {
          SetSearchTableBitLen(backup + x);
          rListLength = 0;
          currentState++;
          maxHitNumber = 0.0f;
          currentThresh = 0.0f;
          hpoc = c_SrchTableLen * 0.777f;
          PrefixIteration(read->Seq, read->length, &CS::PrefixSearch, 0, 0, this, m_PrefixBaseSkip);
          n = CollectResultsStd(read);
        } catch (int) {
          fallback = true;
          x += 1;
        }
      }
      SetSearchTableBitLen(backup);
      if (fallback) n = -1;
    }
    return n;
  }
};

CSProbe* g_probe = 0;

}  // namespace

extern "C" {

// Builds encoded reference + k-mer index from a FASTA file with the reference's own code.
int ref_cs_init(const char* fasta) {
  IConfig* c = new IConfig();
  c->referenceFile = strdup(fasta);
  c->queryFile = strdup(fasta);
  c->outputFile = strdup("/dev/null");
  c->skipSave = true;
  c->progress = false;
  _config = c;
  _Log::Init(0, 0);
  _log = &Log;
  CS::Init();
  SequenceProvider.Init();
  g_table = new CompactPrefixTable();
  g_probe = new CSProbe();
  return 0;
}

// Same, but lets the reference write its on-disk caches next to the FASTA file
// (<fasta>-enc.2.ngm, src/SequenceProvider.cpp:250-272; <fasta>-ht-13-2.2.ngm, src/PrefixTable.cpp:534-567).
int ref_cs_init_save(const char* fasta) {
  IConfig* c = new IConfig();
  c->referenceFile = strdup(fasta);
  c->queryFile = strdup(fasta);
  c->outputFile = strdup("/dev/null");
  c->skipSave = false;
  c->progress = false;
  _config = c;
  _Log::Init(0, 0);
  _log = &Log;
  CS::Init();
  SequenceProvider.Init();
  g_table = new CompactPrefixTable();
  g_probe = new CSProbe();
  return 0;
}

// Same as ref_cs_init / ref_cs_init_save (save != 0), at chosen values of ngmlr's options -k, --kmer-skip,
// --bin-size, -s, --min-kmer-hits (not a command-line option; IConfig's default is 0), --subread-length and
// --subread-corridor. They are set in the configuration before anything reads it. The reference caches several of
// them in function-local statics and singletons on first use (GetBin / ResolveBin, CollectResultsStd, ScoreBuffer,
// SequenceProvider), so one process can serve one option set only.
int ref_cs_init_opts(const char* fasta, int k, int kmer_skip, int bin_size, float sensitivity, int min_kmer_hits,
                     int read_part_length, int read_part_corridor, int save) {
  IConfig* c = new IConfig();
  c->referenceFile = strdup(fasta);
  c->queryFile = strdup(fasta);
  c->outputFile = strdup("/dev/null");
  c->skipSave = save == 0;
  c->progress = false;
  c->kmerLength = k;
  c->kmerSkip = kmer_skip;
  c->binSize = bin_size;
  c->sensitivity = sensitivity;
  c->minKmerHits = min_kmer_hits;
  c->readPartLength = read_part_length;
  c->readPartCorridor = read_part_corridor;
  _config = c;
  _Log::Init(0, 0);
  _log = &Log;
  CS::Init();
  SequenceProvider.Init();
  g_table = new CompactPrefixTable();
  g_probe = new CSProbe();
  return 0;
}

unsigned long long ref_cs_concat_len() { return SequenceProvider.GetConcatRefLen(); }
int ref_cs_ref_count() { return SequenceProvider.GetRefCount(); }
// contig name as SAMWriter prints it ("%.*s" of GetRefName)
int ref_cs_ref_name(int n, char* buf, int cap) {
  int len = 0;
  const char* name = SequenceProvider.GetRefName(n, len);
  if (len < cap) {
    memcpy(buf, name, len);
    buf[len] = 0;
  }
  return len;
}
unsigned long long ref_cs_ref_start(int n) { return SequenceProvider.GetRefStart(n); }
unsigned long long ref_cs_ref_len(int n) { return SequenceProvider.GetRefLen(n); }

// DecodeRefSequence(buffer, 0, offset, len): the call ScoreBuffer makes (src/ScoreBuffer.cpp:110)
int ref_cs_decode(unsigned long long offset, unsigned long long len, char* buf) {
  return SequenceProvider.DecodeRefSequence(buf, 0, offset, len) ? 1 : 0;
}
int ref_cs_decode_exact(unsigned long long offset, unsigned long long len, int corridor, char* buf) {
  return SequenceProvider.DecodeRefSequenceExact(buf, offset, len, corridor) ? 1 : 0;
}

// Raw index of unit 0: packed 5-byte Index records and uint32 locations.
const void* ref_cs_index(unsigned* index_len, const unsigned** ref_table, unsigned* ref_table_len,
                         unsigned long long* unit_offset, unsigned* unit_count) {
  *index_len = (unsigned)pow(4.0, (double)CS::prefixBasecount) + 1;
  *ref_table = reinterpret_cast<const unsigned*>(g_table->m_Units[0].RefTable);
  *ref_table_len = g_table->m_Units[0].cRefTableLen;
  *unit_offset = g_table->m_Units[0].Offset;
  *unit_count = g_table->m_UnitCount;
  return g_table->m_Units[0].RefTableIndex;
}

// Extra probes for multi-threaded timing (one per thread, like one CS task per worker thread in
// the reference). table 2^21 entries: RunRead never asks for more than 2^20.
void* ref_cs_probe_create() { return new CSProbe(21); }
void ref_cs_probe_destroy(void* p) { delete static_cast<CSProbe*>(p); }

// StrippedSW::SingleScore through the full library (src/StrippedSW.cpp:162-202)
void* ref_full_ssw_create() { return new StrippedSW(); }
float ref_full_ssw_score(void* h, const char* ref, const char* qry) {
  float r = -1.0f;
  static_cast<StrippedSW*>(h)->SingleScore(0, 0, ref, qry, r, 0);
  return r;
}

int ref_cs_search_p(void* probe, const char* seq, int len, int table_bits, float* scores,
                    unsigned long long* locs, int* reverse, int cap, float* max_hits);

// ScoreBuffer::topNSE (src/ScoreBuffer.cpp:170-192) on one sub-read's scored candidates. tags[] rides
// in Location.m_Location so that the caller can see the permutation std::sort produced.
int ref_score_select(float* scores, unsigned long long* tags, int n, int* mq) {
  if (!_config) {
    _config = new IConfig();
    _Log::Init(0, 0);
    _log = &Log;
  }
  static ScoreBuffer* sb = new ScoreBuffer(new StrippedSW(), 0);
  MappedRead* read = new MappedRead(0, 16);
  LocationScore* tmp = new LocationScore[n > 0 ? n : 1];
  for (int i = 0; i < n; ++i) {
    tmp[i].Score.f = scores[i];
    tmp[i].Location.m_Location = tags[i];
  }
  read->AllocScores(tmp, n);
  delete[] tmp;
  sb->topNSE(read);
  for (int i = 0; i < n; ++i) {
    scores[i] = read->Scores[i].Score.f;
    tags[i] = read->Scores[i].Location.m_Location;
  }
  *mq = read->mappingQlty;
  int kept = read->Calculated;
  delete read;
  return kept;
}

// One (sub-)read through the reference's vote. Outputs in the reference's emission order.
int ref_cs_search(const char* seq, int len, int table_bits, float* scores, unsigned long long* locs,
                  int* reverse, int cap, float* max_hits) {
  return ref_cs_search_p(g_probe, seq, len, table_bits, scores, locs, reverse, cap, max_hits);
}

int ref_cs_search_p(void* probe_, const char* seq, int len, int table_bits, float* scores,
                    unsigned long long* locs, int* reverse, int cap, float* max_hits) {
  CSProbe* probe = static_cast<CSProbe*>(probe_);
  MappedRead* read = new MappedRead(0, len + 16);
  read->Seq = new char[len + 16];
  memcpy(read->Seq, seq, len);
  read->Seq[len] = 0;
  read->length = len;
  int n = probe->search(read, table_bits);
  *max_hits = probe->maxHitNumber;
  int m = read->numScores();
  if (n >= 0) {
    for (int i = 0; i < m && i < cap; ++i) {
      scores[i] = read->Scores[i].Score.f;
      locs[i] = read->Scores[i].Location.m_Location;
      reverse[i] = read->Scores[i].Location.isReverse() ? 1 : 0;
    }
  }
  delete read;
  return n < 0 ? -1 : m;
}

// ---- corridor builders of the caller (src/AlignmentBuffer.cpp:68-197, 1454-1467) ----------------
}  // extern "C"
CorridorLine* getCorridorLinear(int const corridor, char const* readSeq, int& corridorHeight);
CorridorLine* getCorridorFull(int const corridor, char const* readSeq, int& corridorHeight);
CorridorLine* getCorridorEndpoints(Interval const* interval, int const corridor, char const* refSeq,
                                   char const* readSeq, int& corridorHeight, bool const realign);
extern "C" {

static void ensure_config() {
  if (!_config) {
    IConfig* c = new IConfig();
    c->outputFile = strdup("/dev/null");
    _config = c;
    _Log::Init(0, 0);
    _log = &Log;
  }
}

// AlignmentBuffer's two member functions touch no member data except pacbioDebug; they are called on
// zeroed storage instead of a constructed object (the constructor wants a live SAM writer).
static AlignmentBuffer* fake_alignment_buffer() {
  static void* mem = calloc(1, sizeof(AlignmentBuffer) + 64);
  return static_cast<AlignmentBuffer*>(mem);
}

// kind 0: getCorridorLinear(corridor), 1: getCorridorFull(corridor), 2: getCorridorEndpoints(corridor,
// realign), 3: getCorridorEndpointsWithAnchors(multiplier = corridor). Only strlen of the sequences
// matters. Returns corridorHeight.
int ref_corridor(int kind, int qry_len, int ref_len, int corridor, int realign, int n_anchors,
                 const int* a_on_read, const unsigned long long* a_on_ref, const int* a_rev,
                 unsigned long long on_ref_start, int ext_qstart, int read_part_len, int full_read_len,
                 int* off_out, int* len_out) {
  ensure_config();
  std::vector<char> q((size_t)qry_len + 1, 'A'), r((size_t)ref_len + 1, 'A');
  q[qry_len] = 0;
  r[ref_len] = 0;
  Interval iv;
  std::vector<Anchor> anchors((size_t)(n_anchors > 0 ? n_anchors : 1));
  for (int i = 0; i < n_anchors; ++i) {
    anchors[i].onRead = a_on_read[i];
    anchors[i].onRef = (loc)a_on_ref[i];
    anchors[i].isReverse = a_rev[i] != 0;
  }
  iv.anchors = anchors.data();
  iv.anchorLength = n_anchors;
  iv.onRefStart = (loc)on_ref_start;
  int h = 0;
  CorridorLine* c = 0;
  if (kind == 0) c = getCorridorLinear(corridor, q.data(), h);
  else if (kind == 1) c = getCorridorFull(corridor, q.data(), h);
  else if (kind == 2) c = getCorridorEndpoints(&iv, corridor, r.data(), q.data(), h, realign != 0);
  else c = fake_alignment_buffer()->getCorridorEndpointsWithAnchors(&iv, corridor, r.data(), q.data(), h, ext_qstart,
                                                                  read_part_len, full_read_len, realign != 0);
  for (int i = 0; i < h; ++i) {
    off_out[i] = c[i].offset;
    len_out[i] = c[i].length;
  }
  delete[] c;
  iv.anchors = 0;  // not ours to free in ~Interval
  iv.anchorLength = 0;
  return h;
}

int ref_estimate_corridor(int on_read_start, int on_read_stop, long long on_ref_start, long long on_ref_stop) {
  ensure_config();
  Interval iv;
  iv.onReadStart = on_read_start;
  iv.onReadStop = on_read_stop;
  iv.onRefStart = (loc)on_ref_start;
  iv.onRefStop = (loc)on_ref_stop;
  return fake_alignment_buffer()->estimateCorridor(&iv);
}

// AlignmentBuffer::computeAlignment (src/AlignmentBuffer.cpp:226-465): reference window extraction,
// corridor choice per attempt, SingleAlign, retry with a wider corridor. Needs ref_cs_init (the encoded
// genome). Outputs like ref_convex_single_align of oracle/ref_shim.cpp; returns 1 if an Align came
// back, 0 if the reference gave up (returned 0).
int ref_compute_alignment(unsigned long long on_ref_start, unsigned long long on_ref_stop, int n_anchors,
                          const int* a_on_read, const unsigned long long* a_on_ref, const int* a_rev,
                          int corridor, const char* read_seq, int ext_qstart, int ext_qend, int full_read_len,
                          int realign, int full_alignment, int short_read, int* ints, float* floats,
                          char* cigar_out, int cigar_cap, char* md_out, int md_cap, int* nm_out, int nm_cap) {
  ensure_config();
  AlignmentBuffer* ab = fake_alignment_buffer();
  if (!ab->aligner) {
    ab->aligner = new Convex::ConvexAlignFast(0, Config.getScoreMatch(), Config.getScoreMismatch(),
                                              Config.getScoreGapOpen(), Config.getScoreExtendMax(),
                                              Config.getScoreExtendMin(), Config.getScoreGapDecay());
    *const_cast<int*>(&ab->readPartLength) = Config.getReadPartLength();
  }
  Interval iv;
  std::vector<Anchor> anchors((size_t)(n_anchors > 0 ? n_anchors : 1));
  for (int i = 0; i < n_anchors; ++i) {
    anchors[i].onRead = a_on_read[i];
    anchors[i].onRef = (loc)a_on_ref[i];
    anchors[i].isReverse = a_rev[i] != 0;
  }
  iv.anchors = anchors.data();
  iv.anchorLength = n_anchors;
  iv.onRefStart = (loc)on_ref_start;
  iv.onRefStop = (loc)on_ref_stop;
  MappedRead* read = new MappedRead(0, 16);
  read->name = new char[8];
  strcpy(read->name, "r");
  Align* a = ab->computeAlignment(&iv, corridor, read_seq, strlen(read_seq), ext_qstart, ext_qend, full_read_len,
                                  read, realign != 0, full_alignment != 0, short_read != 0);
  iv.anchors = 0;
  iv.anchorLength = 0;
  delete read;
  if (!a) return 0;
  int n = 0;
  const int v[12] = {0, a->QStart, a->QEnd, a->NM, a->alignmentLength, a->cigarOpCount, a->svType,
                     a->firstPosition.refPosition, a->firstPosition.readPosition, a->lastPosition.refPosition,
                     a->lastPosition.readPosition, (int)a->PositionOffset};
  memcpy(ints, v, sizeof(v));
  floats[0] = a->Score;
  floats[1] = a->Identity;
  snprintf(cigar_out, (size_t)cigar_cap, "%s", a->pBuffer1);
  snprintf(md_out, (size_t)md_cap, "%s", a->pBuffer2);
  (void)nm_out; (void)nm_cap; (void)n;
  a->clearBuffer();
  a->clearNmPerPosition();
  delete a;
  return 1;
}

// Stage 0/2 of one read entirely inside the reference's code (used by bench.py's CPU arm so that no
// Python runs between the calls): every 256-bp sub-read through the CS vote (src/CS.cpp:324-398),
// every candidate through DecodeRefSequence (src/ScoreBuffer.cpp:110-116) and StrippedSW::SingleScore.
// Returns the number of candidates scored.
int ref_stage02_read(void* probe, void* ssw, const char* qry, int len, int part_len, int half_corridor,
                     int ref_max_len) {
  float scores[512];
  unsigned long long locs[512];
  int reverse[512];
  float mh = 0.0f;
  std::vector<char> buf((size_t)ref_max_len + 8), fwd((size_t)part_len + 1), rev((size_t)part_len + 1);
  int n_cand = 0;
  for (int k = 0; k + part_len <= len; k += part_len) {
    memcpy(fwd.data(), qry + k, (size_t)part_len);
    fwd[part_len] = 0;
    const int n = ref_cs_search_p(probe, fwd.data(), part_len, 16, scores, locs, reverse, 512, &mh);
    bool have_rev = false;
    for (int j = 0; j < n && j < 512; ++j) {
      if (!SequenceProvider.DecodeRefSequence(buf.data(), 0, locs[j] - (unsigned long long)half_corridor,
                                              (unsigned long long)ref_max_len)) {
        memset(buf.data(), 'N', (size_t)ref_max_len);
        buf[ref_max_len] = 0;
      }
      const char* q = fwd.data();
      if (reverse[j]) {
        if (!have_rev) {  // MappedRead::computeReverseSeq: complement, reversed
          for (int i = 0; i < part_len; ++i) {
            const char c = fwd[part_len - 1 - i];
            rev[i] = c == 'A' ? 'T' : (c == 'T' ? 'A' : (c == 'C' ? 'G' : (c == 'G' ? 'C' : c)));
          }
          rev[part_len] = 0;
          have_rev = true;
        }
        q = rev.data();
      }
      float r = -1.0f;
      static_cast<StrippedSW*>(ssw)->SingleScore(0, 0, buf.data(), q, r, 0);
      ++n_cand;
    }
  }
  return n_cand;
}

}  // extern "C"

// ---- SAM writer (SURVEY 8(f)4): the UNMODIFIED SAMWriter / GenericReadWriter::WriteRead driven on records
// the test makes up; output captured through a FileWriter that appends every flush to a string.
#include "SAMWriter.h"

namespace {

class CaptureWriter : public FileWriter {
 public:
  std::string text;

 protected:
  void doFlush(int& bufferPosition, int const, char* writeBuffer, bool) override {
    text.append(writeBuffer, (size_t)bufferPosition);
    bufferPosition = 0;
  }
};

}  // namespace

extern "C" {

struct RefSamAln {
  unsigned long long ref_pos;
  int ref_id, reverse;
  float score;
  int mq, nm;
  float identity;
  int qstart, qend, sv_type, primary, skip, cigar_ops;
  const char* cigar;
  const char* md;
};

struct RefSamRead {
  const char* name;
  const char* seq;
  const char* qual;  // NULL: MappedRead::qlty == 0
  int length, n_aln;
  long long first_aln;
  int mapped, empty;
};

// needs ref_cs_init(fasta) (SequenceProvider holds the contig names). rg_id may be NULL.
// what = 0: header only, 1: records only. Returns the number of bytes (copied when they fit cap).
long long ref_sam_write(int what, const RefSamRead* reads, int n_reads, const RefSamAln* alns, int bam_fix,
                        int write_unmapped, const char* rg_id, const char* const* rg_fields, const char* cmdline,
                        char* out, long long cap) {
  IConfig* c = _config;
  c->bamCigarFix = bam_fix != 0;
  c->writeUnmapped = write_unmapped != 0;
  c->rgId = const_cast<char*>(rg_id);
  char** f[11] = {&c->rgSm, &c->rgLb, &c->rgPl, &c->rgDs, &c->rgDt, &c->rgPu, &c->rgPi, &c->rgPg, &c->rgCn, &c->rgFo, &c->rgKs};
  for (int k = 0; k < 11; ++k) *f[k] = rg_fields ? const_cast<char*>(rg_fields[k]) : 0;
  c->fullCommandLineCall = const_cast<char*>(cmdline);
  CaptureWriter cap_writer;
  {
    SAMWriter w(&cap_writer);
    if (what == 0) {
      w.WriteProlog();
    } else {
      for (int i = 0; i < n_reads; ++i) {
        const RefSamRead& r = reads[i];
        MappedRead* read = new MappedRead(i, r.length + 16);
        strncpy(read->name, r.name, 249);
        read->name[249] = 0;
        read->length = r.length;
        read->Seq = new char[r.length + 16];
        memset(read->Seq, 0, r.length + 16);
        memcpy(read->Seq, r.seq, r.length);
        read->computeReverseSeq();
        if (r.qual) {
          const size_t ql = strlen(r.qual);
          read->qlty = new char[ql + 1];
          memcpy(read->qlty, r.qual, ql + 1);
        }
        if (r.empty) read->SetFlag(NGMNames::Empty);
        read->Calculated = r.n_aln;
        if (r.n_aln > 0) {
          read->Scores = new LocationScore[r.n_aln];
          read->Alignments = new Align[r.n_aln];
          for (int j = 0; j < r.n_aln; ++j) {
            const RefSamAln& a = alns[r.first_aln + j];
            read->Scores[j].Score.f = a.score;
            read->Scores[j].Location.m_Location = a.ref_pos;
            read->Scores[j].Location.setRefId(a.ref_id);
            read->Scores[j].Location.setReverse(a.reverse != 0);
            Align& al = read->Alignments[j];
            al.pBuffer1 = new char[strlen(a.cigar) + 1];
            strcpy(al.pBuffer1, a.cigar);
            al.pBuffer2 = new char[strlen(a.md) + 1];
            strcpy(al.pBuffer2, a.md);
            al.MQ = a.mq;
            al.NM = a.nm;
            al.Identity = a.identity;
            al.QStart = a.qstart;
            al.QEnd = a.qend;
            al.svType = a.sv_type;
            al.primary = a.primary != 0;
            al.skip = a.skip != 0;
            al.cigarOpCount = a.cigar_ops;
          }
        }
        w.WriteRead(read, r.mapped != 0);
        delete read;
      }
    }
  }  // ~SAMWriter flushes the rest
  const long long n = (long long)cap_writer.text.size();
  if (out && n <= cap) memcpy(out, cap_writer.text.data(), (size_t)n);
  return n;
}

}  // extern "C"
