// oracle/read_provider_shim.cpp -- TEST INFRASTRUCTURE ONLY.
//
// extern "C" driver around the UNMODIFIED reference's read input, built by oracle/read_provider.mk into
// oracle/_ref/libngmlr_reads.so on top of oracle/_ref/libngmlr_full.so (the whole reference, whose configuration and
// log globals it shares): ReadProvider::GenerateRead -> NextRead -> FastXParser -> kseq_read -> IParser::copyToRead
// (src/ReadProvider.cpp:136-255, src/FastxParser.h, src/IParser.h:51-117, src/kseq.h).
#include <cstdio>
#include <cstdlib>
#include <cstring>

#define private public
#define protected public
#include "IConfig.h"
#undef private
#undef protected
#include "Log.h"
#include "MappedRead.h"
#include "ReadProvider.h"

extern ILog const* _log;
extern IConfig* _config;

extern "C" {

// Reads `path` at --subread-length read_part_length the way _NGM::GetNextReadBatch does (src/NGM.cpp:190-246: until
// GenerateRead returns false) and appends every read to out_path: int32 name length, name, int32 length (MappedRead::
// length), int32 Empty flag, int32 n, n bytes of Seq (length bytes; length - 1 for an Empty read, whose last byte the
// reference leaves uninitialised), int32 m, m bytes of qlty (strlen). A read whose quality length differs ends the
// process: ngmlr's Log.Error("Read %s: Length of read not equal length of quality values.") exits with status 1 -- so
// call this in a process of its own and read the name from its stderr. Returns the number of reads.
int ref_read_file(const char* path, int read_part_length, const char* out_path) {
  IConfig* c = new IConfig();
  c->queryFile = strdup(path);
  c->outputFile = strdup("/dev/null");
  c->readPartLength = read_part_length;
  c->progress = false;
  _config = c;
  _Log::Init(0, 0);
  _log = &Log;
  FILE* out = fopen(out_path, "wb");
  if (!out) return -1;
  ReadProvider* rp = new ReadProvider();
  rp->init();
  int n = 0;
  for (;; ++n) {
    MappedRead* r = 0;
    if (!rp->GenerateRead(n * 2000, r, 0, r)) break;
    const int name_len = (int)strlen(r->name), empty = r->HasFlag(NGMNames::Empty) ? 1 : 0;
    const int seq_len = empty ? r->length - 1 : r->length, qual_len = r->qlty ? (int)strlen(r->qlty) : 0;
    fwrite(&name_len, 4, 1, out);
    fwrite(r->name, 1, (size_t)name_len, out);
    fwrite(&r->length, 4, 1, out);
    fwrite(&empty, 4, 1, out);
    fwrite(&seq_len, 4, 1, out);
    fwrite(r->Seq, 1, (size_t)seq_len, out);
    fwrite(&qual_len, 4, 1, out);
    if (qual_len) fwrite(r->qlty, 1, (size_t)qual_len, out);
    fflush(out);
    rp->DisposeRead(r);
  }
  fclose(out);
  delete rp;
  return n;
}

}  // extern "C"
