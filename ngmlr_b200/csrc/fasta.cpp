// ngmlr_b200/csrc/fasta.cpp -- the reference reader of ngmlr_b200_load_reference.
//
// _SequenceProvider::Init (src/SequenceProvider.cpp:274-400) reads the reference with `while (kseq_read(seq) >= 0)`
// over gzopen(path), so plain and gzip files alike. This reader yields the same records:
//   - a record starts at the first '>' or '@' of the file, or after a FASTQ record at the next '>' or '@' anywhere;
//     after a FASTA record, at a line that starts with '>' or '@';
//   - the name runs up to the first whitespace; the rest of the header line (the comment) is dropped;
//   - sequence lines are concatenated as they are (a '>' inside a line is a sequence character); empty lines are
//     skipped; one '\r' at the end of a line is dropped when the sequence then holds more than one character;
//   - a line that starts with '+' ends the sequence and starts the qualities, which are skipped; a FASTQ record whose
//     qualities are missing or of another length ends the file, as the reader's -2 ends the loop;
//   - the end-of-file tests depend on 16 KiB reads, as they do in the reference, so a final line of a file whose size
//     is a multiple of 16 KiB behaves as it does there.
// A record of 2^31 or more bases is refused: the reference's reader returns its length as an int.
#include "fasta.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace nb {

namespace {

constexpr size_t CHUNK = 16384;

bool is_space(int c) { return c == ' ' || c == '\t' || c == '\n' || c == '\v' || c == '\f' || c == '\r'; }

struct Input {
  StreamFile* f = nullptr;
  unsigned char buf[CHUNK];
  size_t b = 0, e = 0;
  bool eof = false, bad = false;
  ~Input() { close_stream(f); }
  // refill: false when nothing more can be read
  bool fill() {
    const int64_t n = read_stream(f, buf, CHUNK);
    if (n < 0) {
      bad = true;
      eof = true;
      return false;
    }
    b = 0;
    e = (size_t)n;
    if (e < CHUNK) eof = true;
    return e > 0;
  }
  int get() {
    if (b >= e) {
      if (eof || !fill()) return -1;
    }
    return buf[b++];
  }
  // nothing buffered and the last read came up short: a line / token read returns at once
  bool spent() const { return b >= e && eof; }
  // Appends the bytes up to the next '\n' (consumed, not appended) or the end of the file through put(p, n).
  template <typename Put>
  void line(Put put) {
    for (;;) {
      if (b >= e) {
        if (eof || !fill()) return;
      }
      const unsigned char* p = buf + b;
      const unsigned char* nl = static_cast<const unsigned char*>(memchr(p, '\n', e - b));
      const size_t n = nl ? (size_t)(nl - p) : e - b;
      put(reinterpret_cast<const char*>(p), n);
      b += n;
      if (nl) {
        ++b;
        return;
      }
    }
  }
};

}  // namespace

void FastaText::release_text() {
  if (text) {
    if (pinned)
      cudaFreeHost(text);
    else
      free(text);
  }
  text = nullptr;
  size = cap = 0;
}

FastaText::~FastaText() { release_text(); }

uint64_t FastaText::alloc_bytes() const {
  uint64_t size = 1000;
  for (const FastaRecord& r : recs) size += (r.len | 1) + 1 + 1000;
  return ((size / 2) | 1) + 1;
}

uint64_t concat_len_of(const std::vector<uint64_t>& lens) {
  uint64_t bytes = 500;
  for (uint64_t n : lens)
    if (n > 10) bytes += (n + 1) / 2 + 500;
  return bytes * 2 - 1;
}

int read_fasta(const char* path, bool pinned, uint64_t max_concat_len, FastaText& out, std::string& err, int device,
               cudaStream_t stream, StreamCounters* counters) {
  char msg[512];
  auto fail = [&](int rc, const char* fmt, const char* a = "", unsigned long long v = 0) {
    snprintf(msg, sizeof msg, fmt, a, v);
    err = msg;
    return rc;
  };
  FILE* probe = fopen(path, "rb");
  if (!probe) return fail(-2, "cannot open %s", path);
  fseek(probe, 0, SEEK_END);
  const long file_size = ftell(probe);
  fclose(probe);
  Input in;
  auto read_failed = [&]() {
    const std::string& e = stream_error(in.f);
    err = std::string(path) + ": " + (e.empty() ? "read error (corrupt gzip stream?)" : e);
    return -3;
  };
  in.f = open_stream(path);
  if (!in.f) return fail(-2, "cannot open %s", path);
  // a BGZF reference is inflated in rounds of at least 256 MiB: this reader asks for 16 KiB at a time
  if (device >= 0 && !bind_stream_device(in.f, device, stream, 256ll << 20)) return read_failed();
  out.pinned = pinned;
  bool oom = false;
  // room for n more bytes of text: the file size for plain files, grown by doubling for compressed ones
  auto reserve = [&](uint64_t n) {
    if (out.size + n <= out.cap) return true;
    uint64_t want = std::max<uint64_t>(out.cap ? out.cap * 2 : (uint64_t)file_size + 4096, out.size + n);
    char* q = nullptr;
    if (pinned) {
      if (cudaMallocHost(&q, want) != cudaSuccess) q = nullptr;
    } else {
      q = static_cast<char*>(malloc(want));
    }
    if (!q) {
      oom = true;
      return false;
    }
    if (out.size) memcpy(q, out.text, out.size);
    const uint64_t size = out.size;
    out.release_text();
    out.text = q;
    out.size = size;
    out.cap = want;
    return true;
  };
  uint64_t kept_bytes = 500;  // binRefIndex of the records so far (the concatenated genome is 2 x this - 1)
  uint64_t start = 0;         // text offset of the current record's sequence
  bool too_long = false;
  auto append = [&](const char* p, size_t n) {
    if (!n || oom) return;
    if (!reserve(n)) return;
    memcpy(out.text + out.size, p, n);
    out.size += n;
  };
  auto over_limit = [&]() {
    const uint64_t len = out.size - start;
    if (len >= (1ull << 31)) too_long = true;
    return too_long || (len > 10 && (kept_bytes + (len + 1) / 2 + 500) * 2 - 1 > max_concat_len);
  };
  std::string name, qual;
  int head = 0;  // the header character of the next record has been read
  for (;;) {
    if (!head) {
      int c;
      while ((c = in.get()) != -1 && c != '>' && c != '@') {
      }
      if (c == -1) break;
      head = c;
    }
    // name: up to the first whitespace
    if (in.spent()) break;
    name.clear();
    int delim = 0;
    for (int c; (c = in.get()) != -1;) {
      if (is_space(c)) {
        delim = c;
        break;
      }
      name.push_back((char)c);
    }
    if (delim != '\n' && !in.spent()) in.line([](const char*, size_t) {});  // the comment
    // sequence
    start = out.size;
    int c;
    while ((c = in.get()) != -1 && c != '>' && c != '+' && c != '@') {
      if (c == '\n') continue;
      const char ch = (char)c;
      append(&ch, 1);
      if (!in.spent()) {
        in.line(append);
        if (out.size - start > 1 && out.text[out.size - 1] == '\r') --out.size;
      }
      if (oom) break;
      if (over_limit()) break;
    }
    if (oom) return fail(-4, "out of host memory reading %s", path);
    if (too_long) return fail(-5, "%s: a sequence of %llu or more bases (the reference reads lengths as int)", path,
                              1ull << 31);
    if (over_limit())
      return fail(-6, "%s: the genome exceeds %llu positions, the most one k-mer table unit holds", path,
                  (unsigned long long)max_concat_len);
    const uint64_t len = out.size - start;
    head = (c == '>' || c == '@') ? c : head;
    if (c == '+') {
      int d;
      while ((d = in.get()) != -1 && d != '\n') {
      }
      if (d == -1) {  // no quality line: the reference's reader returns -2 and the reference stops reading
        out.size = start;
        break;
      }
      qual.clear();
      while (!in.spent()) {
        in.line([&](const char* p, size_t n) { qual.append(p, n); });
        if (qual.size() > 1 && qual.back() == '\r') qual.pop_back();
        if (qual.size() >= len) break;
      }
      head = 0;
      if (qual.size() != len) {
        out.size = start;
        break;
      }
    }
    if (in.bad) return read_failed();
    out.recs.push_back(FastaRecord{name, start, len});
    if (len > 10) kept_bytes += (len + 1) / 2 + 500;
  }
  if (in.bad) return read_failed();
  if (counters) *counters = stream_counters(in.f);
  return 0;
}

}  // namespace nb
