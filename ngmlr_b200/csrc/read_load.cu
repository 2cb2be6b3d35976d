// ngmlr_b200/csrc/read_load.cu -- reads from a FASTA / FASTQ file, parsed on the device (ngmlr_b200_reads_load).
//
// ngmlr reads its query file with ReadProvider::NextRead -> FastXParser -> kseq_read -> IParser::copyToRead
// (src/ReadProvider.cpp:136-187, src/IParser.h:51-117, src/kseq.h:171-211) on one thread under GetNextReadBatch's
// mutex. Here a chunk of the byte stream (plain, or inflated by zlib on the host) goes to the device once and:
//   1. line table: one warp per 2 KiB segment counts '\n' with ballots; a scan gives every newline its rank and a
//      second pass writes the positions. The same pass notes each segment's first '>' / '@' byte.
//   2. per line: first byte, trailing '\r' count, and what the line adds to a sequence and to a quality string under
//      kseq's '\r' rule (a trailing '\r' goes when the string then holds more than one character); prefix sums.
//   3. every line is resolved as if a record's header sat on it: its sequence lines run to the next line that starts
//      with '>' / '+' / '@' (binary search over those lines); after a '+' line the quality lines are read until they
//      are at least as long as the sequence (binary search on the prefix sums; a thread replays kseq line by line
//      where '\r' runs make the sums inexact); the next header is the next '>' / '@' byte after that. A header may sit
//      inside a line (after a FASTQ record kseq takes the next '>' / '@' byte anywhere), but where a record ends
//      depends only on the line its header is on.
//   4. the true records are the chain of "next" from the chunk's first '>' / '@' byte: stored jumps of 1, 2, 4, ...
//      2^(LEVELS-1) records, one thread walking the longest jumps, and a pass per shorter level marking the records in
//      between (the records k * 2^l along the chain are those at k * 2^(l+1) and one jump of 2^l from them).
//   5. per batch: sequence bytes gathered (one warp per line) into the resident read arena with toupper and the
//      ACGT / N mapping, NUL padded as ngmlr_b200_reads_upload lays them out; the sub-read table written on the device;
//      the normalised bases copied back (sam_format prints them from host memory).
// Names and single-line qualities point into the host copy of the chunk; multi-line qualities are assembled on the
// host by kseq's rule. The bytes after the last complete record move to the front of the next chunk.
//
// End of the stream: kseq reads 16 KiB blocks and notices the end only when a read comes up short. When the stream
// length is a multiple of 16 KiB one more read returns nothing, and three things differ (all at the very end): a
// header character that is the last byte starts an empty record with an empty name; a last line "\r" without newline
// loses its '\r'; a quality string still ending in '\r' after the last line loses one more.
#include <cub/cub.cuh>
#include <zlib.h>

#include "fasta.h"
#include "runtime.h"

using namespace nb;

namespace {

constexpr int SEG = 2048;           // bytes per warp in the line-table pass
constexpr int LEVELS = 8;           // stored jumps along the record chain: 2^0 .. 2^(LEVELS-1) records
constexpr int64_t LINE_BYTES = 32;  // the line table of a chunk holds at most chunk capacity / LINE_BYTES lines
constexpr int NAME_CUT = 249;       // IParser::MAX_READNAME_LENGTH - 1
constexpr int64_t DEFAULT_CHUNK = 256ll << 20;
constexpr int64_t MAX_BASES = 1ll << 31;

enum : int8_t {
  K_NEXT = 0,        // a record; the next header follows in the chunk
  K_END = 1,         // a record; the stream ends after it
  K_TAIL = 2,        // a record; no header follows in the chunk: the next chunk starts where it ends
  K_INCOMPLETE = 3,  // the record runs past the chunk
  K_DROP = 4,        // qualities missing or of another length (kseq's -2): ngmlr drops it and stops reading
  K_NONE = 5,        // a header character that is the stream's last byte (no record unless the length is k x 16 KiB)
};

struct Chunk {
  const uint8_t* c;
  int64_t n;  // bytes resolved (the line table may end before the chunk does)
  const int64_t* nl;
  int n_nl, n_lines;
  const int32_t* tr;   // trailing '\r' characters of each line
  const uint8_t* fb;   // first byte of each line (0 for an empty line)
  const int64_t* sp;   // exclusive prefix sums of the lines' sequence / quality contributions, n_lines + 1
  const int64_t* qp;
  const int32_t* irr;  // exclusive prefix count of lines whose quality contribution depends on what came before
  const int32_t* stops;  // lines starting with '>' / '+' / '@', ascending
  int n_stops;
  const int64_t* seg_mark;  // first '>' / '@' of each segment, or -1
  const int32_t* mark_segs;
  int n_mark_segs;
  int at_eof, late_eof;
};

__device__ __forceinline__ int64_t line_start(const Chunk& k, int j) { return j == 0 ? 0 : k.nl[j - 1] + 1; }
__device__ __forceinline__ int64_t line_end(const Chunk& k, int j) { return j < k.n_nl ? k.nl[j] : k.n; }
__device__ __forceinline__ bool is_marker(uint8_t b) { return b == '>' || b == '@'; }
__device__ __forceinline__ bool is_space(uint8_t b) { return b == ' ' || (b >= '\t' && b <= '\r'); }

template <typename T>
__device__ int lower_bound_dev(const T* a, int n, T v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// the first '>' / '@' byte at or after p, or -1
__device__ int64_t next_marker(const Chunk& k, int64_t p) {
  if (p >= k.n) return -1;
  const int64_t seg = p / SEG, seg_end = min(k.n, (seg + 1) * SEG);
  for (int64_t q = p; q < seg_end; ++q)
    if (is_marker(k.c[q])) return q;
  const int i = lower_bound_dev(k.mark_segs, k.n_mark_segs, (int32_t)(seg + 1));
  if (i >= k.n_mark_segs) return -1;
  const int64_t q = k.seg_mark[k.mark_segs[i]];
  return q < k.n ? q : -1;
}

struct RecInfo {
  int8_t kind, fastq, fix, single_qual;
  int32_t s, stop, first, q0, qk;
  int64_t seq_len, qual_len, next_pos, end;
  int32_t next_line;
};

// kseq_read from a header on line h: where the record's parts lie and where the next header is.
__device__ RecInfo resolve(const Chunk& k, int h) {
  RecInfo r;
  memset(&r, 0, sizeof(r));
  r.next_line = k.n_lines;
  r.next_pos = -1;
  r.qk = -1;
  const bool h_nl = h < k.n_nl;
  if (!h_nl && !k.at_eof) {
    r.kind = K_INCOMPLETE;
    return r;
  }
  const int s = h + 1;
  const int stop_i = lower_bound_dev(k.stops, k.n_stops, (int32_t)s);
  const int stop = stop_i < k.n_stops ? k.stops[stop_i] : k.n_lines;
  int f = s;  // empty lines are skipped
  while (f < stop && line_end(k, f) == line_start(k, f)) ++f;
  r.s = s;
  r.stop = stop;
  r.first = f;
  // a first sequence line "\r" keeps its '\r' (the string holds one character); the per-line sums dropped it
  if (f < stop && line_end(k, f) - line_start(k, f) == 1 && k.tr[f] == 1 && k.sp[f + 1] == k.sp[f]) r.fix = 1;
  r.seq_len = k.sp[stop] - k.sp[s] + r.fix;
  if (stop == k.n_lines) {
    r.kind = k.at_eof ? K_END : K_INCOMPLETE;
    r.end = k.n;
    return r;
  }
  if (k.fb[stop] != '+') {
    r.kind = K_NEXT;
    r.next_line = stop;
    r.next_pos = line_start(k, stop);
    r.end = r.next_pos;
    return r;
  }
  r.fastq = 1;
  if (stop >= k.n_nl) {  // the '+' line has no end: kseq's "no quality string"
    r.kind = k.at_eof ? K_DROP : K_INCOMPLETE;
    return r;
  }
  const int q0 = stop + 1;
  r.q0 = q0;
  if (q0 == k.n_lines) {  // nothing after the '+' line: no quality line is read
    if (!k.at_eof) {
      r.kind = K_INCOMPLETE;
      return r;
    }
    r.qual_len = 0;
    r.qk = stop;
    r.end = k.n;
    r.kind = r.seq_len == 0 ? K_END : K_DROP;
    return r;
  }
  // the first line q0 .. kk whose qualities reach the sequence length (kseq reads at least one line)
  const int64_t target = k.qp[q0] + r.seq_len;
  int lo = q0 + 1, hi = k.n_lines + 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (k.qp[mid] >= target) hi = mid;
    else lo = mid + 1;
  }
  const bool found = lo <= k.n_lines;
  int kk = found ? lo - 1 : k.n_lines - 1;
  if (!k.at_eof && (!found || kk >= k.n_nl)) {
    r.kind = K_INCOMPLETE;
    return r;
  }
  int64_t qlen = k.qp[kk + 1] - k.qp[q0];
  if (k.irr[kk + 1] - k.irr[q0] > 0) {  // replay kseq: Q characters, the last rr of them '\r'
    int64_t Q = 0, rr = 0;
    bool done = false;
    int j = q0;
    for (; j < k.n_lines; ++j) {
      const int64_t m = line_end(k, j) - line_start(k, j), t = k.tr[j];
      Q += m;
      rr = t == m ? rr + m : t;
      if (Q > 1 && rr > 0) --Q, --rr;
      if (Q >= r.seq_len) {
        done = true;
        break;
      }
    }
    if (!done) {
      if (!k.at_eof) {
        r.kind = K_INCOMPLETE;
        return r;
      }
      j = k.n_lines - 1;
      // a stream of k x 16 KiB that ends with '\n': one more read, one more application of the rule
      if (k.late_eof && k.n_lines == k.n_nl && Q > 1 && rr > 0) --Q;
    } else if (!k.at_eof && j >= k.n_nl) {
      r.kind = K_INCOMPLETE;
      return r;
    }
    kk = j;
    qlen = Q;
  } else {
    r.single_qual = kk == q0;
  }
  r.qk = kk;
  r.qual_len = qlen;
  r.end = kk < k.n_nl ? k.nl[kk] + 1 : k.n;
  if (qlen != r.seq_len) {
    r.kind = K_DROP;
    return r;
  }
  const int64_t p = next_marker(k, r.end);
  if (p < 0) {
    r.kind = k.at_eof ? K_END : K_TAIL;
    return r;
  }
  r.kind = K_NEXT;
  r.next_pos = p;
  r.next_line = lower_bound_dev(k.nl, k.n_nl, p);
  return r;
}

// ---- line table ---------------------------------------------------------------------------------------------------
__global__ void k_segments(const uint8_t* __restrict__ c, int64_t n, int64_t n_segs, int64_t* seg_cnt,
                           int64_t* seg_mark) {
  const int64_t seg = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  if (seg >= n_segs) return;
  const int64_t b = seg * SEG, e = min(n, b + SEG);
  int64_t cnt = 0, mark = -1;
  for (int64_t p = b; p < e; p += 32) {
    const uint8_t x = p + lane < e ? c[p + lane] : 0;
    cnt += __popc(__ballot_sync(0xffffffffu, x == '\n'));
    const unsigned mk = __ballot_sync(0xffffffffu, is_marker(x));
    if (mark < 0 && mk) mark = p + __ffs(mk) - 1;
  }
  if (lane == 0) {
    seg_cnt[seg] = cnt;
    seg_mark[seg] = mark;
  }
}

__global__ void k_newlines(const uint8_t* __restrict__ c, int64_t n, int64_t n_segs, const int64_t* seg_base,
                           int64_t limit, int64_t* nl) {
  const int64_t seg = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  if (seg >= n_segs) return;
  const int64_t b = seg * SEG, e = min(n, b + SEG);
  int64_t rank = seg_base[seg];
  if (rank >= limit) return;
  for (int64_t p = b; p < e; p += 32) {
    const bool is_nl = p + lane < e && c[p + lane] == '\n';
    const unsigned m = __ballot_sync(0xffffffffu, is_nl);
    const int64_t r = rank + __popc(m & ((1u << lane) - 1));
    if (is_nl && r < limit) nl[r] = p + lane;
    rank += __popc(m);
  }
}

// per line: first byte, trailing '\r', sequence / quality contributions, the irregular-quality flag, the stop flag
__global__ void k_lines(Chunk k, int64_t* sc, int64_t* qc, int32_t* ir, uint8_t* stop_flag, uint8_t* fb, int32_t* tr) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j > k.n_lines) return;
  if (j == k.n_lines) {  // the sums' last entry
    sc[j] = qc[j] = 0;
    ir[j] = 0;
    return;
  }
  const int64_t b = line_start(k, j), e = line_end(k, j), m = e - b;
  int64_t t = 0;
  while (t < m && k.c[e - 1 - t] == '\r') ++t;
  const uint8_t f = m > 0 ? k.c[b] : 0;
  fb[j] = f;
  tr[j] = (int32_t)(t < 0x7fffffff ? t : 0x7fffffff);
  // the rule is applied after every line except a one-character last line without '\n' at a short-read end
  const bool rule = j < k.n_nl || m > 1 || k.late_eof;
  sc[j] = m == 0 ? 0 : m - (t >= 1 && rule ? 1 : 0);
  qc[j] = m - (t >= 1 ? 1 : 0);
  ir[j] = (t >= 2 || (m == 1 && t == 1)) ? 1 : 0;
  stop_flag[j] = m > 0 && (f == '>' || f == '+' || f == '@');
}

__global__ void k_resolve(Chunk k, int32_t* next0, int64_t* next_pos) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j > k.n_lines) return;
  if (j == k.n_lines) {
    next0[j] = k.n_lines;
    return;
  }
  const RecInfo r = resolve(k, j);
  next0[j] = r.next_line;
  next_pos[j] = r.next_pos;
}

__global__ void k_jump(const int32_t* prev, int32_t* next, int n) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j <= n) next[j] = prev[prev[j]];
}

// the chain's first header, and its records 0, 2^(LEVELS-1), 2 x 2^(LEVELS-1), ...
__global__ void k_chain_start(Chunk k, const int32_t* top, uint8_t* mark, int64_t* first_pos) {
  const int64_t p = next_marker(k, 0);
  *first_pos = p;
  if (p < 0) return;
  int v = lower_bound_dev(k.nl, k.n_nl, p);
  mark[v] = 1;
  while (top[v] != k.n_lines) {
    v = top[v];
    mark[v] = 1;
  }
}

__global__ void k_mark(const int32_t* jump, uint8_t* mark, int n) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n && mark[j] && jump[j] != n) mark[jump[j]] = 1;
}

}  // namespace

// One record of a chunk as the host reads it.
struct LoadRec {
  int64_t hdr, name_end;         // header character, first byte after the name
  int64_t seq_len, qual_len, end;
  int64_t qual_start;            // first quality line (FASTQ)
  int32_t s, stop, first;        // sequence lines [s, stop), the first non-empty one
  int8_t kind, fastq, fix, single_qual;
};

namespace {

__global__ void k_records(Chunk k, const int32_t* rec_lines, int n_recs, const int64_t* next_pos,
                          const int64_t* first_pos, LoadRec* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_recs) return;
  const int h = rec_lines[i];
  const RecInfo r = resolve(k, h);
  LoadRec o;
  o.hdr = i == 0 ? *first_pos : next_pos[rec_lines[i - 1]];
  int64_t q = o.hdr + 1;
  while (q < k.n && !is_space(k.c[q])) ++q;
  o.name_end = q;
  o.seq_len = r.seq_len;
  o.qual_len = r.qual_len;
  o.end = r.end;
  o.qual_start = r.fastq && r.q0 < k.n_lines ? line_start(k, r.q0) : 0;
  o.s = r.s;
  o.stop = r.stop;
  o.first = r.first;
  o.kind = r.kind;
  o.fastq = r.fastq;
  o.fix = r.fix;
  o.single_qual = r.single_qual;
  if (o.hdr == k.n - 1 && k.at_eof && !k.late_eof) o.kind = K_NONE;
  out[i] = o;
}

__device__ __forceinline__ uint8_t base_of(uint8_t x) {
  const uint8_t u = (x >= 'a' && x <= 'z') ? x - 32 : x;
  return (u == 'A' || u == 'C' || u == 'G' || u == 'T') ? u : 'N';
}

// one warp per line of lines [lo, hi): the sequence bytes of records [r0, r1) into the read arena
__global__ void k_gather(Chunk k, const LoadRec* recs, int r0, int r1, int lo, int hi, const uint64_t* read_off,
                         uint8_t* dst) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  const int j = lo + (int)w;
  if (j >= hi) return;
  // the record whose sequence lines hold j: the last of r0 .. r1 - 1 with s <= j
  int a = r0, b = r1;
  while (a < b) {
    const int mid = (a + b) >> 1;
    if (recs[mid].s <= j) a = mid + 1;
    else b = mid;
  }
  const int r = a - 1;
  if (r < r0) return;
  const LoadRec& R = recs[r];
  if (j >= R.stop || j < R.first) return;
  int64_t cnt = k.sp[j + 1] - k.sp[j];
  int64_t off = k.sp[j] - k.sp[R.s];
  if (j == R.first) cnt += R.fix;
  else off += R.fix;
  const uint8_t* src = k.c + line_start(k, j);
  uint8_t* d = dst + read_off[r - r0] + off;
  for (int64_t x = lane; x < cnt; x += 32) d[x] = base_of(src[x]);
}

__global__ void k_subreads(const LoadRec* recs, int r0, int n, const uint64_t* read_off, const uint64_t* sub_start,
                           int read_part_length, uint64_t* soff, int32_t* slen) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int len = (int)recs[r0 + i].seq_len;
  const int parts = len / read_part_length;
  uint64_t s = sub_start[i];
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

struct HasMark {
  const int64_t* seg_mark;
  __device__ bool operator()(int32_t s) const { return seg_mark[s] >= 0; }
};

inline int blocks(int64_t n, int t) { return (int)std::max<int64_t>(1, (n + t - 1) / t); }

}  // namespace

struct ngmlr_b200_read_file {
  std::string path, error, dropped;
  StreamFile* in = nullptr;
  int device = -1;
  int64_t chunk_cap = 0;
  PinBuf<uint8_t> h_chunk;
  int64_t n_host = 0;       // bytes in h_chunk
  int64_t n_res = 0;        // bytes the line table covers
  bool stream_eof = false, late_eof = false;
  int64_t stream_bytes = 0;
  // the records of the current chunk
  std::vector<LoadRec> recs;
  int n_good = 0, next_rec = 0;
  bool ended = false, drop_pending = false, dropped_reported = false;
  int64_t tail = 0;         // where the next chunk starts in h_chunk
  bool resolved = false;
  // device state
  DevBuf<uint8_t> d_chunk, d_tmp, d_fb, d_stop_flag, d_mark;
  DevBuf<int64_t> d_seg_cnt, d_seg_mark, d_nl, d_sp, d_qp, d_next_pos, d_scalar;
  DevBuf<int32_t> d_ir, d_tr, d_stops, d_mark_segs, d_jump, d_rec_lines, d_count;
  DevBuf<LoadRec> d_recs;
  DevBuf<uint64_t> d_layout;
  PinBuf<int64_t> h_small;
  PinBuf<uint64_t> h_layout;
  Chunk k{};
  // the strings of the last load
  PinBuf<uint8_t> h_seq;
  std::vector<std::string> quals;
  int64_t records = 0, device_peak = 0;
  float read_ms = 0, parse_ms = 0, gather_ms = 0;
  size_t device_bytes() const {
    return d_chunk.owned_bytes() + d_tmp.owned_bytes() + d_fb.owned_bytes() + d_stop_flag.owned_bytes() +
           d_mark.owned_bytes() + d_seg_cnt.owned_bytes() + d_seg_mark.owned_bytes() + d_nl.owned_bytes() +
           d_sp.owned_bytes() + d_qp.owned_bytes() + d_next_pos.owned_bytes() + d_scalar.owned_bytes() +
           d_ir.owned_bytes() + d_tr.owned_bytes() + d_stops.owned_bytes() + d_mark_segs.owned_bytes() +
           d_jump.owned_bytes() + d_rec_lines.owned_bytes() + d_count.owned_bytes() + d_recs.owned_bytes() +
           d_layout.owned_bytes();
  }
};

namespace {

using RF = ngmlr_b200_read_file;

#define RCU(call)                                                                                   \
  do {                                                                                              \
    cudaError_t e__ = (call);                                                                       \
    if (e__ != cudaSuccess)                                                                         \
      return ctx->fail("reads_load: %s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

// cub's scratch, grown as needed
template <typename F>
cudaError_t with_tmp(RF* f, F fn) {
  size_t need = 0;
  cudaError_t e = fn(nullptr, need);
  if (e != cudaSuccess) return e;
  if ((e = f->d_tmp.reserve(std::max<size_t>(need, 1))) != cudaSuccess) return e;
  return fn(f->d_tmp.p, need);
}

// Moves the tail to the front and reads more of the stream (the chunk grows when grow is set).
int refill(ngmlr_b200_ctx* ctx, RF* f, bool grow) {
  const double t0 = now_ms();
  const int64_t keep = f->n_host - f->tail;
  if (keep > 0 && f->tail > 0) memmove(f->h_chunk.p, f->h_chunk.p + f->tail, (size_t)keep);
  f->n_host = keep;
  f->tail = 0;
  if (grow) f->chunk_cap *= 2;
  if ((int64_t)f->h_chunk.cap < f->chunk_cap + 1) {
    PinBuf<uint8_t> nb_;
    RCU(nb_.reserve((size_t)f->chunk_cap + 1));
    if (keep) memcpy(nb_.p, f->h_chunk.p, (size_t)keep);
    std::swap(f->h_chunk.p, nb_.p);
    std::swap(f->h_chunk.cap, nb_.cap);
  }
  if (!f->stream_eof) {
    const int64_t want = f->chunk_cap - f->n_host;
    const int64_t got = read_stream(f->in, f->h_chunk.p + f->n_host, (size_t)want);
    if (got < 0) return ctx->fail("reads_load: %s: read error (corrupt gzip stream?)", f->path.c_str());
    f->n_host += got;
    f->stream_bytes += got;
    if (got < want) {
      if (stream_truncated(f->in))
        return ctx->fail("reads_load: %s: the gzip stream is truncated or corrupt", f->path.c_str());
      f->stream_eof = true;
      f->late_eof = f->stream_bytes % 16384 == 0;
    }
  }
  f->h_chunk.p[f->n_host] = 0;  // a name or a quality string may end with the stream
  f->read_ms += (float)(now_ms() - t0);
  return 0;
}

// Line table, record chain and record table of the bytes in h_chunk.
int resolve_chunk(ngmlr_b200_ctx* ctx, RF* f) {
  const double t0 = now_ms();
  cudaStream_t st = ctx->stream;
  const int64_t n = f->n_host;
  const int64_t limit = std::max<int64_t>(f->chunk_cap / LINE_BYTES, 4096);
  RCU(f->d_chunk.reserve((size_t)std::max<int64_t>(f->chunk_cap, n) + 1));
  if (n) RCU(cudaMemcpyAsync(f->d_chunk.p, f->h_chunk.p, (size_t)n, cudaMemcpyHostToDevice, st));
  const int64_t n_segs = std::max<int64_t>(1, (n + SEG - 1) / SEG);
  RCU(f->d_seg_cnt.reserve((size_t)n_segs + 1));
  RCU(f->d_seg_mark.reserve((size_t)n_segs));
  RCU(f->d_nl.reserve((size_t)limit + 1));
  RCU(f->h_small.reserve(8));
  RCU(f->d_scalar.reserve(8));
  k_segments<<<blocks(n_segs * 32, 256), 256, 0, st>>>(f->d_chunk.p, n, n_segs, f->d_seg_cnt.p, f->d_seg_mark.p);
  RCU(cudaMemsetAsync(f->d_seg_cnt.p + n_segs, 0, 8, st));
  int64_t* segc = f->d_seg_cnt.p;
  RCU(with_tmp(f, [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, segc, segc, (int)(n_segs + 1), st);
  }));
  k_newlines<<<blocks(n_segs * 32, 256), 256, 0, st>>>(f->d_chunk.p, n, n_segs, f->d_seg_cnt.p, limit, f->d_nl.p);
  RCU(cudaMemcpyAsync(f->h_small.p, f->d_seg_cnt.p + n_segs, 8, cudaMemcpyDeviceToHost, st));
  RCU(cudaStreamSynchronize(st));
  const int64_t total_nl = f->h_small.p[0];
  const int n_nl = (int)std::min(total_nl, limit);
  int64_t n_res = n, last_nl = -1;
  if (n_nl > 0) {
    RCU(cudaMemcpyAsync(f->h_small.p, f->d_nl.p + n_nl - 1, 8, cudaMemcpyDeviceToHost, st));
    RCU(cudaStreamSynchronize(st));
    last_nl = f->h_small.p[0];
  }
  if (total_nl > limit) n_res = last_nl + 1;
  const int n_lines = n_nl + (n_res > last_nl + 1 ? 1 : 0);
  f->n_res = n_res;
  Chunk& k = f->k;
  k = Chunk{};
  k.c = f->d_chunk.p;
  k.n = n_res;
  k.nl = f->d_nl.p;
  k.n_nl = n_nl;
  k.n_lines = n_lines;
  k.at_eof = f->stream_eof && n_res == n;
  k.late_eof = f->late_eof;
  const size_t L = (size_t)n_lines + 1;
  RCU(f->d_sp.reserve(L));
  RCU(f->d_qp.reserve(L));
  RCU(f->d_ir.reserve(L));
  RCU(f->d_tr.reserve(L));
  RCU(f->d_fb.reserve(L));
  RCU(f->d_stop_flag.reserve(L));
  RCU(f->d_stops.reserve(L));
  RCU(f->d_mark.reserve(L));
  RCU(f->d_next_pos.reserve(L));
  RCU(f->d_jump.reserve(L * LEVELS));
  RCU(f->d_rec_lines.reserve(L));
  RCU(f->d_mark_segs.reserve((size_t)n_segs));
  RCU(f->d_count.reserve(4));
  k.tr = f->d_tr.p;
  k.fb = f->d_fb.p;
  k.sp = f->d_sp.p;
  k.qp = f->d_qp.p;
  k.irr = f->d_ir.p;
  k.seg_mark = f->d_seg_mark.p;
  k_lines<<<blocks((int64_t)L, 256), 256, 0, st>>>(k, f->d_sp.p, f->d_qp.p, f->d_ir.p, f->d_stop_flag.p, f->d_fb.p,
                                                   f->d_tr.p);
  int64_t* sp = f->d_sp.p;
  int64_t* qp = f->d_qp.p;
  int32_t* ir = f->d_ir.p;
  RCU(with_tmp(f, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, sp, sp, (int)L, st); }));
  RCU(with_tmp(f, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, qp, qp, (int)L, st); }));
  RCU(with_tmp(f, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, ir, ir, (int)L, st); }));
  // the lines that end a sequence, and the segments that hold a header character
  cub::CountingInputIterator<int32_t> idx(0);
  int32_t* cnt = f->d_count.p;
  RCU(with_tmp(f, [&](void* t, size_t& b) {
    return cub::DeviceSelect::Flagged(t, b, idx, f->d_stop_flag.p, f->d_stops.p, cnt, n_lines, st);
  }));
  const HasMark has_mark{f->d_seg_mark.p};
  RCU(with_tmp(f, [&](void* t, size_t& b) {
    return cub::DeviceSelect::If(t, b, idx, f->d_mark_segs.p, cnt + 1, (int)n_segs, has_mark, st);
  }));
  int32_t h_cnt[2];
  RCU(cudaMemcpyAsync(h_cnt, cnt, 8, cudaMemcpyDeviceToHost, st));
  RCU(cudaStreamSynchronize(st));
  k.stops = f->d_stops.p;
  k.n_stops = h_cnt[0];
  k.mark_segs = f->d_mark_segs.p;
  k.n_mark_segs = h_cnt[1];
  // every line as a header, then the chain from the first header character
  int32_t* jump = f->d_jump.p;
  k_resolve<<<blocks((int64_t)L, 256), 256, 0, st>>>(k, jump, f->d_next_pos.p);
  for (int l = 1; l < LEVELS; ++l)
    k_jump<<<blocks((int64_t)L, 256), 256, 0, st>>>(jump + (l - 1) * L, jump + l * L, n_lines);
  RCU(cudaMemsetAsync(f->d_mark.p, 0, L, st));
  k_chain_start<<<1, 1, 0, st>>>(k, jump + (LEVELS - 1) * L, f->d_mark.p, f->d_scalar.p);
  for (int l = LEVELS - 2; l >= 0; --l)
    k_mark<<<blocks(n_lines, 256), 256, 0, st>>>(jump + l * L, f->d_mark.p, n_lines);
  RCU(with_tmp(f, [&](void* t, size_t& b) {
    return cub::DeviceSelect::Flagged(t, b, idx, f->d_mark.p, f->d_rec_lines.p, cnt, n_lines, st);
  }));
  RCU(cudaMemcpyAsync(h_cnt, cnt, 4, cudaMemcpyDeviceToHost, st));
  RCU(cudaMemcpyAsync(f->h_small.p, f->d_scalar.p, 8, cudaMemcpyDeviceToHost, st));
  RCU(cudaStreamSynchronize(st));
  const int n_recs = h_cnt[0];
  const int64_t first_pos = f->h_small.p[0];
  RCU(f->d_recs.reserve((size_t)std::max(n_recs, 1)));
  if (n_recs)
    k_records<<<blocks(n_recs, 128), 128, 0, st>>>(k, f->d_rec_lines.p, n_recs, f->d_next_pos.p, f->d_scalar.p,
                                                   f->d_recs.p);
  f->recs.resize((size_t)n_recs);
  if (n_recs)
    RCU(cudaMemcpyAsync(f->recs.data(), f->d_recs.p, (size_t)n_recs * sizeof(LoadRec), cudaMemcpyDeviceToHost, st));
  RCU(cudaStreamSynchronize(st));
  RCU(cudaGetLastError());
  f->device_peak = std::max<int64_t>(f->device_peak, (int64_t)f->device_bytes());
  // what follows the records
  f->n_good = n_recs;
  f->next_rec = 0;
  f->resolved = true;
  if (first_pos < 0) {  // no header character: nothing here is part of a record
    f->tail = n_res;
    if (k.at_eof) f->ended = true;
  } else if (n_recs == 0) {
    f->tail = first_pos;
  } else {
    const LoadRec& last = f->recs.back();
    switch (last.kind) {
      case K_INCOMPLETE:
        f->n_good = n_recs - 1;
        f->tail = last.hdr;
        break;
      case K_TAIL:
        f->tail = last.end;
        break;
      case K_DROP:
        f->n_good = n_recs - 1;
        f->drop_pending = true;
        f->dropped.assign(reinterpret_cast<const char*>(f->h_chunk.p) + last.hdr + 1,
                          (size_t)std::min<int64_t>(last.name_end - last.hdr - 1, NAME_CUT));
        f->ended = true;
        break;
      case K_NONE:
        f->n_good = n_recs - 1;
        f->ended = true;
        break;
      default:
        f->ended = true;  // K_END
    }
  }
  for (int i = 0; i < f->n_good; ++i)
    if (f->recs[i].seq_len >= MAX_BASES)
      return ctx->fail("reads_load: %s: a sequence of %lld or more bases (ngmlr reads lengths as int)", f->path.c_str(),
                       (long long)MAX_BASES);
  if (!f->recs.empty() && f->recs.back().kind == K_INCOMPLETE && f->recs.back().seq_len >= MAX_BASES)
    return ctx->fail("reads_load: %s: a sequence of %lld or more bases (ngmlr reads lengths as int)", f->path.c_str(),
                     (long long)MAX_BASES);
  f->records += f->n_good;
  f->parse_ms += (float)(now_ms() - t0);
  return 0;
}

// kseq's quality string of a multi-line record, from the host copy of the chunk
void assemble_quality(const RF* f, const LoadRec& r, std::string& q) {
  q.clear();
  const char* c = reinterpret_cast<const char*>(f->h_chunk.p);
  const int64_t n = f->n_res;
  for (int64_t p = r.qual_start; p < r.end;) {
    const char* nl = static_cast<const char*>(memchr(c + p, '\n', (size_t)(n - p)));
    const int64_t e = nl ? nl - c : n;
    q.append(c + p, (size_t)(e - p));
    if (q.size() > 1 && q.back() == '\r') q.pop_back();
    p = e + 1;
  }
  // the extra read at the end of a stream of k x 16 KiB
  if ((int64_t)q.size() > r.qual_len && q.size() > 1 && q.back() == '\r') q.pop_back();
}

}  // namespace

extern "C" {

int ngmlr_b200_read_file_open(const char* path, const ngmlr_b200_read_file_options* opts, ngmlr_b200_read_file** out) {
  if (!path || !out) {
    set_error_without_context("read_file_open: path and out must not be NULL");
    return -1;
  }
  *out = nullptr;
  const int64_t chunk = opts && opts->chunk_bytes > 0 ? opts->chunk_bytes : DEFAULT_CHUNK;
  if (chunk < 16) {
    set_error_without_context("read_file_open: chunk_bytes < 16");
    return -1;
  }
  FILE* probe = fopen(path, "rb");
  if (!probe) {
    set_error_without_context(std::string("read_file_open: cannot open ") + path);
    return -2;
  }
  fclose(probe);
  StreamFile* in = open_stream(path);
  if (!in) {
    set_error_without_context(std::string("read_file_open: cannot open ") + path);
    return -2;
  }
  RF* f = new RF;
  f->path = path;
  f->in = in;
  f->chunk_cap = chunk;
  *out = f;
  return 0;
}

void ngmlr_b200_read_file_close(ngmlr_b200_read_file* f) {
  if (!f) return;
  if (f->device >= 0) cudaSetDevice(f->device);
  close_stream(f->in);
  delete f;
}

const char* ngmlr_b200_reads_load_dropped(const ngmlr_b200_read_file* f) {
  return f && f->dropped_reported ? f->dropped.c_str() : nullptr;
}

int ngmlr_b200_read_file_stats(const ngmlr_b200_read_file* f, int64_t* stream_bytes, int64_t* records, float* read_ms,
                               float* parse_ms, float* gather_ms, int64_t* device_bytes) {
  if (!f) return -1;
  if (stream_bytes) *stream_bytes = f->stream_bytes;
  if (records) *records = f->records;
  if (read_ms) *read_ms = f->read_ms;
  if (parse_ms) *parse_ms = f->parse_ms;
  if (gather_ms) *gather_ms = f->gather_ms;
  if (device_bytes) *device_bytes = f->device_peak;
  return 0;
}

int ngmlr_b200_reads_load(ngmlr_b200_ctx* ctx, ngmlr_b200_read_file* f, int max_reads, int64_t max_bases,
                          int read_part_length, ngmlr_b200_sam_read* reads, int* n_reads, int* n_dropped) {
  if (!ctx) return -1;
  if (!f || !reads || !n_reads || !n_dropped) return ctx->fail("reads_load: f, reads, n_reads, n_dropped must be set");
  if (max_reads < 1) return ctx->fail("reads_load: max_reads < 1");
  if (read_part_length < 1) return ctx->fail("reads_load: read_part_length < 1");
  if (!f->error.empty()) return ctx->fail("%s", f->error.c_str());
  *n_reads = 0;
  *n_dropped = 0;
  if (f->device >= 0 && f->device != ctx->device) return ctx->fail("reads_load: the file is being read on another device");
  CU(cudaSetDevice(ctx->device));
  f->device = ctx->device;
  cudaStream_t st = ctx->stream;
  CsState* cs = cs_state(ctx, true);
  f->dropped_reported = false;
  // the next chunk with a record in it
  while (f->next_rec >= f->n_good && !f->ended) {
    // a record that does not fit the chunk (or its line table): a larger chunk
    const bool grow = f->resolved && f->n_good == 0 && f->tail == 0 && (f->n_host >= f->chunk_cap || f->n_res < f->n_host);
    if (refill(ctx, f, grow) || resolve_chunk(ctx, f)) {
      f->error = ctx->error;
      return -1;
    }
  }
  const double t0 = now_ms();
  int r0 = f->next_rec, r1 = r0;
  int64_t bases = 0;
  while (r1 < f->n_good && r1 - r0 < max_reads &&
         (r1 == r0 || max_bases <= 0 || bases + f->recs[r1].seq_len <= max_bases))
    bases += f->recs[r1++].seq_len;
  const int n = r1 - r0;
  f->next_rec = r1;
  if (r1 >= f->n_good && f->drop_pending) {
    f->drop_pending = false;
    f->dropped_reported = true;
    *n_dropped = 1;
  }
  std::vector<int32_t> lens((size_t)n);
  for (int i = 0; i < n; ++i) lens[i] = (int32_t)f->recs[r0 + i].seq_len;
  std::vector<uint64_t> sub_start;
  ReadSetShape shape;
  if (read_set_layout(ctx, "reads_load", n, lens.data(), read_part_length, sub_start, shape)) return -1;
  if (read_set_reserve(ctx, cs, n, shape)) return -1;
  CU(f->h_layout.reserve(2 * ((size_t)n + 1)));
  CU(f->d_layout.reserve(2 * ((size_t)n + 1)));
  memcpy(f->h_layout.p, ctx->read_off.data(), ((size_t)n + 1) * 8);
  memcpy(f->h_layout.p + n + 1, sub_start.data(), ((size_t)n + 1) * 8);
  CU(cudaMemcpyAsync(f->d_layout.p, f->h_layout.p, 2 * ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(ctx->d_read_off.p, f->d_layout.p, ((size_t)n + 1) * 8, cudaMemcpyDeviceToDevice, st));
  CU(cudaMemsetAsync(ctx->d_reads.p, 0, shape.bytes, st));
  if (n) {
    const int lo = f->recs[r0].s, hi = f->recs[r1 - 1].stop;
    if (hi > lo)
      k_gather<<<blocks((int64_t)(hi - lo) * 32, 256), 256, 0, st>>>(f->k, f->d_recs.p, r0, r1, lo, hi, f->d_layout.p,
                                                                   ctx->d_reads.p);
    k_subreads<<<blocks(n, 128), 128, 0, st>>>(f->d_recs.p, r0, n, f->d_layout.p, f->d_layout.p + n + 1,
                                               read_part_length, cs->d_off.p, cs->d_len.p);
  }
  CU(f->h_seq.reserve(shape.bytes + 1));
  if (shape.bytes) CU(cudaMemcpyAsync(f->h_seq.p, ctx->d_reads.p, shape.bytes, cudaMemcpyDeviceToHost, st));
  CU(nb_stream_sync(ctx, st));
  CU(cudaGetLastError());
  read_set_install(ctx, cs, n, shape);
  ctx->reads_h2d_bytes = (int64_t)(2 * ((size_t)n + 1) * 8);
  // the records for sam_format
  static const char kStar[] = "*";
  char* c = reinterpret_cast<char*>(f->h_chunk.p);
  f->quals.resize((size_t)std::max<int>(n, (int)f->quals.size()));
  for (int i = 0; i < n; ++i) {
    const LoadRec& r = f->recs[r0 + i];
    ngmlr_b200_sam_read& o = reads[i];
    memset(&o, 0, sizeof(o));
    c[std::min<int64_t>(r.name_end, r.hdr + 1 + NAME_CUT)] = 0;
    o.name = c + r.hdr + 1;
    o.seq = reinterpret_cast<const char*>(f->h_seq.p) + ctx->read_off[i];
    o.length = (int32_t)r.seq_len;
    o.empty = r.seq_len == 0;
    if (!r.fastq || r.qual_len == 0) {
      o.qual = kStar;
    } else if (r.single_qual) {
      o.qual = c + r.qual_start;
    } else {
      assemble_quality(f, r, f->quals[i]);
      o.qual = f->quals[i].c_str();
    }
  }
  f->gather_ms += (float)(now_ms() - t0);
  *n_reads = n;
  return (int)shape.n_sub;
}

}  // extern "C"

extern "C" {

// Test hook: the resident read set as the device holds it -- read offsets (n_reads + 1), read lengths, the sub-read
// table (offsets, lengths; n_sub entries) and the arena bytes. Sizes always; arrays where not NULL.
int ngmlr_b200_debug_resident_reads(ngmlr_b200_ctx* ctx, int32_t* n_reads, int32_t* n_sub, int64_t* bytes,
                                    uint64_t* read_off, int32_t* read_len, uint64_t* sub_off, int32_t* sub_len,
                                    uint8_t* arena) {
  if (!ctx) return -1;
  CsState* cs = cs_state(ctx, false);
  const int n = ctx->n_reads, m = cs ? cs->rn : 0;
  if (n_reads) *n_reads = n;
  if (n_sub) *n_sub = m;
  if (bytes) *bytes = (int64_t)ctx->reads_bytes;
  CU(cudaSetDevice(ctx->device));
  if (read_off && n) CU(cudaMemcpy(read_off, ctx->d_read_off.p, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost));
  if (read_len && n) memcpy(read_len, ctx->read_len.data(), (size_t)n * 4);
  if (sub_off && m) CU(cudaMemcpy(sub_off, cs->d_off.p, (size_t)m * 8, cudaMemcpyDeviceToHost));
  if (sub_len && m) CU(cudaMemcpy(sub_len, cs->d_len.p, (size_t)m * 4, cudaMemcpyDeviceToHost));
  if (arena && ctx->reads_bytes) CU(cudaMemcpy(arena, ctx->d_reads.p, ctx->reads_bytes, cudaMemcpyDeviceToHost));
  return 0;
}

}  // extern "C"
