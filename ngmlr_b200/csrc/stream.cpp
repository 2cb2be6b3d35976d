// ngmlr_b200/csrc/stream.cpp -- the byte stream ngmlr's gzopen / gzread would give, for the read loader and the
// reference reader (stream.h). A stream has one of three sources, named by StreamFile::mode: the BGZF walker, plain
// gzip rounds on the device, or the host continuation (GzTail, gzread reproduced over the file's bytes), which takes
// any file from its first byte and either device path from the first member it cannot vouch for.
#include "stream.h"

#include <cuda_runtime.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <cerrno>
#include <climits>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <memory>
#include <vector>

#include "inflate.h"

namespace nb {

namespace {

constexpr size_t GZ_BUFFER = 1 << 20;           // gzread's buffers under gzbuffer(1 MiB): reads 1 MiB, inflates 2 MiB
constexpr int64_t READ_BLOCK = 4 << 20;         // read() size of the stage
constexpr int64_t MIN_COMP_ROUND = 1 << 20;     // compressed bytes a round may always take
constexpr int64_t MEMBERS_PER_BYTE = 4096;      // a round holds at most one member per 4 KiB of that budget (>= 64)
constexpr uint32_t GZ_CHUNK = 32 << 10;         // compressed bytes per chunk of a plain gzip round
constexpr int64_t GZ_MIN_ROUND = 4 << 20;       // output a plain gzip round always aims for
constexpr int64_t GZ_SLACK = 9 << 20;           // output a chunk may run past the round's aim: one zlib block
                                                // (at most 32 767 symbols of up to 258 bytes) and more
constexpr int64_t GZ_MARGIN = 2 * GZ_BUFFER;    // the release rule's margin: gzread's inflate fill (see gz_release)
constexpr int64_t GZ_WINDOW = 32768;
constexpr int64_t GZ_PAD = 1024;                // zero bytes after a span: the bit readers look past its end
// The device path runs where it beats gzread (one H100, both paths timed end to end in the same call, DESIGN.md
// §4.9): in rounds of at least 256 MiB of output (in 4 MiB rounds it was 1.4 - 5.8x slower at every ratio measured,
// 3.2 - 8.9; in 256 MiB rounds 1.1 - 1.9x faster up to 6.5), and between these ratios of output to compressed bytes,
// measured over the first round (4x slower on incompressible data, where zlib copies stored blocks; 1.3x slower at
// 8.9 and up to 2x at 114 and 1027, where one warp's serial decode of a chunk's long matches cannot keep up with
// zlib). A stream outside them goes to zlib whole, decided before anything is returned: on the round size before any
// device work, on the ratio after the first round's counting pass.
constexpr int64_t GZ_DEVICE_ROUND = 256ll << 20;
constexpr double GZ_RATIO_LO = 1.5, GZ_RATIO_HI = 6.5;
constexpr int GZ_BATCHED_REDECODES = 8;         // launches of batched re-decodes per round before the serial walk

// Host memory that grows keeping its first `keep` bytes; page-locked once the stream is bound to a device.
struct HostBuf {
  uint8_t* p = nullptr;
  size_t cap = 0;
  bool pinned = false;
  bool reserve(size_t n, size_t keep) {
    if (n <= cap) return true;
    const size_t want = std::max(n, cap + cap / 2);
    uint8_t* q = nullptr;
    if (pinned) {
      if (cudaMallocHost(&q, want) != cudaSuccess) return false;
    } else if (!(q = static_cast<uint8_t*>(malloc(want)))) {
      return false;
    }
    if (keep) memcpy(q, p, keep);
    release();
    p = q;
    cap = want;
    return true;
  }
  bool set_pinned(size_t keep) {
    if (pinned) return true;
    HostBuf b;
    b.pinned = true;
    if (!b.reserve(std::max<size_t>(keep, 1), 0)) return false;
    if (keep) memcpy(b.p, p, keep);
    std::swap(p, b.p);
    std::swap(cap, b.cap);
    std::swap(pinned, b.pinned);
    return true;
  }
  void release() {
    if (p) {
      if (pinned) cudaFreeHost(p);
      else free(p);
    }
    p = nullptr;
    cap = 0;
  }
  ~HostBuf() { release(); }
};

// Device memory sized to the largest round so far (64 KiB granules, no slack: the read loader's bound counts it).
template <typename T>
struct DevMem {
  T* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    const size_t want = (n * sizeof(T) + 65535) / 65536 * 65536 / sizeof(T);
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    const cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
  size_t bytes() const { return cap * sizeof(T); }
  ~DevMem() {
    if (p) cudaFree(p);
  }
};

// gzread over a byte source, from the start of a file (fresh) or from the header of a member that follows another
// one: zlib's gz_read / gz_fetch / gz_decomp / gz_look / gz_avail with gzread's buffer sizes under gzbuffer(1 MiB).
// gzread inflates a member into its 2 MiB buffer as soon as one byte of it is wanted, and reports an error in the call
// that meets it; so this gives the same bytes from the same calls, the same -1 and the same truncation flag.
class GzTail {
 public:
  using Source = std::function<int64_t(uint8_t*, size_t)>;  // up to n bytes; 0 at the end; < 0 on a read error
  GzTail(Source src, bool fresh) : src_(std::move(src)), direct_(fresh), in_(GZ_BUFFER), out_(2 * GZ_BUFFER) {
    memset(&strm_, 0, sizeof strm_);
    ok_ = inflateInit2(&strm_, 15 + 16) == Z_OK;
    if (!ok_) err_ = Z_MEM_ERROR;
  }
  ~GzTail() {
    if (ok_) inflateEnd(&strm_);
  }
  int64_t read(uint8_t* buf, size_t len) {
    if (err_ != Z_OK && err_ != Z_BUF_ERROR) return -1;
    if (len == 0) return 0;
    const size_t r = gz_read(buf, len);
    if (r == 0 && err_ != Z_OK && err_ != Z_BUF_ERROR) return -1;
    return (int64_t)r;
  }
  bool truncated() const { return err_ != Z_OK; }

 private:
  enum { LOOK, COPY, GZIP };
  int load(uint8_t* buf, size_t n, size_t* have) {
    *have = 0;
    int64_t r = 0;
    do {
      r = src_(buf + *have, n - *have);
      if (r <= 0) break;
      *have += (size_t)r;
    } while (*have < n);
    if (r < 0) {
      err_ = Z_ERRNO;
      return -1;
    }
    if (r == 0) eof_ = true;
    return 0;
  }
  int avail() {
    if (err_ != Z_OK && err_ != Z_BUF_ERROR) return -1;
    if (!eof_) {
      if (strm_.avail_in) memmove(in_.data(), strm_.next_in, strm_.avail_in);
      size_t got = 0;
      if (load(in_.data() + strm_.avail_in, GZ_BUFFER - strm_.avail_in, &got) == -1) return -1;
      strm_.avail_in += (unsigned)got;
      strm_.next_in = in_.data();
    }
    return 0;
  }
  int look() {
    if (strm_.avail_in < 2) {
      if (avail() == -1) return -1;
      if (strm_.avail_in == 0) return 0;
    }
    if (strm_.avail_in > 1 && strm_.next_in[0] == 31 && strm_.next_in[1] == 139) {
      inflateReset(&strm_);
      how_ = GZIP;
      direct_ = false;
      return 0;
    }
    if (!direct_) {  // after a gzip member: trailing garbage, ignored
      strm_.avail_in = 0;
      eof_ = true;
      x_have_ = 0;
      return 0;
    }
    x_next_ = out_.data();
    memcpy(x_next_, strm_.next_in, strm_.avail_in);
    x_have_ = strm_.avail_in;
    strm_.avail_in = 0;
    how_ = COPY;
    return 0;
  }
  int decomp() {
    int ret = Z_OK;
    const unsigned had = strm_.avail_out;
    do {
      if (strm_.avail_in == 0 && avail() == -1) return -1;
      if (strm_.avail_in == 0) {
        err_ = Z_BUF_ERROR;  // "unexpected end of file"
        break;
      }
      ret = inflate(&strm_, Z_NO_FLUSH);
      if (ret == Z_STREAM_ERROR || ret == Z_NEED_DICT || ret == Z_MEM_ERROR || ret == Z_DATA_ERROR) {
        err_ = ret == Z_NEED_DICT ? Z_STREAM_ERROR : ret;
        return -1;
      }
    } while (strm_.avail_out && ret != Z_STREAM_END);
    x_have_ = had - strm_.avail_out;
    x_next_ = strm_.next_out - x_have_;
    if (ret == Z_STREAM_END) how_ = LOOK;
    return 0;
  }
  int fetch() {
    do {
      switch (how_) {
        case LOOK:
          if (look() == -1) return -1;
          if (how_ == LOOK) return 0;
          break;
        case COPY: {
          size_t h = 0;
          if (load(out_.data(), out_.size(), &h) == -1) return -1;
          x_have_ = h;
          x_next_ = out_.data();
          return 0;
        }
        case GZIP:
          strm_.avail_out = (unsigned)out_.size();
          strm_.next_out = out_.data();
          if (decomp() == -1) return -1;
      }
    } while (x_have_ == 0 && (!eof_ || strm_.avail_in));
    return 0;
  }
  size_t gz_read(uint8_t* buf, size_t len) {
    size_t got = 0;
    do {
      size_t n = std::min<size_t>(len, UINT_MAX);  // what one pass can hand to zlib, as in zlib's gz_read
      if (x_have_) {
        n = std::min(x_have_, n);
        memcpy(buf, x_next_, n);
        x_next_ += n;
        x_have_ -= n;
      } else if (eof_ && strm_.avail_in == 0) {
        break;
      } else if (how_ == LOOK || n < out_.size()) {
        if (fetch() == -1) return 0;
        continue;
      } else if (how_ == COPY) {
        if (load(buf, n, &n) == -1) return 0;
      } else {
        strm_.avail_out = (unsigned)n;
        strm_.next_out = buf;
        if (decomp() == -1) return 0;
        n = x_have_;
        x_have_ = 0;
      }
      len -= n;
      buf += n;
      got += n;
    } while (len);
    return got;
  }

  Source src_;
  bool direct_, ok_ = false, eof_ = false;
  int how_ = LOOK, err_ = Z_OK;
  z_stream strm_;
  std::vector<uint8_t> in_, out_;
  uint8_t* x_next_ = nullptr;
  size_t x_have_ = 0;
};

// One BGZF member as the walker sees it: file offset, header and total length (BSIZE + 1), trailer, output offset.
struct Member {
  int64_t c = 0, out = 0;
  uint32_t hlen = 0, total = 0, crc = 0, isize = 0;
};

uint32_t le32(const uint8_t* p) { return p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24; }

}  // namespace

struct StreamFile {
  // Where the bytes come from: the BGZF walker, plain gzip rounds on the bound device, or the host continuation. Each
  // device path hands over to HOST (start_host) and never comes back.
  enum Mode { WALK, ROUNDS, HOST } mode = HOST;
  // the file, read sequentially into stage = file bytes [stage_off, stage_off + stage_len)
  int fd = -1;
  HostBuf stage;
  int64_t stage_off = 0, stage_len = 0;
  bool file_eof = false;
  bool gz_plain = false;              // a regular file whose first member is gzip, not BGZF: ROUNDS once bound
  bool used = false;                  // read_stream has been called
  HostBuf out;                        // WALK and ROUNDS output
  // WALK
  int64_t next_c = 0;                 // file offset of the next member to walk
  int64_t hold_b = 0, hold_e = 0;     // inflated bytes out[hold_b, hold_e) not yet returned
  int64_t fallback_c = -1;            // where the host continuation starts once the held bytes are returned
  bool ended = false;                 // the file ends after the held bytes
  z_stream raw;
  bool raw_init = false;
  std::vector<InflateMember> mem;
  std::vector<int32_t> status;
  DevMem<InflateMember> d_mem;
  DevMem<int32_t> d_status;
  // ROUNDS: see "Plain gzip on the device" below
  uint32_t gz_chunk = GZ_CHUNK;
  bool gz_choose = true;             // pick the path by the first round's ratio (off once a chunk size is set)
  uint64_t gz_bit = 0;               // the confirmed chain position (file bit offset) ...
  bool gz_member = true;             // ... is a member header (else a block header)
  int64_t gz_total = 0;              // output decoded on the chain
  int64_t out_base = 0;              // f->out holds output [out_base, gz_total)
  int64_t read_pos = 0, release = 0; // output returned; output that may be returned
  int64_t mem_hdr = 0, mem_out0 = 0; // the member decoding at gz_bit: header file offset, first output offset
  uint32_t mem_crc = 0;
  int64_t avail = 0;                 // output of that member before gz_bit, at most 32 KiB
  int gz_stop = 0;                   // 1: the stream ended cleanly; 2: zlib takes over at prob_hdr
  int64_t prob_hdr = 0;
  double ratio = 4;                  // output / compressed bytes of the last round
  std::deque<int64_t> mem_ends;      // output offsets of verified member ends not yet passed by read_pos
  std::vector<int64_t> portions;     // lengths of the calls answered inside the member at read_pos
  std::vector<uint8_t> win = std::vector<uint8_t>(GZ_WINDOW);  // the last 32 KiB of output
  DevMem<uint16_t> d_sym;
  DevMem<GzChunk> d_chunks;
  DevMem<GzEvent> d_events;
  DevMem<uint32_t> d_pcrc;
  // HOST
  std::unique_ptr<GzTail> tail;
  int64_t tail_pos = 0;               // file offset the continuation reads next
  // the device binding (WALK and ROUNDS)
  int device = -1;
  cudaStream_t st = nullptr;
  int64_t min_round = 0;
  DevMem<uint8_t> d_comp, d_out;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  StreamCounters cnt;
  std::string error;
  ~StreamFile() {
    if (fd >= 0) close(fd);
    if (raw_init) inflateEnd(&raw);
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
  }
};

namespace {

// File bytes up to `end` in the stage: 1, or 0 when the file ends first, or -1 on a read error / no memory.
int stage_cover(StreamFile* f, int64_t end) {
  while (f->stage_off + f->stage_len < end && !f->file_eof) {
    const int64_t want = std::max<int64_t>(end - (f->stage_off + f->stage_len), READ_BLOCK);
    if (!f->stage.reserve((size_t)(f->stage_len + want), (size_t)f->stage_len)) {
      f->error = "out of host memory for the BGZF staging buffer";
      return -1;
    }
    const ssize_t r = read(f->fd, f->stage.p + f->stage_len, (size_t)want);
    if (r < 0) {
      if (errno == EINTR) continue;
      return -1;
    }
    if (r == 0) f->file_eof = true;
    f->stage_len += r;
    f->cnt.compressed_bytes += r;
  }
  return f->stage_off + f->stage_len >= end ? 1 : 0;
}

// The stage keeps nothing before file offset c.
void stage_drop(StreamFile* f, int64_t c) {
  if (c <= f->stage_off) return;
  const int64_t d = std::min(c - f->stage_off, f->stage_len);
  memmove(f->stage.p, f->stage.p + d, (size_t)(f->stage_len - d));
  f->stage_off += d;
  f->stage_len -= d;
}

// The member at file offset c: 1 = a BGZF member whose bytes are staged, ISIZE <= 65536; 2 = the file ends at c;
// 0 = anything else (another header, trailing bytes, a member running past the end of the file); -1 = read error.
int walk_member(StreamFile* f, int64_t c, Member& m) {
  int r = stage_cover(f, c + 18);
  if (r < 0) return -1;
  const int64_t avail = f->stage_off + f->stage_len - c;
  if (avail == 0) return 2;
  if (avail < 18) return 0;
  const uint8_t* p = f->stage.p + (c - f->stage_off);
  if (p[0] != 0x1f || p[1] != 0x8b || p[2] != 8 || p[3] != 4) return 0;
  const uint32_t xlen = p[10] | p[11] << 8;
  if ((r = stage_cover(f, c + 12 + xlen)) <= 0) return r;
  p = f->stage.p + (c - f->stage_off);
  int64_t total = -1;
  for (uint32_t q = 0; q + 4 <= xlen;) {
    const uint8_t* s = p + 12 + q;
    const uint32_t slen = s[2] | s[3] << 8;
    if (s[0] == 'B' && s[1] == 'C' && slen == 2 && q + 6 <= xlen) {
      total = (s[4] | s[5] << 8) + 1;
      break;
    }
    q += 4 + slen;
  }
  if (total < 12 + (int64_t)xlen + 8) return 0;
  if ((r = stage_cover(f, c + total)) <= 0) return r;
  p = f->stage.p + (c - f->stage_off);
  m.c = c;
  m.hlen = 12 + xlen;
  m.total = (uint32_t)total;
  m.crc = le32(p + total - 8);
  m.isize = le32(p + total - 4);
  return m.isize <= 65536 ? 1 : 0;
}

// How many of the round's leading members inflated to what zlib gives (their output is in f->out at m.out).
int inflate_host(StreamFile* f, const std::vector<Member>& ms) {
  if (!f->raw_init) {
    memset(&f->raw, 0, sizeof f->raw);
    if (inflateInit2(&f->raw, -15) != Z_OK) return 0;
    f->raw_init = true;
  }
  int ok = 0;
  for (const Member& m : ms) {
    inflateReset(&f->raw);
    f->raw.next_in = f->stage.p + (m.c - f->stage_off) + m.hlen;
    f->raw.avail_in = m.total - m.hlen - 8;
    f->raw.next_out = f->out.p + m.out;
    f->raw.avail_out = m.isize;
    const int ret = inflate(&f->raw, Z_FINISH);
    if (ret != Z_STREAM_END || f->raw.avail_in || f->raw.avail_out ||
        crc32(0, f->out.p + m.out, m.isize) != m.crc)
      break;
    ++ok;
  }
  return ok;
}

#define SCU(call)                                                                                   \
  do {                                                                                              \
    const cudaError_t e__ = (call);                                                                 \
    if (e__ != cudaSuccess) {                                                                       \
      f->error = std::string(f->mode == StreamFile::WALK ? "BGZF inflate: " : "gzip inflate: ") + #call + \
                 " failed: " + cudaGetErrorString(e__);                                             \
      return -1;                                                                                    \
    }                                                                                               \
  } while (0)

// The same on the bound device: one warp per member (inflate.cu). Returns -1 on a CUDA error.
int inflate_device(StreamFile* f, const std::vector<Member>& ms, int64_t out_bytes) {
  const int n = (int)ms.size();
  const int64_t c0 = ms.front().c, c1 = ms.back().c + ms.back().total;
  f->mem.resize(n);
  f->status.assign(n, -1);
  for (int i = 0; i < n; ++i) {
    const Member& m = ms[i];
    f->mem[i] = InflateMember{(uint64_t)(m.c - c0 + m.hlen), (uint64_t)m.out, m.total - m.hlen - 8, m.isize, m.crc, 0};
  }
  SCU(cudaSetDevice(f->device));
  SCU(f->d_comp.reserve((size_t)(c1 - c0) + 64));
  SCU(f->d_out.reserve((size_t)out_bytes + 1));
  SCU(f->d_mem.reserve(n));
  SCU(f->d_status.reserve(n));
  SCU(cudaMemcpyAsync(f->d_comp.p, f->stage.p + (c0 - f->stage_off), (size_t)(c1 - c0), cudaMemcpyHostToDevice, f->st));
  SCU(cudaMemcpyAsync(f->d_mem.p, f->mem.data(), n * sizeof(InflateMember), cudaMemcpyHostToDevice, f->st));
  SCU(cudaEventRecord(f->ev[0], f->st));
  SCU(launch_inflate(f->d_comp.p, f->d_mem.p, n, f->d_out.p, f->d_status.p, f->st));
  SCU(cudaEventRecord(f->ev[1], f->st));
  if (out_bytes) SCU(cudaMemcpyAsync(f->out.p, f->d_out.p, (size_t)out_bytes, cudaMemcpyDeviceToHost, f->st));
  SCU(cudaMemcpyAsync(f->status.data(), f->d_status.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, f->st));
  SCU(cudaStreamSynchronize(f->st));
  float ms_ = 0;
  SCU(cudaEventElapsedTime(&ms_, f->ev[0], f->ev[1]));
  f->cnt.inflate_ms += ms_;
  int ok = 0;
  while (ok < n && f->status[ok] == 0) ++ok;
  f->cnt.device_members += ok;
  return ok;
}

// One round from next_c: the members whose output starts within `want` bytes (at least min_round) of it, inflated
// together; the vouched prefix becomes the held bytes. Returns -1 on a read or device error.
int run_round(StreamFile* f, int64_t want) {
  stage_drop(f, f->next_c);
  const int64_t target = std::max(want, f->min_round);
  const int64_t comp_cap = std::max(target, MIN_COMP_ROUND);
  const size_t max_members = (size_t)std::max<int64_t>(64, comp_cap / MEMBERS_PER_BYTE);
  std::vector<Member> ms;
  int64_t out = 0, comp = 0, c = f->next_c;
  int stop = 1;  // 1: the round is full; 2: the file ends at c; 0: the member at c is not for the walker
  while (out < target && ms.size() < max_members) {
    Member m;
    const int r = walk_member(f, c, m);
    if (r < 0) return -1;
    if (r != 1) {
      stop = r;
      break;
    }
    if (!ms.empty() && comp + m.total > comp_cap) break;
    m.out = out;
    ms.push_back(m);
    out += m.isize;
    comp += m.total;
    c += m.total;
  }
  int ok = 0;
  if (!ms.empty()) {
    if (!f->out.reserve((size_t)out + 1, 0)) {
      f->error = "out of host memory for the BGZF output round";
      return -1;
    }
    ok = f->device >= 0 ? inflate_device(f, ms, out) : inflate_host(f, ms);
    if (ok < 0) return -1;
  }
  f->hold_b = 0;
  if (ok < (int)ms.size()) {
    f->hold_e = ms[ok].out;
    f->next_c = f->fallback_c = ms[ok].c;
  } else {
    f->hold_e = out;
    f->next_c = c;
    if (stop == 0) f->fallback_c = c;
    if (stop == 2) f->ended = true;
  }
  return 0;
}

// The host continuation takes the stream from file offset c: gzread from there (fresh at the file's first byte),
// after replaying the sizes of the calls already answered inside the member at c (their output is discarded; it is
// identical by construction).
void start_host(StreamFile* f, int64_t c) {
  f->mode = StreamFile::HOST;
  f->tail_pos = c;
  f->tail.reset(new GzTail(
      [f](uint8_t* b, size_t k) -> int64_t {
        while (f->tail_pos < f->stage_off) {  // a regular file whose stage moved past the continuation's start
          const ssize_t r = pread(f->fd, b, std::min<size_t>(k, (size_t)(f->stage_off - f->tail_pos)), f->tail_pos);
          if (r < 0 && errno == EINTR) continue;
          if (r <= 0) return -1;
          f->cnt.compressed_bytes += r;
          f->tail_pos += r;
          return r;
        }
        const int64_t staged = f->stage_off + f->stage_len - f->tail_pos;
        if (staged > 0) {
          const size_t m = std::min<size_t>(k, (size_t)staged);
          memcpy(b, f->stage.p + (f->tail_pos - f->stage_off), m);
          f->tail_pos += (int64_t)m;
          return (int64_t)m;
        }
        if (f->file_eof) return 0;
        for (;;) {
          const ssize_t r = read(f->fd, b, k);
          if (r < 0 && errno == EINTR) continue;
          if (r < 0) return -1;
          if (r == 0) f->file_eof = true;
          f->cnt.compressed_bytes += r;
          f->tail_pos += r;
          return r;
        }
      },
      c == 0));
  std::vector<uint8_t> scratch;
  for (int64_t p : f->portions) {
    scratch.resize((size_t)std::max<int64_t>(p, (int64_t)scratch.size()));
    f->tail->read(scratch.data(), (size_t)p);
  }
  f->portions.clear();
}

int64_t read_host(StreamFile* f, uint8_t* buf, size_t n) {
  const int64_t r = f->tail->read(buf, n);
  if (r > 0) f->cnt.host_bytes += r;
  return r;
}

int64_t read_walker(StreamFile* f, uint8_t* buf, size_t n) {
  size_t got = 0;
  while (got < n) {
    if (f->hold_b < f->hold_e) {
      const size_t k = std::min<size_t>(n - got, (size_t)(f->hold_e - f->hold_b));
      memcpy(buf + got, f->out.p + f->hold_b, k);
      f->hold_b += (int64_t)k;
      got += k;
      continue;
    }
    if (f->fallback_c >= 0) {
      start_host(f, f->fallback_c);
      const int64_t r = read_host(f, buf + got, n - got);
      return r < 0 ? -1 : (int64_t)got + r;
    }
    if (f->ended) break;
    if (run_round(f, (int64_t)(n - got)) < 0) return -1;
  }
  return (int64_t)got;
}

// ---- Plain gzip on the device -----------------------------------------------------------------------------------------
// A stream whose first member is not BGZF, once bound to a device, is read with read() and inflated in rounds
// (gzip_inflate.cu has the kernels). gz_round confirms the speculative chunks of a round: chunk 0 starts at the
// confirmed position; chunk k + 1 is confirmed when chunk k is and ends exactly at its start, else it is decoded again
// from chunk k's true end (a false boundary costs time, never bytes). Chunks are placed while their output fits the
// round, output offsets are prefix sums, and the rest of the span is carried to the next round.
//
// Release rule. A caller must not be able to tell this path from gzread, so zlib decides every unusual case: from the
// member where the device finds anything it cannot vouch for (a decode error, truncation, a bad header, trailing
// bytes, a CRC / ISIZE mismatch, a chunk too large to place), a GzTail started at that member's header continues the
// stream, after replaying the sizes of the calls already answered inside that member (their output is discarded; it
// is identical by construction). gzread reports an error in the call that meets it and loses every byte of the 2 MiB
// inflate fill in which it meets it (of the whole call for calls of 2 MiB or more). zlib meets an error at or after
// the output offset where the bad symbol, header or trailer lies, and an inflate fill that holds byte R - 1 ends no
// later than R - 1 + 2 MiB. So a member's first R bytes may be returned only when the chain has verified the member
// to at least R + 2 MiB of output, or verified its trailer: then no gzread call that returns one of them can fail.
// A call returns its full n bytes unless the stream ends, running further rounds as needed.

using namespace inflate_status;

bool gz_decode_error(int32_t st) { return st != ST_OK && st != GZ_END && st != GZ_SPAN && st != GZ_MEMBER; }

float gz_elapsed(StreamFile* f) {
  float ms = 0;
  cudaEventElapsedTime(&ms, f->ev[0], f->ev[1]);
  return ms;
}

// Pass A over chunks [0, n) of f->d_chunks; results and events back into c / ev.
int gz_pass_a(StreamFile* f, GzChunk* c, GzEvent* ev, int n, uint64_t span, bool final_span, int64_t soft,
              int64_t hard) {
  SCU(cudaMemcpyAsync(f->d_chunks.p, c, n * sizeof(GzChunk), cudaMemcpyHostToDevice, f->st));
  SCU(cudaEventRecord(f->ev[0], f->st));
  SCU(launch_gz_decode(false, f->d_comp.p, span, final_span, f->d_chunks.p, f->d_events.p, n, nullptr, (uint32_t)soft,
                       (uint32_t)hard, f->st));
  SCU(cudaEventRecord(f->ev[1], f->st));
  SCU(cudaMemcpyAsync(c, f->d_chunks.p, n * sizeof(GzChunk), cudaMemcpyDeviceToHost, f->st));
  SCU(cudaMemcpyAsync(ev, f->d_events.p, (size_t)n * GZ_EVENTS * sizeof(GzEvent), cudaMemcpyDeviceToHost, f->st));
  SCU(cudaStreamSynchronize(f->st));
  f->cnt.gzip_ms += gz_elapsed(f);
  return 0;
}

// One round over the compressed span [c0, c0 + span). Returns 1 when it moved the stream on (or stopped it), 0 when
// nothing could be placed without more input, -1 on a CUDA error.
int gz_try(StreamFile* f, int64_t c0, uint64_t span, bool final_span, int64_t budget) {
  const int64_t hard = budget + GZ_SLACK;
  const int J = (int)std::max<uint64_t>(1, (span + f->gz_chunk - 1) / f->gz_chunk);
  const uint64_t start0 = f->gz_bit - (uint64_t)c0 * 8;
  SCU(cudaSetDevice(f->device));
  SCU(f->d_comp.reserve(span + GZ_PAD));
  SCU(f->d_chunks.reserve(J));
  SCU(f->d_events.reserve((size_t)J * GZ_EVENTS));
  SCU(cudaMemcpyAsync(f->d_comp.p, f->stage.p + (c0 - f->stage_off), span, cudaMemcpyHostToDevice, f->st));
  SCU(cudaMemsetAsync(f->d_comp.p + span, 0, GZ_PAD, f->st));
  std::vector<GzChunk> all((size_t)J);
  for (GzChunk& c : all) c.start = GZ_NONE;
  all[0].start = start0;
  all[0].start_member = f->gz_member;
  SCU(cudaMemcpyAsync(f->d_chunks.p, all.data(), J * sizeof(GzChunk), cudaMemcpyHostToDevice, f->st));
  SCU(cudaEventRecord(f->ev[0], f->st));
  SCU(launch_gz_find(f->d_comp.p, span, f->gz_chunk, J, f->d_chunks.p, f->st));
  SCU(cudaEventRecord(f->ev[1], f->st));
  SCU(cudaMemcpyAsync(all.data(), f->d_chunks.p, J * sizeof(GzChunk), cudaMemcpyDeviceToHost, f->st));
  SCU(cudaStreamSynchronize(f->st));
  f->cnt.gzip_ms += gz_elapsed(f);
  std::vector<GzChunk> L;
  for (const GzChunk& c : all)
    if (c.start != GZ_NONE && (L.empty() || c.start > L.back().start)) L.push_back(c);
  for (size_t i = 0; i < L.size(); ++i) L[i].stop = i + 1 < L.size() ? L[i + 1].start : GZ_NONE;
  std::vector<GzEvent> E(L.size() * GZ_EVENTS);
  if (gz_pass_a(f, L.data(), E.data(), (int)L.size(), span, final_span, budget, hard)) return -1;
  std::vector<std::vector<GzEvent>> LE(L.size());
  for (size_t i = 0; i < L.size(); ++i) LE[i].assign(E.begin() + i * GZ_EVENTS, E.begin() + (i + 1) * GZ_EVENTS);
  // Batched re-decodes: every chunk (up to the round's output) whose decode ends short of or past the next start gets
  // a chunk decoded from its end, all of them in one launch, until the speculative chain has no gap left. A chunk
  // that started at a false boundary only adds a chunk the walk drops; the walk still confirms every link.
  auto first_from = [&](uint64_t bit) {
    return (size_t)(std::lower_bound(L.begin(), L.end(), bit, [](const GzChunk& c, uint64_t b) { return c.start < b; }) -
                    L.begin());
  };
  for (int round = 0; round < GZ_BATCHED_REDECODES; ++round) {
    std::vector<GzChunk> add;
    int64_t out = 0;
    for (size_t i = 0; i < L.size() && out < hard; ++i) {
      const GzChunk& c = L[i];
      out += c.out_len;
      if (c.status != ST_OK) continue;
      size_t k = first_from(c.end);
      bool linked = false;
      for (; k < L.size() && L[k].start == c.end; ++k) linked |= L[k].start_member == c.end_member;
      if (linked || (!add.empty() && add.back().start == c.end)) continue;
      GzChunk n{};
      n.start = c.end;
      n.start_member = c.end_member;
      n.stop = k < L.size() ? L[k].start : GZ_NONE;
      add.push_back(n);
    }
    if (add.empty()) break;
    std::sort(add.begin(), add.end(), [](const GzChunk& a, const GzChunk& b) { return a.start < b.start; });
    add.erase(std::unique(add.begin(), add.end(), [](const GzChunk& a, const GzChunk& b) { return a.start == b.start; }),
              add.end());
    std::vector<GzEvent> ae(add.size() * GZ_EVENTS);
    if (gz_pass_a(f, add.data(), ae.data(), (int)add.size(), span, final_span, budget, hard)) return -1;
    f->cnt.gzip_redecoded += (int64_t)add.size();
    for (size_t a = 0; a < add.size(); ++a) {
      const size_t at = first_from(add[a].start);
      L.insert(L.begin() + at, add[a]);
      LE.insert(LE.begin() + at, std::vector<GzEvent>(ae.begin() + a * GZ_EVENTS, ae.begin() + (a + 1) * GZ_EVENTS));
    }
  }
  // the walk: confirm, place, decode again after a false start
  int64_t prefix = 0, avail = f->avail, hdr = f->mem_hdr;
  size_t placed = 0;
  int stop = 0;  // 1: clean end; 2: zlib from prob (file offset)
  int64_t prob = 0;
  for (size_t i = 0; i < L.size();) {
    GzChunk& c = L[i];
    if (c.status == ST_INPUT && !final_span) break;
    if (gz_decode_error(c.status) || c.reach > avail) {
      // the prefix up to the last member header before the error is sound; zlib takes that member
      int h = -1;
      if (c.reach <= avail)
        for (int k = 0; k < (int)c.n_ev; ++k)
          if (LE[i][k].kind == 0) h = k;
      stop = 2;
      prob = hdr;
      if (h >= 0 && (i == 0 || (prefix < budget && prefix + LE[i][h].out <= hard))) {
        c.end = c.stop = LE[i][h].bit;
        c.end_member = 1;
        c.out_len = LE[i][h].out;
        c.n_ev = (uint32_t)h;
        c.status = GZ_MEMBER;
        c.out_off = (uint64_t)(prefix + GZ_WINDOW);
        prefix += c.out_len;
        ++placed;
        prob = c0 + (int64_t)(c.end >> 3);
      }
      break;
    }
    if (i > 0 && (prefix >= budget || prefix + c.out_len > hard)) break;
    c.out_off = (uint64_t)(prefix + GZ_WINDOW);
    prefix += c.out_len;
    ++placed;
    int last_start = -1;
    for (uint32_t k = 0; k < c.n_ev; ++k)
      if (LE[i][k].kind == 0) {
        last_start = (int)LE[i][k].out;
        hdr = c0 + (int64_t)(LE[i][k].bit >> 3);
      }
    avail = std::min<int64_t>(GZ_WINDOW, last_start >= 0 ? c.out_len - last_start : avail + c.out_len);
    if (c.status == GZ_END) {
      stop = 1;
      break;
    }
    if (c.status == GZ_MEMBER) {
      stop = 2;
      prob = c0 + (int64_t)(c.end >> 3);
      break;
    }
    if (c.status == GZ_SPAN) break;
    const size_t j = i + 1;
    size_t k = j;
    while (k < L.size() && (L[k].start < c.end || (L[k].start == c.end && L[k].start_member != c.end_member))) ++k;
    L.erase(L.begin() + j, L.begin() + k);
    LE.erase(LE.begin() + j, LE.begin() + k);
    if (j < L.size() && L[j].start == c.end) {
      i = j;
      continue;
    }
    if (prefix >= budget) break;  // the round is full: the next round starts at c.end
    GzChunk n{};
    n.start = c.end;
    n.start_member = c.end_member;
    n.stop = j < L.size() ? L[j].start : GZ_NONE;
    std::vector<GzEvent> ne(GZ_EVENTS);
    if (gz_pass_a(f, &n, ne.data(), 1, span, final_span, budget, hard)) return -1;
    ++f->cnt.gzip_redecoded;
    L.insert(L.begin() + j, n);
    LE.insert(LE.begin() + j, ne);
    i = j;
  }
  const uint64_t end_bit = placed ? L[placed - 1].end : start0;
  if (!stop && end_bit == start0) return 0;
  const uint64_t used = (end_bit - start0) / 8;
  if (used && prefix) f->ratio = std::max(1.0, (double)prefix / (double)used);
  if (f->gz_choose && stop == 0 && f->gz_total == 0 && (f->ratio < GZ_RATIO_LO || f->ratio > GZ_RATIO_HI)) {
    // the first round of a stream the device path is slower on, known from its counting pass: zlib from the first
    // byte (nothing was returned), before the writing pass and the resolve
    f->gz_stop = 2;
    f->prob_hdr = 0;
    return 1;
  }
  f->cnt.gzip_chunks += (int64_t)placed;
  std::vector<uint32_t> pcrc(placed * (GZ_EVENTS + 1));
  const int64_t held = f->gz_total - f->out_base;
  if (placed) {
    SCU(f->d_sym.reserve((size_t)(GZ_WINDOW + prefix)));
    SCU(f->d_out.reserve((size_t)prefix + 1));
    SCU(f->d_pcrc.reserve(pcrc.size()));
    std::vector<uint16_t> w16(GZ_WINDOW);
    for (int64_t i = 0; i < GZ_WINDOW; ++i) w16[i] = f->win[i];
    SCU(cudaMemcpyAsync(f->d_sym.p, w16.data(), GZ_WINDOW * 2, cudaMemcpyHostToDevice, f->st));
    SCU(cudaMemcpyAsync(f->d_chunks.p, L.data(), placed * sizeof(GzChunk), cudaMemcpyHostToDevice, f->st));
    SCU(cudaEventRecord(f->ev[0], f->st));
    SCU(launch_gz_decode(true, f->d_comp.p, span, final_span, f->d_chunks.p, f->d_events.p, (int)placed, f->d_sym.p,
                         (uint32_t)budget, (uint32_t)hard, f->st));
    SCU(launch_gz_resolve(f->d_chunks.p, f->d_events.p, (int)placed, f->d_sym.p, f->d_out.p, f->d_pcrc.p, f->st));
    SCU(cudaEventRecord(f->ev[1], f->st));
    if (prefix)
      SCU(cudaMemcpyAsync(f->out.p + held, f->d_out.p, (size_t)prefix, cudaMemcpyDeviceToHost, f->st));
    SCU(cudaMemcpyAsync(pcrc.data(), f->d_pcrc.p, pcrc.size() * 4, cudaMemcpyDeviceToHost, f->st));
    SCU(cudaStreamSynchronize(f->st));
    f->cnt.gzip_ms += gz_elapsed(f);
  }
  // members: CRC32 and ISIZE of every trailer
  int64_t prob_out0 = -1, prob_len = 0;
  for (size_t k = 0; k < placed && prob_out0 < 0; ++k) {
    const GzChunk& c = L[k];
    const int64_t g = f->gz_total + (int64_t)c.out_off - GZ_WINDOW;
    uint32_t pb = 0;
    int piece = 0;
    for (uint32_t q = 0; q <= c.n_ev; ++q) {
      const GzEvent* e = q < c.n_ev ? &LE[k][q] : nullptr;
      if (e && e->kind == 0) {
        f->mem_hdr = c0 + (int64_t)(e->bit >> 3);
        f->mem_out0 = g + e->out;
        f->mem_crc = 0;
        continue;
      }
      const uint32_t pe = e ? e->out : c.out_len;
      f->mem_crc = (uint32_t)crc32_combine64(f->mem_crc, pcrc[k * (GZ_EVENTS + 1) + piece++], pe - pb);
      pb = pe;
      if (!e) break;
      const int64_t len = g + e->out - f->mem_out0;
      if (f->mem_crc != e->crc || (uint32_t)len != e->isize) {
        prob_out0 = f->mem_out0;
        prob_len = len;
        stop = 2;
        prob = f->mem_hdr;
        break;
      }
      f->mem_ends.push_back(g + e->out);
    }
  }
  f->gz_total += prefix;
  // the window: the last 32 KiB of output
  const uint8_t* fresh = f->out.p + held;
  if (prefix >= GZ_WINDOW) {
    memcpy(f->win.data(), fresh + prefix - GZ_WINDOW, GZ_WINDOW);
  } else if (prefix) {
    memmove(f->win.data(), f->win.data() + prefix, (size_t)(GZ_WINDOW - prefix));
    memcpy(f->win.data() + GZ_WINDOW - prefix, fresh, (size_t)prefix);
  }
  f->gz_bit = (uint64_t)c0 * 8 + end_bit;
  f->gz_member = placed ? L[placed - 1].end_member : f->gz_member;
  f->avail = avail;
  if (stop == 1) {
    f->gz_stop = 1;
    f->release = f->gz_total;
  } else if (stop == 2) {
    f->gz_stop = 2;
    f->prob_hdr = prob;
    if (prob_out0 < 0) {  // a member at gz_bit's position (a decode problem) or a bad boundary
      prob_out0 = f->gz_member ? f->gz_total : f->mem_out0;
      prob_len = f->gz_total - prob_out0;
    }
    f->release = std::max(f->release, prob_out0 + std::max<int64_t>(0, prob_len - GZ_MARGIN));
  } else {
    f->release = std::max(f->release, f->gz_member ? f->gz_total
                                                   : f->mem_out0 + std::max<int64_t>(0, f->gz_total - f->mem_out0 - GZ_MARGIN));
  }
  return 1;
}

// Rounds until the chain has moved on (or stopped), aiming at `want` more bytes past what is held.
int gz_round(StreamFile* f, int64_t want) {
  const int64_t need = f->read_pos + want + GZ_MARGIN + 65536 - f->gz_total;
  const int64_t budget = std::min<int64_t>(std::max({need, f->min_round, GZ_MIN_ROUND}), 1 << 30);
  if (f->gz_choose && f->gz_total == 0 && budget < GZ_DEVICE_ROUND) {  // rounds too small to beat gzread: zlib whole
    f->gz_stop = 2;
    f->prob_hdr = 0;
    return 0;
  }
  // the held output keeps nothing before read_pos
  const int64_t drop = f->read_pos - f->out_base, held = f->gz_total - f->read_pos;
  if (drop > 0 && held > 0) memmove(f->out.p, f->out.p + drop, (size_t)held);
  f->out_base = f->read_pos;
  if (!f->out.reserve((size_t)(held + budget + GZ_SLACK + 1), (size_t)held)) {
    f->error = "out of host memory for the gzip output round";
    return -1;
  }
  // the stage keeps nothing behind the chain (the file is regular: zlib rereads a member with pread)
  const int64_t c0 = (int64_t)(f->gz_bit >> 3);
  stage_drop(f, c0);
  int64_t S = std::min<int64_t>(budget + MIN_COMP_ROUND, std::max<int64_t>(MIN_COMP_ROUND, (int64_t)(budget / f->ratio)));
  for (;;) {
    if (stage_cover(f, c0 + S) < 0) return -1;
    const int64_t have = f->stage_off + f->stage_len - c0;
    const uint64_t span = (uint64_t)std::min(S, have);
    const bool final_span = f->file_eof && (int64_t)span == have;
    const int r = gz_try(f, c0, span, final_span, budget);
    if (r != 0) return r < 0 ? -1 : 0;
    if (final_span) {  // cannot happen: at the end of the file every chunk is placed or stops the stream
      f->gz_stop = 2;
      f->prob_hdr = f->mem_hdr;
      return 0;
    }
    S *= 2;
  }
}

int64_t read_gz(StreamFile* f, uint8_t* buf, size_t n) {
  size_t got = 0, g0 = 0;  // g0: where this call entered the member at read_pos
  while (got < n) {
    while (!f->mem_ends.empty() && f->mem_ends.front() <= f->read_pos) {
      f->mem_ends.pop_front();
      f->portions.clear();
      g0 = got;
    }
    if (f->release > f->read_pos) {
      int64_t k = std::min<int64_t>((int64_t)(n - got), f->release - f->read_pos);
      if (!f->mem_ends.empty()) k = std::min(k, f->mem_ends.front() - f->read_pos);
      memcpy(buf + got, f->out.p + (f->read_pos - f->out_base), (size_t)k);
      f->read_pos += k;
      got += (size_t)k;
      f->cnt.gzip_bytes += k;
      continue;
    }
    if (f->gz_stop == 1) return (int64_t)got;
    if (f->gz_stop == 2) {  // zlib from the member at read_pos: replay the calls it answered, then this one
      start_host(f, f->prob_hdr);
      const int64_t r = read_host(f, buf + g0, n - g0);
      if (r < 0) return -1;
      f->cnt.gzip_bytes -= (int64_t)(got - g0);
      return (int64_t)(g0 + r);
    }
    if (gz_round(f, (int64_t)(n - got)) < 0) return -1;
  }
  if (n > g0) f->portions.push_back((int64_t)(n - g0));
  return (int64_t)got;
}

}  // namespace

StreamFile* open_stream(const char* path) {
  std::unique_ptr<StreamFile> f(new StreamFile);
  f->fd = open(path, O_RDONLY);
  if (f->fd < 0) return nullptr;
  Member m;
  const int r = walk_member(f.get(), 0, m);
  if (r == 1) {
    f->mode = StreamFile::WALK;
    return f.release();
  }
  // anything else: the host continuation from the first byte, or device rounds for a gzip member that is not BGZF in
  // a regular file when a device is bound before the first read (see bind_stream_device)
  struct stat sb;
  f->gz_plain = r == 0 && fstat(f->fd, &sb) == 0 && S_ISREG(sb.st_mode) && f->stage_len >= 3 &&
                f->stage.p[0] == 0x1f && f->stage.p[1] == 0x8b && f->stage.p[2] == 8;
  start_host(f.get(), 0);
  return f.release();
}

void close_stream(StreamFile* f) { delete f; }

int64_t read_stream(StreamFile* f, void* buf, size_t n) {
  f->used = true;
  uint8_t* b = static_cast<uint8_t*>(buf);
  switch (f->mode) {
    case StreamFile::WALK: return read_walker(f, b, n);
    case StreamFile::ROUNDS: return read_gz(f, b, n);
    case StreamFile::HOST: return read_host(f, b, n);
  }
  return -1;
}

bool stream_truncated(StreamFile* f) { return f->tail && f->tail->truncated(); }

bool bind_stream_device(StreamFile* f, int device, cudaStream_t stream, int64_t min_round) {
  f->device = device;
  f->st = stream;
  f->min_round = min_round;
  // plain gzip in a regular file: inflate on the device from here on. A pipe stays with the gzread continuation: zlib
  // may have to reread a member from its header, which a pipe could only offer by holding every compressed byte of
  // the current member, a whole single-member file, in page-locked memory.
  if (f->gz_plain && !f->used && f->mode == StreamFile::HOST) {
    f->tail.reset();
    f->mode = StreamFile::ROUNDS;
    if (const char* e = getenv("NGMLR_B200_DEBUG_GZIP_CHUNK")) set_gzip_chunk(f, atoll(e));
  }
  if (f->mode == StreamFile::HOST) return true;
  cudaError_t e = cudaSetDevice(device);
  for (cudaEvent_t& ev : f->ev)
    if (e == cudaSuccess && !ev) e = cudaEventCreate(&ev);
  if (e != cudaSuccess) {
    f->error = std::string("BGZF inflate: ") + cudaGetErrorString(e);
    return false;
  }
  if (!f->stage.set_pinned((size_t)f->stage_len) || !f->out.set_pinned(0)) {
    f->error = "BGZF inflate: out of page-locked host memory";
    return false;
  }
  return true;
}

StreamCounters stream_counters(const StreamFile* f) { return f->cnt; }

size_t stream_device_bytes(const StreamFile* f) {
  return f->d_comp.bytes() + f->d_out.bytes() + f->d_mem.bytes() + f->d_status.bytes() + f->d_sym.bytes() +
         f->d_chunks.bytes() + f->d_events.bytes() + f->d_pcrc.bytes();
}

void set_gzip_chunk(StreamFile* f, int64_t chunk_bytes) {
  if (chunk_bytes < 64) return;
  f->gz_chunk = (uint32_t)std::min<int64_t>(chunk_bytes, 1 << 24);
  f->gz_choose = false;
}

const std::string& stream_error(const StreamFile* f) { return f->error; }

}  // namespace nb
