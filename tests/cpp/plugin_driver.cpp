// tests/cpp/plugin_driver.cpp -- exercises libngmlr_b200.so exactly the way ngmlr would: dlopen,
// CreateAlignment(gpu_id), then calls through the IAlignment vtable (SingleAlign with
// CorridorLine[], BatchAlign with NgmlrB200BatchAlignArgs, BatchScore, SingleScore) with
// caller-allocated Align buffers (src/AlignmentBuffer.cpp:271-278). Problems are read from a
// simple text file written by tests/test_gpu_plugin.py, results are printed one line per problem
// for comparison with the oracle. An optional third argument runs the SingleAlign calls from that many threads at
// once (with NGMLR_B200_BATCH_WINDOW_US set the cross-thread batcher then serves several of them per launch).
#include <dlfcn.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <thread>
#include <vector>

#include "ngmlr_b200_ialignment.h"

struct Problem {
  std::string ref, qry;
  std::vector<CorridorLine> lines;
  int qs, qe;
};

static void print_align(const char* tag, int i, int ret, const Align& a) {
  unsigned bits, ibits;
  memcpy(&bits, &a.Score, 4);
  memcpy(&ibits, &a.Identity, 4);
  if (ret < 0) {
    printf("%s %d ret=-1 score_bits=%u\n", tag, i, bits);
    return;
  }
  printf("%s %d ret=%d score_bits=%u identity_bits=%u pos=%d qstart=%d qend=%d nm=%d alen=%d ops=%d sv=%d "
         "first=%d,%d last=%d,%d cigar=%s md=%s\n",
         tag, i, ret, bits, ibits, a.PositionOffset, a.QStart, a.QEnd, a.NM, a.alignmentLength,
         a.cigarOpCount, a.svType, a.firstPosition.refPosition, a.firstPosition.readPosition,
         a.lastPosition.refPosition, a.lastPosition.readPosition, a.pBuffer1, a.pBuffer2);
}

// nmPerPosition (the triples ngmlr's SV logic reads): count and FNV-1a over (refPosition, readPosition, nm) as
// little-endian int32s, on a line of its own so that the lines above keep their format. The Align record carries no
// count, so alloc_align fills the array with a pattern no triple can take; the written entries are the ones before it.
static const int32_t kNmUnset = INT32_MIN;
static void print_nm(const char* tag, int i, int ret, const Align& a) {
  if (ret < 0) return;
  int count = 0;
  uint32_t h = 2166136261u;
  while (a.nmPerPosition && count < a.nmPerPostionLength && a.nmPerPosition[count].nm != kNmUnset) {
    const PositionNM& p = a.nmPerPosition[count++];
    const int32_t v[3] = {p.refPosition, p.readPosition, p.nm};
    const unsigned char* b = reinterpret_cast<const unsigned char*>(v);
    for (int x = 0; x < 12; ++x) h = (h ^ b[x]) * 16777619u;
  }
  printf("nm %s %d count=%d fnv=%u\n", tag, i, count, h);
}

static void alloc_align(Align& a, size_t readLength) {
  a.maxBufferLength = (int)readLength * 4 + 8;
  a.maxMdBufferLength = (int)readLength * 4 + 8;
  a.pBuffer1 = new char[a.maxBufferLength];
  a.pBuffer2 = new char[a.maxMdBufferLength];
  a.pBuffer1[0] = a.pBuffer2[0] = '\0';
  a.nmPerPostionLength = ((int)readLength + 1) * 2;
  a.nmPerPosition = new PositionNM[a.nmPerPostionLength];
  for (int k = 0; k < a.nmPerPostionLength; ++k) a.nmPerPosition[k].refPosition = a.nmPerPosition[k].readPosition =
      a.nmPerPosition[k].nm = kNmUnset;
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  void* h = dlopen(argv[1], RTLD_NOW);
  if (!h) { fprintf(stderr, "dlopen: %s\n", dlerror()); return 3; }
  pfCreateAlignment create = (pfCreateAlignment)dlsym(h, "CreateAlignment");
  pfDeleteAlignment destroy = (pfDeleteAlignment)dlsym(h, "DeleteAlignment");
  if (!create || !destroy) return 4;
  IAlignment* al = create(0);
  if (!al) { fprintf(stderr, "CreateAlignment returned NULL (no device?)\n"); return 5; }

  FILE* f = fopen(argv[2], "r");
  int n = 0;
  if (fscanf(f, "%d", &n) != 1) return 6;
  std::vector<Problem> ps(n);
  for (int i = 0; i < n; ++i) {
    int rl, ql;
    if (fscanf(f, "%d %d %d %d", &rl, &ql, &ps[i].qs, &ps[i].qe) != 4) return 6;
    std::vector<char> buf((size_t)std::max(rl, ql) + 2);
    if (fscanf(f, "%s", buf.data()) != 1) return 6;
    ps[i].ref = buf.data();
    if (fscanf(f, "%s", buf.data()) != 1) return 6;
    ps[i].qry = buf.data();
    ps[i].lines.resize(ql);
    for (int y = 0; y < ql; ++y)
      if (fscanf(f, "%d %d", &ps[i].lines[y].offset, &ps[i].lines[y].length) != 2) return 6;
  }
  fclose(f);

  printf("batchsize %d %d\n", al->GetScoreBatchSize(), al->GetAlignBatchSize());
  // 1) one blocking SingleAlign per problem, as computeAlignment does (from `threads` worker threads)
  {
    const int threads = argc > 3 ? std::max(1, atoi(argv[3])) : 1;
    std::vector<Align> as(n);
    std::vector<int> rets(n, -2);
    for (int i = 0; i < n; ++i) {
      alloc_align(as[i], ps[i].qry.size());
      as[i].svType = 1234;  // "read id" hack of the caller (:363)
    }
    auto work = [&](int t) {
      for (int i = t; i < n; i += threads) {
        try {
          rets[i] = al->SingleAlign(i, ps[i].lines.data(), (int)ps[i].lines.size(), ps[i].ref.c_str(),
                                    ps[i].qry.c_str(), as[i], ps[i].qs, ps[i].qe, 0);
        } catch (...) {
          rets[i] = -3;
        }
      }
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; ++t) pool.emplace_back(work, t);
    work(0);
    for (auto& t : pool) t.join();
    for (int i = 0; i < n; ++i) {
      print_align("single", i, rets[i], as[i]);
      print_nm("single", i, rets[i], as[i]);
      unsigned long expect = 0;
      bool ok = true;
      for (size_t y = 0; y < ps[i].lines.size(); ++y) {  // prepare() publishes offsetInMatrix
        ok = ok && ps[i].lines[y].offsetInMatrix == expect;
        expect += (unsigned long)ps[i].lines[y].length;
      }
      printf("offsetInMatrix %d %s\n", i, ok ? "ok" : "BAD");
      delete[] as[i].pBuffer1; delete[] as[i].pBuffer2; delete[] as[i].nmPerPosition;
    }
  }
  // 2) the same problems through BatchAlign
  {
    std::vector<Align> as(n);
    std::vector<const char*> refs(n), qrys(n);
    std::vector<NgmlrB200BatchAlignArgs> args(n);
    for (int i = 0; i < n; ++i) {
      alloc_align(as[i], ps[i].qry.size());
      refs[i] = ps[i].ref.c_str();
      qrys[i] = ps[i].qry.c_str();
      args[i] = {ps[i].lines.data(), (int)ps[i].lines.size(), ps[i].qs, ps[i].qe};
    }
    int rc = al->BatchAlign(0, n, refs.data(), qrys.data(), as.data(), args.data());
    printf("batchalign rc=%d\n", rc);
    for (int i = 0; i < n; ++i) {
      // BatchAlign reports a failed problem the way SingleAlign does: Score == -1
      print_align("batch", i, as[i].Score == -1.0f ? -1 : 0, as[i]);
      print_nm("batch", i, as[i].Score == -1.0f ? -1 : 0, as[i]);
      delete[] as[i].pBuffer1; delete[] as[i].pBuffer2; delete[] as[i].nmPerPosition;
    }
  }
  // 3) BatchScore / SingleScore on (ref prefix, read prefix) pairs
  {
    std::vector<std::string> r(n), q(n);
    std::vector<const char*> rp(n), qp(n);
    std::vector<float> out(n, -1.0f);
    for (int i = 0; i < n; ++i) {
      r[i] = ps[i].ref.substr(0, 306);
      q[i] = ps[i].qry.substr(0, 256);
      rp[i] = r[i].c_str();
      qp[i] = q[i].c_str();
    }
    int rc = al->BatchScore(0, n, rp.data(), qp.data(), out.data(), 0);
    printf("batchscore rc=%d\n", rc);
    for (int i = 0; i < n; ++i) {
      float s = -7.0f;
      int r1 = al->SingleScore(10, 0, rp[i], qp[i], s, 0);
      printf("score %d %g %g %d\n", i, out[i], s, r1);
    }
  }
  // 4) the unimplemented overload throws, like the reference
  {
    Align a;
    bool threw = false;
    try { al->SingleAlign(0, 40, "ACGT", "ACGT", a, 0); } catch (...) { threw = true; }
    printf("single_int_corridor_throws %d\n", threw ? 1 : 0);
  }
  destroy(al);
  return 0;
}
