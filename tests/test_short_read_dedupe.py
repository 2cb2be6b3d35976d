"""Host half of ngmlr's short-read scoring (ScoreBuffer::scoreShortRead, src/ScoreBuffer.cpp:216-286): duplicate
removal after std::sort by location, then std::sort by score + computeMQ. Compared with a program compiled here that
runs libstdc++'s std::sort with the reference's comparators on records of the reference's LocationScore layout, so
that the order of tied locations and tied scores is checked, not assumed."""
import ctypes as C
import shutil
import subprocess

import numpy as np
import pytest

from ngmlr_b200 import _lib, select_candidates

PROG = r"""
#include <algorithm>
#include <cmath>
#include <cstdio>
typedef unsigned long long uloc;
struct SequenceLocation { uloc m_Location; unsigned int m_RefId; };
struct LocationScore { union { float f; int i; } Score; SequenceLocation Location; int Read; };
bool sortLocationScore(LocationScore a, LocationScore b) { return a.Score.f > b.Score.f; }
bool sortLocationScoreLocation(LocationScore a, LocationScore b) { return a.Location.m_Location < b.Location.m_Location; }
int main() {
  int n;
  while (scanf("%d", &n) == 1) {
    LocationScore* s = new LocationScore[n > 0 ? n : 1];
    for (int i = 0; i < n; ++i) { scanf("%llu %f", &s[i].Location.m_Location, &s[i].Score.f); s[i].Read = i; }
    std::sort(s, s + n, sortLocationScoreLocation);
    LocationScore* t = new LocationScore[n > 0 ? n : 1];
    int m = 0;
    uloc last = 0;
    for (int i = 0; i < n; ++i) {
      if (last - s[i].Location.m_Location > 256) t[m++] = s[i];
      last = s[i].Location.m_Location;
    }
    std::sort(t, t + m, sortLocationScore);
    int mq = 60;
    if (m > 1) mq = ceil(60.0f * (t[0].Score.f - t[1].Score.f) / t[0].Score.f);
    printf("%d %d", m, mq);
    for (int i = 0; i < m; ++i) printf(" %d", t[i].Read);
    printf("\n");
    delete[] s;
    delete[] t;
  }
}
"""


def _cases():
    rng = np.random.default_rng(3)
    out = []
    for m in [1, 2, 16, 17, 40, 41, 64, 200] * 6:
        bins = rng.integers(0, max(2, m // 3), m) * 16 + 1000   # many forward/reverse pairs of one bin
        locs = bins.astype(np.uint64)
        if rng.integers(0, 4) == 0:
            locs[0] = 0                                        # a first candidate at location 0
        scores = rng.integers(10, 14, m).astype(np.float32)     # many tied scores
        out.append((locs, scores))
    return out


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_dedupe_order_mq_match_std_sort(tmp_path):
    exe = tmp_path / "ref_sort"
    src = tmp_path / "ref_sort.cpp"
    src.write_text(PROG)
    subprocess.run(["g++", "-O2", "-o", str(exe), str(src)], check=True)
    cases = _cases()
    inp = "".join(f"{len(l)} " + " ".join(f"{int(a)} {float(b):.1f}" for a, b in zip(l, s)) + "\n" for l, s in cases)
    want = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout.splitlines()

    lib = _lib.load()
    starts = np.cumsum([0] + [len(l) for l, _ in cases]).astype(np.int64)
    locs = np.concatenate([l for l, _ in cases]).astype(np.uint64)
    scores = np.concatenate([s for _, s in cases]).astype(np.float32)
    kept = np.zeros(locs.size, dtype=np.int32)
    kstart = np.zeros(len(cases) + 1, dtype=np.int64)
    assert lib.ngmlr_b200_dedupe_short_read_candidates(
        len(cases), starts.ctypes.data_as(C.POINTER(C.c_int64)), locs.ctypes.data_as(C.POINTER(C.c_uint64)), 256,
        kept.ctypes.data_as(C.POINTER(C.c_int32)), kstart.ctypes.data_as(C.POINTER(C.c_int64))) == len(cases)
    ks = kept[:kstart[-1]]
    order, _kept, mq = select_candidates(kstart, scores[ks])
    for i, line in enumerate(want):
        w = [int(x) for x in line.split()]
        b, e = int(kstart[i]), int(kstart[i + 1])
        got_ids = [int(ks[o]) - int(starts[i]) for o in order[b:e]]
        assert [e - b, int(mq[i]) if e > b else 60] + got_ids == w, i
