"""ngmlr's short-read path (reads of at most --subread-length = 256 bases: ScoreBuffer::scoreShortRead ->
AlignmentBuffer::processShortRead -> WriteRead) on the resident pipeline: reads_upload -> cs_run ->
map_short_reads -> sam_format must print the records the unmodified ngmlr binary prints for those reads, byte for
byte. Plus the short-read scorer against the oracle, and cs_run / cs_fetch unchanged by the new call."""
import os
import subprocess

import numpy as np
import pytest

from ngmlr_b200 import B200Aligner, samtext, synth
from oracle_lib import CsOracle, Oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLAIN = os.path.join(ROOT, "oracle", "_ref", "ngmlr")
FIXTURE = os.path.join(ROOT, "tests", "golden", "ref_fixtures", "test_2")
need_plain = pytest.mark.skipif(not os.path.exists(PLAIN),
                                reason="oracle/_ref/ngmlr not built (needs the reference sources at build time)")


def _contigs(seed=21):
    rng = np.random.default_rng(seed)
    c1 = synth.random_genome(120_000, seed + 1)
    c2 = synth.random_genome(80_001, seed + 2)
    seg = synth.random_genome(230, seed + 3)
    # one segment planted 2 and 4 times: tied scores, MQ 0 and the alignIndex < 2 continuation
    for c, where in ((c1, (20_000, 50_000, 90_000)), (c2, (30_000,))):
        for w in where:
            c[w:w + seg.size] = seg
    c1[60_000:60_040] = ord("N")  # an N run in the reference
    return [c1, c2], seg, rng


def _reads(contigs, seg, rng, n=2400):
    reads = []
    for i in range(n):
        kind = i % 10
        c = contigs[i % 2]
        L = int(rng.integers(5, 258))
        if i < 40:
            L = (256, 257, 255, 12, 5)[i % 5]
        if kind == 0:                      # random, unmappable
            r = synth.random_genome(L, 1000 + i)
        elif kind == 1:                    # the planted segment
            a = int(rng.integers(0, max(1, seg.size - min(L, seg.size) + 1)))
            r = seg[a:a + L].copy()
        elif kind == 2:                    # contig ends: the window runs into the spacer
            r = c[:L].copy() if i % 4 == 2 else c[c.size - L:].copy()
        else:
            s = int(rng.integers(0, c.size - L))
            r = c[s:s + L].copy()
            if kind in (3, 4, 5):          # sequencing errors
                r, _ = synth.mutate(r, rng, err=0.08 if kind != 5 else 0.2)
            if kind == 6 and r.size > 40:  # an N run in the read
                a = int(rng.integers(0, r.size - 20))
                r[a:a + 15] = ord("N")
        r = np.ascontiguousarray(r[:257], dtype=np.uint8)
        if r.size == 0:
            r = np.frombuffer(b"ACGTA", dtype=np.uint8).copy()
        if rng.integers(0, 2):
            r = synth.revcomp(r)
        reads.append(r.tobytes())
    return reads


def _write(dirpath, contigs, reads):
    ref = os.path.join(dirpath, "ref.fa")
    with open(ref, "w") as f:
        for i, c in enumerate(contigs):
            f.write(f">chr{i + 1}\n")
            s = c.tobytes().decode()
            for k in range(0, len(s), 80):
                f.write(s[k:k + 80] + "\n")
    fq = os.path.join(dirpath, "reads.fq")
    quals = []
    with open(fq, "w") as f:
        for i, r in enumerate(reads):
            q = "".join(chr(33 + (7 * i + 3 * k) % 40) for k in range(len(r)))
            quals.append(q.encode())
            f.write(f"@r{i}\n{r.decode()}\n+\n{q}\n")
    return ref, fq, quals


def _plain_records(ref, fq, tmp):
    sam = os.path.join(tmp, "plain.sam")
    r = subprocess.run([PLAIN, "-r", ref, "-q", fq, "-o", sam, "-t", "1", "--skip-write", "--no-progress"],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    recs = {}
    for line in open(sam, "rb"):
        if not line.startswith(b"@"):
            recs.setdefault(line.split(b"\t", 1)[0], []).append(line)
    return recs


def _library_records(contigs, reads, quals, names):
    a = B200Aligner(0)
    try:
        enc = a.encode_reference([c.tobytes() for c in contigs], fetch=False)
        a.build_index(enc)
        a.reads_upload(reads)
        a.cs_run()
        res = a.map_short_reads(256, 0.25)
    finally:
        a.close()
    ref_names = [b"chr1", b"chr1", b"chr2", b"chr2"]  # SequenceProvider's list: every contig twice
    out = {}
    for i, r in enumerate(res):
        if r is None:
            out[names[i]] = None
            continue
        mapped, al = r
        text = samtext.sam_format([samtext.Read(names[i], reads[i], quals[i], al, mapped)], ref_names, threads=1)
        out[names[i]] = text.splitlines(keepends=True)
    return out


@need_plain
def test_short_reads_sam_identical_to_plain_binary(tmp_path):
    contigs, seg, rng = _contigs()
    reads = _reads(contigs, seg, rng)
    ref, fq, quals = _write(str(tmp_path), contigs, reads)
    names = [f"r{i}".encode() for i in range(len(reads))]
    want = _plain_records(ref, fq, str(tmp_path))
    got = _library_records(contigs, reads, quals, names)
    n_mapped = n_multi = n_mq0 = 0
    for i, r in enumerate(reads):
        if len(r) > 256:
            assert got[names[i]] is None, f"read {i} ({len(r)} bp) must be reported as not handled"
            continue
        w = want.get(names[i], [])
        assert got[names[i]] == w, f"read {i} ({len(r)} bp) differs:\nngmlr: {w}\nlib  : {got[names[i]]}"
        if w and not (int(w[0].split(b"\t")[1]) & 4):
            n_mapped += 1
            n_multi += len(w) > 1
            n_mq0 += any(x.split(b"\t")[4] == b"0" for x in w)
    # the data reach the interesting branches
    assert n_mapped > 500 and n_multi > 10 and n_mq0 > 10, (n_mapped, n_multi, n_mq0)


@need_plain
def test_fixture_short_reads(tmp_path):
    """test_2's 100bp and 200bp reads reproduce the plain binary's records (expected.bed: 8913-9010 and
    8913-9109, MAPQ 60, +)."""
    contigs, names = [], []
    for line in open(os.path.join(FIXTURE, "ref_chr21_20kb.fa"), "rb"):
        line = line.strip()
        if line.startswith(b">"):
            names.append(line[1:].split()[0])
            contigs.append(bytearray())
        elif line:
            contigs[-1] += line.upper()
    reads, rnames = [], []
    for line in open(os.path.join(FIXTURE, "reads_100_2200bp.fa"), "rb"):
        line = line.strip()
        if line.startswith(b">"):
            rnames.append(line[1:].split()[0])
            reads.append(bytearray())
        elif line:
            reads[-1] += line.upper()
    reads = [bytes(b if b in b"ACGT" else ord("N") for b in r) for r in reads]
    ref = os.path.join(str(tmp_path), "ref.fa")
    with open(ref, "wb") as f:
        for n, c in zip(names, contigs):
            f.write(b">" + n + b"\n" + bytes(c) + b"\n")
    fq = os.path.join(str(tmp_path), "reads.fq")
    quals = [b"I" * len(r) for r in reads]
    with open(fq, "wb") as f:
        for n, r, q in zip(rnames, reads, quals):
            f.write(b"@" + n + b"\n" + r + b"\n+\n" + q + b"\n")
    want = _plain_records(ref, fq, str(tmp_path))
    a = B200Aligner(0)
    try:
        enc = a.encode_reference([bytes(c) for c in contigs], fetch=False)
        a.build_index(enc)
        a.reads_upload(reads)
        a.cs_run()
        res = a.map_short_reads()
    finally:
        a.close()
    ref_names = [n for n in names for _ in (0, 1)]
    checked = 0
    for i, r in enumerate(res):
        if r is None:
            continue
        text = samtext.sam_format([samtext.Read(rnames[i], reads[i], quals[i], r[1], r[0])], ref_names, threads=1)
        assert text.splitlines(keepends=True) == want[rnames[i]]
        if rnames[i] in (b"100bp", b"200bp"):
            f = text.split(b"\t")
            assert f[1] == b"0" and f[3] == b"8914" and f[4] == b"60", text[:200]
            checked += 1
    assert checked == 2


def test_short_read_scores_match_oracle():
    """The scorer on >= 5000 pairs: 588-column windows, windows past the concatenated genome's end ('N'),
    reverse candidates; all through the ungapped path."""
    rng = np.random.default_rng(5)
    contigs = [synth.random_genome(30_000, 51), synth.random_genome(20_001, 52)]
    cso = CsOracle([c.tobytes() for c in contigs])
    orc = Oracle()
    a = B200Aligner(0)
    try:
        a.encode_reference([c.tobytes() for c in contigs], fetch=False)
        lens = [256, 255, 1, 13] + [int(x) for x in rng.integers(1, 257, 396)]
        reads = []
        for L in lens:
            r = synth.random_genome(L, int(rng.integers(1 << 30)))
            if rng.integers(0, 3) == 0 and L > 20:
                c = contigs[0]
                s = int(rng.integers(0, c.size - L))
                r, _ = synth.mutate(c[s:s + L].copy(), rng, err=0.05)
                r = np.ascontiguousarray(r[:256], dtype=np.uint8)
            reads.append(r.tobytes() or b"A")
        a.reads_upload(reads)
        cl = cso.concat_len
        n = 6000
        ri = rng.integers(0, len(reads), n).astype(np.int32)
        loc = rng.integers(0, cl, n).astype(np.uint64)
        loc[:300] = cl - rng.integers(0, 400, 300).astype(np.uint64)   # window runs past the end
        loc[300:400] = cl + rng.integers(0, 1000, 100).astype(np.uint64)  # decoding fails: 'N' window
        loc[400:450] = rng.integers(0, 200, 50).astype(np.uint64)       # loc - corridor/2 wraps below 0
        ri[:600] = 0                                                    # 256 bases: 588-column windows
        rv = rng.integers(0, 2, n).astype(np.uint8)
        got = a.score_short_reads(ri, loc, rv)
        assert a.lib.ngmlr_b200_debug_short_read_general_pairs(a.h) == 0
    finally:
        a.close()
    for j in range(n):
        q = reads[ri[j]]
        L = len(q)
        corridor = int(L * 0.3 + 256)
        w = cso.decode((int(loc[j]) - (corridor >> 1)) % (1 << 64), L + corridor) or b"N" * (L + corridor)
        qq = synth.revcomp_upper(np.frombuffer(q, dtype=np.uint8)).tobytes() if rv[j] else q
        assert float(got[j]) == orc.ssw_score(w, qq), (j, L, int(loc[j]), int(rv[j]))
    cso.close()


def test_cs_run_unchanged_by_map_short_reads():
    genome = synth.random_genome(200_000, 61)
    contigs = [genome[:100_000], genome[100_000:]]
    rng = np.random.default_rng(62)
    reads = []
    for i in range(64):
        L = int(rng.integers(20, 257)) if i % 2 else int(rng.integers(300, 3000))
        s = int(rng.integers(0, 100_000 - L))
        r, _ = synth.mutate(contigs[i % 2][s:s + L].copy(), rng, err=0.05)
        reads.append(np.ascontiguousarray(r, dtype=np.uint8).tobytes())
    a = B200Aligner(0)
    try:
        enc = a.encode_reference([c.tobytes() for c in contigs], fetch=False)
        a.build_index(enc)
        a.reads_upload(reads)
        a.cs_run()
        before = a.cs_fetch()
        res = a.map_short_reads()
        after = a.cs_fetch()
        a.cs_run()
        again = a.cs_fetch()
    finally:
        a.close()
    for x, y, z in zip(before, after, again):
        assert np.array_equal(x, y) and np.array_equal(x, z)
    assert [r is None for r in res] == [len(r) > 256 for r in reads]
    assert sum(1 for r in res if r is not None and r[0]) > 20
