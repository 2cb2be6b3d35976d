"""ngmlr_b200_reads_load (B200Aligner.load_reads) on the GPU:
  - record parity: for every case of read_loader_cases, plain and gzip, the concatenated batches equal the reads the
    unmodified ReadProvider makes (name, bases, qualities, length, empty flag) and the dropped read, at the default
    chunk, 4 KiB and a chunk smaller than one record, with max_reads 1 / 7 / all and a small max_bases;
  - resident equivalence: after each load the read arena, read offsets, read lengths, sub-read table and cs_run /
    cs_fetch arrays are those of reads_upload of the reference's strings, at --subread-length 256 and 1000;
  - file to SAM: load -> cs_run -> map_short_reads -> sam_format prints the plain ngmlr binary's SAM body for test_2's
    short reads and for 2 000 synthetic FASTQ reads of 5-257 bases (lowercase, IUPAC, CRLF, multi-line, empty
    records), plain and gzip;
  - errors: a missing file, a truncated gzip stream and a record of 2^31 bases return an error."""
import gzip
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import read_loader_cases as R
from ngmlr_b200 import B200Aligner, samtext

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLAIN = os.path.join(ROOT, "oracle", "_ref", "ngmlr")
FIX = os.path.join(ROOT, "tests", "golden", "ref_fixtures", "test_2")
need_full = pytest.mark.skipif(not os.path.exists(R.FULL), reason="oracle/_ref/libngmlr_reads.so not built")
need_plain = pytest.mark.skipif(not os.path.exists(PLAIN), reason="oracle/_ref/ngmlr not built")


@pytest.fixture(scope="module")
def aligner():
    a = B200Aligner(0)
    yield a
    a.close()


def _load_all(a, path, **kw):
    reads, dropped, sizes = [], [], []
    for b in a.load_reads(path, **kw):
        reads += [(r.name, r.seq, r.qual, len(r.seq), int(r.empty)) for r in b.reads]
        dropped += b.dropped
        sizes.append(len(b.reads))
    return reads, dropped, sizes


@need_full
@pytest.mark.parametrize("gz", [False, True])
def test_records_equal_reference_reader(aligner, tmp_path, gz):
    checked = 0
    for name in R.CASES:
        path = R.write_case(tmp_path, name, gz)
        oracle, odrop = R.oracle_reads(R.write_case(tmp_path / "o", name))
        want = R.as_loaded(oracle)
        longest = max([len(r[1]) * 2 + 300 for r in want] + [300])
        chunks = [0, 4096] if name in R.BIG else [0, 4096, max(16, longest // 4)]
        for chunk in chunks:
            for max_reads, max_bases in ((1, 0), (7, 0), (100_000, 0), (100_000, 150)):
                got, drop, sizes = _load_all(aligner, path, chunk_bytes=chunk, max_reads=max_reads, max_bases=max_bases)
                where = f"{name} gz={gz} chunk={chunk} max_reads={max_reads} max_bases={max_bases}"
                assert len(got) == len(want), where
                for i, (g, w) in enumerate(zip(got, want)):
                    assert g == w, f"{where} read {i}: {g[:1]} {g[3:]} vs {w[:1]} {w[3:]}"
                assert drop == odrop, where
                assert all(s <= max_reads for s in sizes), where
                checked += 1
    assert checked >= 20 * 3 * 4


def _oracle_strings(path, rpl):
    return [s for _, s, _, _, _ in R.as_loaded(R.oracle_reads(path, rpl)[0], rpl)]


@need_full
@pytest.mark.parametrize("rpl", [256, 1000])
def test_resident_set_equals_reads_upload(tmp_path, rpl):
    ref = shutil.copyfile(os.path.join(FIX, "ref_chr21_20kb.fa"), str(tmp_path / "ref.fa"))
    a, b = B200Aligner(0), B200Aligner(0)
    try:
        a.load_reference(ref, skip_write=True)
        b.load_reference(ref, skip_write=True)
        # at --subread-length 1000 ngmlr's Empty reads overrun their buffer (src/IParser.h:80) badly enough to abort
        names = ("fuzz_a", "fastq_multi", "crlf", "empty", "iupac") if rpl == 256 else \
            ("fastq_multi", "fasta_multi", "crlf", "iupac", "kb32_no_nl")
        for name in names:
            path = R.write_case(tmp_path, name)
            want = _oracle_strings(path, rpl)
            k = 0
            for batch in a.load_reads(path, read_part_length=rpl, max_reads=64, chunk_bytes=8192):
                seqs = want[k:k + len(batch.reads)]
                k += len(batch.reads)
                assert [r.seq for r in batch.reads] == seqs
                n_sub = b.reads_upload(seqs, read_part_length=rpl)
                assert batch.n_sub == n_sub
                for x, y in zip(a.resident_reads(), b.resident_reads()):
                    assert np.array_equal(x, y), name
                ra, rb = a.cs_run(read_part_length=rpl), b.cs_run(read_part_length=rpl)
                assert ra[0] == rb[0]
                for x, y in zip(a.cs_fetch(), b.cs_fetch()):
                    assert np.array_equal(x, y), name
            assert k == len(want)
    finally:
        a.close()
        b.close()


def _ngmlr_sam(ref_dir, query, out, rpl):
    ref = shutil.copyfile(os.path.join(FIX, "ref_chr21_20kb.fa"), os.path.join(ref_dir, "ref.fa"))
    cmd = [PLAIN, "-r", ref, "-q", query, "-o", out, "-t", "1", "--no-progress", "--skip-write",
           "--subread-length", str(rpl)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    return [l for l in open(out, "rb").read().split(b"\n") if l and not l.startswith(b"@")]


def _library_sam(tmp_path, query, rpl):
    ref = shutil.copyfile(os.path.join(FIX, "ref_chr21_20kb.fa"), str(tmp_path / "lib_ref.fa"))
    a = B200Aligner(0)
    try:
        loaded = a.load_reference(ref, skip_write=True)
        out = b""
        for batch in a.load_reads(query, read_part_length=rpl, max_reads=500):
            a.cs_run(read_part_length=rpl)
            res = a.map_short_reads(read_part_length=rpl)
            recs = [samtext.Read(r.name, r.seq, r.qual, m[1], m[0], r.empty) for r, m in zip(batch.reads, res)]
            out += samtext.sam_format(recs, loaded.sam_ref_names(), threads=1)
    finally:
        a.close()
    return [l for l in out.split(b"\n") if l]


def _short_reads_file(path, seed=5, n=2000):
    genome = b"".join(l.strip() for l in open(os.path.join(FIX, "ref_chr21_20kb.fa"), "rb") if not l.startswith(b">"))
    rng = random.Random(seed)
    comp = bytes.maketrans(b"ACGTacgt", b"TGCAtgca")
    out = []
    for i in range(n):
        L = rng.randint(5, 257)
        p = rng.randrange(0, len(genome) - L)
        s = bytearray(genome[p:p + L])
        for _ in range(rng.randint(0, 4)):
            s[rng.randrange(L)] = rng.choice(b"ACGTNRYK")
        if rng.random() < 0.5:
            s = bytearray(bytes(s).translate(comp)[::-1])
        if rng.random() < 0.2:
            s = bytearray(bytes(s).lower())
        nl = b"\r\n" if rng.random() < 0.1 else b"\n"
        w = rng.choice([60, 1000])
        lines = nl.join(bytes(s[j:j + w]) for j in range(0, L, w))
        if rng.random() < 0.02:
            out.append(b">empty%d%s" % (i, nl))
        else:  # FASTQ only: ngmlr's writer overruns the "*" quality of a reverse-strand FASTA read
            q = bytes(rng.choice(b"#+5?@>AEI") for _ in range(L))
            ql = nl.join(q[j:j + w] for j in range(0, L, w))
            out.append(b"@s%d%s%s%s+%s%s%s" % (i, nl, lines, nl, nl, ql, nl))
    with open(path, "wb") as f:
        f.write(b"".join(out))
    return path


def _test2_short_fastq(path):
    names, reads = [], []
    for line in open(os.path.join(FIX, "reads_100_2200bp.fa"), "rb"):
        line = line.strip()
        if line.startswith(b">"):
            names.append(line[1:].split()[0])
            reads.append(b"")
        elif line:
            reads[-1] += line
    with open(path, "wb") as f:
        for n, s in zip(names, reads):
            if len(s) <= 256:
                f.write(b"@" + n + b"\n" + s + b"\n+\n" + b"I" * len(s) + b"\n")
    return path


@need_plain
@pytest.mark.parametrize("which,rpl", [("test_2", 256), ("synthetic", 257)])
@pytest.mark.parametrize("gz", [False, True])
def test_file_to_sam_equals_plain_ngmlr(tmp_path, which, rpl, gz):
    src = str(tmp_path / "reads.fq")
    if which == "test_2":
        _test2_short_fastq(src)
    else:
        _short_reads_file(src)
    query = src
    if gz:
        query = src + ".gz"
        with open(src, "rb") as f, gzip.open(query, "wb") as g:
            g.write(f.read())
    want = _ngmlr_sam(str(tmp_path), query, str(tmp_path / "plain.sam"), rpl)
    got = _library_sam(tmp_path, query, rpl)
    assert len(want) >= 2
    assert got == want


def test_errors_return_a_message(aligner, tmp_path):
    with pytest.raises(RuntimeError, match="cannot open"):
        list(aligner.load_reads(str(tmp_path / "missing.fq")))
    data = gzip.compress(R.CASES["fuzz_a"])
    bad = str(tmp_path / "truncated.fq.gz")
    with open(bad, "wb") as f:
        f.write(data[: len(data) // 2])
    with pytest.raises(RuntimeError, match="truncated or corrupt"):
        list(aligner.load_reads(bad))
    # one record of 2^31 bases (a sparse run of NUL bytes, which kseq takes as sequence characters)
    big = str(tmp_path / "big.fa")
    with open(big, "wb") as f:
        f.write(b">big\n")
        f.truncate(5 + (1 << 31))
        f.seek(0, 2)
        f.write(b"\n")
    with pytest.raises(RuntimeError, match="2147483648 or more bases"):
        list(aligner.load_reads(big, chunk_bytes=512 << 20))
    # the context still loads a good file afterwards
    reads, _, _ = _load_all(aligner, R.write_case(tmp_path, "fasta_single"))
    assert [r[0] for r in reads] == [b"r1", b"r2", b"r3"]
