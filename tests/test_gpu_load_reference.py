"""ngmlr_b200_load_reference (B200Aligner.load_reference, python -m ngmlr_b200.index) on the GPU:
  - the caches it writes for a fresh copy of a FASTA file are the ones the plain ngmlr binary writes for that copy
    (the index file byte for byte; the encoded reference up to the end of the used part of binRef, behind which the
    reference writes uninitialised memory), for FASTA / FASTQ / gzip inputs with edge cases, the reference's own
    fixtures and one non-default -k / --kmer-skip pair;
  - with the caches present a second load reads them and writes nothing, installs the same arrays and gives the same
    candidates; a truncated or foreign index file is rebuilt;
  - ngmlr started from caches written by `python -m ngmlr_b200.index` writes the SAM it writes when it builds its own
    index, and load_reference -> reads_upload -> cs_run -> map_short_reads -> sam_header + sam_format with the names
    of reference_contigs reproduces its SAM file, header included, for test_2's short reads;
  - failures (missing file, empty FASTA, genome over the single-unit limit) return an error and leave the context as
    it was."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from ngmlr_b200 import B200Aligner, ngmfiles, samtext
from test_fasta_reader import CASES, write_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLAIN = os.path.join(ROOT, "oracle", "_ref", "ngmlr")
FIX = os.path.join(ROOT, "tests", "golden", "ref_fixtures")
need_plain = pytest.mark.skipif(not os.path.exists(PLAIN), reason="oracle/_ref/ngmlr not built")


def _query(dirpath):
    q = os.path.join(str(dirpath), "q.fa")
    with open(q, "w") as f:
        f.write(">q\n" + "ACGTTGCA" * 40 + "\n")
    return q


def _ngmlr(ref, query, out, *extra, skip_write=False):
    cmd = [PLAIN, "-r", ref, "-q", query, "-o", out, "-t", "1", "--no-progress", *extra]
    if skip_write:
        cmd.append("--skip-write")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    return r


def _copy(src, dst_dir, name):
    os.makedirs(dst_dir, exist_ok=True)
    dst = os.path.join(dst_dir, name)
    shutil.copyfile(src, dst)
    return dst


def _sources(tmp_path):
    out = {}
    for name, gz in (("mixed", False), ("crlf_blank", True), ("fastq", False), ("inline_gt", False)):
        out[f"{name}{'.gz' if gz else ''}"] = write_case(tmp_path / "src", name, gz)
    out["test_2"] = os.path.join(FIX, "test_2", "ref_chr21_20kb.fa")
    out["test_4"] = os.path.join(FIX, "test_4", "reference.fasta.gz")
    return out


def _compare_caches(ours, theirs, k, skip):
    ht = f"-ht-{k}-{skip}.2.ngm"
    assert open(ours + ht, "rb").read() == open(theirs + ht, "rb").read()
    mine, ref = open(ours + "-enc.2.ngm", "rb").read(), open(theirs + "-enc.2.ngm", "rb").read()
    n = int(np.frombuffer(mine[4:8], dtype="<u4")[0])
    used = int(np.frombuffer(mine[8:16], dtype="<u8")[0]) // 2
    defined = 24 + 128 * n + used
    assert len(mine) == len(ref) and mine[:defined] == ref[:defined]


@need_plain
@pytest.mark.parametrize("which", ["mixed", "crlf_blank.gz", "fastq", "inline_gt", "test_2", "test_4"])
def test_caches_byte_identical_to_plain_ngmlr(tmp_path, which):
    src = _sources(tmp_path)[which]
    name = os.path.basename(src)
    ours, theirs = _copy(src, str(tmp_path / "ours"), name), _copy(src, str(tmp_path / "theirs"), name)
    a = B200Aligner(0)
    try:
        got = a.load_reference(ours)
    finally:
        a.close()
    assert (got.reference_read, got.reference_written, got.index_read, got.index_written) == (False, True, False, True)
    _ngmlr(theirs, _query(tmp_path), str(tmp_path / "o.sam"))
    _compare_caches(ours, theirs, 13, 2)
    ref, names = ngmfiles.read_encoded_reference(theirs + "-enc.2.ngm")
    assert [n.encode() for n in names] == got.names
    assert ref.ref_start == got.starts and ref.ref_len == got.lens and ref.concat_len == got.concat_len


@need_plain
def test_non_default_kmer_length_and_skip(tmp_path):
    src = os.path.join(FIX, "test_2", "ref_chr21_20kb.fa")
    ours, theirs = _copy(src, str(tmp_path / "ours"), "r.fa"), _copy(src, str(tmp_path / "theirs"), "r.fa")
    r = subprocess.run([sys.executable, "-m", "ngmlr_b200.index", ours, "-k", "12", "--kmer-skip", "1"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "ms" in r.stdout and "written" in r.stdout
    _ngmlr(theirs, _query(tmp_path), str(tmp_path / "o.sam"), "-k", "12", "--kmer-skip", "1")
    _compare_caches(ours, theirs, 12, 1)


def _state(a):
    """The context's encoded genome, concat length and k-mer index."""
    import ctypes as C
    a.lib.ngmlr_b200_cs_get_reference.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                                  C.POINTER(C.c_uint64)]
    nb, cl = C.c_uint64(0), C.c_uint64(0)
    a._check(a.lib.ngmlr_b200_cs_get_reference(a.h, None, 0, C.byref(nb), C.byref(cl)))
    ref = np.zeros(nb.value, np.uint8)
    a._check(a.lib.ngmlr_b200_cs_get_reference(a.h, ref.ctypes.data_as(C.c_void_p), ref.size, None, None))
    idx = a.get_index()
    return ref, cl.value, idx


def _reads():
    seq = b"".join(l.strip() for l in open(os.path.join(FIX, "test_2", "ref_chr21_20kb.fa"), "rb") if not l.startswith(b">"))
    seq = seq.upper()
    rng = np.random.default_rng(4)
    out = []
    for i in range(40):
        L = (150, 600, 2000)[i % 3]
        s = int(rng.integers(0, len(seq) - L))
        out.append(seq[s:s + L])
    return out


def test_second_load_reads_the_caches_and_installs_the_same_arrays(tmp_path):
    src = _copy(os.path.join(FIX, "test_2", "ref_chr21_20kb.fa"), str(tmp_path), "r.fa")
    reads = _reads()
    a, b = B200Aligner(0), B200Aligner(0)
    try:
        first = a.load_reference(src)
        assert first.reference_written and first.index_written
        s1 = _state(a)
        a.reads_upload(reads)
        a.cs_run()
        c1 = a.cs_fetch()
        files = [src + "-enc.2.ngm", src + "-ht-13-2.2.ngm"]
        mtimes = [os.stat(f).st_mtime_ns for f in files]
        second = b.load_reference(src)
        assert (second.reference_read, second.reference_written, second.index_read, second.index_written) == \
            (True, False, True, False)
        assert [os.stat(f).st_mtime_ns for f in files] == mtimes
        assert (second.names, second.starts, second.lens, second.concat_len) == \
            (first.names, first.starts, first.lens, first.concat_len)
        s2 = _state(b)
        assert np.array_equal(s1[0], s2[0]) and s1[1] == s2[1]
        for x, y in ((s1[2].tab, s2[2].tab), (s1[2].rci, s2[2].rci), (s1[2].pos, s2[2].pos)):
            assert np.array_equal(x, y)
        b.reads_upload(reads)
        b.cs_run()
        c2 = b.cs_fetch()
        assert int(c1[0][-1]) > 0
        for x, y in zip(c1, c2):
            assert np.array_equal(x, y)
        # a context sharing the loaded reference keeps working
        c = B200Aligner(0)
        try:
            c.share_reference(b)
            c.reads_upload(reads)
            c.cs_run()
            for x, y in zip(c1, c.cs_fetch()):
                assert np.array_equal(x, y)
        finally:
            c.close()
        # a truncated and a foreign index file are rebuilt (and rewritten as before)
        good = open(files[1], "rb").read()
        for bad in (good[:len(good) // 2], b"\x00" * 64 + good[64:]):
            open(files[1], "wb").write(bad)
            r = b.load_reference(src)
            assert r.reference_read and not r.index_read and r.index_written
            assert open(files[1], "rb").read() == good
        r = b.load_reference(src, rebuild=True, skip_write=True)
        assert not (r.reference_read or r.reference_written or r.index_read or r.index_written)
    finally:
        a.close()
        b.close()


@need_plain
def test_ngmlr_from_gpu_caches_and_library_sam_file(tmp_path):
    fa = os.path.join(FIX, "test_2", "ref_chr21_20kb.fa")
    reads_fa = os.path.join(FIX, "test_2", "reads_100_2200bp.fa")
    gpu_ref, own_ref = _copy(fa, str(tmp_path / "gpu"), "ref.fa"), _copy(fa, str(tmp_path / "own"), "ref.fa")
    r = subprocess.run([sys.executable, "-m", "ngmlr_b200.index", gpu_ref], capture_output=True, text=True, timeout=600,
                       cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    # the unmodified ngmlr reads the caches the GPU wrote (it leaves them untouched) and writes the SAM of its own build
    caches = [gpu_ref + "-enc.2.ngm", gpu_ref + "-ht-13-2.2.ngm"]
    mtimes = [os.stat(f).st_mtime_ns for f in caches]
    _ngmlr(gpu_ref, reads_fa, str(tmp_path / "gpu.sam"))
    assert [os.stat(f).st_mtime_ns for f in caches] == mtimes
    _ngmlr(own_ref, reads_fa, str(tmp_path / "own.sam"), skip_write=True)
    body = lambda p: [l for l in open(p, "rb") if not l.startswith(b"@")]
    sq = lambda p: [l for l in open(p, "rb") if l.startswith(b"@SQ")]
    assert body(tmp_path / "gpu.sam") == body(tmp_path / "own.sam") and len(body(tmp_path / "own.sam")) >= 10
    assert sq(tmp_path / "gpu.sam") == sq(tmp_path / "own.sam")
    # the library from the same FASTA file to the SAM file of the short reads
    names, reads = [], []
    for line in open(reads_fa, "rb"):
        line = line.strip()
        if line.startswith(b">"):
            names.append(line[1:].split()[0])
            reads.append(b"")
        elif line:
            reads[-1] += line
    clean = lambda s: bytes(b if b in b"ACGT" else ord("N") for b in s.upper())
    short = [(n, clean(s)) for n, s in zip(names, reads) if len(s) <= 256]
    assert [n for n, _ in short] == [b"100bp", b"200bp"]
    fq = str(tmp_path / "short.fq")
    with open(fq, "wb") as f:
        for n, s in short:
            f.write(b"@" + n + b"\n" + s + b"\n+\n" + b"I" * len(s) + b"\n")
    plain_sam = str(tmp_path / "short.sam")
    _ngmlr(_copy(fa, str(tmp_path / "plain"), "ref.fa"), fq, plain_sam, skip_write=True)
    want = open(plain_sam, "rb").read()
    pg = [l for l in want.split(b"\n") if l.startswith(b"@PG")][0]
    version, cmdline = pg.split(b"\t")[3][3:], pg.split(b"\tCL:", 1)[1]
    a = B200Aligner(0)
    try:
        ref = a.load_reference(_copy(fa, str(tmp_path / "fresh"), "ref.fa"), skip_write=True)
        a.reads_upload([s for _, s in short])
        a.cs_run()
        res = a.map_short_reads()
    finally:
        a.close()
    header = samtext.sam_header(ref.names, ref.lens, version, cmdline)
    recs = b"".join(samtext.sam_format([samtext.Read(n, s, b"I" * len(s), r[1], r[0])], ref.sam_ref_names(), threads=1)
                    for (n, s), r in zip(short, res))
    assert header + recs == want


def test_failures_leave_the_context_as_it_was(tmp_path):
    src = _copy(os.path.join(FIX, "test_2", "ref_chr21_20kb.fa"), str(tmp_path), "r.fa")
    a = B200Aligner(0)
    try:
        good = a.load_reference(src, skip_write=True)
        before = _state(a)
        open(tmp_path / "empty.fa", "wb").close()
        with open(tmp_path / "short.fa", "wb") as f:
            f.write(b">a\nACGT\n>b\nACGTACGTAC\n")
        # a cached genome over the single-unit limit: a header claiming 2^32 positions
        big = str(tmp_path / "big.fa")
        with open(big, "wb") as f:
            f.write(b">x\nACGTACGTACGTACGT\n")
        with open(big + "-enc.2.ngm", "wb") as f:
            f.write(np.array([0x74656, 1], "<u4").tobytes() + np.array([1 << 32, 1 << 31], "<u8").tobytes()
                    + bytes(128))   # one RefIdx record; the genome's bytes are never read
        for path, msg in ((str(tmp_path / "missing.fa"), "cannot open"), (str(tmp_path / "empty.fa"), "no sequence"),
                          (str(tmp_path / "short.fa"), "no sequence"), (big, "table unit")):
            with pytest.raises(RuntimeError, match=msg):
                a.load_reference(path)
        assert not os.path.exists(str(tmp_path / "empty.fa-enc.2.ngm"))
        after = _state(a)
        assert np.array_equal(before[0], after[0]) and before[1] == after[1]
        assert np.array_equal(before[2].pos, after[2].pos) and np.array_equal(before[2].tab, after[2].tab)
        assert a.lib.ngmlr_b200_reference_contigs(a.h, None, None, None, None) == len(good.names)
        # another call that replaces the reference ends the contig table
        a.encode_reference([b"ACGT" * 100], fetch=False)
        assert a.lib.ngmlr_b200_reference_contigs(a.h, None, None, None, None) < 0
    finally:
        a.close()
