"""BAM input of ngmlr_b200_reads_load (B200Aligner.load_reads) on the GPU, against ngmlr's ReadProvider reading the
text `samtools fastq -n` writes for the same records (tests/bam_cases.py):
  - record parity: every case as BGZF (4 KiB members, so headers and records straddle members), plain gzip and an
    uncompressed stream, at the default chunk, 4 KiB and a chunk smaller than one record (which must grow), with
    max_reads 1 / 7 / all and a small max_bases; the BAM counters per case; a chunk end on every byte of one record's
    36-byte fixed part;
  - resident equivalence: the read arena, offsets, sub-read table and cs_run / cs_fetch equal reads_upload's of the
    reference reader's strings at --subread-length 256 and 1000;
  - file to SAM: test_2's short reads and 2 000 synthetic short reads as BAM, half stored reverse-complemented under
    0x10, with secondary and supplementary copies: load -> cs_run -> map_short_reads -> sam_format prints the plain
    ngmlr binary's SAM body for the equivalent FASTQ;
  - errors: every malformed stream fails with a message naming its offset, the handle stays failed, the context
    loads a good file afterwards;
  - memory: the handle's peak device memory stays under the header's bound for BGZF BAM at two chunk sizes."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import bam_cases as B
import read_loader_cases as R
import test_gpu_read_loader as T
from ngmlr_b200 import B200Aligner, _lib
from ngmlr_b200.samtext import SamRead

pytestmark = pytest.mark.gpu
need_full = pytest.mark.skipif(not os.path.exists(R.FULL), reason="oracle/_ref/libngmlr_reads.so not built")
need_plain = pytest.mark.skipif(not os.path.exists(T.PLAIN), reason="oracle/_ref/ngmlr not built")


@pytest.fixture(scope="module")
def aligner():
    a = B200Aligner(0)
    yield a
    a.close()


def _load_all(a, path, **kw):
    reads, sizes, last = [], [], None
    for b in a.load_reads(path, **kw):
        reads += [(r.name, r.seq, r.qual, len(r.seq), int(r.empty)) for r in b.reads]
        sizes.append(len(b.reads))
        last = b
    return reads, sizes, last


def _write(tmp_path, name, mode):
    return B.write_case(tmp_path / mode, name, mode, block=4096)


def _check(a, path, want, counters, where, **kw):
    got, sizes, last = _load_all(a, path, **kw)
    assert len(got) == len(want), where
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{where} read {i}: {g[:1]} {g[3:]} vs {w[:1]} {w[3:]}"
    assert all(s <= kw.get("max_reads", 100_000) for s in sizes), where
    assert last.format == _lib.READ_FORMAT_BAM, where
    # the last batch's counters are those of the records walked so far (skipped records may follow it)
    seen = (last.bam_header_bytes, last.bam_records, last.bam_skipped, last.bam_reversed, last.bam_no_quality)
    assert seen[0] == counters[0] and all(x <= y for x, y in zip(seen, counters)), where
    assert last.records == len(want), where
    if kw.get("max_reads") == 100_000 and not kw.get("max_bases"):
        assert _raw_counters(a, path, kw.get("chunk_bytes", 0)) == counters, where
    return last


def _raw_counters(a, path, chunk):
    """ngmlr_b200_read_file_bam_stats once reads_load has reached the end of the file."""
    lib = a.lib
    f = C.c_void_p()
    opts = _lib.ReadFileOptions(chunk)
    assert lib.ngmlr_b200_read_file_open(os.fsencode(path), C.byref(opts), C.byref(f)) == 0
    assert lib.ngmlr_b200_read_file_format(f) == -1
    recs = (SamRead * 100_000)()
    n, nd = C.c_int32(0), C.c_int32(0)
    try:
        while True:
            assert a._check(lib.ngmlr_b200_reads_load(a.h, f, 100_000, 0, 256, recs, C.byref(n), C.byref(nd))) >= 0
            if n.value == 0:
                break
        assert lib.ngmlr_b200_read_file_format(f) == _lib.READ_FORMAT_BAM
        st = [C.c_int64(0) for _ in range(5)]
        assert lib.ngmlr_b200_read_file_bam_stats(f, *[C.byref(x) for x in st]) == 0
        return tuple(x.value for x in st)
    finally:
        lib.ngmlr_b200_read_file_close(f)


@need_full
@pytest.mark.parametrize("mode", ["bgzf", "gzip", "plain"])
def test_records_equal_reference_reader(aligner, tmp_path, mode):
    checked = 0
    for name in B.CASES:
        hdr, recs = B.CASES[name]
        path = _write(tmp_path, name, mode)
        want = R.as_loaded(R.oracle_reads(B.write_text(tmp_path / "o", name))[0])
        counters = B.counters(hdr, recs)
        longest = max(len(B.record(r)) for r in recs)
        small = max(16, longest // 4)
        if name in B.BIG:
            plan = [(0, 100_000, 0), (4096, 100_000, 0), (4096, 1000, 5000), (small, 100_000, 0)]
        else:
            plan = [(c, m, b) for c in (0, 4096, small) for m, b in ((1, 0), (7, 0), (100_000, 0), (100_000, 150))]
        for chunk, max_reads, max_bases in plan:
            where = f"{name} {mode} chunk={chunk} max_reads={max_reads} max_bases={max_bases}"
            last = _check(aligner, path, want, counters, where, chunk_bytes=chunk, max_reads=max_reads,
                          max_bases=max_bases)
            if chunk == small and longest > 4 * 16:
                assert last.grows > 0, where
            checked += 1
    assert checked >= 8 * 12 + 3 * 4


@need_full
@pytest.mark.parametrize("mode", ["bgzf", "plain"])
def test_chunk_end_on_every_fixed_byte(aligner, tmp_path, mode):
    hdr, recs = B.CASES["aligned"]
    path = _write(tmp_path, "aligned", mode)
    want = R.as_loaded(R.oracle_reads(B.write_text(tmp_path / "o", "aligned"))[0])
    first = len(hdr) + len(B.record(recs[0]))
    for k in range(37):  # the chunk ends k bytes into the second record (its block_size and fixed fields)
        _check(aligner, path, want, B.counters(hdr, recs), f"{mode} chunk end +{k}", chunk_bytes=first + k,
               max_reads=5)


@need_full
@pytest.mark.parametrize("rpl", [256, 1000])
def test_resident_set_equals_reads_upload(tmp_path, rpl):
    ref = T.shutil.copyfile(os.path.join(T.FIX, "ref_chr21_20kb.fa"), str(tmp_path / "ref.fa"))
    a, b = B200Aligner(0), B200Aligner(0)
    try:
        a.load_reference(ref, skip_write=True)
        b.load_reference(ref, skip_write=True)
        # at --subread-length 1000 ngmlr's Empty reads overrun their buffer badly enough to abort (as in the text tests)
        names = ("aligned", "odd", "codes", "empty", "pacbio") if rpl == 256 else ("aligned", "odd", "pacbio", "long_read")
        for name in names:
            path = _write(tmp_path, name, "bgzf")
            want = [s for _, s, _, _, _ in R.as_loaded(R.oracle_reads(B.write_text(tmp_path / "o", name), rpl)[0], rpl)]
            k = 0
            for batch in a.load_reads(path, read_part_length=rpl, max_reads=16, chunk_bytes=8192):
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


def _as_bam_records(reads, seed):
    """BAM records of (name, seq, qual) reads: half stored reverse-complemented under 0x10 (only reads with qualities:
    ngmlr's writer overruns the "*" of a reverse FASTA read), with secondary and supplementary copies between them."""
    rng = random.Random(seed)
    recs = []
    for name, seq, qual, _length, empty in reads:
        s = seq.decode()
        q = None if qual == b"*" else [c - 33 for c in qual]
        if empty:
            s, q = "", []
        r = B.Rec(name, s, q, flag=4)
        if q and rng.random() < 0.5:
            r = B.Rec(name, B._revcomp(s), q[::-1], flag=0x10, ref_id=0, pos=rng.randrange(10000), mapq=30,
                      cigar=[(len(s), 0)])
        recs.append(r)
        if rng.random() < 0.1:
            junk = "".join(rng.choice("ACGTN") for _ in range(rng.randint(1, 200)))
            recs.append(B.Rec(name, junk, [30] * len(junk), flag=rng.choice([0x100, 0x800, 0x110, 0x810])))
    return recs


@need_full
@need_plain
@pytest.mark.parametrize("which,rpl", [("test_2", 256), ("synthetic", 257)])
def test_file_to_sam_equals_plain_ngmlr(tmp_path, which, rpl):
    src = str(tmp_path / "reads.fq")
    if which == "test_2":
        T._test2_short_fastq(src)
    else:
        T._short_reads_file(src)
    # test_2 has two short reads: a seed that stores both reversed and adds a secondary copy
    recs = _as_bam_records(R.as_loaded(R.oracle_reads(src)[0]), 4 if which == "test_2" else 3)
    kept = [r for r in recs if not r.flag & B.SKIP]
    assert sum(1 for r in kept if r.flag & 0x10) >= len(kept) // 3 and len(kept) < len(recs)
    hdr = B.header(b"@HD\tVN:1.6\n", [(b"chr21", 20000)])
    query = B.write(str(tmp_path / "reads.bam"), B.bam_stream(hdr, recs), "bgzf")
    text = str(tmp_path / "equivalent.fq")
    with open(text, "wb") as f:
        f.write(B.fastq_text(recs))
    want = T._ngmlr_sam(str(tmp_path), text, str(tmp_path / "plain.sam"), rpl)
    got = T._library_sam(tmp_path, query, rpl)
    assert len(want) >= 2
    assert got == want


def _raw_load(a, path, chunk=0):
    """reads_load through the C ABI until it fails or the file ends: ([return values], [messages])."""
    lib = a.lib
    f = C.c_void_p()
    opts = _lib.ReadFileOptions(chunk)
    assert lib.ngmlr_b200_read_file_open(os.fsencode(path), C.byref(opts), C.byref(f)) == 0
    recs = (SamRead * 64)()
    n, nd = C.c_int32(0), C.c_int32(0)
    rets, msgs = [], []
    try:
        for _ in range(100):
            r = lib.ngmlr_b200_reads_load(a.h, f, 64, 0, 256, recs, C.byref(n), C.byref(nd))
            rets.append(r)
            if r < 0:
                msgs.append(lib.ngmlr_b200_last_error(a.h).decode())
                if len(msgs) == 2:
                    break
            elif n.value == 0:
                break
    finally:
        lib.ngmlr_b200_read_file_close(f)
    return rets, msgs


@pytest.mark.parametrize("mode", ["bgzf", "plain"])
def test_errors_name_the_offset(aligner, tmp_path, mode):
    for name, (data, at, pattern) in B.ERRORS.items():
        path = B.write(str(tmp_path / f"{name}.bam"), data, mode, block=4096)
        for chunk in (0, 64):
            rets, msgs = _raw_load(aligner, path, chunk)
            where = f"{name} {mode} chunk={chunk}: {rets} {msgs}"
            assert len(msgs) == 2 and rets[-1] < 0 and rets[-2] < 0, where
            assert pattern in msgs[0] and f"stream offset {at}" in msgs[0], where
            assert msgs[1] == msgs[0], where
    # the context still loads a good file
    hdr, recs = B.CASES["odd"]
    got, _, _ = _load_all(aligner, _write(tmp_path, "odd", mode))
    assert [g[0] for g in got] == [r.name for r in recs]


@pytest.mark.parametrize("name", ["many_short", "long_read"])
def test_device_memory_under_bound(aligner, tmp_path, name):
    path = _write(tmp_path, name, "bgzf")
    for chunk in (64 << 10, 4 << 20):
        got, _, last = _load_all(aligner, path, chunk_bytes=chunk, max_reads=100_000)
        assert len(got) == sum(1 for r in B.CASES[name][1] if not r.flag & B.SKIP)
        assert 0 < last.device_bytes < 8 * max(last.chunk_cap, 1 << 20), (name, chunk, last.device_bytes,
                                                                          last.chunk_cap)
