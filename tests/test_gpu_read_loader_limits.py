"""ngmlr_b200_reads_load (B200Aligner.load_reads) at the limits of its chunk path, record for record against the
unmodified ReadProvider (read_loader_cases.oracle_reads). Each test asserts the chunk counters that show it reached the
branch it is about:
  - line-limited chunks: files whose lines average under 32 bytes (SRA-style 36 bp FASTQ, one-line and narrowly
    wrapped FASTA, blank-line runs, the loader fuzz text repeated) at 256 KiB, 1 MiB and 1 MiB + 13, and at one chunk
    holding the whole file; the limit-th newline on a chunk's last byte, its second-to-last, or before a header;
  - growth: a record with more lines than the line table (FASTA at width 1, FASTQ at width 2) first, in the middle,
    last and without a trailing newline; a record longer than the chunk and one with too many lines in one file; the
    expected doublings, the grown capacity and the device memory bound against it (plain and BGZF);
  - chunk boundaries: every chunk size from 16 bytes for the small read_loader_cases, the 16 / 32 KiB cases within
    64 bytes of 16 KiB and of their length, and BGZF copies at one size in seven;
  - segment edges: headers at offsets 2047 / 2048 / 4095 / 4096, junk runs over several 2 KiB segments;
  - scale: about 40 MB of mixed reads in one chunk of ~10^5 records, in 1 MiB and 300 001-byte chunks, gzip, BGZF;
  - file to SAM: 10 000 SRA-style short reads through a line-limited chunk to the plain ngmlr binary's SAM body."""
import gzip
import os

import pytest

import bgzf_cases as B
import read_loader_cases as R
import read_loader_limits as X
import test_gpu_read_loader as T
from ngmlr_b200 import B200Aligner

pytestmark = [pytest.mark.gpu, T.need_full]
KiB, MiB = X.KiB, X.MiB


@pytest.fixture(scope="module")
def aligner():
    a = B200Aligner(0)
    yield a
    a.close()


def _write(path, blob):
    with open(path, "wb") as f:
        f.write(blob)
    return str(path)


def _oracle(tmp_path, name, data):
    reads, dropped = R.oracle_reads(_write(tmp_path / (name + ".oracle.fq"), data))
    return R.as_loaded(reads), dropped


def _load(a, path, **kw):
    """The concatenated records, the dropped names and the last batch (its counters are the handle's)."""
    reads, dropped, last = [], [], None
    for b in a.load_reads(path, **kw):
        reads += [(r.name, r.seq, r.qual, len(r.seq), int(r.empty)) for r in b.reads]
        dropped += b.dropped
        last = b
    return reads, dropped, last


def _check(a, path, want, where, **kw):
    """Loads path, compares with the oracle's (reads, dropped) and returns the last batch."""
    got, drop, last = _load(a, path, **kw)
    reads, dropped = want
    assert len(got) == len(reads), where
    for i, (g, w) in enumerate(zip(got, reads)):
        assert g == w, f"{where} read {i}: {g[:1]} {g[3:]} vs {w[:1]} {w[3:]}"
    assert drop == dropped, where
    assert last is not None and last.records == len(got), where
    return last


def _ctr(b):
    return {k: getattr(b, k) for k in ("records", "device_bytes", "chunks", "line_limited", "grows", "chunk_cap",
                                       "device_members", "host_bytes")}


def _bound(last, bgzf=False):
    if bgzf:
        return 0 < last.device_bytes < 11 * max(last.chunk_cap, MiB)
    return 0 < last.device_bytes < 9 * max(last.chunk_cap, 128 * KiB)


# ---- line-limited chunks ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["sra36", "fasta_oneline", "fasta_wrapped", "blank_runs", "fuzz_repeat"])
def test_line_limited_chunks(aligner, tmp_path, name):
    data = X.dense()[name]
    path = _write(tmp_path / (name + ".fq"), data)
    want = _oracle(tmp_path, name, data)
    for chunk in (256 * KiB, MiB, MiB + 13, len(data) + 1):
        where = f"{name} chunk={chunk}"
        last = _check(aligner, path, want, where, chunk_bytes=chunk)
        # len(data) + 1: the whole file is read at once, so the stream has ended while its first chunk is line-limited
        assert last.line_limited >= (1 if chunk > len(data) else 2), (where, _ctr(last))
        assert last.grows == 0 and last.chunk_cap == chunk, (where, _ctr(last))
        assert _bound(last), (where, last.device_bytes)


@pytest.mark.parametrize("capacity", [256 * KiB, MiB + 13])
@pytest.mark.parametrize("fastq", [False, True])
def test_limit_th_newline_at_chunk_end(aligner, tmp_path, capacity, fastq):
    for where in X.LIMIT_EDGES:
        data = X.limit_edge(capacity, where, fastq)
        path = _write(tmp_path / f"{where}.fq", data)
        want = _oracle(tmp_path, where, data)
        last = _check(aligner, path, want, f"{where} fastq={fastq} capacity={capacity}", chunk_bytes=capacity)
        assert last.line_limited >= 1 and last.grows == 0, (where, _ctr(last))


# ---- growth ----------------------------------------------------------------------------------------------------------
GROWTH = {"fasta1": 12_000, "fastq2": 24_002}  # lines: one doubling at 256 KiB (limit 8192), two


@pytest.mark.parametrize("kind", ["fasta1", "fastq2"])
def test_growth_by_lines(aligner, tmp_path, kind):
    chunk = 256 * KiB
    rec = X.long_record(kind, GROWTH[kind])
    expect = X.doublings(chunk, GROWTH[kind] + 2)
    assert expect == {"fasta1": 1, "fastq2": 2}[kind]
    for where in ("first", "middle", "last", "last_no_nl"):
        data = X.around(rec, where)
        path = _write(tmp_path / f"{where}.fq", data)
        want = _oracle(tmp_path, where, data)
        assert any(len(r[1]) > 10_000 for r in want[0])
        tag = f"{kind} {where}"
        last = _check(aligner, path, want, tag, chunk_bytes=chunk)
        assert last.grows == expect and last.chunk_cap == chunk << expect, (tag, _ctr(last))
        assert _bound(last), (tag, last.device_bytes, last.chunk_cap)
        packed = _write(tmp_path / f"{where}.fq.gz", B.bgzf(data, 1))
        last = _check(aligner, packed, want, tag + " bgzf", chunk_bytes=chunk)
        assert last.grows == expect and last.chunk_cap == chunk << expect and last.device_members > 0, (tag, _ctr(last))
        assert _bound(last, bgzf=True), (tag, last.device_bytes, last.chunk_cap)


def test_growth_by_bytes_and_lines(aligner, tmp_path):
    chunk = 256 * KiB
    wide, long_ = X.wide_record(600_000), X.long_record("fasta1", 40_000)
    cases = {"bytes": (X.around(wide, "middle"), X.doublings(chunk, nbytes=600_010)),
             "bytes_then_lines": (X.around(wide, "first") + long_ + X.sra_fastq(5, 500),
                                  X.doublings(chunk, lines=40_002, nbytes=600_010)),
             "lines_then_bytes": (X.around(long_, "first") + wide + X.sra_fastq(6, 500),
                                  X.doublings(chunk, lines=40_002, nbytes=600_010))}
    assert [c[1] for c in cases.values()] == [2, 3, 3]
    for name, (data, expect) in cases.items():
        path = _write(tmp_path / f"{name}.fq", data)
        want = _oracle(tmp_path, name, data)
        last = _check(aligner, path, want, name, chunk_bytes=chunk)
        assert last.grows == expect and last.chunk_cap == chunk << expect, (name, _ctr(last))
        assert _bound(last), (name, last.device_bytes, last.chunk_cap)
        packed = _write(tmp_path / f"{name}.fq.gz", B.bgzf(data, 1))
        last = _check(aligner, packed, want, name + " bgzf", chunk_bytes=chunk)
        assert last.grows == expect and _bound(last, bgzf=True), (name, _ctr(last))


# ---- chunk boundaries ------------------------------------------------------------------------------------------------
def test_chunk_boundary_sweep(aligner, tmp_path):
    loads = 0
    for name, data in R.CASES.items():
        if len(data) >= 2 * KiB:
            continue
        path = R.write_case(tmp_path, name)
        packed = _write(tmp_path / f"{name}.bgzf.gz", B.bgzf(data, 6, block=97))
        want = _oracle(tmp_path, name, data)
        for chunk in range(16, min(len(data) + 1, 600) + 1):
            where = f"{name} chunk={chunk}"
            last = _check(aligner, path, want, where, chunk_bytes=chunk)
            assert _bound(last), (where, last.device_bytes)
            # a first chunk of a quarter of the file can end the load only by a dropped read, which needs more bytes
            assert last.chunks >= (2 if chunk <= len(data) // 4 else 1), (where, _ctr(last))
            if chunk % 10 == 0:
                _check(aligner, path, want, where + " max_reads=1", chunk_bytes=chunk, max_reads=1)
            if chunk % 7 == 0:
                _check(aligner, packed, want, where + " bgzf", chunk_bytes=chunk)
            loads += 1
    assert loads > 3000


def test_chunk_boundary_sweep_16k(aligner, tmp_path):
    for name, data in R.CASES.items():
        if name not in ("kb16_nl", "kb32_no_nl", "kb16_header_last", "kb16_lone_cr_last", "kb16_cr_qual"):
            continue
        path = R.write_case(tmp_path, name)
        packed = _write(tmp_path / f"{name}.bgzf.gz", B.bgzf(data, 6, block=5000))
        want = _oracle(tmp_path, name, data)
        sizes = sorted(set(range(16384 - 64, 16384 + 65)) | set(range(len(data) - 64, len(data) + 65)))
        for i, chunk in enumerate(sizes):
            where = f"{name} chunk={chunk}"
            last = _check(aligner, path, want, where, chunk_bytes=chunk)
            assert last.chunks >= (2 if chunk < len(data) else 1), (where, _ctr(last))
            if i % 7 == 0:
                _check(aligner, packed, want, where + " bgzf", chunk_bytes=chunk)


# ---- segment edges ---------------------------------------------------------------------------------------------------
def test_segment_edges(aligner, tmp_path):
    for name, data in X.segment_edges().items():
        path = _write(tmp_path / f"{name}.fq", data)
        want = _oracle(tmp_path, name, data)
        assert want[0], name
        last = _check(aligner, path, want, name)
        assert last.chunks == 1, (name, _ctr(last))
        last = _check(aligner, path, want, name + " chunk=4097", chunk_bytes=4097)
        assert last.chunks >= len(data) // 4097, (name, _ctr(last))


# ---- scale -----------------------------------------------------------------------------------------------------------
def test_scale_fuzz(aligner, tmp_path):
    data = X.scale_fuzz()
    path = _write(tmp_path / "scale.fq", data)
    want = _oracle(tmp_path, "scale", data)
    assert len(want[0]) > 100_000 and want[1] == [b"bad"]
    last = _check(aligner, path, want, "scale default chunk")
    assert last.chunks == 1, _ctr(last)
    for chunk in (MiB, 300_001):
        last = _check(aligner, path, want, f"scale chunk={chunk}", chunk_bytes=chunk)
        assert last.chunks > (100 if chunk < MiB else 30), (chunk, _ctr(last))
    gz = str(tmp_path / "scale.fq.gz")
    with gzip.open(gz, "wb", compresslevel=1) as f:
        f.write(data)
    last = _check(aligner, gz, want, "scale gzip", chunk_bytes=MiB)
    assert last.chunks > 30, _ctr(last)
    packed = _write(tmp_path / "scale.bgzf.gz", B.bgzf(data, 1))
    last = _check(aligner, packed, want, "scale bgzf", chunk_bytes=MiB)
    assert last.chunks > 30 and last.device_members > 0 and last.host_bytes == 0, _ctr(last)
    assert _bound(last, bgzf=True), _ctr(last)


# ---- file to SAM -----------------------------------------------------------------------------------------------------
@T.need_plain
def test_file_to_sam_through_line_limited_chunks(tmp_path):
    genome = b"".join(l.strip() for l in open(os.path.join(T.FIX, "ref_chr21_20kb.fa"), "rb") if not l.startswith(b">"))
    data = X.sra_fastq(41, 10_000, 24, 36, genome=genome.upper())
    assert X.mean_line(data) < 32
    query = _write(tmp_path / "sra.fq", data)
    a = B200Aligner(0)
    try:
        batches = list(a.load_reads(query, chunk_bytes=256 * KiB, max_reads=500))
    finally:
        a.close()
    assert batches[-1].line_limited >= 1 and batches[-1].records == 10_000, _ctr(batches[-1])
    want = T._ngmlr_sam(str(tmp_path), query, str(tmp_path / "plain.sam"), 256)
    got = T._library_sam(tmp_path, query, 256, chunk_bytes=256 * KiB)
    assert len(want) >= 1000
    assert got == want
