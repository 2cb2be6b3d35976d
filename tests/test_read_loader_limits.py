"""CPU checks of the generators of read_loader_limits: each file reaches the part of the loader's chunk path that
tests/test_gpu_read_loader_limits.py uses it for, and (where oracle/_ref/libngmlr_reads.so is built) ngmlr's
ReadProvider parses it."""
import os
import re

import pytest

import read_loader_cases as R
import read_loader_limits as X

KiB, MiB = X.KiB, X.MiB
need_full = pytest.mark.skipif(not os.path.exists(R.FULL), reason="oracle/_ref/libngmlr_reads.so not built")


def _parses(tmp_path, name, data):
    path = str(tmp_path / (name + ".fq"))
    with open(path, "wb") as f:
        f.write(data)
    return R.oracle_reads(path)


def test_limit_and_doublings():
    assert X.limit(256 * KiB) == 8192 and X.limit(MiB + 13) == 32768 and X.limit(4096) == 4096
    assert X.doublings(256 * KiB, lines=8192) == 0 and X.doublings(256 * KiB, lines=8193) == 1
    assert X.doublings(256 * KiB, nbytes=600_000) == 2 and X.doublings(256 * KiB, 40_002, 600_000) == 3


def test_dense_files_overflow_the_line_table():
    for name, data in X.dense().items():
        assert X.mean_line(data) < 32, name
        for chunk in (256 * KiB, MiB, MiB + 13):
            # every full chunk holds more newlines than its line table
            assert data[:chunk].count(b"\n") > X.limit(chunk), (name, chunk)
            assert len(data) > 2 * chunk, (name, chunk)
        assert data.count(b"\n") > X.limit(len(data) + 1), name
    sra = X.sra_fastq(1, 100)
    assert sra.split(b"\n")[2] == b"+" + sra.split(b"\n")[0][1:] and len(sra.split(b"\n")[1]) == 36


@pytest.mark.parametrize("capacity", [256 * KiB, MiB + 13])
@pytest.mark.parametrize("fastq", [False, True])
def test_limit_edges(capacity, fastq):
    L = X.limit(capacity)
    for where in X.LIMIT_EDGES:
        data = X.limit_edge(capacity, where, fastq)
        nl = [i for i, c in enumerate(data[:capacity]) if c == 10]
        p = nl[L - 1]  # the limit-th newline of the first chunk
        after = data[p + 1:p + 2]
        if where == "last":
            assert p == capacity - 1 and len(nl) == L
        elif where == "second_last_nl":
            assert p == capacity - 2 and after == b"\n" and len(nl) == L + 1
        elif where == "second_last_hdr":
            assert p == capacity - 2 and after == (b"@" if fastq else b">") and len(nl) == L
        else:
            assert p == capacity - 101 and after == (b"@" if fastq else b">") and len(nl) > L
        # the chunks after the first are line-limited
        assert data[capacity:2 * capacity].count(b"\n") > L, where


def test_long_records():
    for kind, lines in (("fasta1", 12_000), ("fastq2", 24_002), ("fasta1", 40_000)):
        rec = X.long_record(kind, lines)
        assert rec.count(b"\n") == lines, kind
        parts = rec.split(b"\n")
        assert max(len(x) for x in parts[1:]) <= (1 if kind == "fasta1" else 2)
    assert X.limit(256 * KiB) < 12_000 < X.limit(512 * KiB) < 24_002 < X.limit(MiB) < 40_000 < X.limit(2 * MiB)
    wide = X.wide_record(600_000)
    assert wide.count(b"\n") == 2 and len(wide) > 2 * 256 * KiB
    rec = X.long_record("fasta1", 12_000)
    for where in ("first", "middle", "last", "last_no_nl"):
        data = X.around(rec, where)
        assert (rec[:-1] if where == "last_no_nl" else rec) in data
        assert data.endswith(b"\n") == (where != "last_no_nl")


def test_segment_edges():
    files = X.segment_edges()
    for tag, offsets in X.EDGE_OFFSETS.items():
        for kind in ("hdr_at_edges_", "fastq_at_edges_"):
            marks = set(X.first_markers(files[kind + tag]))
            assert set(offsets) <= marks, (kind, tag)
            data = files[kind + tag]
            for off in offsets:
                assert data[off:off + 2] in (b">h", b"@m")
                if kind == "hdr_at_edges_":
                    assert data[off - 1:off] == b"\n"
    assert {2047, 2048, 4095, 4096} <= {o for t in X.EDGE_OFFSETS.values() for o in t}
    for name in ("junk_runs", "junk_runs_markers"):
        data = files[name]
        assert len(data) > 12 * 2 * KiB
        junk = re.sub(rb"@j\d+\n[ACGT]{50}\n\+\n[^\n]{50}\n", b"", data)
        assert len(junk) > 12 * 2 * KiB and b"\n+\n" not in junk
        assert bool(X.first_markers(junk)) == (name == "junk_runs_markers"), name
    # a FASTQ record followed by more than three whole segments without '>' / '@'
    data = files["marker_free_segments"]
    marks = X.first_markers(data)
    gaps = [b - a for a, b in zip(marks, marks[1:])]
    assert max(gaps) > 4 * X.SEG


def test_scale_fuzz():
    data = X.scale_fuzz()
    assert 40 * MiB <= len(data) < 42 * MiB
    assert data.count(b"\r\n") > 10_000 and data.count(b"\n+\n@") + data.count(b"\n+\r\n@") > 100
    assert max(len(x) for x in data.split(b"\n")) < 100_001
    assert data.rfind(b"@bad\n") > len(data) - 200


@need_full
def test_oracle_parses_every_generated_file(tmp_path):
    files = dict(X.dense())
    files.update(X.segment_edges())
    files["edge"] = X.limit_edge(256 * KiB, "hdr_after", True)
    files["long"] = X.around(X.long_record("fastq2", 24_002), "middle")
    files["scale"] = X.scale_fuzz()
    for name, data in files.items():
        reads, dropped = _parses(tmp_path, name, data)
        assert len(reads) >= 3, name
        assert dropped == ([b"bad"] if name == "scale" else []), name
