"""The read loader's CPU side: the query-file cases and what the unmodified ReadProvider (oracle/_ref/libngmlr_reads.so)
makes of them -- the rules the device loader (tests/test_gpu_read_loader.py) is held to -- and the C ABI's error paths
that need no device."""
import ctypes as C
import os

import pytest

import read_loader_cases as R
from ngmlr_b200 import _lib

need_full = pytest.mark.skipif(not os.path.exists(R.FULL), reason="oracle/_ref/libngmlr_reads.so not built")


def test_enough_cases_and_every_stream_size_rule():
    assert len(R.CASES) >= 20
    sizes = {n: len(b) for n, b in R.CASES.items()}
    assert sizes["kb16_nl"] == R.KB16 and sizes["kb32_no_nl"] == 2 * R.KB16 and sizes["kb16_cr_qual"] == R.KB16
    assert sizes["kb16_header_last"] == R.KB16 and R.CASES["kb16_header_last"].endswith(b">")
    assert not R.CASES["kb32_no_nl"].endswith(b"\n")


@need_full
def test_reference_reader_rules(tmp_path):
    got = {}
    for name in ("names", "empty", "mismatch_mid", "kb16_header_last", "header_last", "lone_cr_last",
                 "kb16_lone_cr_last", "iupac", "junk_between"):
        got[name] = R.oracle_reads(R.write_case(tmp_path, name))
    names = [r[0] for r in got["names"][0]]
    assert names[:3] == [b"n" * 249, b"o" * 249, b"p" * 249] and names[3:5] == [b"t1", b"v1"]
    # an empty record: read_part_length + 16 N's, flagged Empty; the reads after a -2 are never read
    assert [(r[0], r[3], r[4]) for r in got["empty"][0]][:2] == [(b"e1", 272, 1), (b"e2", 272, 1)]
    assert got["empty"][1] == [b"e5"] and got["mismatch_mid"][1] == [b"m2"] and len(got["mismatch_mid"][0]) == 1
    # the end of a stream of k x 16 KiB
    assert got["kb16_header_last"][0][-1][::4] == (b"", 1) and len(got["header_last"][0]) == 1
    assert got["lone_cr_last"][0][-1][1].endswith(b"N") and got["kb16_lone_cr_last"][0][-1][1].endswith(b"A")
    assert got["iupac"][0][0][1] == b"ACGTN" + b"N" * 26 + b"ACGT"
    assert [r[0] for r in got["junk_between"][0]] == [b"j1", b"j2", b"j3"]


@need_full
def test_gzip_copy_reads_the_same(tmp_path):
    for name in ("fastq_multi", "crlf", "kb16_nl"):
        assert R.oracle_reads(R.write_case(tmp_path, name)) == R.oracle_reads(R.write_case(tmp_path, name, gz=True))


def test_open_errors_need_no_device(tmp_path):
    lib = _lib.load()
    f = C.c_void_p()
    assert lib.ngmlr_b200_read_file_open(str(tmp_path / "missing.fq").encode(), None, C.byref(f)) < 0
    assert b"cannot open" in lib.ngmlr_b200_last_error(None)
    p = R.write_case(tmp_path, "fasta_single")
    assert lib.ngmlr_b200_read_file_open(p.encode(), None, C.byref(f)) == 0
    nbytes, nrec = C.c_int64(-1), C.c_int64(-1)
    assert lib.ngmlr_b200_read_file_stats(f, C.byref(nbytes), C.byref(nrec), None, None, None, None) == 0
    assert (nbytes.value, nrec.value) == (0, 0)
    assert lib.ngmlr_b200_reads_load_dropped(f) is None
    lib.ngmlr_b200_read_file_close(f)
