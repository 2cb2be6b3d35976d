"""The reference reader of ngmlr_b200_load_reference (csrc/fasta.cpp) against the unmodified reference's own
_SequenceProvider::Init (kseq_read over gzopen) on FASTA / FASTQ files built here, plain and gzip: lower case, IUPAC
codes, N runs, contigs of 0 / 10 / 11 bases, names longer than 100 characters with comments, a FASTQ-formatted
reference, blank lines, '\\r', records without sequence, '>' inside a line, text before the first header, FASTQ
records with missing or short qualities, and files whose size is a multiple of the reader's 16 KiB block.
For each file the reader's kept records (names cut to 100 characters), their numpy encoding, the contig table and the
allocation size the reference writes into <fasta>-enc.2.ngm equal the file the reference writes. No GPU needed."""
import ctypes as C
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest

from ngmlr_b200 import _lib, ngmfiles, refindex, synth
from oracle_lib import CsReference

FULL_LIMIT = 0xffff0000 - 1


def read_fasta(path, max_concat_len=FULL_LIMIT):
    """-> (records [(name, sequence bytes)], alloc_bytes) through ngmlr_b200_debug_read_fasta."""
    lib = _lib.load()
    n, tsz, nsz, alloc = C.c_int64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
    err = C.create_string_buffer(512)
    args = (os.fsencode(path), max_concat_len, C.byref(n), C.byref(tsz), C.byref(nsz), C.byref(alloc))
    rc = lib.ngmlr_b200_debug_read_fasta(*args, None, None, None, None, err, 512)
    if rc:
        raise ValueError(rc, err.value.decode())
    nl = np.zeros(max(n.value, 1), dtype=np.int64)
    rl = np.zeros(max(n.value, 1), dtype=np.uint64)
    names = C.create_string_buffer(nsz.value + 1)
    text = C.create_string_buffer(tsz.value + 1)
    rc = lib.ngmlr_b200_debug_read_fasta(*args, nl.ctypes.data_as(C.POINTER(C.c_int64)),
                                         rl.ctypes.data_as(C.POINTER(C.c_uint64)), names, text, err, 512)
    assert rc == 0
    recs, a, b = [], 0, 0
    for i in range(n.value):
        recs.append((names.raw[a:a + int(nl[i])], text.raw[b:b + int(rl[i])]))
        a += int(nl[i])
        b += int(rl[i])
    return recs, alloc.value


def _wrap(seq, width=60, eol=b"\n"):
    return b"".join(seq[i:i + width] + eol for i in range(0, len(seq), width))


def _cases():
    rng = np.random.default_rng(17)
    g = lambda n, s: synth.random_genome(n, s).tobytes()
    iupac = bytes(rng.choice(np.frombuffer(b"ACGTacgtNnRYKMSWBDHVrykmswbdhv-*.", dtype=np.uint8), 3001))
    long_name = b"x" * 140
    cases = {}
    cases["mixed"] = (b">chr1 the first contig\n" + _wrap(g(5000, 1).lower()) + b">empty\n"
                      + b">ten\nACGTACGTAC\n>eleven\tcomment\nACGTACGTACG\n>iupac\n" + _wrap(iupac, 77)
                      + b">" + long_name + b" a comment after a long name\n" + _wrap(g(2001, 2))
                      + b">nrun\n" + _wrap(g(1000, 3) + b"N" * 3000 + g(999, 4)) + b">last\n" + g(30, 5) + b"\n")
    q = lambda s: bytes(33 + (i % 40) for i in range(len(s)))
    s1, s2, s3 = g(4000, 6), g(12, 7), g(3001, 8)
    cases["fastq"] = (b"@read1 comment\n" + s1 + b"\n+\n" + q(s1) + b"\n@r2\n" + s2 + b"\n+r2\n" + q(s2)
                      + b"\n@r3\n" + s3[:1500] + b"\n" + s3[1500:] + b"\n+\n" + q(s3)[:1000] + b"\n" + q(s3)[1000:] + b"\n")
    cases["crlf_blank"] = (b"\r\n\n>c1 x\r\n" + _wrap(g(3000, 9), 70, b"\r\n") + b"\r\n\n\r\n" + b">c2\r\n\r\nACGTACGTACGTA\r\r\n"
                           + b">c3\n\r\n" + _wrap(g(500, 10), 50, b"\r\n") + b">\n" + g(40, 11) + b"\n> spaced name\n"
                           + g(41, 12) + b"\r")
    cases["inline_gt"] = (b"junk before the first header\n>a\n" + g(100, 13) + b">not a header\n" + g(100, 14)
                          + b"\n@b\n" + g(200, 15) + b"\n>c\nAC>GT\n" + g(64, 16) + b"\n>no_newline_at_end\n" + g(77, 17))
    # a FASTQ record whose quality string is short: the reference's reader returns -2 and ngmlr stops reading there
    cases["fastq_short_qual"] = (b">f1\n" + g(300, 18) + b"\n@q1\n" + g(50, 19) + b"\n+\n" + b"I" * 49 + b"\n>f2\n"
                                 + g(300, 20) + b"\n")
    # file sizes that are multiples of the 16 KiB read block, ending in "\r" as the first character of a line and
    # in a one-character line
    for name, tail in (("block_cr", b"\n\r"), ("block_char", b"\nG")):
        body = b">blk\n" + _wrap(g(20000, 21))
        fill = (-(len(body) - 1 + len(tail))) % 16384
        data = body[:-1] + b"A" * fill + tail
        assert len(data) % 16384 == 0
        cases[name] = data
    return cases


CASES = _cases()


def _reference_files(path):
    code = "import ctypes, sys; lib = ctypes.CDLL(sys.argv[1]); sys.exit(lib.ref_cs_init_save(sys.argv[2].encode()))"
    run = subprocess.run([sys.executable, "-c", code, CsReference.PATH, path], capture_output=True, text=True,
                         timeout=600)
    assert run.returncode == 0, run.stderr[-2000:]
    os.remove(path + "-ht-13-2.2.ngm")
    with open(path + "-enc.2.ngm", "rb") as f:
        alloc = int(np.frombuffer(f.read(24), dtype="<u8")[2])
    return ngmfiles.read_encoded_reference(path + "-enc.2.ngm"), alloc


def write_case(dirpath, name, gz):
    os.makedirs(str(dirpath), exist_ok=True)
    path = os.path.join(str(dirpath), name + (".fa.gz" if gz else ".fa"))
    with (gzip.open(path, "wb") if gz else open(path, "wb")) as f:
        f.write(CASES[name])
    return path


@pytest.mark.skipif(not CsReference.available(), reason="oracle/_ref/libngmlr_full.so not built")
@pytest.mark.parametrize("gz", [False, True], ids=["plain", "gzip"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_reader_equals_reference_sequence_provider(tmp_path, name, gz):
    path = write_case(tmp_path, name, gz)
    recs, alloc = read_fasta(path)
    (want, want_names), want_alloc = _reference_files(path)
    kept = [(n[:100], s) for n, s in recs if len(s) > 10]
    assert [n for n, _ in kept] == [n.encode() for n in want_names]
    got = refindex.encode_reference([s for _, s in recs])
    assert got.ref_start == want.ref_start and got.ref_len == want.ref_len and got.concat_len == want.concat_len
    assert np.array_equal(got.enc, want.enc)
    assert alloc == want_alloc


def test_reader_edge_cases_pinned(tmp_path):
    """What the reference comparison above relies on, stated directly (runs without the compiled reference)."""
    g = lambda n, s: synth.random_genome(n, s).tobytes()
    recs = read_fasta(write_case(tmp_path, "crlf_blank", False))[0]
    assert recs == [(b"c1", g(3000, 9)),
                    # a '\r' is dropped at the end of a line only once the sequence holds two characters
                    (b"c2", b"\rACGTACGTACGTA\r"), (b"c3", b"\r" + g(500, 10)),
                    (b"", g(40, 11)), (b"", g(41, 12))]      # ">" alone and "> spaced name": empty names
    recs = read_fasta(write_case(tmp_path, "inline_gt", True))[0]
    assert [n for n, _ in recs] == [b"a", b"b", b"c", b"no_newline_at_end"]
    assert recs[0][1] == g(100, 13) + b">not a header" + g(100, 14)   # '>' inside a line is sequence
    assert recs[2][1].startswith(b"AC>GT") and recs[3][1] == g(77, 17)
    assert [n for n, _ in read_fasta(write_case(tmp_path, "fastq_short_qual", False))[0]] == [b"f1"]
    fq = read_fasta(write_case(tmp_path, "fastq", False))[0]
    assert [(n, len(s)) for n, s in fq] == [(b"read1", 4000), (b"r2", 12), (b"r3", 3001)]
    # the final "\r" line of a file that ends on a 16 KiB block boundary is dropped (elsewhere it would stay)
    assert read_fasta(write_case(tmp_path, "block_cr", False))[0][0][1].endswith(b"AAA")
    assert read_fasta(write_case(tmp_path, "block_char", False))[0][0][1].endswith(b"AG")
    mixed = read_fasta(write_case(tmp_path, "mixed", True))
    assert [len(n) for n, _ in mixed[0]][5] == 140                 # the reader keeps whole names; the load cuts them
    lens = [len(s) for _, s in mixed[0]]
    assert mixed[1] == ngmfiles.reference_alloc_bytes([n for n in lens if n > 10], [n for n in lens if n <= 10])


def test_reader_errors(tmp_path):
    with pytest.raises(ValueError, match="cannot open"):
        read_fasta(str(tmp_path / "missing.fa"))
    path = write_case(tmp_path, "mixed", False)
    recs, _ = read_fasta(path)
    lens = [len(s) for _, s in recs]
    need = refindex.encode_reference([s for _, s in recs]).concat_len
    assert read_fasta(path, need)[0] == recs                        # exactly at the limit: read
    with pytest.raises(ValueError, match="exceeds"):                # one position less: refused while reading
        read_fasta(path, need - 1)
    assert sum(lens) > 0
    open(tmp_path / "empty.fa", "wb").close()
    assert read_fasta(str(tmp_path / "empty.fa")) == ([], ngmfiles.reference_alloc_bytes([]))
