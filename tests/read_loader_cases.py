"""Query files for the read loader (ngmlr_b200_reads_load) and the reference's own reading of them.

CASES maps a name to the bytes of a FASTA / FASTQ stream that exercises one of kseq's rules (src/kseq.h:171-211) or
IParser::copyToRead's (src/IParser.h:51-117). oracle_reads() runs the unmodified ReadProvider::GenerateRead loop
(ref_read_file of oracle/_ref/libngmlr_reads.so, built from oracle/read_provider_shim.cpp) in a process of its own:
ngmlr's error for a quality string of another length exits the process, and its message names the dropped read."""
import gzip
import os
import random
import re
import struct
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FULL = os.path.join(ROOT, "oracle", "_ref", "libngmlr_reads.so")
KB16 = 16384


def _rand_seq(rng, n, alphabet="ACGT"):
    return "".join(rng.choice(alphabet) for _ in range(n))


def _qual(rng, n, alphabet="!#+5?@>ABCDEFGHIJ"):
    return "".join(rng.choice(alphabet) for _ in range(n))


def _wrap(s, w):
    return "\n".join(s[i:i + w] for i in range(0, len(s), w)) if s else ""


def _pad_to(text, size, filler_name="pad"):
    """text + one FASTA record whose sequence makes the stream exactly `size` bytes (text ends with a newline)."""
    head = f">{filler_name}\n"
    n = size - len(text.encode()) - len(head)
    assert n > 1
    return text + head + "A" * (n - 1) + "\n"


def _fuzz(seed, n_records):
    rng = random.Random(seed)
    out = []
    for i in range(n_records):
        n = rng.choice([0, 1, 5, 60, 150, 257, 300, 1200])
        seq = _rand_seq(rng, n, "ACGTacgtNRYKMn.0") if rng.random() < 0.3 else _rand_seq(rng, n)
        nl = "\r\n" if rng.random() < 0.2 else "\n"
        name = f"f{seed}_{i}" + (f"\tcomment {i}" if rng.random() < 0.2 else "")
        if rng.random() < 0.5:
            body = _wrap(seq, rng.choice([7, 60, 100000])).replace("\n", nl)
            out.append(f">{name}{nl}{body}{nl}" if n else f">{name}{nl}")
        else:
            q = _qual(rng, n)
            w = rng.choice([9, 80, 100000])
            plus = "+" + (name.split()[0] if rng.random() < 0.3 else "")
            out.append(f"@{name}{nl}{_wrap(seq, w).replace(chr(10), nl)}{nl}{plus}{nl}"
                       f"{_wrap(q, w).replace(chr(10), nl)}{nl}")
    return "".join(out)


def _cases():
    rng = random.Random(11)
    s = lambda n: _rand_seq(rng, n)
    q = lambda n: _qual(rng, n)
    c = {}
    c["fasta_single"] = f">r1 the comment\n{s(120)}\n>r2\n{s(300)}\n>r3\n{s(7)}\n"
    c["fasta_multi"] = f">m1\n{_wrap(s(500), 60)}\n>m2 x\n{_wrap(s(61), 60)}\n\n\n>m3\n\n{_wrap(s(130), 13)}\n"
    c["fastq_4line"] = "".join(f"@q{i}\n{x}\n+\n{q(len(x))}\n" for i, x in enumerate([s(100), s(1), s(256), s(257)]))
    c["fastq_multi"] = "".join(f"@w{i}\n{_wrap(x, 50)}\n+\n{_wrap(q(len(x)), 33)}\n"
                               for i, x in enumerate([s(130), s(700), s(50)]))
    # quality lines that start with '@', '>' or '+' (single and multi-line)
    c["qual_markers"] = (f"@a1\nACGTA\n+\n@@@@@\n@a2\nACGT\n+\n>III\n@a3\nAC\n+\n++\n"
                         f"@a4\nACGTACGT\n+\n@III\n>III\n@a5\nACGTAC\n+\n+II\n@II\n>x\nACGT\n")
    c["plus_name"] = "".join(f"@p{i} c\n{x}\n+p{i} c\n{q(len(x))}\n" for i, x in enumerate([s(40), s(90)]))
    c["crlf"] = (f">c1 x\r\n{s(60)}\r\n{s(20)}\r\n@c2\r\n{s(30)}\r\n+\r\n{q(30)}\r\n"
                 f"@c3\r\n{_wrap(s(45), 20)}\r\n+\r\n{_wrap(q(45), 10)}\r\n".replace("\n", "\r\n").replace("\r\r", "\r"))
    c["lone_cr"] = (f">l1\n\r\n{s(10)}\n\r\n{s(5)}\n>l2\n\r\n>l3\n{s(4)}\r\r\n\r\n"
                    f"@l4\nACGT\n+\n\r\nII\r\nII\n@l5\nACG\n+\nII\r\r\nI\n@l6\nAC\n+\n\r\n\r\nII\n>l7\nAC\n")
    c["iupac"] = ">i1\nacgtnRYKMSWBDHVN.-0123456789xX*acgt\n@i2\nacgtRYn.9\n+\n" + q(9) + "\n>i3\n\x01\x7f\xe9ACGT\n"
    c["empty"] = f">e1\n>e2\n\n>e3\n{s(10)}\n@e4\n\n+\n\n@e5\n+\n>e6\n"
    c["names"] = (f">{'n' * 249}\n{s(10)}\n>{'o' * 250} c\n{s(10)}\n>{'p' * 400}\n{s(10)}\n"
                  f">t1\tcom ment\n{s(10)}\n>v1\x0bx\n{s(10)}\n>\n{s(3)}\n> spaced\n{s(3)}\n")
    c["mismatch_mid"] = f"@m1\n{s(10)}\n+\n{q(10)}\n@m2\n{s(10)}\n+\n{q(9)}\n@m3\n{s(10)}\n+\n{q(10)}\n"
    c["mismatch_long"] = f"@m1\n{s(10)}\n+\n{q(10)}\n@m2\n{s(10)}\n+\n{q(12)}\n@m3\n{s(10)}\n+\n{q(10)}\n"
    c["mismatch_end"] = f">m0\n{s(20)}\n@m1\n{s(10)}\n+\n{q(10)}\n@m2\n{s(10)}\n+\n{q(7)}\n"
    c["no_quality"] = f"@m1\n{s(10)}\n+\n{q(10)}\n@m2\n{s(10)}\n+"
    c["no_trailing_nl_fasta"] = f">z1\n{s(50)}\n>z2\n{s(33)}"
    c["no_trailing_nl_fastq"] = f"@z1\n{s(50)}\n+\n{q(50)}\n@z2\n{s(33)}\n+\n{q(33)}"
    c["junk_lead"] = f"junk line\nmore junk x>y\n{s(5)}\n>j1\n{s(40)}\n"
    c["junk_between"] = f"@j1\n{s(8)}\n+\n{q(8)}\njunk@j2 c\n{s(6)}\n+\n{q(6)}\nzz\n\n>j3\n{s(5)}\n"
    # streams of exactly k x 16 KiB: kseq's end-of-file tests see one more (empty) read
    c["kb16_nl"] = _pad_to(f">k1\n{s(100)}\n", KB16)
    c["kb32_no_nl"] = _pad_to(f">k1\n{s(100)}\n", 2 * KB16 + 1)[:-1]
    c["kb16_header_last"] = _pad_to(f">k1\n{s(100)}\n", KB16 - 1) + ">"
    c["kb16_lone_cr_last"] = _pad_to(f">k1\n{s(100)}\n", KB16 - 1) + "\r"
    c["kb16_cr_qual"] = _pad_to(f">k0\n{s(10)}\n", KB16 - 15) + "@k\nACGT\n+\nII\r\r\n"
    c["header_last"] = f">k1\n{s(100)}\n>"
    c["lone_cr_last"] = f">k1\n{s(100)}\n\r"
    c["fuzz_a"] = _fuzz(1, 300)
    c["fuzz_b"] = _fuzz(2, 120)
    return {k: v.encode("latin-1") for k, v in c.items()}


CASES = _cases()
BIG = ("fuzz_a", "fuzz_b")  # the cases only read with the larger chunk sizes


def write_case(dirpath, name, gz=False):
    os.makedirs(dirpath, exist_ok=True)
    path = os.path.join(str(dirpath), name + (".fq.gz" if gz else ".fq"))
    data = CASES[name]
    if gz:
        with gzip.open(path, "wb") as f:
            f.write(data)
    else:
        with open(path, "wb") as f:
            f.write(data)
    return path


_SCRIPT = r"""
import ctypes, sys
lib = ctypes.CDLL(sys.argv[1])
lib.ref_read_file.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p]
sys.exit(0 if lib.ref_read_file(sys.argv[2].encode(), int(sys.argv[3]), sys.argv[4].encode()) >= 0 else 3)
"""


def oracle_reads(path, read_part_length=256, tmp=None):
    """[(name, seq, qual, length, empty)] as ngmlr's ReadProvider makes them, and the names ngmlr drops."""
    out = (tmp or path) + ".oracle"
    r = subprocess.run([sys.executable, "-c", _SCRIPT, FULL, path, str(read_part_length), out], capture_output=True,
                       timeout=300)
    assert r.returncode in (0, 1), r.stderr[-2000:]
    dropped = re.findall(rb"Read (.*): Length of read not equal length of quality values\.", r.stderr)
    assert (r.returncode == 1) == bool(dropped), r.stderr[-2000:]
    data = open(out, "rb").read()
    os.unlink(out)
    reads, p = [], 0
    u32 = lambda: struct.unpack_from("<i", data, p)[0]
    while p < len(data):
        nl = u32(); p += 4
        name = data[p:p + nl]; p += nl
        length = u32(); p += 4
        empty = u32(); p += 4
        sl = u32(); p += 4
        seq = data[p:p + sl]; p += sl
        ql = u32(); p += 4
        qual = data[p:p + ql]; p += ql
        reads.append((name, seq, qual, length, empty))
    return reads, dropped


def as_loaded(oracle, read_part_length=256):
    """The oracle's reads as the loader gives them: an Empty read (read_part_length + 16 N's in ngmlr, the last one
    uninitialised) has length 0 and no bases."""
    out = []
    for name, seq, qual, length, empty in oracle:
        if empty:
            assert length == read_part_length + 16 and seq == b"N" * (length - 1) and qual == b"*"
            out.append((name, b"", b"*", 0, 1))
        else:
            out.append((name, seq, qual, length, 0))
    return out
