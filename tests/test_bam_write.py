"""ngmlr_b200_bam_header / ngmlr_b200_bam_format against the SAMv1 restatement of tests/bam_write_cases.py applied to
the SAM text the library writes for the same records (CPU only)."""
import copy
import struct

import numpy as np
import pytest

import bam_write_cases as bw
import sam_cases
from ngmlr_b200 import samtext as st

NAMES = [b"chr1", b"chrUn_gl000220", b"2", b"scaffold_with_a_long_name.0042|len=77"]
LENS = [1500, 2**31 - 1, 7, 123456]


# ---- the oracle against hand-worked values ----

def test_reg2bin_hand_values():
    assert bw.reg2bin(-1, 0) == 4680
    assert bw.reg2bin(0, 1) == 4681
    assert bw.reg2bin(16383, 16384) == 4681
    assert bw.reg2bin(16383, 16385) == 585          # crosses a 16 KiB bin: the 128 KiB level
    assert bw.reg2bin(2**29 - 1, 2**29) == 4681 + (2**29 - 1 >> 14)


@pytest.mark.parametrize("v,typ,raw", [
    (-129, b"s", struct.pack("<h", -129)), (-128, b"c", struct.pack("<b", -128)), (-1, b"c", b"\xff"),
    (0, b"C", b"\0"), (255, b"C", b"\xff"), (256, b"S", struct.pack("<H", 256)),
    (65535, b"S", b"\xff\xff"), (65536, b"I", struct.pack("<I", 65536)), (-32768, b"s", struct.pack("<h", -32768)),
    (-32769, b"i", struct.pack("<i", -32769)),
])
def test_integer_tag_types(v, typ, raw):
    assert bw.tag(b"XX:i:%d" % v) == b"XX" + typ + raw


def test_float_tags_round_trip_the_printed_text():
    assert bw.tag(b"XI:f:0.98") == b"XIf" + bytes.fromhex("48e17a3f")
    assert bw.tag(b"CV:f:100.000000") == b"CVf" + bytes.fromhex("0000c842")
    assert bw.tag(b"XI:f:0.3333") == b"XIf" + struct.pack("<f", np.float32(0.3333))


def test_hand_worked_record():
    line = b"r1\t16\tchr1\t10\t60\t3M1I1M\t*\t0\t0\tACGTN\t!!I#+\tNM:i:1\tMD:Z:4"
    body = struct.pack("<iiBBHHHiiii", 0, 9, 3, 60, 4681, 3, 16, 5, -1, -1, 0) + b"r1\0"
    body += struct.pack("<III", 3 << 4 | 0, 1 << 4 | 1, 1 << 4 | 0)
    body += bytes([0x12, 0x48, 0xF0]) + bytes([0, 0, 40, 2, 10])
    body += b"NMC\x01" + b"MDZ4\0"
    assert bw.record(line, [b"chr1"]) == struct.pack("<i", len(body)) + body


def test_hand_worked_header():
    text = b"@HD\tVN:1.0\n@SQ\tSN:c\tLN:5\n"
    assert bw.header(text) == b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<ii", 1, 2) + b"c\0" + \
        struct.pack("<i", 5)


# ---- the library against the oracle ----

def _printable(reads):
    """The reads with every alignment whose printed POS (low 32 bits of ref_pos + 1) exceeds 2^31 moved below it."""
    out = copy.deepcopy(reads)
    for r in out:
        for a in r.alignments:
            if ((a.ref_pos + 1) & 0xFFFFFFFF) > 2**31:
                a.ref_pos = a.ref_pos % 2**31
    return out


def _configs():
    for name, opts in sam_cases.CONFIGS:
        for fix in (False, True):
            for threads in (1, 2, 3, 4, 5):
                yield name, opts, fix, threads


@pytest.mark.parametrize("name,opts,fix,threads", list(_configs()))
def test_records_equal_the_oracle_of_the_sam_text(name, opts, fix, threads):
    reads = _printable(sam_cases.config_reads(name))
    kw = dict(write_unmapped=opts["write_unmapped"], bam_cigar_fix=opts["bam_cigar_fix"], rg_id=opts["rg_id"],
              fix_quality_orientation=fix, threads=threads)
    text = st.sam_format(reads, NAMES, **kw)
    got = st.bam_format(reads, NAMES, NAMES, **kw)
    want = bw.records(text, NAMES)
    assert bw.split_records(got) == bw.split_records(want)


@pytest.mark.parametrize("name", [c[0] for c in sam_cases.CONFIGS])
def test_header_equals_the_oracle_of_the_sam_header(name):
    opts = dict(sam_cases.CONFIGS)[name]
    fields = [b"s1", None, b"ILLUMINA", None, None, None, None, None, None, None, b"TCAG"]
    rg = dict(rg_id=opts["rg_id"], rg_fields=fields if opts["rg_id"] else None)
    text = st.sam_header(NAMES, LENS, b"0.2.8", b"ngmlr -r x -q y", **rg)
    assert st.bam_header(NAMES, LENS, b"0.2.8", b"ngmlr -r x -q y", **rg) == bw.header(text)


def test_contigs_named_twice_map_to_one_header_entry():
    reads = _printable(sam_cases.make_reads(21))
    twice = [n for n in NAMES for _ in range(2)]
    for r in reads:
        for a in r.alignments:
            a.ref_id = a.ref_id * 2 + (a.ref_id & 1)
    text = st.sam_format(reads, twice)
    assert st.bam_format(reads, twice, NAMES) == bw.records(text, NAMES)


def _long_read(n_ops, fix):
    rng = np.random.default_rng(5)
    cigar = b"".join(b"%d%s" % (1 + k % 3, b"MID"[k % 3:k % 3 + 1]) for k in range(n_ops))
    length = sum(1 + k % 3 for k in range(n_ops) if k % 3 != 2)
    seq = bytes(rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), length))
    a = st.Alignment(ref_pos=4000, ref_id=1, reverse=False, score=9.0, mq=20, nm=3, identity=0.5, qstart=0, qend=0,
                     cigar=cigar, md=b"10", cigar_ops=n_ops)
    return st.Read(b"long", seq, b"I" * length, [a])


@pytest.mark.parametrize("n_ops", [65535, 65536, 70001])
@pytest.mark.parametrize("fix", [False, True])
def test_long_cigars(n_ops, fix):
    reads = [_long_read(n_ops, fix)]
    text = st.sam_format(reads, NAMES, bam_cigar_fix=fix)
    got = st.bam_format(reads, NAMES, NAMES, bam_cigar_fix=fix)
    assert got == bw.records(text, NAMES)
    n_cigar = struct.unpack_from("<H", got, 16)[0]
    if n_ops > 65535:
        assert n_cigar == (1 if fix else 2)
        assert b"CGBI" + struct.pack("<i", n_ops) in got
    else:
        assert n_cigar == n_ops


def _one(ref_pos=10, name=b"r", ref_id=0, mq=7):
    a = st.Alignment(ref_pos=ref_pos, ref_id=ref_id, reverse=False, score=1.0, mq=mq, nm=0, identity=1.0, qstart=0,
                     qend=0, cigar=b"4M", md=b"4")
    return [st.Read(name, b"ACGT", b"IIII", [a])]


@pytest.mark.parametrize("reads,fragment", [
    (_one(ref_pos=2**31), b"POS"), (_one(ref_pos=2**31 + 7), b"POS"), (_one(ref_pos=2**32 - 2), b"POS"),
    (_one(ref_id=1), b"RNAME"), (_one(name=b"n" * 255), b"name"), (_one(mq=256), b"MAPQ"),
])
def test_records_bam_cannot_hold_fail_naming_the_read(reads, fragment):
    with pytest.raises(RuntimeError) as e:
        st.bam_format(reads, [b"chr1", b"elsewhere"], [b"chr1"])
    assert reads[0].name[:20].decode() in str(e.value) and fragment.decode() in str(e.value)
    text = st.sam_format(reads, [b"chr1", b"elsewhere"])
    with pytest.raises(bw.BamError):
        bw.records(text, [b"chr1"])


def test_limits_that_still_fit():
    reads = _one(ref_pos=2**31 - 1, name=b"n" * 254, mq=255)
    text = st.sam_format(reads, [b"chr1"])
    assert st.bam_format(reads, [b"chr1"]) == bw.records(text, [b"chr1"])


@pytest.mark.parametrize("ln", [2**31, 2**32 + 5])
def test_header_refuses_lengths_bam_cannot_hold(ln):
    with pytest.raises(RuntimeError, match="LN"):
        st.bam_header([b"a", b"b"], [5, ln])


def test_size_query():
    reads = _printable(sam_cases.config_reads("default"))
    full = st.bam_format(reads, NAMES, NAMES)
    rc, need, out = st.bam_format(reads, NAMES, NAMES, cap=len(full) - 1)
    assert (rc, need, out) == (-2, len(full), b"")
    rc, need, out = st.bam_format(reads, NAMES, NAMES, cap=len(full))
    assert (rc, need, out) == (0, len(full), full)


def test_unmapped_record_without_bases():
    reads = [st.Read(b"nothing", b"*", b"*", []), st.Read(b"fasta", b"ACGTA", b"*", [])]
    text = st.sam_format(reads, NAMES)
    got = st.bam_format(reads, NAMES, NAMES)
    assert got == bw.records(text, NAMES)
    assert struct.unpack_from("<i", got, 20)[0] == 0   # l_seq of SEQ "*"
