"""BAM input for the read loader (ngmlr_b200_reads_load): a small BAM writer, the text `samtools fastq -n` writes for
the same records, and named cases (tests/test_bam_cases.py on the CPU, tests/test_gpu_bam.py on the GPU).

  - Rec / header() / record() / bam_stream(): the BAM layout of the SAM specification (§4.2): magic, l_text, text,
    n_ref and reference entries, then per record block_size, the 32 bytes of fixed fields, read_name with its NUL,
    CIGAR, 4-bit packed seq, qual and aux fields of every type (A c C s S i I f Z H and B arrays of each subtype);
  - write(): the stream as BGZF (bgzf_cases.bgzf, at a chosen member size so headers and records straddle members),
    plain gzip or uncompressed;
  - fastq_text(): what `samtools fastq -n` writes: records flagged 0x100 / 0x800 left out, seq and qual
    reverse-complemented back under 0x10, a '>' record when the first quality byte is 0xFF;
  - CASES, ERRORS: the named record sets and the malformed streams, each with the offset its error names."""
import gzip
import os
import random
import struct
from dataclasses import dataclass, field

import bgzf_cases

NT16 = "=ACMGRSVTWYHKDBN"
COMP = dict(zip(NT16, "=TGKCYSBAWRDMHVN"))  # htslib's seq_nt16 complement
SKIP = 0x900


@dataclass
class Rec:
    """One BAM record as stored: seq in NT16 letters, qual as Phred values (None: absent, stored as 0xFF bytes)."""
    name: bytes
    seq: str
    qual: list = None
    flag: int = 4
    ref_id: int = -1
    pos: int = -1
    mapq: int = 255
    cigar: list = field(default_factory=list)  # [(length, op index)]
    aux: bytes = b""
    next_ref_id: int = -1
    next_pos: int = -1
    tlen: int = 0


def aux_all_types(rng):
    """Aux fields of every type, B arrays of every subtype included."""
    out = b"XAA" + b"z"
    out += b"Xcc" + struct.pack("<b", -5) + b"XCC" + struct.pack("<B", 200)
    out += b"Xss" + struct.pack("<h", -300) + b"XSS" + struct.pack("<H", 60000)
    out += b"Xii" + struct.pack("<i", -70000) + b"XII" + struct.pack("<I", 4000000000)
    out += b"Xff" + struct.pack("<f", 0.25)
    out += b"XZZ" + b"a Z string\0" + b"XHH" + b"1AE301\0"
    for sub, fmt in (("c", "b"), ("C", "B"), ("s", "h"), ("S", "H"), ("i", "i"), ("I", "I"), ("f", "f")):
        vals = [rng.randint(0, 100) for _ in range(rng.randint(0, 5))]
        out += b"B" + sub.encode() + b"B" + sub.encode() + struct.pack("<i", len(vals)) + \
            struct.pack("<" + fmt * len(vals), *vals)
    return out


def header(text=b"", refs=()):
    out = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    for name, length in refs:
        out += struct.pack("<i", len(name) + 1) + name + b"\0" + struct.pack("<i", length)
    return out


def pack_seq(seq):
    codes = [NT16.index(c) for c in seq]
    if len(codes) % 2:
        codes.append(0)
    return bytes((codes[i] << 4) | codes[i + 1] for i in range(0, len(codes), 2))


def record(r, block_size=None, l_name=None, l_seq=None, name_nul=True):
    """The record's bytes, block_size first (the overrides make the error variants)."""
    name = r.name + (b"\0" if name_nul else b"")
    qual = bytes(r.qual) if r.qual is not None else b"\xff" * len(r.seq)
    body = (struct.pack("<iiBBHHHiiii", r.ref_id, r.pos, len(name) if l_name is None else l_name, r.mapq, 4680,
                        len(r.cigar), r.flag, len(r.seq) if l_seq is None else l_seq, r.next_ref_id, r.next_pos,
                        r.tlen)
            + name + b"".join(struct.pack("<I", n << 4 | op) for n, op in r.cigar) + pack_seq(r.seq) + qual + r.aux)
    return struct.pack("<i", len(body) if block_size is None else block_size) + body


def bam_stream(hdr, recs):
    return hdr + b"".join(record(r) for r in recs)


def write(path, data, mode="bgzf", block=bgzf_cases.BLOCK):
    """data as BGZF (members of `block` input bytes), plain gzip ("gzip") or as it is ("plain")."""
    with open(path, "wb") as f:
        if mode == "bgzf":
            f.write(bgzf_cases.bgzf(data, level=1, block=block))
        elif mode == "gzip":
            f.write(gzip.compress(data, 1))
        else:
            f.write(data)
    return path


def stored_to_read(r):
    """(seq, qual) as `samtools fastq` prints them: reverse-complemented back under 0x10; qual None when absent."""
    seq, qual = r.seq, r.qual
    if r.flag & 0x10:
        seq = "".join(COMP[c] for c in reversed(seq))
        qual = None if qual is None else list(reversed(qual))
    return seq, qual


def fastq_text(recs):
    out = []
    for r in recs:
        if r.flag & SKIP:
            continue
        seq, qual = stored_to_read(r)
        if qual is None and seq:
            out.append(b">" + r.name + b"\n" + seq.encode() + b"\n")
        else:
            out.append(b"@" + r.name + b"\n" + seq.encode() + b"\n+\n" + bytes(q + 33 for q in (qual or [])) + b"\n")
    return b"".join(out)


def counters(hdr, recs):
    """(header bytes, records, skipped, reversed, no quality) as ngmlr_b200_read_file_bam_stats counts them."""
    kept = [r for r in recs if not r.flag & SKIP]
    return (len(hdr), len(recs), len(recs) - len(kept), sum(1 for r in kept if r.flag & 0x10),
            sum(1 for r in kept if r.seq and r.qual is None))


def _seq(rng, n, alphabet="ACGT"):
    return "".join(rng.choice(alphabet) for _ in range(n))


def _qual(rng, n):
    return [rng.randint(0, 60) for _ in range(n)]


def _revcomp(seq):
    return "".join(COMP[c] for c in reversed(seq))


def _cases():
    rng = random.Random(23)
    c = {}
    refs = [(b"chr1", 248956422), (b"chr2", 242193529)]
    # unaligned PacBio-style records (subreads.bam / hifi_reads.bam)
    recs = []
    for i in range(12):
        n = rng.randint(300, 6000)
        recs.append(Rec(b"m64011_190830_220126/%d/ccs" % (1000 + i), _seq(rng, n), _qual(rng, n), flag=4,
                        aux=b"np" + b"i" + struct.pack("<i", 7) + b"rqf" + struct.pack("<f", 0.999) + aux_all_types(rng)))
    c["pacbio"] = (header(b"@HD\tVN:1.6\tSO:unknown\n@RG\tID:x\tPL:PACBIO\n"), recs)
    # aligned forward and reverse, reverse with and without qualities
    recs = []
    for i in range(40):
        n = rng.randint(1, 400)
        rev = rng.random() < 0.5
        qual = None if rng.random() < 0.25 else _qual(rng, n)
        recs.append(Rec(b"al%d" % i, _seq(rng, n, "ACGTN" if i % 5 == 0 else "ACGT"), qual, flag=0x10 if rev else 0,
                        ref_id=i % 2, pos=1000 * i, mapq=60, cigar=[(n, 0)] if n > 3 else [(1, 4), (n - 1, 0)] if n > 1
                        else [(1, 0)], aux=aux_all_types(rng) if i % 3 == 0 else b"NMi" + struct.pack("<i", 1)))
    c["aligned"] = (header(b"@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:chr1\tLN:248956422\n@SQ\tSN:chr2\tLN:242193529\n",
                           refs), recs)
    # secondary and supplementary records mixed in
    recs = []
    for i in range(30):
        n = rng.randint(20, 300)
        flag = rng.choice([0, 0x10, 0x100, 0x110, 0x800, 0x810, 0x900, 4])
        recs.append(Rec(b"sx%d" % i, _seq(rng, n), _qual(rng, n) if rng.random() < 0.8 else None, flag=flag,
                        ref_id=0 if flag != 4 else -1, pos=5 * i if flag != 4 else -1, cigar=[(n, 0)] if flag != 4 else []))
    recs.append(Rec(b"last_secondary", _seq(rng, 50), _qual(rng, 50), flag=0x100))
    c["secondary"] = (header(b"", refs), recs)
    # odd l_seq: the last nibble unused
    recs = [Rec(b"odd%d" % n, _seq(rng, n, NT16[1:]), _qual(rng, n), flag=rng.choice([0, 0x10]))
            for n in (1, 3, 5, 33, 255, 1023, 1025, 2049)]
    c["odd"] = (header(), recs)
    # l_seq = 0
    c["empty"] = (header(), [Rec(b"e1", "", []), Rec(b"e2", "ACGT", _qual(rng, 4)), Rec(b"e3", "", [], flag=0x10),
                             Rec(b"e4", "", [], flag=0x100), Rec(b"e5", "GATTACA", None)])
    # names of 1, 249, 250 and 254 characters, with a space, with a tab, with '\v' and '\r'
    names = [b"a", b"n" * 249, b"o" * 250, b"p" * 254, b"sp ace", b"t\tab", b"v\x0bx", b"cr\rx", b"@odd>name+"]
    c["names"] = (header(), [Rec(nm, _seq(rng, 10), _qual(rng, 10)) for nm in names])
    # all 16 sequence codes, forward and reverse
    allc = NT16 * 3 + NT16[::-1]
    c["codes"] = (header(), [Rec(b"c_fwd", allc, _qual(rng, len(allc))), Rec(b"c_rev", allc, _qual(rng, len(allc)),
                                                                             flag=0x10),
                             Rec(b"c_rev_noq", allc, None, flag=0x10), Rec(b"c_fwd_noq", allc, None)])
    # Phred 0 and 93
    c["phred"] = (header(), [Rec(b"q0", "ACGT", [0, 93, 0, 93]), Rec(b"q1", "ACGTA", [93] * 5, flag=0x10),
                             Rec(b"q2", "ACG", [0, 0, 0])])
    # a 1 MB header: @CO lines, and reference entries
    text = b"@HD\tVN:1.6\n" + b"".join(b"@CO\t" + _seq(rng, 1000).encode() + b"\n" for _ in range(1000))
    many = [(b"contig_%d" % i, 1000 + i) for i in range(3000)]
    c["big_header"] = (header(text, many), [Rec(b"bh%d" % i, _seq(rng, 80), _qual(rng, 80), flag=rng.choice([0, 16]),
                                                ref_id=i % 3000, pos=i, cigar=[(80, 0)]) for i in range(50)])
    # a 300 kb read over many members, between short ones
    c["long_read"] = (header(b"@HD\tVN:1.6\n"), [Rec(b"s1", _seq(rng, 50), _qual(rng, 50)),
                                                 Rec(b"long", _seq(rng, 300_000), _qual(rng, 300_000), flag=0x10),
                                                 Rec(b"s2", _seq(rng, 70), None)])
    # 10^5 short records (SRA-like 36 bp)
    r2 = random.Random(5)
    recs = []
    acgt = bytes(b"ACGT"[i % 4] for i in range(256))
    for i in range(100_000):
        s = r2.randbytes(36).translate(acgt).decode()
        recs.append(Rec(b"SRR000001.%d" % i, s, [2 + q % 39 for q in r2.randbytes(36)],
                        flag=(0x10 if i % 2 else 0) | (0x100 if i % 97 == 0 else 0)))
    c["many_short"] = (header(b"@HD\tVN:1.6\n"), recs)
    return c


CASES = _cases()
BIG = ("big_header", "long_read", "many_short")  # read with fewer chunk sizes and batch limits


def case_stream(name):
    hdr, recs = CASES[name]
    return bam_stream(hdr, recs)


def write_case(dirpath, name, mode="bgzf", block=bgzf_cases.BLOCK):
    os.makedirs(dirpath, exist_ok=True)
    return write(os.path.join(str(dirpath), f"{name}.{mode}.bam"), case_stream(name), mode, block)


def write_text(dirpath, name):
    """The case's `samtools fastq -n` text, for ngmlr's ReadProvider."""
    os.makedirs(dirpath, exist_ok=True)
    path = os.path.join(str(dirpath), name + ".fq")
    with open(path, "wb") as f:
        f.write(fastq_text(CASES[name][1]))
    return path


def _errors():
    """name -> (stream, the stream offset the error names, a pattern of its message)."""
    rng = random.Random(9)
    good = [Rec(b"g%d" % i, _seq(rng, 30), _qual(rng, 30)) for i in range(3)]
    hdr = header(b"@HD\tVN:1.6\n", [(b"chr1", 1000)])
    head = bam_stream(hdr, good)
    bad = Rec(b"bad", _seq(rng, 21), _qual(rng, 21))
    rb = record(bad)
    at = len(head)
    e = {}
    e["header_cut_text"] = (hdr[:30], 30, "header cut off")
    e["header_cut_refs"] = (hdr[:-3], len(hdr) - 3, "header cut off")
    e["header_l_text_negative"] = (b"BAM\1" + struct.pack("<i", -1), 0, "l_text < 0")
    e["record_cut_block_size"] = (head + rb[:2], at, "record cut off")
    e["record_cut_fixed"] = (head + rb[:20], at, "record cut off")
    e["record_cut_seq"] = (head + rb[:50], at, "record cut off")
    e["block_size_31"] = (head + record(bad, block_size=31) + rb, at, "block_size < 32")
    e["fixed_over_block"] = (head + record(bad, l_seq=40) + rb, at, "do not fit its block_size")
    e["l_read_name_0"] = (head + record(bad, l_name=0) + rb, at, "l_read_name = 0")
    e["name_without_nul"] = (head + record(Rec(b"badx", bad.seq, bad.qual), name_nul=False) + rb, at, "lacks its NUL")
    e["l_seq_negative"] = (head + record(bad, l_seq=-1) + rb, at, "l_seq < 0")
    e["phred_94"] = (head + record(Rec(b"q94", "ACGT", [30, 94, 30, 30])) + rb, at, "quality value above 93")
    e["phred_255_late"] = (head + record(Rec(b"q255", "ACGT", [30, 255, 30, 30])) + rb, at, "quality value above 93")
    return e


ERRORS = _errors()
