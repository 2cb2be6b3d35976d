"""SAM text -> BAM, restated from SAMv1 section 4.2 (and the integer-type and placeholder rules htslib applies when
`samtools view -b` converts a SAM file): the oracle that tests/test_bam_write.py and tests/test_gpu_bgzf_write.py
hold ngmlr_b200_bam_header / ngmlr_b200_bam_format against. It reads only the text, never the library."""
import re
import struct

NT16 = b"=ACMGRSVTWYHKDBN"
CIGAR_OPS = b"MIDNSHP=X"
_CIGAR_RE = re.compile(rb"(\d+)([MIDNSHP=X])")


class BamError(ValueError):
    pass


def reg2bin(beg, end):
    """SAMv1 section 5.3 (Python's >> on negative numbers is arithmetic, as C's on int64 here)."""
    end -= 1
    if beg >> 14 == end >> 14:
        return ((1 << 15) - 1) // 7 + (beg >> 14)
    if beg >> 17 == end >> 17:
        return ((1 << 12) - 1) // 7 + (beg >> 17)
    if beg >> 20 == end >> 20:
        return ((1 << 9) - 1) // 7 + (beg >> 20)
    if beg >> 23 == end >> 23:
        return ((1 << 6) - 1) // 7 + (beg >> 23)
    if beg >> 26 == end >> 26:
        return ((1 << 3) - 1) // 7 + (beg >> 26)
    return 0


def int_tag(key, v):
    """An i tag in htslib's smallest type: c / s / i below 0, C / S / I otherwise."""
    if v < 0:
        for t, fmt, lo in ((b"c", "<b", -128), (b"s", "<h", -32768), (b"i", "<i", -2**31)):
            if v >= lo:
                return key + t + struct.pack(fmt, v)
        raise BamError("integer tag below INT32_MIN")
    for t, fmt, hi in ((b"C", "<B", 255), (b"S", "<H", 65535), (b"I", "<I", 2**32 - 1)):
        if v <= hi:
            return key + t + struct.pack(fmt, v)
    raise BamError("integer tag above UINT32_MAX")


def tag(field):
    key, typ, val = field[:2], field[3:4], field[5:]
    if typ == b"i":
        return int_tag(key, int(val))
    if typ == b"f":
        return key + b"f" + struct.pack("<f", float(val))   # strtod, then narrowed to float
    if typ == b"Z":
        return key + b"Z" + val + b"\0"
    if typ == b"A":
        return key + b"A" + val[:1]
    if typ == b"B":
        parts = val.split(b",")
        sub, nums = parts[0], [int(x) for x in parts[1:]]
        fmt = {b"I": "<I", b"i": "<i", b"S": "<H", b"s": "<h", b"C": "<B", b"c": "<b"}[sub]
        if sub == b"I":
            nums = [x & 0xFFFFFFFF for x in nums]
        return key + b"B" + sub + struct.pack("<i", len(nums)) + b"".join(struct.pack(fmt, x) for x in nums)
    raise BamError("tag type %r" % typ)


def parse_cigar(text):
    if text == b"*":
        return []
    ops = _CIGAR_RE.findall(text)
    if b"".join(a + b for a, b in ops) != text:
        raise BamError("malformed CIGAR")
    return [(int(n), CIGAR_OPS.index(op)) for n, op in ops]


def record(line, names):
    """One SAM line (without its newline) -> the BAM record with its block_size. names: the header's @SQ SNs."""
    f = line.split(b"\t")
    qname, flag, rname, pos, mapq, cigar, rnext, pnext, tlen, seq, qual = f[:11]
    if len(qname) > 254:
        raise BamError("read name longer than 254 bytes")
    if rname == b"*":
        ref = -1
    elif rname in names:
        ref = names.index(rname)
    else:
        raise BamError("RNAME not in the header")
    if int(pos) > 2**31:
        raise BamError("POS above 2^31")
    pos, flag, mapq = int(pos) - 1, int(flag), int(mapq)
    if not 0 <= mapq <= 255:
        raise BamError("MAPQ outside 0..255")
    ops = parse_cigar(cigar)
    l_seq = 0 if seq == b"*" else len(seq)
    tags = [tag(x) for x in f[11:]]
    if len(ops) > 65535:    # SAMv1 4.2.2: <l_seq>S<rlen>N, the CIGAR itself as CG:B:I appended last
        rlen = sum(n for n, op in ops if op in (0, 2, 3, 7, 8))
        tags.append(b"CGBI" + struct.pack("<i", len(ops)) + b"".join(struct.pack("<I", n << 4 | op) for n, op in ops))
        ops = [(l_seq, 4), (rlen, 3)]
    rlen = sum(n for n, op in ops if op in (0, 2, 3, 7, 8))
    bin_ = 4680 if flag & 4 else reg2bin(pos, pos + max(rlen, 1))
    next_ref = -1 if rnext == b"*" else (ref if rnext == b"=" else names.index(rnext))
    codes = [NT16.index(c) if c in NT16 else 15 for c in seq.upper()] if l_seq else []
    codes += [0] * (len(codes) & 1)
    packed = bytes(codes[k] << 4 | codes[k + 1] for k in range(0, len(codes), 2))
    if qual == b"*":
        qbytes = b"\xff" * l_seq
    else:
        if len(qual) != l_seq:
            raise BamError("QUAL and SEQ differ in length")
        qbytes = bytes(c - 33 for c in qual)
    body = struct.pack("<iiBBHHHiiii", ref, pos, len(qname) + 1, mapq, bin_, len(ops), flag, l_seq, next_ref,
                       int(pnext) - 1, int(tlen))
    body += qname + b"\0" + b"".join(struct.pack("<I", n << 4 | op) for n, op in ops) + packed + qbytes
    body += b"".join(tags)
    return struct.pack("<i", len(body)) + body


def header_names(text):
    """(SN, LN) of every @SQ line of a header text."""
    out = []
    for line in text.split(b"\n"):
        if line.startswith(b"@SQ\t"):
            kv = dict(x.split(b":", 1) for x in line.split(b"\t")[1:])
            out.append((kv[b"SN"], int(kv[b"LN"])))
    return out


def header(text):
    """SAM header text -> the BAM header: magic, l_text, text, n_ref and (l_name, name NUL, l_ref) per @SQ."""
    refs = header_names(text)
    out = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    for name, ln in refs:
        if ln > 2**31 - 1:
            raise BamError("LN above 2^31 - 1")
        out += struct.pack("<i", len(name) + 1) + name + b"\0" + struct.pack("<i", ln)
    return out


def records(text, names):
    """Every line of a SAM body -> its BAM records, back to back."""
    return b"".join(record(line, names) for line in text.split(b"\n") if line)


def split_records(blob):
    """BAM records back to back -> the list of records (each with its block_size)."""
    out, i = [], 0
    while i < len(blob):
        n = struct.unpack_from("<i", blob, i)[0]
        out.append(blob[i:i + 4 + n])
        i += 4 + n
    return out


def walk_qualities(rng, n):
    """A seeded quality random walk: a Phred value in 2..60 that moves by -6..+6 with probability 0.15 per base."""
    import numpy as np
    moves = np.flatnonzero(rng.random(n) < 0.15)
    steps = rng.integers(-6, 7, moves.size)
    q = np.empty(n, dtype=np.uint8)
    v, last = int(rng.integers(2, 61)), 0
    for at, s in zip(moves.tolist(), steps.tolist()):
        q[last:at] = v
        v = min(60, max(2, v + s))
        last = at
    q[last:] = v
    return (q + 33).tobytes()


def mapped_synthetic_reads(n=2000, seed=17, median=2000):
    """n synth.simulate_reads reads, each one mapped record at its true position with an all-M CIGAR and ngmlr's tag
    set, qualities from walk_qualities: (samtext.Read list, contig names, contig lengths)."""
    import numpy as np
    from ngmlr_b200 import samtext, synth
    contig = 1_000_000
    genome = synth.random_genome(2 * contig, seed)
    reads, ivs = synth.simulate_reads(n, genome, contig, seed + 1, median=median, lo=300, hi=6000)
    rng = np.random.default_rng(seed + 2)
    out = []
    for k, iv in enumerate(ivs[:n]):
        seq = bytes(reads[iv.read])
        L = len(seq)
        ref_id = 2 * (iv.ref_start // contig)
        a = samtext.Alignment(ref_pos=iv.ref_start % contig, ref_id=ref_id, reverse=bool(iv.reverse),
                              score=float(L * 0.8), mq=60, nm=int(L * 0.1), identity=0.9, qstart=0, qend=0,
                              cigar=b"%dM" % L, md=b"%d" % L)
        out.append(samtext.Read(b"sim_%d" % k, seq, walk_qualities(rng, L), [a]))
    return out, [b"sim_a", b"sim_a", b"sim_b", b"sim_b"], [contig, contig]
