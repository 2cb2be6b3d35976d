"""Query files that drive the read loader (ngmlr_b200_reads_load) to the limits of its chunk path.

A chunk's line table holds at most limit(capacity) = max(capacity / 32, 4096) newlines. A chunk with more is resolved
up to its limit-th newline and the rest moves to the next chunk ("line-limited"); a chunk whose first record does not
fit its bytes or its line table doubles. The generators here make files that reach those branches on purpose:
  - dense(): short-read files whose lines average under 32 bytes, so that every full chunk is line-limited;
  - limit_edge(): the limit-th newline of the first chunk on its last byte, on its second-to-last byte, or followed
    by a header character;
  - long_record() / growth files: one record with more lines than the limit (or more bytes than the chunk) among
    ordinary records;
  - segment_edges(): header characters at the 2 KiB segment edges of the newline / marker pass, junk runs of several
    segments with and without '>' / '@' in them;
  - scale_fuzz(): about 40 MB of mixed short and long reads, CRLF, empty records, junk and a dropped read at the end.
Every generator is seeded and builds its bytes with numpy and bytes.join."""
import numpy as np

import read_loader_cases as R

KiB, MiB = 1 << 10, 1 << 20
SEG = 2048  # bytes per warp of the loader's newline / marker pass


def limit(capacity):
    """Newlines the line table of a chunk of this capacity holds."""
    return max(capacity // 32, 4096)


def doublings(capacity, lines=0, nbytes=0):
    """Doublings of a chunk of this capacity until `lines` newlines fit its line table and `nbytes` its bytes."""
    d = 0
    while limit(capacity << d) < lines or (capacity << d) < nbytes:
        d += 1
    return d


class _Gen:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)

    def bases(self, n, alphabet=b"ACGT"):
        a = np.frombuffer(alphabet, np.uint8)
        return a[self.rng.integers(0, len(a), n)].tobytes()

    def qual(self, n, alphabet=b"!#+5?@>ABCDEFGHIJ"):
        return self.bases(n, alphabet)

    def pick(self, lo, hi, n):
        return self.rng.integers(lo, hi + 1, n).tolist()


def _wrap(s, w, nl=b"\n"):
    return nl.join(s[i:i + w] for i in range(0, len(s), w))


def _mutate(g, s, k):
    s = bytearray(s)
    for p in g.pick(0, len(s) - 1, k):
        s[p] = g.bases(1)[0]
    return bytes(s)


# ---- (a) dense files -------------------------------------------------------------------------------------------------
def sra_fastq(seed, n, lo=36, hi=36, genome=None, name=b"SRR062634"):
    """SRA-style FASTQ: '@SRR062634.i' with the name repeated on the '+' line. From `genome` (bytes) the reads are
    drawn from both strands with a few substitutions."""
    g = _Gen(seed)
    comp = bytes.maketrans(b"ACGT", b"TGCA")
    lens = g.pick(lo, hi, n)
    out = []
    for i, L in enumerate(lens):
        if genome is None:
            s = g.bases(L)
        else:
            p = int(g.rng.integers(0, len(genome) - L))
            s = _mutate(g, genome[p:p + L], int(g.rng.integers(0, 3)))
            if g.rng.random() < 0.5:
                s = s.translate(comp)[::-1]
        nm = b"%s.%d" % (name, i + 1)
        out.append(b"@%s\n%s\n+%s\n%s\n" % (nm, s, nm, g.qual(L)))
    return b"".join(out)


def fasta_oneline(seed, n):
    """One-line FASTA of 20-40 bp reads."""
    g = _Gen(seed)
    return b"".join(b">r%d\n%s\n" % (i, g.bases(L)) for i, L in enumerate(g.pick(20, 40, n)))


def fasta_wrapped(seed, n):
    """FASTA of 20-200 bp reads wrapped at widths 1-8."""
    g = _Gen(seed)
    lens, widths = g.pick(20, 200, n), g.pick(1, 8, n)
    return b"".join(b">w%d\n%s\n" % (i, _wrap(g.bases(L), w)) for i, (L, w) in enumerate(zip(lens, widths)))


def blank_runs(seed, n):
    """FASTA and FASTQ records separated by runs of 1-40 blank lines, '\\n' or '\\r\\n'."""
    g = _Gen(seed)
    out = []
    for i in range(n):
        L = int(g.rng.integers(1, 60))
        if g.rng.random() < 0.5:
            out.append(b">b%d\n%s\n" % (i, g.bases(L)))
        else:
            out.append(b"@b%d\n%s\n+\n%s\n" % (i, g.bases(L), g.qual(L)))
        out.append((b"\r\n" if g.rng.random() < 0.5 else b"\n") * int(g.rng.integers(1, 41)))
    return b"".join(out)


def fuzz_repeat(size=10 * MiB):
    """read_loader_cases' fuzz_a + fuzz_b, repeated to about `size` bytes."""
    text = R.CASES["fuzz_a"] + R.CASES["fuzz_b"]
    return text * max(1, size // len(text))


def dense():
    """name -> bytes of the files whose full chunks are line-limited at 256 KiB and 1 MiB."""
    return {
        "sra36": sra_fastq(1, 40_000),
        "fasta_oneline": fasta_oneline(2, 100_000),
        "fasta_wrapped": fasta_wrapped(3, 20_000),
        "blank_runs": blank_runs(4, 50_000),
        "fuzz_repeat": fuzz_repeat(),
    }


def mean_line(data):
    return len(data) / max(1, data.count(b"\n"))


# ---- (a) the limit-th newline at the end of the first chunk ----------------------------------------------------------
def _lines_exact(g, n_lines, nbytes, fastq):
    """Records of exactly n_lines lines (a multiple of 2 / 4) and nbytes bytes, the last byte a newline."""
    per = 4 if fastq else 2
    assert n_lines % per == 0
    n = n_lines // per
    rec = nbytes // n
    out, used = [], 0
    for i in range(n):
        want = rec if i < n - 1 else nbytes - used
        head = b"@e%d" % i if fastq else b">e%d" % i
        if fastq:  # head\n seq\n +\n qual\n
            L = (want - len(head) - 5) // 2
            head += b"x" * (want - len(head) - 5 - 2 * L)
            r = b"%s\n%s\n+\n%s\n" % (head, g.bases(L), g.qual(L))
        else:
            L = want - len(head) - 2
            r = b"%s\n%s\n" % (head, g.bases(L))
        assert len(r) == want
        out.append(r)
        used += want
    return b"".join(out)


def limit_edge(capacity, where, fastq, seed=9):
    """A file whose first chunk (capacity bytes) has its limit-th newline on the chunk's last byte ('last'), on its
    second-to-last byte followed by a blank line ('second_last_nl') or by a header character ('second_last_hdr'), or
    100 bytes before the chunk's end followed by a header character ('hdr_after'). Dense records follow, so the
    later chunks are line-limited."""
    g = _Gen(seed)
    L = limit(capacity)
    end = {"last": capacity, "second_last_nl": capacity - 1, "second_last_hdr": capacity - 1,
           "hdr_after": capacity - 100}[where]
    head = _lines_exact(g, L, end, fastq)
    assert head.count(b"\n") == L and len(head) == end and head[-1:] == b"\n"
    rest = sra_fastq(seed + 1, 20_000, 20, 30) if fastq else fasta_oneline(seed + 1, 40_000)
    if where == "second_last_nl":
        rest = b"\n" + rest
    return head + rest


LIMIT_EDGES = ("last", "second_last_nl", "second_last_hdr", "hdr_after")


# ---- (b) growth ------------------------------------------------------------------------------------------------------
def long_record(kind, lines, seed=12):
    """One record of about `lines` lines: 'fasta1' (FASTA at width 1) or 'fastq2' (FASTQ, sequence and quality at
    width 2)."""
    g = _Gen(seed)
    if kind == "fasta1":
        return b">long\n" + _wrap(g.bases(lines - 1), 1) + b"\n"
    L = lines - 2  # L / 2 sequence and L / 2 quality lines
    return b"@long\n" + _wrap(g.bases(L), 2) + b"\n+\n" + _wrap(g.qual(L), 2) + b"\n"


def wide_record(nbytes, seed=13):
    """One FASTA record of one sequence line of nbytes bases."""
    return b">wide\n" + _Gen(seed).bases(nbytes) + b"\n"


def around(record, where, seed=14, n=3000):
    """record among ordinary short reads: first, in the middle or last ('last_no_nl': without its trailing newline)."""
    before = sra_fastq(seed, n, 20, 40, name=b"pre")
    after = sra_fastq(seed + 1, n, 20, 40, name=b"post")
    if where == "first":
        return record + after
    if where == "middle":
        return before + record + after
    if where == "last":
        return before + record
    assert where == "last_no_nl"
    return before + record[:-1]


# ---- (d) segment edges -----------------------------------------------------------------------------------------------
EDGE_OFFSETS = {"a": (2047, 4096, 6143), "b": (2048, 4095, 8192)}


def _fill_to(g, text, offset):
    """text + a FASTA filler record (wrapped at 70) that ends exactly at `offset`."""
    head = b">fill%d\n" % len(text)
    n = offset - len(text) - len(head) - 1
    assert n >= 1
    seq = g.bases(n)
    body = bytearray(_wrap(seq, 70))[:n]  # keep the byte count: newlines replace bases
    return text + head + bytes(body) + b"\n"


def _junk(g, n, markers):
    alphabet = b"acgtxyz0123 =.;" + (b">@" if markers else b"")
    s = bytearray(g.bases(n, alphabet))
    for p in range(int(g.rng.integers(20, 60)), n, int(g.rng.integers(40, 120))):
        s[p] = ord("\n")
    return bytes(s)


def segment_edges(seed=21):
    """name -> bytes: header characters at offsets 2047, 2048, 4095 and 4096 (and 6143, 8192) at line starts of FASTA
    records ('hdr_at_edges_a' / '_b') and after junk inside a line following a FASTQ record ('fastq_at_edges_a' /
    '_b'); junk runs of 2-10 KiB before the first record and between FASTQ records, with and without '>' / '@' in
    them; a FASTQ record followed by more than three marker-free segments, and another by three."""
    g = _Gen(seed)
    out = {}
    for tag, offsets in EDGE_OFFSETS.items():
        t = b""
        for off in offsets:
            t = _fill_to(g, t, off)
            t += b">h%d\n%s\n" % (off, g.bases(30))
        out["hdr_at_edges_" + tag] = t
        t = b""
        for off in offsets:
            rec = b"@q%d\n%s\n+\n%s\n" % (len(t), g.bases(20), g.qual(20))
            t += rec + _junk(g, off - len(t) - len(rec), False)
            t += b"@m%d\n%s\n+\n%s\n" % (off, g.bases(20), g.qual(20))
        out["fastq_at_edges_" + tag] = t
    recs = [b"@j%d\n%s\n+\n%s\n" % (i, g.bases(50), g.qual(50)) for i in range(12)]
    for markers in (False, True):
        run = lambda: _junk(g, int(g.rng.integers(2 * KiB, 10 * KiB)), markers) + b"\n"
        parts = [run()]
        for r in recs:
            parts += [r, run()]
        parts.append(recs[0])
        out["junk_runs_markers" if markers else "junk_runs"] = b"".join(parts)
    # a record, then junk covering at least three whole segments, then records (twice, at two alignments)
    t = b"@a\n" + g.bases(40) + b"\n+\n" + g.qual(40) + b"\n" + _junk(g, 4 * SEG + 100, False)
    t += b"@b\nACGT\n+\nIIII\n" + _junk(g, 3 * SEG + 1, False) + b">c\nACGT\n"
    out["marker_free_segments"] = t
    return out


def first_markers(data):
    """Offsets of the bytes '>' / '@' that start a line or follow junk (every '>' / '@' in data)."""
    a = np.frombuffer(data, np.uint8)
    return np.flatnonzero((a == ord(">")) | (a == ord("@"))).tolist()


# ---- (e) scale fuzz --------------------------------------------------------------------------------------------------
def scale_fuzz(seed=31, size=40 * MiB):
    """About `size` bytes: short-read FASTQ (some CRLF, some with quality lines starting '@' / '>' / '+'), multi-line
    FASTA / FASTQ long reads up to 100 kb, empty records, junk between FASTQ records; near the end one FASTQ record
    whose quality is one character short (ngmlr drops it and stops), and a few records after it."""
    g = _Gen(seed)
    out, total, i = [], 0, 0
    while total < size:
        u = g.rng.random()
        nl = b"\r\n" if g.rng.random() < 0.1 else b"\n"
        if u < 0.002:  # long read
            L = int(g.rng.integers(1_000, 100_001))
            w = int(g.rng.choice([60, 80, 1000]))
            s = _wrap(g.bases(L), w, nl)
            if g.rng.random() < 0.5:
                r = b">long%d%s%s%s" % (i, nl, s, nl)
            else:
                r = b"@long%d%s%s%s+%s%s%s" % (i, nl, s, nl, nl, _wrap(g.qual(L), w, nl), nl)
        elif u < 0.01:
            r = b">empty%d%s" % (i, nl) if g.rng.random() < 0.5 else b"@empty%d%s%s+%s%s" % (i, nl, nl, nl, nl)
        elif u < 0.02:
            r = _junk(g, int(g.rng.integers(1, 3000)), False) + b"\n"
            if out and out[-1][:1] != b"@":
                r = b""  # junk only after a FASTQ record (after FASTA it would be sequence)
        else:
            L = int(g.rng.integers(30, 151))
            q = g.qual(L)
            if g.rng.random() < 0.05:
                q = bytes([b"@>+"[int(g.rng.integers(0, 3))]]) + q[1:]
            if g.rng.random() < 0.1:  # two quality lines, the second starting with a marker
                k = int(g.rng.integers(1, L))
                q = q[:k] + nl + bytes([b"@>+"[int(g.rng.integers(0, 3))]]) + q[k + 1:]
            r = b"@s%d x%s%s%s+%s%s%s" % (i, nl, g.bases(L), nl, nl, q, nl)
        out.append(r)
        total += len(r)
        i += 1
    out.append(b"@bad\nACGTACGTAC\n+\nIIIIIIIII\n")
    out += [b"@after%d\nACGT\n+\nIIII\n" % k for k in range(5)]
    return b"".join(out)
