"""BGZF fixtures for the stream layer's tests (tests/test_bgzf_stream.py on the CPU, tests/test_gpu_bgzf.py on the GPU).

  - bgzf(): htslib's writer layout -- members of at most 0xff00 input bytes, each a gzip member with FLG.FEXTRA and a
    BC subfield holding BSIZE, optionally followed by the 28-byte EOF marker -- at a zlib level and strategy per file,
    optionally with several deflate blocks per member (Z_FULL_FLUSH / Z_SYNC_FLUSH);
  - BitWriter and the hand-built members: what zlib's encoder never emits (a code-length repeat that crosses from the
    literal / length lengths into the distance lengths, a single distance code of length 1, distance 32 768) and one
    member for each deflate error zlib reports;
  - inspect(): a small inflate that lists each member's block types, longest code, longest match, farthest distance
    and distance-1 matches, so the tests can show which parts of deflate the fixture set reaches;
  - stream_read(): ngmlr_b200_debug_stream_read (gzread, the stream layer without a device, or on a context's device).
"""
import ctypes as C
import gzip
import os
import random
import struct
import zlib

EOF_MARKER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
BLOCK = 0xff00


def member(deflate, data, crc=None, isize=None, bsize=None, flg=4, extra=None):
    """One BGZF member around a raw deflate stream (trailer from `data` unless overridden)."""
    extra = extra if extra is not None else b"BC\x02\x00" + b"\0\0"
    total = 12 + len(extra) + len(deflate) + 8
    if extra.startswith(b"BC"):
        extra = extra[:4] + struct.pack("<H", (bsize if bsize is not None else total - 1) & 0xffff) + extra[6:]
    head = b"\x1f\x8b\x08" + bytes([flg]) + b"\0\0\0\0\0\xff" + struct.pack("<H", len(extra)) + extra
    if flg & 8:
        head += b"name.fq\0"
    crc = zlib.crc32(data) if crc is None else crc
    isize = len(data) if isize is None else isize
    return head + deflate + struct.pack("<II", crc & 0xffffffff, isize & 0xffffffff)


def deflate_raw(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flush=None, pieces=4):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    if flush is None:
        return c.compress(data) + c.flush()
    step = max(1, len(data) // pieces)
    out = b""
    for i in range(0, len(data), step):
        out += c.compress(data[i:i + step]) + c.flush(flush)
    return out + c.flush()


def bgzf(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, eof=True, flush=None, block=BLOCK):
    out = []
    for i in range(0, len(data), block):
        chunk = data[i:i + block]
        m = member(deflate_raw(chunk, level, strategy, flush), chunk)
        if len(m) > 65536:  # htslib stores what does not compress into one block
            m = member(deflate_raw(chunk, 0), chunk)
        out.append(m)
    return b"".join(out) + (EOF_MARKER if eof else b"")


def members(blob):
    """[(offset, bytes)] of a BGZF file's members (BSIZE chain)."""
    out, p = [], 0
    while p + 18 <= len(blob):
        xlen = struct.unpack_from("<H", blob, p + 10)[0]
        bsize = struct.unpack_from("<H", blob, p + 16)[0] if xlen >= 6 else None
        if blob[p:p + 4] != b"\x1f\x8b\x08\x04" or bsize is None:
            break
        out.append((p, blob[p:p + bsize + 1]))
        p += bsize + 1
    return out


def _compress_piece(args):
    data, level, blocked = args
    return bgzf(data, level, eof=False) if blocked else gzip.compress(data, level)


def compress_file(src, dst, level=6, blocked=True, piece=BLOCK * 256):
    """src compressed to dst by a process pool: BGZF (with the EOF marker), or multi-member gzip without BC subfields
    (one member per `piece` bytes, which gzread reads like any gzip file). Returns dst's size."""
    from concurrent.futures import ProcessPoolExecutor

    def pieces(f):
        while True:
            c = f.read(piece)
            if not c:
                return
            yield c, level, blocked
    with open(src, "rb") as f, open(dst, "wb") as g, ProcessPoolExecutor() as ex:
        for out in ex.map(_compress_piece, pieces(f), chunksize=2):
            g.write(out)
        if blocked:
            g.write(EOF_MARKER)
    return os.path.getsize(dst)


# ---- a deflate bit writer ------------------------------------------------------------------------------------------
class BitWriter:
    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def bits(self, v, n):
        self.acc |= (v & ((1 << n) - 1)) << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 0xff)
            self.acc >>= 8
            self.n -= 8

    def code(self, c, n):  # a Huffman code goes out most significant bit first
        self.bits(int(format(c, f"0{n}b")[::-1], 2), n)

    def align(self):
        if self.n:
            self.bits(0, 8 - self.n)

    def done(self):
        self.align()
        return bytes(self.out)


def canonical(lens):
    """{symbol: (code, length)} for code lengths (RFC 1951 3.2.2)."""
    bl = [0] * 16
    for l in lens:
        bl[l] += 1
    bl[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = {}
    for s, l in enumerate(lens):
        if l:
            out[s] = (nxt[l], l)
            nxt[l] += 1
    return out


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


def put_match(w, lit, dist, length, distance):
    s = max(i for i in range(29) if LEN_BASE[i] <= length)
    w.code(*lit[257 + s])
    w.bits(length - LEN_BASE[s], LEN_EXTRA[s])
    d = max(i for i in range(30) if DIST_BASE[i] <= distance)
    w.code(*dist[d])
    w.bits(distance - DIST_BASE[d], DIST_EXTRA[d])


def dynamic_header(w, nlit, ndist, cl_syms, cl_lens):
    """Block header of a dynamic block: code-length code cl_lens (19, by symbol) and the symbol stream cl_syms
    [(symbol, extra value)]."""
    ncl = max(i for i in range(19) if cl_lens[CL_ORDER[i]] or i < 4) + 1
    w.bits(nlit - 257, 5)
    w.bits(ndist - 1, 5)
    w.bits(ncl - 4, 4)
    for i in range(ncl):
        w.bits(cl_lens[CL_ORDER[i]], 3)
    cl = canonical(cl_lens)
    for s, x in cl_syms:
        w.code(*cl[s])
        if s == 16:
            w.bits(x - 3, 2)
        elif s == 17:
            w.bits(x - 3, 3)
        elif s == 18:
            w.bits(x - 11, 7)


def cl_stream(lens):
    """Run-length code-length symbols for a list of lengths (16 / 17 / 18 wherever they fit)."""
    out, i = [], 0
    while i < len(lens):
        v, r = lens[i], 1
        while i + r < len(lens) and lens[i + r] == v:
            r += 1
        if v == 0 and r >= 11:
            k = min(r, 138)
            out.append((18, k))
        elif v == 0 and r >= 3:
            k = min(r, 10)
            out.append((17, k))
        else:
            k = 1
            out.append((v, 0))
            if r >= 4:
                k += min(r - 1, 6)
                out.append((16, k - 1))
        i += k
    return out


def complete_cl_lens():
    """A complete code-length code over all 19 symbols: 13 of 4 bits and 6 of 5 bits (13/16 + 6/32 = 1)."""
    lens = [4] * 19
    for s in (1, 2, 3, 4, 5, 6):
        lens[s] = 5
    return lens


def dynamic_member(lit_lens, dist_lens, body, data, final=True, cl_syms=None, cl_lens=None, **kw):
    """A member of one dynamic block; body(w, lit, dist) writes its symbols (end-of-block included)."""
    w = BitWriter()
    w.bits(int(final), 1)
    w.bits(2, 2)
    cl_lens = cl_lens or complete_cl_lens()
    dynamic_header(w, len(lit_lens), len(dist_lens), cl_syms or cl_stream(lit_lens + dist_lens), cl_lens)
    body(w, canonical(lit_lens), canonical(dist_lens))
    return member(w.done(), data, **kw)


def fixed_member(body, data, **kw):
    w = BitWriter()
    w.bits(1, 1)
    w.bits(1, 2)
    body(w, canonical(FIXED_LIT), canonical([5] * 32))
    return member(w.done(), data, **kw)


def _lits(w, lit, s):
    for b in s:
        w.code(*lit[b])


def _lit3():  # 'A' (1 bit), end-of-block and length symbol 257 (2 bits each)
    lens = [0] * 258
    lens[65], lens[256], lens[257] = 1, 2, 2
    return lens


def cross_repeat_member():
    """Literal / length lengths end with 2, 2 and the distance lengths are 2, 2, 2, 2: one repeat code 16 covers
    symbols 257 .. 261, crossing into the distance lengths. Output 'A' then a copy of 3 at distance 1."""
    lit, dist = _lit3(), [2, 2, 2, 2]
    syms = [(18, 65), (1, 0), (18, 138), (18, 52), (2, 0), (16, 5)]
    assert sum(x if s >= 16 else 1 for s, x in syms) == 262

    def body(w, L, D):
        w.code(*L[65])
        put_match(w, L, D, 3, 1)
        w.code(*L[256])
    return dynamic_member(lit, dist, body, b"AAAA", cl_syms=syms)


def single_distance_member():
    """One distance code, of length 1 (incomplete: zlib's one allowed case)."""
    def body(w, L, D):
        w.code(*L[65])
        put_match(w, L, D, 3, 1)
        put_match(w, L, D, 3, 1)
        w.code(*L[256])
    return dynamic_member(_lit3(), [1], body, b"A" * 7)


def far_distance_member(seed=3):
    """A stored block of 32 768 bytes, then a fixed block copying 258 bytes from distance 32 768 (zlib's encoder stops
    at 32 506)."""
    rng = random.Random(seed)
    raw = bytes(rng.randrange(256) for _ in range(32768))
    w = BitWriter()
    w.bits(0, 1)
    w.bits(0, 2)
    w.align()
    w.bits(len(raw), 16)
    w.bits(~len(raw) & 0xffff, 16)
    for b in raw:
        w.bits(b, 8)
    w.bits(1, 1)
    w.bits(1, 2)
    L, D = canonical(FIXED_LIT), canonical([5] * 32)
    put_match(w, L, D, 258, 32768)
    w.code(*L[256])
    return member(w.done(), raw + raw[:258])


def reject_members():
    """{name: member} for every deflate error zlib reports; each trailer is that of b"AAAA"."""
    d = b"AAAA"
    out = {}
    w = BitWriter()
    w.bits(1, 1)
    w.bits(3, 2)
    out["block_type_3"] = member(w.done() + b"\0" * 8, d)
    w = BitWriter()
    w.bits(1, 1)
    w.bits(0, 2)
    w.align()
    w.bits(4, 16)
    w.bits(0x1234, 16)
    out["stored_nlen"] = member(w.done() + d, d)
    for name, nlit, ndist in (("hlit_287", 287, 2), ("hdist_31", 258, 31)):
        w = BitWriter()
        w.bits(1, 1)
        w.bits(2, 2)
        w.bits(nlit - 257, 5)
        w.bits(ndist - 1, 5)
        w.bits(15, 4)
        for _ in range(19):
            w.bits(4, 3)
        out[name] = member(w.done() + b"\0" * 64, d)
    over = [0] * 258
    over[65] = over[66] = over[256] = 1

    # sets zlib refuses: only their code-length streams are written (no symbol could be coded with them)
    def raw_lens(lens, dist, tail):
        w = BitWriter()
        w.bits(1, 1)
        w.bits(2, 2)
        dynamic_header(w, len(lens), len(dist), cl_stream(lens + dist), complete_cl_lens())
        w.bits(tail, 16)
        return member(w.done() + b"\0" * 16, d)
    out["oversubscribed"] = raw_lens(over, [1], 0)
    inc = [0] * 258
    inc[65], inc[256] = 2, 2
    out["incomplete"] = raw_lens(inc, [1], 0)
    out["incomplete_distance"] = raw_lens(_lit3(), [2], 0)
    for name, syms in (("repeat_first", [(16, 3)] + cl_stream(_lit3()[3:] + [1])),
                       ("repeat_overrun", cl_stream(_lit3() + [1])[:-1] + [(18, 20)])):
        w = BitWriter()
        w.bits(1, 1)
        w.bits(2, 2)
        dynamic_header(w, 258, 1, syms, complete_cl_lens())
        out[name] = member(w.done() + b"\0" * 16, d)
    no_eob = [0] * 258
    no_eob[65], no_eob[66] = 1, 1
    out["no_end_of_block"] = raw_lens(no_eob, [1], 0)
    w = BitWriter()
    w.bits(1, 1)
    w.bits(2, 2)
    w.bits(1, 5)
    w.bits(0, 5)
    w.bits(15, 4)
    for i in range(19):
        w.bits(5 if i == 0 else 0, 3)  # one code-length code of 5 bits: incomplete
    out["incomplete_cl_code"] = member(w.done() + b"\0" * 16, d)
    for name, sym in (("literal_286", 286), ("literal_287", 287)):
        def body(w, L, D, sym=sym):
            w.code(*L[65])
            w.code(*L[sym])
            w.code(*L[256])
        out[name] = fixed_member(body, d)
    for name, ds in (("distance_30", 30), ("distance_31", 31)):
        def body(w, L, D, ds=ds):
            _lits(w, L, b"AA")
            w.code(*L[257])
            w.code(*D[ds])
            w.code(*L[256])
        out[name] = fixed_member(body, d)

    def too_far(w, L, D):
        w.code(*L[65])
        put_match(w, L, D, 3, 2)
        w.code(*L[256])
    out["distance_too_far"] = fixed_member(too_far, d)

    def not_final(w, L, D):  # a block that is not the last, then the trailer: the stream has no end
        _lits(w, L, d)
        w.code(*L[256])
    w = BitWriter()
    w.bits(0, 1)
    w.bits(1, 2)
    not_final(w, canonical(FIXED_LIT), None)
    out["no_final_block"] = member(w.done(), d)
    return out


# ---- the fixture set -----------------------------------------------------------------------------------------------
def _fastq(seed, n):
    rng = random.Random(seed)
    out = []
    for i in range(n):
        L = rng.choice([50, 150, 300, 1000])
        s = "".join(rng.choice("ACGT") for _ in range(L))
        q = "".join(rng.choice("#+5?@>AEI") for _ in range(L))
        out.append(f"@r{seed}_{i} c\n{s}\n+\n{q}\n")
    return "".join(out).encode()


def _fib_text():
    """Symbol frequencies of consecutive Fibonacci numbers, shuffled: Huffman-only coding gives 15-bit codes."""
    a, b, out = 1, 1, []
    for i in range(22):
        out += [33 + i] * a
        a, b = b, a + b
    rng = random.Random(5)
    rng.shuffle(out)
    return bytes(out)


def sources():
    """{name: source bytes} of the clean fixtures."""
    rng = random.Random(9)
    runs = b"".join(bytes([rng.choice(b"ACGTN")]) * rng.choice([1, 5, 300, 2000]) for _ in range(300))
    return {"fastq": _fastq(1, 400), "runs": runs, "fib": _fib_text()[:60000], "random": rng.randbytes(150000),
            "small": _fastq(2, 3)}


def clean_files():
    """{name: (file bytes, source bytes)}: every level / strategy / flush / EOF variant the set needs."""
    src = sources()
    f = {}
    for lvl in (0, 1, 6, 9):
        f[f"fastq_l{lvl}"] = (bgzf(src["fastq"], lvl), src["fastq"])
    f["fastq_noeof"] = (bgzf(src["fastq"], 6, eof=False), src["fastq"])
    f["runs_rle"] = (bgzf(src["runs"], 6, zlib.Z_RLE), src["runs"])
    f["runs_l9"] = (bgzf(src["runs"], 9), src["runs"])
    f["fib_huffman"] = (bgzf(src["fib"], 6, zlib.Z_HUFFMAN_ONLY), src["fib"])
    f["fastq_fixed"] = (bgzf(src["fastq"], 6, zlib.Z_FIXED), src["fastq"])
    f["fastq_full_flush"] = (bgzf(src["fastq"], 6, flush=zlib.Z_FULL_FLUSH), src["fastq"])
    f["fastq_sync_flush"] = (bgzf(src["fastq"], 1, flush=zlib.Z_SYNC_FLUSH), src["fastq"])
    f["random"] = (bgzf(src["random"], 6), src["random"])
    f["small"] = (bgzf(src["small"], 6), src["small"])
    f["eof_only"] = (EOF_MARKER, b"")
    far = far_distance_member()
    blob = bgzf(src["small"], 6, eof=False) + cross_repeat_member() + single_distance_member() + far + EOF_MARKER
    f["hand_built"] = (blob, src["small"] + b"AAAA" + b"A" * 7 + gzip.decompress(far))
    return f


def edge_files():
    """{name: file bytes} of files the device path must hand to zlib (or that end early / oddly)."""
    src = sources()
    good = bgzf(src["fastq"], 6, eof=False)
    ms = members(good)
    k = len(ms) // 2
    head = b"".join(m for _, m in ms[:k])
    tail = b"".join(m for _, m in ms[k:])
    mid = ms[k][1]
    e = {}
    for name, m in reject_members().items():
        e["reject_" + name] = head + m + tail + EOF_MARKER
    bad = bytearray(mid)
    bad[-8] ^= 1
    e["crc"] = head + bytes(bad) + tail + EOF_MARKER
    bad = bytearray(mid)
    bad[-4] ^= 1
    e["isize"] = head + bytes(bad) + tail + EOF_MARKER
    bad = bytearray(mid)
    bad[-4:] = struct.pack("<I", 70000)
    e["isize_over_64k"] = head + bytes(bad) + tail + EOF_MARKER
    bad = bytearray(mid)
    struct.pack_into("<H", bad, 16, len(mid) + 1)  # BSIZE one byte long
    e["bsize_long"] = head + bytes(bad) + tail + EOF_MARKER
    bad = bytearray(mid)
    struct.pack_into("<H", bad, 16, len(mid) - 3)
    e["bsize_short"] = head + bytes(bad) + tail + EOF_MARKER
    e["bsize_past_end"] = head + mid[:len(mid) // 2]
    e["truncated_mid_member"] = head + mid[:len(mid) // 2]
    e["truncated_in_trailer"] = head + mid[:-3]
    e["truncated_at_member"] = head
    e["truncated_header"] = head + mid[:11]
    e["eof_marker_middle"] = head + EOF_MARKER + tail + EOF_MARKER
    e["eof_markers_only_mid"] = head + EOF_MARKER * 5 + tail
    e["plain_gzip_after"] = head + gzip.compress(src["small"]) + tail + EOF_MARKER
    e["garbage_one_byte"] = good + EOF_MARKER + b"x"
    e["garbage_1f"] = good + EOF_MARKER + b"\x1f"
    e["garbage_text"] = good + EOF_MARKER + b"@not a member\nACGT\n"
    e["garbage_magic"] = good + EOF_MARKER + b"\x1f\x8b\x08\x00junk"
    e["fname_middle"] = head + member(deflate_raw(b"ACGT\n"), b"ACGT\n", flg=0x0c) + tail + EOF_MARKER
    e["fname_first"] = member(deflate_raw(src["small"]), src["small"], flg=0x0c) + good + EOF_MARKER
    e["fhcrc_first"] = gzip.compress(src["small"])  # single-member gzip: gzread throughout
    e["extra_without_bc"] = member(deflate_raw(src["small"]), src["small"], extra=b"XY\x02\x00ab") + good
    e["empty"] = b""
    e["plain_text"] = src["small"]
    e["bad_crc_eof_marker"] = good + EOF_MARKER[:-8] + b"\x01\0\0\0\0\0\0\0"
    return e


# ---- an inflate that reports what it decodes ------------------------------------------------------------------------
class _Bits:
    def __init__(self, b):
        self.b, self.p = b, 0

    def get(self, n):
        v = 0
        for i in range(n):
            v |= ((self.b[self.p >> 3] >> (self.p & 7)) & 1) << i
            self.p += 1
        return v


def _decoder(lens):
    codes = {(l, c): s for s, (c, l) in canonical(lens).items()}
    return codes


def _sym(br, table):
    c = 0
    for l in range(1, 16):
        c = (c << 1) | br.get(1)
        if (l, c) in table:
            return table[(l, c)], l
    raise ValueError("bad code")


def inspect(deflate):
    """(output, info) of one raw deflate stream: info = block types, longest code, longest match, farthest distance,
    number of distance-1 matches."""
    br, out = _Bits(deflate), bytearray()
    info = {"types": [], "max_code": 0, "max_len": 0, "max_dist": 0, "dist1": 0}
    while True:
        last, t = br.get(1), br.get(2)
        info["types"].append(t)
        if t == 0:
            br.p = (br.p + 7) & ~7
            n = br.get(16)
            br.get(16)
            out += deflate[br.p >> 3:(br.p >> 3) + n]
            br.p += 8 * n
        else:
            if t == 1:
                ll, dl = FIXED_LIT, [5] * 32
            else:
                nlit, ndist, ncl = br.get(5) + 257, br.get(5) + 1, br.get(4) + 4
                cl = [0] * 19
                for i in range(ncl):
                    cl[CL_ORDER[i]] = br.get(3)
                clt, lens = _decoder(cl), []
                while len(lens) < nlit + ndist:
                    s, _ = _sym(br, clt)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + br.get(2))
                    elif s == 17:
                        lens += [0] * (3 + br.get(3))
                    else:
                        lens += [0] * (11 + br.get(7))
                ll, dl = lens[:nlit], lens[nlit:]
            info["max_code"] = max(info["max_code"], max(ll), max(dl))
            lt, dt = _decoder(ll), _decoder(dl)
            while True:
                s, _ = _sym(br, lt)
                if s < 256:
                    out.append(s)
                elif s == 256:
                    break
                else:
                    n = LEN_BASE[s - 257] + br.get(LEN_EXTRA[s - 257])
                    d, _ = _sym(br, dt)
                    dist = DIST_BASE[d] + br.get(DIST_EXTRA[d])
                    for _ in range(n):
                        out.append(out[-dist])
                    info["max_len"] = max(info["max_len"], n)
                    info["max_dist"] = max(info["max_dist"], dist)
                    info["dist1"] += dist == 1
        if last:
            return bytes(out), info


def member_deflate(m):
    xlen = struct.unpack_from("<H", m, 10)[0]
    return m[12 + xlen:-8]


# ---- the stream layer through the C ABI ----------------------------------------------------------------------------
GZREAD, HOST, DEVICE = 0, 1, 2


def stream_read(lib, path, mode, read_size, ctx=None, cap=None):
    """(bytes, error, truncated, (compressed bytes, device members, host bytes), inflate ms) of
    ngmlr_b200_debug_stream_read."""
    cap = cap if cap is not None else max(os.path.getsize(path) * 8, 1 << 20) if os.path.exists(path) else 1 << 20
    buf = (C.c_uint8 * cap)()
    n, err, tr = C.c_int64(0), C.c_int32(0), C.c_int32(0)
    cnt = (C.c_int64 * 3)()
    ms = C.c_float(0)
    rc = lib.ngmlr_b200_debug_stream_read(os.fsencode(path), mode, ctx, int(read_size), buf, cap, C.byref(n),
                                          C.byref(err), C.byref(tr), cnt, C.byref(ms))
    assert rc == 0, lib.ngmlr_b200_last_error(None)
    assert n.value <= cap, (path, n.value, cap)
    return bytes(buf[:n.value]), err.value, tr.value, tuple(cnt), ms.value
