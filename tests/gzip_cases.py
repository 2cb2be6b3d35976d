"""Plain gzip streams (one deflate stream per member, as gzip, pigz and Python's gzip write) for the device gzip path:
clean streams across zlib's levels, strategies, flushes and header flags, member layouts, hand-built deflate, a
stored block that hides a valid dynamic block header (a guaranteed false block start), and refusals zlib decides.
The deflate bit writer and the reject members come from bgzf_cases."""
import ctypes as C
import os
import random
import struct
import zlib

import bgzf_cases as B

MiB = 1 << 20
# stream.cpp: the compression ratios and the round size at which a stream stays on the device
GZ_RATIO_LO, GZ_RATIO_HI, GZ_DEVICE_ROUND = 1.5, 6.5, 256 * MiB


def header(flg=0, extra=b"", name=b"", comment=b""):
    h = bytearray(b"\x1f\x8b\x08" + bytes([flg]) + b"\0\0\0\0\0\xff")
    if flg & 4:
        h += struct.pack("<H", len(extra)) + extra
    if flg & 8:
        h += name + b"\0"
    if flg & 16:
        h += comment + b"\0"
    if flg & 2:
        h += struct.pack("<H", zlib.crc32(bytes(h)) & 0xffff)
    return bytes(h)


def wrap(deflate, data, crc=None, isize=None, **hdr):
    crc = zlib.crc32(data) if crc is None else crc
    isize = len(data) & 0xffffffff if isize is None else isize
    return header(**hdr) + deflate + struct.pack("<II", crc, isize)


def gz(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, mem=8, flush=None, pieces=8, **hdr):
    """One member of data compressed by zlib; flush (Z_SYNC_FLUSH / Z_FULL_FLUSH) between `pieces` parts."""
    c = zlib.compressobj(level, zlib.DEFLATED, -15, mem, strategy)
    out = []
    step = max(1, len(data) // pieces)
    for i in range(0, len(data), step):
        out.append(c.compress(data[i:i + step]))
        if flush is not None:
            out.append(c.flush(flush))
    out.append(c.flush())
    return wrap(b"".join(out), data, **hdr)


def fastq(nbytes, seed=5):
    """pacbio50-shaped FASTQ: reads of a few kb with qualities."""
    rng = random.Random(seed)
    out, n = [], 0
    i = 0
    while n < nbytes:
        L = rng.randint(2000, 12000)
        s = bytes(rng.choice(b"ACGT") for _ in range(64)) * (L // 64 + 1)
        s = s[:L]
        q = bytes(rng.choice(b"#$%&'()*+,-./0123456789:;<=>?") for _ in range(32)) * (L // 32 + 1)
        rec = b"@m54/%d/0_%d\n%s\n+\n%s\n" % (i, L, s, q[:L])
        out.append(rec)
        n += len(rec)
        i += 1
    return b"".join(out)


def false_start_stream():
    """A stored block whose payload is copies of a small compressed dynamic block (the finder accepts each copy's
    header, one in every chunk, so the chunk holding the stored block's true end starts at a false one), then a
    dynamic final block: (member, data)."""
    text = B.sources()["fastq"][:200_000]
    c = zlib.compressobj(9, zlib.DEFLATED, -15)
    dyn = c.compress(text[:3000]) + c.flush(zlib.Z_FULL_FLUSH)  # one non-final block, byte aligned
    assert len(dyn) < 2000
    payload = (dyn * (60_000 // len(dyn) + 1))[:60_000]
    stored = b"\x00" + struct.pack("<HH", len(payload), len(payload) ^ 0xffff) + payload
    rest = text[:50_000]
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    tail = c.compress(rest) + c.flush()
    data = payload + rest
    return wrap(stored + tail, data), data


def clean():
    """{name: (file bytes, inflated bytes)}."""
    src = B.sources()["fastq"]
    rnd = random.Random(7).randbytes(3 * MiB)
    out = {}
    for level in (0, 1, 6, 9):
        out[f"level{level}"] = (gz(src, level), src)
    for name, st in (("rle", zlib.Z_RLE), ("huffman", zlib.Z_HUFFMAN_ONLY), ("filtered", zlib.Z_FILTERED),
                     ("fixed", zlib.Z_FIXED)):
        out[name] = (gz(src, 6, st), src)
    out["mem9"] = (gz(src, 6, mem=9), src)
    out["sync_flush"] = (gz(src, 6, flush=zlib.Z_SYNC_FLUSH), src)
    out["full_flush"] = (gz(src, 6, flush=zlib.Z_FULL_FLUSH), src)
    out["header_flags"] = (gz(src, 6, flg=2 | 4 | 8 | 16, extra=b"ab\x02\x00xy", name=b"reads.fq",
                              comment=b"a comment"), src)
    half = len(src) // 2
    out["two_members"] = (gz(src[:half]) + gz(src[half:], 1), src)
    small = [src[i:i + 3000] for i in range(0, 300 * 3000, 3000)]
    out["300_members"] = (b"".join(gz(s) for s in small), b"".join(small))
    out["empty_member"] = (gz(src[:5000]) + gz(b"") + gz(src[5000:20000]), src[:20000])
    out["random"] = (gz(rnd), rnd)
    n = b"N" * (64 * 10 ** 6)
    out["n_64mb"] = (gz(n), n)
    for name, m in (("far_distance", B.far_distance_member()), ("cross_repeat", B.cross_repeat_member())):
        d = B.member_deflate(m)
        out[name] = (wrap(d, zlib.decompress(d, -15)), zlib.decompress(d, -15))
    fs, fd = false_start_stream()
    out["false_start"] = (fs, fd)
    return out


def big_fastq():
    data = fastq(40 * 10 ** 6)
    return gz(data, 1), data


# refusals with a clean prefix the device may return: a whole clean member first (every after_* case too), or many
# MB of a member before its corruption (the release rule holds back the last 2 MiB before any problem)
CLEAN_PREFIX = {"deep_flip", "trailing_garbage", "trailing_magic", "trunc_second_header", "distance_before_member"}


def refusals():
    """{name: file bytes} zlib refuses, truncates or reads on from."""
    src = B.sources()["fastq"]
    big = gz(src)
    out = {}
    for name, m in B.reject_members().items():
        bad = wrap(B.member_deflate(m), b"AAAA")
        out["start_" + name] = bad
        out["after_" + name] = big + bad
    raw = gz(src * 40)  # about 13 MB in one member
    flip = bytearray(raw)
    flip[int(len(raw) * 0.7)] ^= 0x5a
    out["deep_flip"] = bytes(flip)
    bad_crc = bytearray(big)
    bad_crc[-8] ^= 1
    out["crc"] = bytes(bad_crc) + gz(src[:1000])
    bad_isize = bytearray(big)
    bad_isize[-4] ^= 1
    out["isize"] = bytes(bad_isize)
    out["trunc_mid_block"] = big[:len(big) // 2]
    out["trunc_trailer"] = big[:-3]
    out["trunc_second_header"] = big + gz(src[:1000])[:6]
    out["trailing_garbage"] = big + b"garbage after the member"
    out["trailing_magic"] = big + b"\x1f\x8b\x09junk"
    out["distance_before_member"] = big + _far_member()
    return out


def _far_member():
    """A member whose first block reaches one byte before its first output byte."""
    data = b"xyz" * 10
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    good = c.compress(data) + c.flush()
    # the dictionary trick: compress with a preset dictionary so the stream references bytes before its start
    c = zlib.compressobj(6, zlib.DEFLATED, -15, 8, zlib.Z_DEFAULT_STRATEGY, b"xyz" * 100)
    dep = c.compress(data) + c.flush()
    assert dep != good
    return wrap(dep, data)


def stream_read(lib, path, ctx, read_size, chunk=0, cap=1 << 20):
    """(bytes, error, truncated, (compressed, device members, host bytes), (gzip bytes, chunks, redecoded, us)) of up to
    cap bytes."""
    buf = (C.c_uint8 * cap)()
    n, err, tr = C.c_int64(0), C.c_int32(0), C.c_int32(0)
    cnt, g = (C.c_int64 * 3)(), (C.c_int64 * 4)()
    rc = lib.ngmlr_b200_debug_gzip_stream_read(os.fsencode(path), ctx, int(read_size), int(chunk), buf, cap,
                                               C.byref(n), C.byref(err), C.byref(tr), cnt, g)
    assert rc == 0, lib.ngmlr_b200_last_error(None)
    return bytes(buf[:n.value]), err.value, tr.value, tuple(cnt), tuple(g)
