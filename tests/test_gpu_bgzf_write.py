"""The BGZF writer with the deflate on the device (ngmlr_b200_bgzf_*): member framing, determinism, the ratio against
zlib level 1, BAM read back through this repository's own loader, the file-to-BAM flow, errors and device memory."""
import os
import random
import struct
import zlib

import numpy as np
import pytest

import bam_write_cases as bw
import bgzf_cases as G
import test_gpu_read_loader as T
from ngmlr_b200 import B200Aligner, samtext

pytestmark = pytest.mark.gpu
BLOCK = 0xff00


@pytest.fixture(scope="module")
def aligner():
    a = B200Aligner(0)
    yield a
    a.close()


def _write(a, path, pieces, chunk_bytes=0, flush_after=()):
    with a.bgzf_writer(path, chunk_bytes=chunk_bytes) as w:
        for k, p in enumerate(pieces):
            w.write(p)
            if k in flush_after:
                w.flush()
    return open(path, "rb").read(), w.stats()


def _check_members(blob):
    """Every member's framing, CRC32, ISIZE and inflate; returns [(member bytes, inflated piece)]."""
    assert blob.endswith(G.EOF_MARKER)
    ms = G.members(blob[:-len(G.EOF_MARKER)])
    assert sum(len(m) for _, m in ms) == len(blob) - len(G.EOF_MARKER)
    out = []
    for off, m in ms:
        assert m[:12] == bytes.fromhex("1f8b08040000000000ff0600") and m[12:16] == b"BC\x02\x00"
        assert struct.unpack_from("<H", m, 16)[0] == len(m) - 1 and len(m) <= 65536
        data = zlib.decompressobj(-15)
        piece = data.decompress(m[18:-8])
        assert data.eof and data.unused_data == b"", off
        crc, isize = struct.unpack_from("<II", m, len(m) - 8)
        assert crc == zlib.crc32(piece) and isize == len(piece), off
        out.append((m, piece))
    return out


def _framing_inputs():
    rng = np.random.default_rng(1)
    rand8 = rng.integers(0, 256, 8 << 20, dtype=np.uint8).tobytes()
    base = rng.integers(0, 256, 40000, dtype=np.uint8).tobytes()
    far = base[:32768] + base[:300] + base[40000 - 20000:]        # a 300-byte repeat at distance exactly 32 768
    farther = base[:32769] + base[:300] + base[40000 - 20000:]    # ... and at 32 769 (out of reach)
    runs = b"".join(bytes([c]) * n for c, n in zip(rng.integers(0, 256, 400).tolist(),
                                                     rng.integers(1, 1200, 400).tolist()))
    return {
        "empty": b"", "one": b"x", "block-1": rand8[:BLOCK - 1], "block": rand8[:BLOCK], "block+1": rand8[:BLOCK + 1],
        "random8M": rand8, "zeros8M": bytes(8 << 20), "runs": runs, "dist32768": far, "dist32769": farther,
        "text": b"".join(b"line %d of some text\tACGT%s\n" % (i, b"AC" * (i % 50)) for i in range(100000)),
    }


@pytest.mark.parametrize("name", list(_framing_inputs()))
def test_members_inflate_to_their_pieces(aligner, tmp_path, name):
    data = _framing_inputs()[name]
    blob, st = _write(aligner, str(tmp_path / "o.gz"), [data])
    ms = _check_members(blob)
    assert b"".join(p for _, p in ms) == data
    assert [len(p) for _, p in ms] == [min(BLOCK, len(data) - i) for i in range(0, len(data), BLOCK)]
    assert st["bytes_in"] == len(data) and st["blocks"] == len(ms)
    assert st["bytes_out"] == len(blob) - len(G.EOF_MARKER)
    if name.startswith("random") or name.startswith("block"):
        assert all(len(m) <= len(p) + 31 for m, p in ms)
        assert st["stored_blocks"] == sum(len(p) >= 1024 for _, p in ms)   # a byte or two costs less as fixed
    if name == "zeros8M":
        assert all(len(m) < 200 for m, _ in ms)


def _btype(member):
    """BTYPE of the member's (only) deflate block: 0 stored, 1 fixed, 2 dynamic."""
    return (member[18] >> 1) & 3


def test_fixed_blocks_with_high_literals(aligner, tmp_path):
    """Short flushed pieces come out as fixed Huffman blocks; literals 0x90..0xFF take the fixed code's 9-bit codes."""
    reads, names, _ = bw.mapped_synthetic_reads(n=3, seed=2, median=400)
    record = bw.split_records(samtext.bam_format(reads, names, [b"sim_a", b"sim_b"]))[0]
    every = bytes(range(256))
    pieces = [b"\x90", b"\xff", b"\x8f\x90\xff\x00"]
    pieces += [every[i:i + k] for k in (1, 2, 3, 5, 8, 13) for i in range(0, 256, k)]
    pieces += [record[:40], record]
    blob, _ = _write(aligner, str(tmp_path / "fixed.gz"), pieces, flush_after=set(range(len(pieces))))
    ms = _check_members(blob)
    assert [p for _, p in ms] == pieces
    fixed = [p for m, p in ms if _btype(m) == 1]
    assert b"\x90" in fixed and b"\xff" in fixed
    assert set(b"".join(fixed)) >= set(range(0x90, 0x100))


def test_short_pieces_of_every_kind_inflate(aligner, tmp_path):
    """Pieces of 1 - 4000 bytes over alphabets of 1 - 256 symbols, each flushed: stored, fixed and dynamic blocks."""
    rng = np.random.default_rng(8)
    pieces = []
    for _ in range(400):
        n = int(rng.integers(1, 4000))
        k = int(rng.choice([1, 2, 4, 16, 64, 256]))
        lo = int(rng.integers(0, 257 - k))
        piece = rng.integers(lo, lo + k, n, dtype=np.uint8)
        if rng.random() < 0.3:   # repeats for the match finder
            piece = np.tile(piece[:max(1, n // 7)], 7)[:n]
        pieces.append(piece.tobytes())
    blob, st = _write(aligner, str(tmp_path / "short.gz"), pieces, flush_after=set(range(len(pieces))))
    ms = _check_members(blob)
    assert [p for _, p in ms] == pieces
    kinds = {_btype(m) for m, _ in ms}
    assert kinds == {0, 1, 2}, kinds
    assert st["stored_blocks"] == sum(_btype(m) == 0 for m, _ in ms)


def test_flush_ends_a_block_and_nothing_else_does(aligner, tmp_path):
    rng = np.random.default_rng(2)
    pieces = [rng.integers(0, 4, int(n), dtype=np.uint8).tobytes() for n in (100, 70000, 5, 0, 130000)]
    blob, _ = _write(aligner, str(tmp_path / "f.gz"), pieces, flush_after={0, 2, 3})
    sizes = [len(p) for _, p in _check_members(blob)]
    assert sizes == [100, BLOCK, 70005 - BLOCK, BLOCK, 130000 - BLOCK]


def test_file_depends_only_on_bytes_and_flush_points(aligner, tmp_path):
    rng = random.Random(3)
    reads, names, _ = bw.mapped_synthetic_reads(n=600, seed=5, median=3000)
    data = samtext.bam_format(reads, names, [b"sim_a", b"sim_b"])
    data = data + bytes(np.random.default_rng(4).integers(0, 256, 3 << 20, dtype=np.uint8)) + data
    want = None
    for chunk in (1 << 20, 7 << 20, 64 << 20):
        for trial in range(2):
            cuts = sorted(rng.randrange(len(data)) for _ in range(rng.choice([0, 3, 40])))
            pieces = [data[a:b] for a, b in zip([0] + cuts, cuts + [len(data)])]
            blob, _ = _write(aligner, str(tmp_path / f"d{chunk}_{trial}.gz"), pieces, chunk_bytes=chunk)
            if want is None:
                want = blob
                assert b"".join(p for _, p in _check_members(blob)) == data
            assert blob == want, (chunk, trial)
    # a second context / handle on the same device
    b = B200Aligner(0)
    try:
        blob, _ = _write(b, str(tmp_path / "other.gz"), [data])
    finally:
        b.close()
    assert blob == want


def _zlib1(pieces):
    total = 0
    for p in pieces:
        c = zlib.compressobj(1, zlib.DEFLATED, -15)
        total += len(c.compress(p) + c.flush())
    return total


@pytest.mark.parametrize("fmt", ["bam", "sam"])
def test_ratio_not_worse_than_zlib_level_1(aligner, tmp_path, fmt):
    reads, names, lens = bw.mapped_synthetic_reads()
    targets = [b"sim_a", b"sim_b"]
    if fmt == "bam":
        head, body = samtext.bam_header(targets, lens), samtext.bam_format(reads, names, targets)
    else:
        head, body = samtext.sam_header(targets, lens), samtext.sam_format(reads, names)
    blob, _ = _write(aligner, str(tmp_path / f"r.{fmt}"), [head, body], flush_after={0})
    ms = _check_members(blob)
    assert b"".join(p for _, p in ms) == head + body
    ours = sum(len(m) - 26 for m, _ in ms)
    z1 = _zlib1([p for _, p in ms])
    print(f"{fmt}: {len(head + body)} bytes, device deflate {ours}, zlib-1 {z1}, ratio {ours / z1:.4f}")
    assert ours <= z1, (ours, z1)


def test_bam_round_trip_through_the_read_loader(aligner, tmp_path):
    reads, names, lens = bw.mapped_synthetic_reads(n=500, seed=9, median=1500)
    targets = [b"sim_a", b"sim_b"]
    for r in reads[::3]:   # a secondary copy after some reads: the loader skips 0x900
        r.alignments.append(samtext.Alignment(ref_pos=5, ref_id=0, reverse=not r.alignments[0].reverse, score=1.0,
                                              mq=0, nm=0, identity=0.5, qstart=0, qend=0,
                                              cigar=b"%dM" % len(r.seq), md=b"0", primary=False))
    path = str(tmp_path / "rt.bam")
    with aligner.bgzf_writer(path) as w:
        w.write(samtext.bam_header(targets, lens))
        w.flush()
        w.write(samtext.bam_format(reads, names, targets, fix_quality_orientation=True))
    got, last = [], None
    for batch in aligner.load_reads(path, read_part_length=256, max_reads=10_000):
        got += [(r.name, r.seq, r.qual) for r in batch.reads]
        last = batch
    norm = bytes.maketrans(b"acgtRYKMSWBDHVN", b"ACGTNNNNNNNNNNN")
    want = [(r.name, bytes(r.seq).translate(norm), r.qual) for r in reads]
    assert got == want
    assert last.device_members >= len(G.members(open(path, "rb").read()[:-28])) and last.host_bytes == 0


def _map_file(a, query, loaded, rpl):
    out = []
    for batch in a.load_reads(query, read_part_length=rpl, max_reads=500):
        a.cs_run(read_part_length=rpl)
        res = a.map_short_reads(read_part_length=rpl)
        out.append([samtext.Read(r.name, r.seq, r.qual, m[1], m[0], r.empty) for r, m in zip(batch.reads, res)])
    return out


@pytest.mark.parametrize("which,rpl", [("test_2", 256), ("synthetic", 257)])
def test_file_to_bam(tmp_path, which, rpl):
    src = str(tmp_path / "reads.fq")
    if which == "test_2":
        T._test2_short_fastq(src)
    else:
        T._short_reads_file(src)
    ref = T.shutil.copyfile(os.path.join(T.FIX, "ref_chr21_20kb.fa"), str(tmp_path / "ref.fa"))
    a = B200Aligner(0)
    try:
        loaded = a.load_reference(ref, skip_write=True)
        targets = list(dict.fromkeys(loaded.sam_ref_names()))
        lens = [int(x) for x in loaded.lens]
        path = str(tmp_path / "out.bam")
        text = b""
        with a.bgzf_writer(path, chunk_bytes=1 << 20) as w:
            w.write(samtext.bam_header(targets, lens))
            w.flush()
            for recs in _map_file(a, src, loaded, rpl):
                w.write(samtext.bam_format(recs, loaded.sam_ref_names(), targets, threads=2))
                text += samtext.sam_format(recs, loaded.sam_ref_names(), threads=1)
    finally:
        a.close()
    blob = open(path, "rb").read()
    data = b"".join(p for _, p in _check_members(blob))
    head = bw.header(samtext.sam_header(targets, lens))
    assert data[:len(head)] == head
    body = data[len(head):]
    assert len(text.split(b"\n")) > 2
    assert bw.split_records(body) == bw.split_records(bw.records(text, targets))
    if os.path.exists(T.PLAIN):
        plain = T._ngmlr_sam(str(tmp_path), src, str(tmp_path / "plain.sam"), rpl)
        assert bw.split_records(body) == bw.split_records(bw.records(b"\n".join(plain) + b"\n", targets))


def test_errors(aligner, tmp_path):
    with pytest.raises(RuntimeError, match="cannot open"):
        aligner.bgzf_writer(str(tmp_path / "missing" / "x.bam"))
    if os.path.exists("/dev/full"):
        w = aligner.bgzf_writer("/dev/full", chunk_bytes=1 << 20)
        with pytest.raises(RuntimeError, match="write failed"):
            w.write(bytes(3 << 20))
            w.flush()
        with pytest.raises(RuntimeError, match="write failed"):
            w.close()
    # the context still writes a good file
    blob, _ = _write(aligner, str(tmp_path / "ok.gz"), [b"abc" * 1000])
    assert b"".join(p for _, p in _check_members(blob)) == b"abc" * 1000


@pytest.mark.parametrize("chunk", [1 << 20, 16 << 20])
def test_device_memory_under_bound(aligner, tmp_path, chunk):
    import torch
    data = bytes(np.random.default_rng(6).integers(0, 4, 3 * chunk, dtype=np.uint8))
    free0, _ = torch.cuda.mem_get_info(0)
    with aligner.bgzf_writer(str(tmp_path / "m.gz"), chunk_bytes=chunk) as w:
        w.write(data)
        free1, _ = torch.cuda.mem_get_info(0)
        held = w.stats()["device_bytes"]
    assert 0 < held < 20 * chunk + (64 << 20), held
    assert free0 - free1 < 20 * chunk + (64 << 20) + (32 << 20), (free0 - free1)
