"""Plain gzip (one deflate stream per member) inflated on the device (csrc/gzip_inflate.cu through the stream layer
of csrc/stream.cpp), with zlib's gzread (mode 0 of the stream hook) as the oracle:
  - clean streams give gzread's bytes and flags at read sizes 4 KiB, 65 535, 3 MiB and the whole file, at 32 KiB
    (the default) and 4 KiB chunks given explicitly, which keep a stream on the device: every byte from the device;
  - path choice: without a chunk size, a stream read in rounds too small for the device, or whose first round
    inflates at a ratio where gzread is faster, goes to zlib whole; one inside both stays on the device; all give
    gzread's bytes;
  - a stored block hiding a valid dynamic header is a false block start: decoded again, same bytes;
  - refusals (every reject member at the start and after a clean member, a flipped byte deep in a member, CRC / ISIZE
    corruption, truncation, trailing bytes, a distance before the member's start) give gzread's bytes, -1 in the same
    call and the same truncation flag; at 4 KiB chunks each of those that holds a clean prefix has it served by the
    device and the rest by zlib;
  - pipes: a gzip file read through a FIFO stays with the gzread continuation (no member bytes are held for zlib to
    reread) and gives gzread's bytes, -1 and truncation flag, clean or refused;
  - loaders: the read loader's cases as gzip at small chunks give ReadProvider's records; a gzip reference installs
    the genome and index of its plain FASTA; the read loader's device memory stays under its stated bound."""
import ctypes as C
import gzip
import os

import numpy as np
import pytest

import bgzf_cases as B
import gzip_cases as G
import read_loader_cases as R
import test_gpu_read_loader as T
from ngmlr_b200 import B200Aligner

pytestmark = pytest.mark.gpu
MiB = 1 << 20
SIZES = [4096, 65535, 3 * MiB, 0]


@pytest.fixture(scope="module")
def aligner():
    a = B200Aligner(0)
    yield a
    a.close()


@pytest.fixture(scope="module")
def clean():
    return G.clean()


def _write(path, blob):
    with open(path, "wb") as f:
        f.write(blob)
    return str(path)


def _gzread(a, path, rs, cap):
    return B.stream_read(a.lib, path, B.GZREAD, rs, cap=cap)


@pytest.mark.parametrize("chunk", [32768, 4096])
def test_clean_streams_equal_gzread(aligner, tmp_path, clean, chunk):
    for name, (blob, data) in clean.items():
        path = _write(tmp_path / (name + ".gz"), blob)
        cap = len(data) + MiB
        for size in SIZES:
            rs = size or len(data) + 1
            want = _gzread(aligner, path, rs, cap)
            got = G.stream_read(aligner.lib, path, aligner.h, rs, chunk, cap)
            where = (name, chunk, size, len(got[0]), got[1:3], want[1:3], got[3], got[4])
            assert got[:3] == want[:3], where
            assert got[0] == data, where
            assert got[4][0] == len(data) and got[3][2] == 0, where
            if name == "false_start":
                assert got[4][2] > 0, where


def test_pacbio_shaped_fastq(aligner, tmp_path):
    blob, data = G.big_fastq()
    path = _write(tmp_path / "pb.fq.gz", blob)
    for size, chunk in ((65535, 32768), (3 * MiB, 32768), (4096, 8192), (0, 32768)):
        rs = size or len(data) + 1
        got = G.stream_read(aligner.lib, path, aligner.h, rs, chunk, len(data) + MiB)
        assert got[0] == data and got[1:3] == (0, 0), (size, chunk, got[3], got[4])
        assert got[4][0] == len(data) and got[3][2] == 0 and got[4][1] > 1, (size, chunk, got[4])


def test_path_follows_round_size_and_ratio(aligner, tmp_path):
    import random
    rng = random.Random(4)
    quals = b"".join(b"@r\n%s\n+\n%s\n" % (bytes(rng.choice(b"ACGT") for _ in range(2000)),
                                            bytes(rng.randrange(33, 75) for _ in range(2000))) for _ in range(2500))
    rnd = np.random.default_rng(3).bytes(300 * MiB)  # more than one round: the ratio decides after the first
    big = G.GZ_DEVICE_ROUND
    for name, data, level, size, device in (("fastq", quals, 6, big, True), ("fastq", quals, 6, 3 * MiB, False),
                                            ("random", rnd, 1, big, False)):
        blob = G.gz(data, level)
        ratio = len(data) / len(blob)
        assert (G.GZ_RATIO_LO <= ratio <= G.GZ_RATIO_HI) == (name == "fastq"), (name, ratio)
        path = _write(tmp_path / (name + ".gz"), blob)
        want = _gzread(aligner, path, size, len(data) + MiB)
        got = G.stream_read(aligner.lib, path, aligner.h, size, 0, len(data) + MiB)
        assert got[:3] == want[:3] and got[0] == data, (name, size)
        assert (got[4][0], got[3][2]) == ((len(data), 0) if device else (0, len(data))), (name, size, got[3], got[4])


def test_refusals_equal_gzread(aligner, tmp_path):
    for name, blob in G.refusals().items():
        path = _write(tmp_path / (name + ".gz"), blob)
        cap = 64 * MiB
        for size in SIZES:
            rs = size or len(blob) * 8 + 1
            want = _gzread(aligner, path, rs, cap)
            for chunk in (0, 4096):
                got = G.stream_read(aligner.lib, path, aligner.h, rs, chunk, cap)
                where = (name, size, chunk, len(got[0]), len(want[0]), got[1:3], want[1:3], got[3], got[4])
                assert got[:3] == want[:3], where
                if chunk and name != "trailing_garbage":  # zlib ignores bytes after a member that are no header
                    # zlib continued: it returned bytes, or reported the error or the truncation itself
                    assert got[3][2] > 0 or got[1] == 1 or got[2] == 1, where
                    if name in G.CLEAN_PREFIX or name.startswith("after_"):
                        assert got[4][0] > 0, where  # the clean prefix came from the device


def _through_fifo(tmp_path, path, fn):
    import threading
    fifo = str(tmp_path / "fifo")
    if os.path.exists(fifo):
        os.unlink(fifo)
    os.mkfifo(fifo)
    data = open(path, "rb").read()

    def feed():
        with open(fifo, "wb") as f:
            for i in range(0, len(data), 7000):
                f.write(data[i:i + 7000])
    t = threading.Thread(target=feed)
    t.start()
    try:
        return fn(fifo)
    finally:
        t.join()


def test_pipe_equals_gzread(aligner, tmp_path, clean):
    refused = G.refusals()
    cases = {"level6": clean["level6"][0], "two_members": clean["two_members"][0],
             "after_distance_too_far": refused["after_distance_too_far"], "trunc_mid_block": refused["trunc_mid_block"],
             "crc": refused["crc"]}
    for name, blob in cases.items():
        path = _write(tmp_path / (name + ".gz"), blob)
        for size in (4096, 65535):
            want = _gzread(aligner, path, size, 64 * MiB)
            for chunk in (0, 4096):
                got = _through_fifo(tmp_path, path,
                                    lambda p: G.stream_read(aligner.lib, p, aligner.h, size, chunk, 64 * MiB))
                where = (name, size, chunk, len(got[0]), len(want[0]), got[1:3], want[1:3], got[3], got[4])
                assert got[:3] == want[:3], where
                assert got[4][0] == 0 and got[3][2] == len(got[0]), where


@T.need_full
def test_read_loader_records_equal_reference_reader(aligner, tmp_path, monkeypatch):
    monkeypatch.setenv("NGMLR_B200_DEBUG_GZIP_CHUNK", "2048")
    checked = 0
    for name in R.CASES:
        path = _write(tmp_path / (name + ".fq.gz"), gzip.compress(R.CASES[name], 6))
        oracle, odrop = R.oracle_reads(R.write_case(tmp_path / "o", name))
        want = R.as_loaded(oracle)
        for chunk in ([0, 4096] if name in R.BIG else [0, 4096, 300]):
            got, drop, sizes = T._load_all(aligner, path, chunk_bytes=chunk, max_reads=7, max_bases=0)
            assert got == want and drop == odrop, (name, chunk)
            checked += 1
    assert checked >= 28 * 2
    batches = list(aligner.load_reads(path))
    assert batches[-1].gzip_bytes == len(R.CASES[name]) and batches[-1].host_bytes == 0


def test_read_loader_memory_bound(aligner, tmp_path, monkeypatch):
    from ngmlr_b200 import _lib, samtext
    monkeypatch.setenv("NGMLR_B200_DEBUG_GZIP_CHUNK", "32768")  # both files compress far beyond the device's window
    fq = G.fastq(30 * 10 ** 6)
    for name, text in (("fastq", fq), ("n", b">n\n" + b"N" * (200 * 10 ** 6) + b"\n")):
        path = _write(tmp_path / (name + ".gz"), gzip.compress(text, 6))
        chunk = 1 << 20
        f = C.c_void_p()
        opts = _lib.ReadFileOptions(chunk)
        assert aligner.lib.ngmlr_b200_read_file_open(os.fsencode(path), C.byref(opts), C.byref(f)) == 0
        try:
            recs = (samtext.SamRead * 100_000)()
            n, nd = C.c_int32(0), C.c_int32(0)
            while True:
                assert aligner.lib.ngmlr_b200_reads_load(aligner.h, f, 100_000, 0, 256, recs, C.byref(n),
                                                         C.byref(nd)) >= 0
                if n.value == 0:
                    break
            dev, cap, gb = C.c_int64(0), C.c_int64(0), C.c_int64(0)
            aligner.lib.ngmlr_b200_read_file_stats(f, None, None, None, None, None, C.byref(dev))
            aligner.lib.ngmlr_b200_debug_read_file_chunks(f, None, None, None, C.byref(cap))
            aligner.lib.ngmlr_b200_read_file_gzip_stats(f, C.byref(gb), None, None, None)
        finally:
            aligner.lib.ngmlr_b200_read_file_close(f)
        assert gb.value == len(text), name
        assert 0 < dev.value < 13 * max(cap.value, MiB) + 48 * MiB, (name, dev.value, cap.value)


@pytest.mark.parametrize("which", ["test_2", "synthetic", "n_run"])
def test_reference_from_gzip_equals_plain(tmp_path, which, monkeypatch):
    import test_gpu_bgzf as TB
    monkeypatch.setenv("NGMLR_B200_DEBUG_GZIP_CHUNK", "32768")  # the N run compresses beyond the device's window
    import test_gpu_load_reference as L
    if which == "test_2":
        text = open(os.path.join(TB.FIX, "ref_chr21_20kb.fa"), "rb").read()
    elif which == "synthetic":
        text = TB._synthetic_fasta()
    else:
        text = TB._synthetic_fasta(contigs=2, size=200_000) + b">gap\n" + b"N" * 5_000_000 + b"\nACGT" * 3000 + b"\n"
    for d in ("plain", "gz"):
        os.makedirs(tmp_path / d)
    plain = _write(tmp_path / "plain" / "r.fa", text)
    packed = _write(tmp_path / "gz" / "r.fa.gz", gzip.compress(text, 6))
    a = B200Aligner(0)
    try:
        want = a.load_reference(plain)
        s_want = TB._state(a)
        got = a.load_reference(packed)
        s_got = TB._state(a)
    finally:
        a.close()
    assert (got.names, got.starts, got.lens, got.concat_len) == (want.names, want.starts, want.lens, want.concat_len)
    assert np.array_equal(s_got[0], s_want[0]) and s_got[1] == s_want[1]
    for x, y in ((s_got[2].tab, s_want[2].tab), (s_got[2].rci, s_want[2].rci), (s_got[2].pos, s_want[2].pos)):
        assert np.array_equal(x, y)
    assert got.gzip_bytes == len(text) and got.host_bytes == 0 and got.gzip_chunks > 0
    L._compare_caches(packed, plain, 13, 2)
