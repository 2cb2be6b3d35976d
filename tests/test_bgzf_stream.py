"""The BGZF stream layer on the CPU (csrc/stream.cpp without a device binding):
  - the fixtures of bgzf_cases are valid gzip, and together they reach stored, fixed and dynamic blocks, a 15-bit
    code, length 258, distance 32 768, distance-1 runs (Z_RLE), Z_HUFFMAN_ONLY and several blocks in one member;
  - the walker (members inflated with zlib's raw inflate on the host, the gzread continuation from the first member it
    cannot vouch for) returns gzread's byte stream, error and truncation flag at read sizes 1, 4 KiB, 65 535 and the
    whole file, on every clean, reject and edge file, and from a pipe;
  - the unmodified ReadProvider reads BGZF copies of the read loader's cases to the records of the plain files."""
import os
import threading
import zlib

import pytest

import bgzf_cases as B
import read_loader_cases as R
from ngmlr_b200 import _lib

SIZES = [1, 4096, 65535, 0]  # 0: the whole file in one call


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("bgzf")
    out = {}
    for name, (blob, _) in B.clean_files().items():
        out[name] = str(d / (name + ".gz"))
        open(out[name], "wb").write(blob)
    for name, blob in B.edge_files().items():
        out[name] = str(d / (name + ".gz"))
        open(out[name], "wb").write(blob)
    return out


def test_python_gzip_reads_every_fixture():
    import gzip
    for name, (blob, src) in B.clean_files().items():
        assert gzip.decompress(blob) == src, name
    for name, m in B.reject_members().items():
        with pytest.raises(zlib.error):
            zlib.decompress(m, 31)


def test_fixtures_reach_every_part_of_deflate():
    info = {}
    for name, (blob, src) in B.clean_files().items():
        got = b""
        for _, m in B.members(blob):
            out, i = B.inspect(B.member_deflate(m))
            got += out
            info.setdefault(name, []).append(i)
        assert got == src, name
    allm = [i for v in info.values() for i in v]
    assert {t for i in allm for t in i["types"]} == {0, 1, 2}
    assert max(i["max_code"] for i in allm) == 15
    assert max(i["max_len"] for i in allm) == 258
    assert max(i["max_dist"] for i in allm) == 32768
    assert all(i["max_dist"] <= 1 for i in info["runs_rle"]) and sum(i["dist1"] for i in info["runs_rle"]) > 100
    assert all(i["max_len"] == 0 for i in info["fib_huffman"]) and max(i["max_code"] for i in info["fib_huffman"]) == 15
    for name in ("fastq_full_flush", "fastq_sync_flush"):
        assert max(len(i["types"]) for i in info[name]) > 4, name
    assert all(set(i["types"]) == {1} for i in info["fastq_fixed"])


def _size(path, s):
    return s or max(os.path.getsize(path) * 8, 1)


@pytest.mark.parametrize("size", SIZES)
def test_walker_without_device_equals_gzread(files, size):
    lib = _lib.load()
    clean = B.clean_files()
    for name, path in files.items():
        rs = _size(path, size)
        want = B.stream_read(lib, path, B.GZREAD, rs)
        got = B.stream_read(lib, path, B.HOST, rs)
        assert got[:3] == want[:3], (name, size, len(got[0]), len(want[0]), got[1:3], want[1:3])
        if name in clean:
            assert got[0] == clean[name][1] and got[3][2] == 0, name  # every member vouched: no host continuation
    # where the walker hands over: everything after the plain gzip member, and after the FNAME member
    for name in ("plain_gzip_after", "fname_middle", "bsize_long"):
        assert B.stream_read(lib, files[name], B.HOST, 65536)[3][2] > 0, name
    # a file that is not BGZF: the host continuation returns every byte, and every byte of the file is read
    text = files["plain_text"]
    got = B.stream_read(lib, text, B.HOST, _size(text, size))
    assert got[3] == (os.path.getsize(text), 0, len(got[0])) and len(got[0]) == os.path.getsize(text), got[3]


def _through_pipe(tmp_path, path, mode, size):
    fifo = str(tmp_path / "pipe")
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
        return B.stream_read(_lib.load(), fifo, mode, size, cap=max(len(data) * 8, 1 << 20))
    finally:
        t.join()


@pytest.mark.parametrize("name", ["fastq_l6", "reject_distance_too_far", "plain_gzip_after", "fhcrc_first",
                                  "plain_text", "garbage_text", "truncated_mid_member", "empty"])
def test_walker_reads_a_pipe_as_gzread_reads_the_file(files, tmp_path, name):
    lib = _lib.load()
    for size in (4096, 65535):
        want = B.stream_read(lib, files[name], B.GZREAD, size)
        got = _through_pipe(tmp_path, files[name], B.HOST, size)
        assert got[:3] == want[:3], (name, size, len(got[0]), len(want[0]), got[1:3], want[1:3])


@pytest.mark.skipif(not os.path.exists(R.FULL), reason="oracle/_ref/libngmlr_reads.so not built")
def test_read_provider_reads_bgzf_copies_as_plain_files(tmp_path):
    for name in R.CASES:
        plain = R.write_case(tmp_path / "plain", name)
        path = str(tmp_path / (name + ".fq.gz"))
        open(path, "wb").write(B.bgzf(R.CASES[name], 6, block=5000))
        assert R.oracle_reads(path, tmp=str(tmp_path / "o")) == R.oracle_reads(plain), name
