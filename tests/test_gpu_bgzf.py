"""BGZF inflated on the device (csrc/inflate.cu through the stream layer of csrc/stream.cpp):
  - byte stream: the device walker returns gzread's bytes, error and truncation flag on every fixture of bgzf_cases;
  - counters: on clean files every member was inflated on the device (no host continuation), on a file with a bad
    member the device stops exactly at that member;
  - records: BGZF copies of every read_loader_cases file load to the unmodified ReadProvider's records at the chunk
    sizes and max_reads / max_bases settings of test_gpu_read_loader; the resident set equals reads_upload's;
  - file to SAM: a BGZF query gives the plain ngmlr binary's SAM body (test_2's short reads, 2 000 synthetic reads);
  - reference: a BGZF reference (test_2's and a multi-contig synthetic of a few Mb over many members) installs the
    genome and index of its plain FASTA and writes the same caches, which the plain binary also writes from it;
  - memory: a handle reading BGZF stays below 11 x chunk_bytes of device memory."""
import ctypes as C
import os
import random
import shutil

import numpy as np
import pytest

import bgzf_cases as B
import read_loader_cases as R
import test_gpu_read_loader as T
from ngmlr_b200 import B200Aligner

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "ref_fixtures", "test_2")


@pytest.fixture(scope="module")
def aligner():
    a = B200Aligner(0)
    yield a
    a.close()


def _write(path, blob):
    with open(path, "wb") as f:
        f.write(blob)
    return str(path)


@pytest.mark.parametrize("size", [4096, 65535, 0])
def test_device_stream_equals_gzread(aligner, tmp_path, size):
    clean, edge = B.clean_files(), B.edge_files()
    for name, blob in [(k, v[0]) for k, v in clean.items()] + list(edge.items()):
        path = _write(tmp_path / (name + ".gz"), blob)
        rs = size or max(len(blob) * 8, 1)
        want = B.stream_read(aligner.lib, path, B.GZREAD, rs)
        got = B.stream_read(aligner.lib, path, B.DEVICE, rs, ctx=aligner.h)
        assert got[:3] == want[:3], (name, size, len(got[0]), len(want[0]), got[1:3], want[1:3])
        if name in clean:
            assert got[0] == clean[name][1], name
            assert got[3][1] == len(B.members(blob)) and got[3][2] == 0, (name, got[3])


def test_device_stops_at_the_bad_member(aligner, tmp_path):
    good = B.members(B.bgzf(B.sources()["fastq"], 6, eof=False))
    k = len(good) // 2
    for name, blob in B.edge_files().items():
        if not (name.startswith("reject_") or name in ("crc", "isize", "isize_over_64k", "bsize_long", "bsize_short",
                                                        "plain_gzip_after", "fname_middle")):
            continue
        got = B.stream_read(aligner.lib, _write(tmp_path / "f.gz", blob), B.DEVICE, 1 << 30, ctx=aligner.h)
        assert got[3][1] == k, (name, got[3])
        if name.startswith("reject_") or name in ("crc", "isize", "isize_over_64k"):
            assert got[1] == 1, name  # zlib reports the error
        else:
            assert got[1] == 0 and got[3][2] > 0, name  # zlib reads on from that member


def _bgzf_case(tmp_path, name, block=3000):
    return _write(tmp_path / (name + ".fq.gz"), B.bgzf(R.CASES[name], 6, block=block))


@T.need_full
def test_records_equal_reference_reader(aligner, tmp_path):
    checked = 0
    for name in R.CASES:
        path = _bgzf_case(tmp_path, name)
        oracle, odrop = R.oracle_reads(R.write_case(tmp_path / "o", name))
        want = R.as_loaded(oracle)
        longest = max([len(r[1]) * 2 + 300 for r in want] + [300])
        chunks = [0, 4096] if name in R.BIG else [0, 4096, max(16, longest // 4)]
        for chunk in chunks:
            for max_reads, max_bases in ((1, 0), (7, 0), (100_000, 0), (100_000, 150)):
                got, drop, sizes = T._load_all(aligner, path, chunk_bytes=chunk, max_reads=max_reads,
                                               max_bases=max_bases)
                where = f"{name} chunk={chunk} max_reads={max_reads} max_bases={max_bases}"
                assert got == want, where
                assert drop == odrop, where
                assert all(s <= max_reads for s in sizes), where
                checked += 1
    assert checked >= 20 * 3 * 4
    # the batches report the device inflate
    batches = list(aligner.load_reads(_bgzf_case(tmp_path, "fuzz_a")))
    assert batches[-1].device_members == len(B.members(open(str(tmp_path / "fuzz_a.fq.gz"), "rb").read()))
    assert batches[-1].host_bytes == 0 and batches[-1].compressed_bytes > 0


@T.need_full
def test_resident_set_equals_reads_upload(tmp_path):
    ref = shutil.copyfile(os.path.join(FIX, "ref_chr21_20kb.fa"), str(tmp_path / "ref.fa"))
    a, b = B200Aligner(0), B200Aligner(0)
    try:
        a.load_reference(ref, skip_write=True)
        b.load_reference(ref, skip_write=True)
        for name in ("fuzz_a", "fastq_multi", "crlf", "empty", "iupac"):
            path = _bgzf_case(tmp_path, name)
            want = T._oracle_strings(R.write_case(tmp_path, name), 256)
            k = 0
            for batch in a.load_reads(path, max_reads=64, chunk_bytes=8192):
                seqs = want[k:k + len(batch.reads)]
                k += len(batch.reads)
                assert [r.seq for r in batch.reads] == seqs
                assert batch.n_sub == b.reads_upload(seqs)
                for x, y in zip(a.resident_reads(), b.resident_reads()):
                    assert np.array_equal(x, y), name
            assert k == len(want)
    finally:
        a.close()
        b.close()


@T.need_plain
@pytest.mark.parametrize("which,rpl", [("test_2", 256), ("synthetic", 257)])
def test_file_to_sam_equals_plain_ngmlr(tmp_path, which, rpl):
    src = str(tmp_path / "reads.fq")
    if which == "test_2":
        T._test2_short_fastq(src)
    else:
        T._short_reads_file(src)
    query = _write(tmp_path / "reads.fq.gz", B.bgzf(open(src, "rb").read(), 6))
    want = T._ngmlr_sam(str(tmp_path), query, str(tmp_path / "plain.sam"), rpl)
    got = T._library_sam(tmp_path, query, rpl)
    assert len(want) >= 2
    assert got == want


def _synthetic_fasta(seed=8, contigs=12, size=300_000):
    rng = random.Random(seed)
    out = []
    for i in range(contigs):
        s = "".join(rng.choice("ACGTacgtN") if rng.random() < 0.01 else rng.choice("ACGT") for _ in range(size))
        out.append(f">chr{i} synthetic\n" + "\n".join(s[j:j + 60] for j in range(0, len(s), 60)) + "\n")
    return "".join(out).encode()


def _state(a):
    nb, cl = C.c_uint64(0), C.c_uint64(0)
    a.lib.ngmlr_b200_cs_get_reference.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                                  C.POINTER(C.c_uint64)]
    a._check(a.lib.ngmlr_b200_cs_get_reference(a.h, None, 0, C.byref(nb), C.byref(cl)))
    ref = np.zeros(nb.value, np.uint8)
    a._check(a.lib.ngmlr_b200_cs_get_reference(a.h, ref.ctypes.data_as(C.c_void_p), ref.size, None, None))
    idx = a.get_index()
    return ref, cl.value, idx


@pytest.mark.parametrize("which", ["test_2", "synthetic"])
def test_reference_from_bgzf_equals_plain(tmp_path, which):
    import test_gpu_load_reference as L
    text = open(os.path.join(FIX, "ref_chr21_20kb.fa"), "rb").read() if which == "test_2" else _synthetic_fasta()
    for d in ("plain", "bgzf", "theirs"):
        os.makedirs(tmp_path / d)
    plain = _write(tmp_path / "plain" / "r.fa", text)
    blob = B.bgzf(text, 6)
    packed = _write(tmp_path / "bgzf" / "r.fa.gz", blob)
    a = B200Aligner(0)
    try:
        want = a.load_reference(plain)
        s_want = _state(a)
        got = a.load_reference(packed)
        s_got = _state(a)
    finally:
        a.close()
    assert (got.names, got.starts, got.lens, got.concat_len) == (want.names, want.starts, want.lens, want.concat_len)
    assert np.array_equal(s_got[0], s_want[0]) and s_got[1] == s_want[1]
    for x, y in ((s_got[2].tab, s_want[2].tab), (s_got[2].rci, s_want[2].rci), (s_got[2].pos, s_want[2].pos)):
        assert np.array_equal(x, y)
    assert got.device_members == len(B.members(blob)) and got.host_bytes == 0 and got.compressed_bytes == len(blob)
    assert want.device_members == 0
    L._compare_caches(packed, plain, 13, 2)
    if os.path.exists(L.PLAIN):
        theirs = _write(tmp_path / "theirs" / "r.fa.gz", blob)
        L._ngmlr(theirs, L._query(tmp_path), str(tmp_path / "o.sam"))
        L._compare_caches(packed, theirs, 13, 2)


def test_device_memory_bound(aligner, tmp_path):
    text = b"".join(R.CASES[n] for n in R.BIG) * 60
    path = _write(tmp_path / "big.fq.gz", B.bgzf(text, 6))
    chunk = 1 << 20
    f = C.c_void_p()
    from ngmlr_b200 import _lib, samtext
    opts = _lib.ReadFileOptions(chunk)
    assert aligner.lib.ngmlr_b200_read_file_open(os.fsencode(path), C.byref(opts), C.byref(f)) == 0
    try:
        recs = (samtext.SamRead * 100_000)()
        n, nd = C.c_int32(0), C.c_int32(0)
        total = 0
        while True:
            assert aligner.lib.ngmlr_b200_reads_load(aligner.h, f, 100_000, 0, 256, recs, C.byref(n), C.byref(nd)) >= 0
            total += n.value
            if n.value == 0:
                break
        dev = C.c_int64(0)
        dm = C.c_int64(0)
        aligner.lib.ngmlr_b200_read_file_stats(f, None, None, None, None, None, C.byref(dev))
        aligner.lib.ngmlr_b200_read_file_inflate_stats(f, None, C.byref(dm), None, None)
    finally:
        aligner.lib.ngmlr_b200_read_file_close(f)
    assert total > 1000 and dm.value == len(B.members(open(path, "rb").read()))
    assert 0 < dev.value < 11 * chunk
