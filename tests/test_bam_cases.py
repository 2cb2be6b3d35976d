"""The BAM fixtures of tests/bam_cases.py, without a GPU:
  - the writer's output is valid: gzip reads its BGZF and gzip forms back, members are split where asked, and an
    independent struct-based reader recovers every field of every record;
  - ngmlr's ReadProvider (read_loader_cases.oracle_reads) reads each case's `samtools fastq -n` text, and its reads
    are those the BAM rules give (name cut, ACGT / N, reverse complement, qualities), so each case's expectation comes
    from the unmodified reader;
  - every malformed stream differs from a valid one where its error says."""
import gzip
import os
import struct

import pytest

import bam_cases as B
import bgzf_cases
import read_loader_cases as R

need_full = pytest.mark.skipif(not os.path.exists(R.FULL), reason="oracle/_ref/libngmlr_reads.so not built")


def read_bam(data):
    """(text, refs, [Rec]) of an uncompressed BAM stream, field by field."""
    assert data[:4] == b"BAM\1"
    p = 4
    (l_text,) = struct.unpack_from("<i", data, p)
    text = data[p + 4:p + 4 + l_text]
    p += 4 + l_text
    (n_ref,) = struct.unpack_from("<i", data, p)
    p += 4
    refs = []
    for _ in range(n_ref):
        (ln,) = struct.unpack_from("<i", data, p)
        refs.append((data[p + 4:p + 4 + ln - 1], struct.unpack_from("<i", data, p + 4 + ln)[0]))
        p += 8 + ln
    recs = []
    while p < len(data):
        bs, ref_id, pos, l_name, mapq, _bin, n_cig, flag, l_seq, nref, npos, tlen = \
            struct.unpack_from("<iiiBBHHHiiii", data, p)
        q = p + 36
        name = data[q:q + l_name]
        assert name.endswith(b"\0")
        q += l_name
        cigar = [(v >> 4, v & 15) for v in struct.unpack_from("<%dI" % n_cig, data, q)]
        q += 4 * n_cig
        packed = data[q:q + (l_seq + 1) // 2]
        seq = "".join(B.NT16[b >> 4] + B.NT16[b & 15] for b in packed)[:l_seq]
        q += (l_seq + 1) // 2
        qual = list(data[q:q + l_seq])
        q += l_seq
        aux = data[q:p + 4 + bs]
        recs.append(B.Rec(name[:-1], seq, None if l_seq and qual[0] == 0xff else qual, flag, ref_id, pos, mapq, cigar,
                          aux, nref, npos, tlen))
        p += 4 + bs
    assert p == len(data)
    return text, refs, recs


@pytest.mark.parametrize("name", list(B.CASES))
def test_writer_round_trip(tmp_path, name):
    hdr, recs = B.CASES[name]
    stream = B.case_stream(name)
    for mode in ("bgzf", "gzip", "plain"):
        path = B.write_case(tmp_path, name, mode, block=4096 if mode == "bgzf" else bgzf_cases.BLOCK)
        raw = open(path, "rb").read()
        assert (gzip.decompress(raw) if mode != "plain" else raw) == stream
        if mode == "bgzf":
            ms = bgzf_cases.members(raw)
            assert len(ms) == (len(stream) + 4095) // 4096 + 1  # and the EOF marker
    text, refs, got = read_bam(stream)
    assert B.header(text, refs) == hdr
    assert got == recs


def test_cases_reach_what_they_name():
    names = [r.name for r in B.CASES["names"][1]]
    assert {1, 249, 250, 254} <= {len(n) for n in names} and b"sp ace" in names and b"t\tab" in names
    assert set("".join(r.seq for r in B.CASES["codes"][1])) == set(B.NT16)
    assert {q for r in B.CASES["phred"][1] for q in r.qual} == {0, 93}
    assert len(B.CASES["big_header"][0]) > 1 << 20
    assert max(len(r.seq) for r in B.CASES["long_read"][1]) == 300_000
    assert len(B.CASES["many_short"][1]) == 100_000
    flags = {r.flag for r in B.CASES["secondary"][1]}
    assert flags & {0x100, 0x110} and flags & {0x800, 0x810} and flags & {0, 0x10}
    assert any(len(r.seq) % 2 for r in B.CASES["odd"][1])
    assert any(not r.seq for r in B.CASES["empty"][1])
    al = B.CASES["aligned"][1]
    assert any(r.flag & 0x10 and r.qual is None for r in al) and any(r.flag & 0x10 and r.qual for r in al)
    aux = B.CASES["pacbio"][1][0].aux
    for tag in (b"XAA", b"Xcc", b"XCC", b"Xss", b"XSS", b"Xii", b"XII", b"Xff", b"XZZ", b"XHH", b"BcB", b"BfB"):
        assert tag in aux


def expected_reads(recs):
    """The BAM rules of ngmlr_b200_reads_load, restated: (name, bases, qualities, length, empty)."""
    out = []
    norm = bytes(c if c in b"ACGT" else ord("N") for c in range(256))
    for r in recs:
        if r.flag & B.SKIP:
            continue
        seq, qual = B.stored_to_read(r)
        name = r.name
        for i, c in enumerate(name):
            if c == 32 or 9 <= c <= 13:
                name = name[:i]
                break
        name = name[:249]
        if not seq:
            out.append((name, b"", b"*", 0, 1))
        else:
            q = b"*" if qual is None else bytes(x + 33 for x in qual)
            out.append((name, seq.encode().translate(norm), q, len(seq), 0))
    return out


@need_full
@pytest.mark.parametrize("name", list(B.CASES))
def test_reference_reader_reads_the_equivalent_text(tmp_path, name):
    oracle, dropped = R.oracle_reads(B.write_text(tmp_path, name))
    assert not dropped
    assert R.as_loaded(oracle) == expected_reads(B.CASES[name][1])


@pytest.mark.parametrize("err", list(B.ERRORS))
def test_error_streams(err):
    data, at, _msg = B.ERRORS[err]
    if err.startswith("header"):
        with pytest.raises(Exception):
            read_bam(data)
        return
    # everything before the named offset is a valid BAM stream
    text, refs, recs = read_bam(data[:at])
    assert len(recs) == 3 and refs == [(b"chr1", 1000)]
    assert len(data) > at
