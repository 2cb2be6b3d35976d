"""The device at ngmlr's non-default options (cs_cases.OPTION_SETS), against the C restatement that
test_cs_options.py pins to the reference at the same options:
  - the k-mer index built on the device (k 10..15, --kmer-skip 0..3, --bin-size 0..6);
  - the candidate search (ties at -s 1 and 0, min_kmer_hits, vote tables in the arena);
  - the sub-read scorer in gather mode on the branches the defaults never take: odd window starts, sw_ungapped<5>
    (sub-reads of 257-320 bases), the gapped path with one and with several passes (windows of more than 384
    columns, queries of more than 288 characters);
  - the resident pipeline (reads_upload -> cs_run -> cs_fetch) with sub-reads of --subread-length bases;
  - compute_alignments with anchors of read_part_length 128 and 512;
  - ngmlr's short-read path and the cache files through the plain ngmlr binary at non-default options.
Each test asserts that its data reach the branches its option set is there for."""
import os

import numpy as np
import pytest

import cs_cases
from ngmlr_b200 import B200Aligner, refindex, samtext, synth
from oracle_lib import CsOracle, same_alignment

pytestmark = pytest.mark.gpu

CS_SMEM_CAP = 512        # csrc/kernels.h: vote tables up to this many entries live in shared memory
SW_COLS = 384            # widest window of the ungapped scorer
SW_PASS_ROWS = 288       # query characters per pass of the gapped scorer (32 lanes x 9 rows)
K15_MEMORY = 32 << 30    # host memory a 15-mer index needs here: the oracle's copy, the fetched copy, their arrays


def _mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def _contigs():
    return cs_cases.genome_contigs() + cs_cases.repeat_contigs()


def _hits(sub, idx, k):
    """Index positions the search visits for a sub-read (both strands of every N-free k-mer), ignoring the one
    window the reference may drop at the end: a lower bound of the count that sizes the vote table."""
    code = {ord("A"): 0, ord("C"): 1, ord("T"): 2, ord("G"): 3}
    s = np.frombuffer(sub, dtype=np.uint8)
    total = 0
    for p in range(len(s) - k):
        w = s[p:p + k]
        if (w == ord("N")).any():
            continue
        f = 0
        for c in w:
            f = (f << 2) | code[int(c)]
        r = 0
        for c in w[::-1]:
            r = (r << 2) | (code[int(c)] ^ 2)
        for x in (f, r):
            if idx.rci[x] != 0:
                total += int(idx.tab[x + 1]) - int(idx.tab[x])
    return total


def _window(orc, o, loc):
    n = cs_cases.ref_max_len(o)
    pos = (loc - (o["corridor"] >> 1)) % (1 << 64)
    return pos, orc.decode(pos, n) or b"N" * n


@pytest.mark.parametrize("set_name", list(cs_cases.OPTION_SETS))
def test_device_equals_oracle_at_options(set_name, oracle):
    o = cs_cases.OPTION_SETS[set_name]
    if o["k"] == 15 and _mem_available() < K15_MEMORY:
        pytest.skip("a 15-mer index needs ~32 GB of free host memory for the comparison")
    contigs = _contigs()
    orc = CsOracle([c.tobytes() for c in contigs], k=o["k"], skip=o["skip"], bin_shift=o["bin"])
    enc = refindex.encode_reference(contigs)
    a = B200Aligner(0)
    try:
        a.set_reference(enc)
        # ---- the index ----
        idx = a.build_index(enc, o["k"], o["skip"], o["bin"], fetch=True)
        tab, rci, pos = orc.index()
        assert tab.size == 4 ** o["k"] + 1
        assert np.array_equal(idx.tab, tab) and np.array_equal(idx.rci, rci) and np.array_equal(idx.pos, pos)
        del tab, rci, pos
        # ---- the search ----
        seed = 100 + ord(set_name)
        subs = cs_cases.option_subreads(contigs, o, seed)
        n_direct = len(subs) - sum(len(cs_cases.split_read(r, o["rpl"]))
                                   for r in cs_cases.option_reads(contigs, o["rpl"], 60, seed + 1))
        want = [orc.search(s, o["s"], o["min_hits"]) for s in subs]
        got, mx = a.cs_search(subs, o["s"], o["min_hits"])
        for i, s in enumerate(subs):
            assert got[i] == want[i][0], (i, len(s))
            assert mx[i] == np.float32(want[i][1]), i
        n_cand = sum(len(w[0]) for w in want)
        assert n_cand > 100, n_cand
        # ---- search + sub-read scores ----
        scored, mx2 = a.cs_score(subs, o["s"], o["min_hits"], o["corridor"], o["rpl"])
        assert np.array_equal(mx2, mx)
        reach = dict(gapped=0, multi_pass=0, ungapped5=0, odd_start=0, arena=0)
        for i, s in enumerate(subs):
            assert [g[:3] for g in scored[i]] == want[i][0], i
            for (_cs, loc, rev, sw) in scored[i]:
                start, window = _window(orc, o, loc)
                q = synth.revcomp_upper(np.frombuffer(s, dtype=np.uint8)).tobytes() if rev else s
                assert sw == oracle.ssw_score(window, q), (i, loc, rev)
                gapped = len(q) > 320 or len(window) > SW_COLS
                reach["gapped"] += gapped
                reach["multi_pass"] += gapped and len(q) + 1 > SW_PASS_ROWS
                reach["ungapped5"] += not gapped and len(q) > 256
                reach["odd_start"] += start % 2 == 1 and start < orc.concat_len
        if set_name == "A":
            reach["arena"] = sum(1 for s in subs if 2 * _hits(s, idx, o["k"]) + 2 > CS_SMEM_CAP)
        # ---- the resident pipeline on whole reads: sub-reads of rpl bases ----
        reads = cs_cases.option_reads(contigs, o["rpl"], 60, seed + 1)
        assert a.reads_upload(reads, o["rpl"]) == len(subs) - n_direct
        m, _ms = a.cs_run(o["s"], o["min_hits"], o["corridor"], o["rpl"])
        start, sc, lo, rv, sw, mx3 = a.cs_fetch()
        assert m == start[-1]
        for j, w in enumerate(scored[n_direct:]):
            assert [(sc[x], int(lo[x]), int(rv[x]), sw[x]) for x in range(start[j], start[j + 1])] == w, j
        assert np.array_equal(mx3, mx[n_direct:])
    finally:
        a.close()
        orc.close()
    # each set reaches what it is there for
    need = dict(A=["arena"], B=["odd_start"], C=["ungapped5"], E=["gapped", "multi_pass"]).get(set_name, [])
    for key in need:
        assert reach[key] > 10, (set_name, reach)
    if set_name == "E":
        assert reach["gapped"] > reach["multi_pass"] > 0   # single-pass gapped pairs too (windows > 384, short queries)
    if o["s"] == 1.0:
        assert all(c[0] == w[1] for w in want for c in w[0])   # ties: every candidate reaches the maximum


@pytest.mark.parametrize("rpl", [128, 512])
def test_compute_alignments_read_part_length(rpl, oracle):
    """ngmlr_b200_compute_alignments with anchors of rpl bases (the anchor rows of getCorridorEndpointsWithAnchors)
    == the Python mirror over the CPU oracle, which test_cs_options.py pins to the reference at the same rpl."""
    from ngmlr_b200.intervals import compute_alignments
    from test_cs_oracle import _OracleBackend, _interval_tasks
    contigs = cs_cases.genome_contigs()
    orc = CsOracle([c.tobytes() for c in contigs])
    enc = refindex.encode_reference(contigs)
    tasks = _interval_tasks(contigs, enc, rpl)
    a = B200Aligner(0)
    try:
        a.set_reference(enc)
        got, calls = a.compute_alignments(tasks, rpl)
        got = list(got)
    finally:
        a.close()
    want, want_calls = compute_alignments(_OracleBackend(orc, oracle), _interval_tasks(contigs, enc, rpl))
    orc.close()
    assert list(calls) == want_calls
    n_valid = n_rev = 0
    for t, w, g in zip(tasks, want, got):
        assert (w is None) == (g.ret < 0)
        if w is None:
            continue
        n_valid += 1
        n_rev += any(x[2] for x in t.anchors) and not t.realign
        assert same_alignment(w, dict(g.as_dict(), nm_positions=w["nm_positions"])) == []
    assert n_valid >= 24 and n_rev >= 5, (n_valid, n_rev)


# ---- through ngmlr itself -------------------------------------------------------------------------------------------
from test_gpu_short_reads import PLAIN, _contigs as _sr_contigs, _reads as _sr_reads, _write as _sr_write  # noqa: E402

need_plain = pytest.mark.skipif(not os.path.exists(PLAIN), reason="oracle/_ref/ngmlr not built")

SHORT_READ_SETS = {
    "B": cs_cases.OPTION_SETS["B"],
    "G": dict(k=12, skip=2, bin=3, s=0.7, min_hits=0, rpl=200, corridor=60),
}


def _plain_records(ref, fq, tmp, o):
    import subprocess
    sam = os.path.join(tmp, "plain.sam")
    r = subprocess.run([PLAIN, "-r", ref, "-q", fq, "-o", sam, "-t", "1", "--skip-write", "--no-progress",
                        "-k", str(o["k"]), "--kmer-skip", str(o["skip"]), "--bin-size", str(o["bin"]),
                        "-s", str(o["s"]), "--subread-length", str(o["rpl"]), "--subread-corridor", str(o["corridor"])],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    recs = {}
    for line in open(sam, "rb"):
        if not line.startswith(b"@"):
            recs.setdefault(line.split(b"\t", 1)[0], []).append(line)
    return recs


@need_plain
@pytest.mark.parametrize("set_name", list(SHORT_READ_SETS))
def test_short_reads_at_options_identical_to_plain_binary(set_name, tmp_path):
    o = SHORT_READ_SETS[set_name]
    contigs, seg, rng = _sr_contigs(31)
    reads = _sr_reads(contigs, seg, rng, n=1200)
    reads[:6] = [r[:L] for r, L in zip(reads[:6], (o["rpl"] - 1, o["rpl"], o["rpl"] + 1) * 2)]
    ref, fq, quals = _sr_write(str(tmp_path), contigs, reads)
    names = [f"r{i}".encode() for i in range(len(reads))]
    want = _plain_records(ref, fq, str(tmp_path), o)
    a = B200Aligner(0)
    try:
        enc = a.encode_reference([c.tobytes() for c in contigs], fetch=False)
        a.build_index(enc, o["k"], o["skip"], o["bin"])
        a.reads_upload(reads, o["rpl"])
        # ngmlr declares -s but never reads it (ArgParser.cpp assigns every other option, not sensitivity): the binary
        # searches at its default 0.8 whatever -s says, so the library does too here
        a.cs_run(0.8, 0.0, o["corridor"], o["rpl"])
        res = a.map_short_reads(o["rpl"], 0.25)
    finally:
        a.close()
    ref_names = [b"chr1", b"chr1", b"chr2", b"chr2"]
    n_mapped = n_long = 0
    for i, r in enumerate(reads):
        if len(r) > o["rpl"]:
            assert res[i] is None, f"read {i} ({len(r)} bp) must be reported as not handled"
            n_long += 1
            continue
        mapped, al = res[i]
        text = samtext.sam_format([samtext.Read(names[i], r, quals[i], al, mapped)], ref_names, threads=1)
        w = want.get(names[i], [])
        assert text.splitlines(keepends=True) == w, f"read {i} ({len(r)} bp) differs:\nngmlr: {w}\nlib  : {text}"
        n_mapped += bool(w) and not int(w[0].split(b"\t")[1]) & 4
    assert n_mapped > 200 and n_long > 50, (n_mapped, n_long)


@need_plain
def test_caches_at_bin_size_6_k14_skip3(tmp_path):
    """load_reference(bin_shift=6, k=14, kmer_skip=3) writes the cache files `ngmlr --bin-size 6 -k 14 --kmer-skip 3`
    writes. The bin size enters the index (its repeat filter compares bins) but not the file name, here as in ngmlr:
    <fasta>-ht-14-3.2.ngm."""
    from test_gpu_load_reference import FIX, _compare_caches, _copy, _ngmlr, _query
    src = os.path.join(FIX, "test_2", "ref_chr21_20kb.fa")
    ours, theirs = _copy(src, str(tmp_path / "ours"), "r.fa"), _copy(src, str(tmp_path / "theirs"), "r.fa")
    a = B200Aligner(0)
    try:
        got = a.load_reference(ours, k=14, kmer_skip=3, bin_shift=6)
    finally:
        a.close()
    assert got.index_written and got.reference_written
    _ngmlr(theirs, _query(tmp_path), str(tmp_path / "o.sam"), "--bin-size", "6", "-k", "14", "--kmer-skip", "3")
    _compare_caches(ours, theirs, 14, 3)
