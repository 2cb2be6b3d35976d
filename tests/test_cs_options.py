"""CPU tests of the candidate-search row at ngmlr's non-default options (cs_cases.OPTION_SETS): the unmodified
reference (oracle/_ref/libngmlr_full.so), initialised at each option set, against the C restatement
(oracle/cs_oracle.c) and the numpy index builder (ngmlr_b200/refindex.py). This pins the restatement at the options
before the device tests (test_gpu_options.py) compare the library with it.

The reference keeps options in function-local statics and singletons that are set on first use (GetBin /
ResolveBin's bin size, CollectResultsStd's minimum k-mer hits, ScoreBuffer's sub-read length, SequenceProvider), so
every option set runs in a process of its own."""
import ctypes as C
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import cs_cases
from oracle_lib import CsOracle, CsReference


def _has_init_opts():
    return hasattr(C.CDLL(CsReference.PATH), "ref_cs_init_opts")


# build() rebuilds the library where the reference sources are present; without them an older _ref/ may remain
pytestmark = [pytest.mark.skipif(not CsReference.available(), reason="oracle/_ref/libngmlr_full.so not built"),
              pytest.mark.skipif(CsReference.available() and not _has_init_opts(),
                                 reason="oracle/_ref/libngmlr_full.so predates ref_cs_init_opts")]

TESTS = os.path.dirname(os.path.abspath(__file__))
GENOMES = {"mixed": cs_cases.genome_contigs, "repeats": cs_cases.repeat_contigs}
RUNS = [(s, g) for s in cs_cases.OPTION_SETS if s != "F" for g in GENOMES] + [("F", "mixed")]
ALIGN_RPL = {"B": 128, "E": 512}   # sets whose sub-read length differs from 256: computeAlignment's anchor rows


def _decode_positions(o, cands, concat_len):
    """Sub-read windows (ScoreBuffer: DecodeRefSequence(loc - corridor / 2, refMaxLen)) of the candidates, plus
    windows around contig ends and at both parities."""
    half = o["corridor"] >> 1
    pos = {(loc - half) % (1 << 64) for c in cands for (_s, loc, _r) in c}
    pos |= {1, 2, 999, 1000, 1001, 5555, 5556, concat_len - 300, concat_len - 301, concat_len - 1, concat_len}
    return sorted(pos)


def _reference_worker(set_name, genome, out):
    """Runs in a subprocess: the reference at one option set on one genome -> pickle at `out`."""
    from ngmlr_b200 import refindex
    o = cs_cases.OPTION_SETS[set_name]
    contigs = GENOMES[genome]()
    fasta = out + ".fa"
    with open(fasta, "w") as f:
        for i, c in enumerate(contigs):
            f.write(f">c{i}\n{c.tobytes().decode()}\n")
    ref = CsReference(fasta, options=o)
    tab, rci, pos = ref.index()
    used = np.flatnonzero((tab != 0) | (rci != 0))   # every other entry is zero in both arrays
    res = dict(concat_len=ref.concat_len, ref_starts=ref.ref_starts(), n_index=int(tab.size), used=used,
               tab_used=tab[used], rci_used=rci[used], pos=pos)
    del tab, rci
    subs = cs_cases.option_subreads(contigs, o, seed=100 + ord(set_name))
    res["search16"] = [ref.search(s, table_bits=16) for s in subs]
    res["search8"] = [ref.search(s, table_bits=8) for s in subs]
    positions = _decode_positions(o, [c for c, _ in res["search16"]], ref.concat_len)
    res["decode"] = [(p, ref.decode(p, cs_cases.ref_max_len(o))) for p in positions]
    if set_name in ALIGN_RPL and genome == "mixed":
        enc = refindex.encode_reference(contigs)
        from test_cs_oracle import _interval_tasks
        res["align"] = [_ref_compute_alignment(ref.lib, t) for t in _interval_tasks(contigs, enc, ALIGN_RPL[set_name])]
    with open(out, "wb") as f:
        pickle.dump(res, f)


def _ref_compute_alignment(lib, t):
    """AlignmentBuffer::computeAlignment of the reference on one IntervalTask -> None or the record's fields."""
    n = len(t.anchors)
    a0 = (C.c_int * max(n, 1))(*[a[0] for a in t.anchors])
    a1 = (C.c_ulonglong * max(n, 1))(*[a[1] for a in t.anchors])
    a2 = (C.c_int * max(n, 1))(*[a[2] for a in t.anchors])
    ints = (C.c_int * 12)()
    fl = (C.c_float * 2)()
    cap = 8 * len(t.read_seq) + 64
    cig, md = C.create_string_buffer(cap), C.create_string_buffer(cap)
    ok = lib.ref_compute_alignment(C.c_ulonglong(t.on_ref_start), C.c_ulonglong(t.on_ref_stop), n, a0, a1, a2,
                                   t.corridor, t.read_seq, t.ext_qstart, t.ext_qend, t.full_read_length,
                                   int(t.realign), int(t.full_alignment), int(t.short_read), ints, fl,
                                   cig, cap, md, cap, None, 0)
    if not ok:
        return None
    return dict(cigar=cig.value.decode(), md=md.value.decode(), qstart=ints[1], qend=ints[2], nm=ints[3],
                alignment_length=ints[4], cigar_op_count=ints[5], position_offset=ints[11],
                score_bits=int(np.float32(fl[0]).view(np.uint32)), identity_bits=int(np.float32(fl[1]).view(np.uint32)))


def _start(set_name, genome, tmp):
    out = os.path.join(tmp, f"{set_name}-{genome}.pkl")
    code = ("import sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]; "
            "import test_cs_options as t; t._reference_worker(*sys.argv[3:])")
    p = subprocess.Popen([sys.executable, "-c", code, TESTS, os.path.dirname(TESTS), set_name, genome, out],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return p, out


def _finish(p, out):
    text, _ = p.communicate(timeout=900)
    assert p.returncode == 0, text[-3000:]
    with open(out, "rb") as f:
        return pickle.load(f)


@pytest.fixture(scope="module")
def reference_runs(tmp_path_factory):
    """The reference's results at every option set, computed in parallel processes. Set F (a 15-mer index needs
    ~5.4 GB per builder) runs only where the host has the memory for it."""
    tmp = str(tmp_path_factory.mktemp("cs_options"))
    procs = {(s, g): _start(s, g, tmp) for s, g in RUNS if s != "F" or _mem_available() >= K15_MEMORY}
    return {key: _finish(*v) for key, v in procs.items()}


def _check_index(res, tab, rci, pos):
    assert tab.size == res["n_index"] and rci.size == res["n_index"]
    used = np.flatnonzero((tab != 0) | (rci != 0))
    assert np.array_equal(used, res["used"])
    assert np.array_equal(tab[used], res["tab_used"]) and np.array_equal(rci[used], res["rci_used"])
    assert np.array_equal(pos, res["pos"])


def _compare(set_name, genome, res, numpy_builder=True):
    from ngmlr_b200 import refindex
    o = cs_cases.OPTION_SETS[set_name]
    contigs = GENOMES[genome]()
    orc = CsOracle([c.tobytes() for c in contigs], k=o["k"], skip=o["skip"], bin_shift=o["bin"])
    try:
        assert orc.concat_len == res["concat_len"] and orc.ref_starts() == res["ref_starts"]
        tab, rci, pos = orc.index()
        _check_index(res, tab, rci, pos)
        assert pos.size > 1000
        del tab, rci
        if numpy_builder:
            idx = refindex.build_index(refindex.encode_reference(contigs), o["k"], o["skip"], o["bin"], 1000)
            _check_index(res, idx.tab, idx.rci, idx.pos)
        subs = cs_cases.option_subreads(contigs, o, seed=100 + ord(set_name))
        n_cand = n_ties = 0
        for i, s in enumerate(subs):
            want = orc.search(s, o["s"], o["min_hits"])
            assert res["search16"][i] == want, (i, len(s))
            assert res["search8"][i] == want, (i, len(s))    # overflow -> retry with a larger table
            n_cand += len(want[0])
            n_ties += sum(1 for c in want[0] if c[0] == want[1])
        assert n_cand > 100, n_cand
        if o["s"] == 1.0:
            assert n_ties == n_cand   # at s = 1 only the bins that reach the maximum are listed
        win = cs_cases.ref_max_len(o)
        n_odd = 0
        for p, text in res["decode"]:
            assert orc.decode(p, win) == text, p
            n_odd += p % 2 == 1 and text is not None
        if o["bin"] < 2 or (o["corridor"] >> 1) % 2:   # windows of candidates start at odd positions too
            assert n_odd > 50, n_odd
        if "align" in res:
            _check_alignments(contigs, orc, res["align"], ALIGN_RPL[set_name])
    finally:
        orc.close()


def _check_alignments(contigs, orc, want, rpl):
    """ngmlr_b200.intervals.compute_alignments over the CPU oracle (the mirror the device is compared with) ==
    the reference's computeAlignment with readPartLength = rpl."""
    from ngmlr_b200 import refindex
    from ngmlr_b200.intervals import compute_alignments
    from oracle_lib import Oracle
    from test_cs_oracle import _OracleBackend, _interval_tasks
    tasks = _interval_tasks(contigs, refindex.encode_reference(contigs), rpl)
    got, _calls = compute_alignments(_OracleBackend(orc, Oracle()), tasks)
    n_rev = 0
    for t, w, g in zip(tasks, want, got):
        assert (w is None) == (g is None), t.corridor
        if w is None:
            continue
        for key, v in w.items():
            assert g[key] == v, key
        n_rev += any(a[2] for a in t.anchors) and not t.realign
    assert sum(w is not None for w in want) >= 24 and n_rev >= 5, n_rev


@pytest.mark.parametrize("set_name,genome", [r for r in RUNS if r[0] != "F"])
def test_reference_equals_oracle_at_options(set_name, genome, reference_runs):
    # the numpy builder costs seconds per 4^k entries: at k >= 14 it runs on one genome
    o = cs_cases.OPTION_SETS[set_name]
    _compare(set_name, genome, reference_runs[(set_name, genome)], numpy_builder=o["k"] < 14 or genome == "mixed")


K15_MEMORY = 24 << 30   # two 15-mer builders and their copies


def _mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def test_reference_equals_oracle_at_k15(reference_runs):
    """Set F: a 15-mer index (4^15 + 1 entries, ~5.4 GB for each builder), against the C restatement only."""
    if ("F", "mixed") not in reference_runs:
        pytest.skip("a 15-mer index needs ~24 GB of free host memory (two builders and their copies)")
    _compare("F", "mixed", reference_runs[("F", "mixed")], numpy_builder=False)
