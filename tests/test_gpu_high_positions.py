"""Every device stage on a reference whose real contigs lie beyond 2^31 concatenated positions, where about a third of a
human genome lies. The CPU oracle cannot index a genome of that size in test time, so the expected values come from
a small genome through a relation that holds by construction:

  - R: the real contigs, about 3 Mb: three contigs of 1 000 000 bases (so that synth.simulate_reads can draw reads
    from them) with the edge features of cs_cases.genome_contigs / repeat_contigs (N runs, a homopolymer, a tandem
    repeat, a final run of exactly k characters behind an N run, and 1100 copies of one 99-base unit, so that the
    maxPrefixFreq cutoff fires), one contig of odd length, and one of 8 bases that both layouts drop.
  - P: nine padding contigs of pure N, about 239 Mb each (each below 2^31 bases: longer records are refused as the
    reference's reader refuses them).
  - Layout L = R; layout H = P followed by R. The padding lengths put the first real contig across 2^31 (it starts
    about 0.5 Mb below it) and every later real contig wholly above it, make D = ref_start_H(first real contig) -
    ref_start_L(first real contig) a multiple of 64, and keep concat_len(H) below 0xffff0000 (one table unit).

An all-N contig gives no k-mer callback, so H's index holds the k-mers of R only. Every rule on the path works
relative to a contig or to a read: the repeat filter compares 16-bp bins of consecutive callbacks of one contig; the
candidate vote bins are (loc - corr) >> bin_shift; the ScoreBuffer window sits at loc - 20 and its odd term depends on
the parity of loc; corridors are built from onRef - onRefStart; short-read windows are built from the candidate
location; the is_mapped test is *up - loc >= 1000; SAM positions are relative to the contig. With D a multiple of 64
(bin shifts up to 6, even parity), every output at H is therefore the output at L with locations shifted by D, and the
output at L comes from the CPU oracle (CsOracle, Oracle and the Python computeAlignment mirror, which
test_cs_oracle.py pins to the compiled reference). Where the plain ngmlr binary was built, it checks the argument
itself: its own caches of H equal ours, and its SAM body from our H caches equals its SAM body on L.

The load of H needs about 17 B of device memory per position (about 37 GB); the tests that need it are skipped with
the reason when less is free."""
import os
import shutil
import subprocess
import threading
import time
import zlib

import numpy as np
import pytest

import cs_cases
from ngmlr_b200 import B200Aligner, IntervalBatch, ngmfiles, samtext, synth
from ngmlr_b200.intervals import compute_alignments
from oracle_lib import CsOracle, same_alignment
from test_cs_oracle import _OracleBackend
from test_gpu_load_reference import _compare_caches

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLAIN = os.path.join(ROOT, "oracle", "_ref", "ngmlr")
need_plain = pytest.mark.skipif(not os.path.exists(PLAIN), reason="oracle/_ref/ngmlr not built")

TWO31 = 1 << 31
CONTIG = 1_000_000
N_PAD = 9
LINE = 1 << 16                  # FASTA line length of the padding
BLOCK_LINES = 256               # padding lines per pre-compressed gzip member (16 MiB of text)
BYTES_PER_POSITION = 17         # device memory at the peak of load_reference (51.8 GB at 3 Gb)
REAL_NAMES = [b"r0", b"r1", b"tiny", b"r2", b"odd"]


def _real_contigs():
    r0 = synth.random_genome(CONTIG, 101)
    r1 = synth.random_genome(CONTIG, 102)
    r2 = synth.random_genome(CONTIG, 103)
    r0[0:3] = ord("N")
    r0[20:25] = ord("N")
    r0[5000:5010] = ord("N")
    r0[7000:7400] = ord("A")                                              # homopolymer
    r0[499_000:499_040] = ord("N")                                        # N run just below 2^31 at H
    r1[100:160] = np.tile(np.frombuffer(b"ACGTAC", dtype=np.uint8), 10)  # tandem repeat
    r1[600_000:600_300] = ord("N")
    unit = synth.random_genome(99, 104)                                   # 99 = 3 * 33: every copy gives the same
    r2[400_000:400_000 + 99 * 1100] = np.tile(unit, 1100)                 # callbacks -> frequency > maxPrefixFreq
    r2[-18:-13] = ord("N")                                                # a final run of exactly k = 13 characters
    odd = synth.random_genome(30_001, 105)
    odd[50:70] = ord("N")
    tiny = np.frombuffer(b"ACGTACGT", dtype=np.uint8).copy()
    return [r0, r1, tiny, r2, odd]


def _padding_lengths():
    """N_PAD even lengths: the first real contig starts at 1000 + D in H with D a multiple of 64 about 0.5 Mb below
    2^31 (each padding contig takes its length plus a 1000-N spacer)."""
    d = (TWO31 - 500_000 - 1000) // 64 * 64
    total = d - 1000 * N_PAD
    each = total // N_PAD // 2 * 2
    return [each] * (N_PAD - 1) + [total - each * (N_PAD - 1)], d


def _gz_member(text):
    c = zlib.compressobj(1, zlib.DEFLATED, 31)
    return c.compress(text) + c.flush()


def _write_fasta(path, real, pads):
    """gzip FASTA of H. A gzip file may hold several members one after another; the padding is written as one
    pre-compressed member repeated, so that writing 2 Gb of N takes a second."""
    block = _gz_member((b"N" * LINE + b"\n") * BLOCK_LINES)
    with open(path, "wb") as f:
        for i, n in enumerate(pads):
            f.write(_gz_member(b">pad%d padding\n" % i))
            full, rest = divmod(n, LINE * BLOCK_LINES)
            for _ in range(full):
                f.write(block)
            lines, tail = divmod(rest, LINE)
            f.write(_gz_member((b"N" * LINE + b"\n") * lines + (b"N" * tail + b"\n" if tail else b"")))
        for name, c in zip(REAL_NAMES, real):
            s = c.tobytes()
            f.write(_gz_member(b">" + name + b"\n" + b"".join(s[k:k + 10_000] + b"\n"
                                                             for k in range(0, len(s), 10_000))))


def _write_plain_fasta(path, names, contigs):
    with open(path, "wb") as f:
        for name, c in zip(names, contigs):
            f.write(b">" + name + b"\n" + bytes(c) + b"\n")


class _Peak:
    """Device memory in use on the card (all processes), sampled every 2 ms while the block runs."""

    def __enter__(self):
        import torch
        self.torch = torch
        self.free0, self.total = torch.cuda.mem_get_info(0)
        self.peak = self.total - self.free0
        self.done = threading.Event()

        def sample():
            while not self.done.is_set():
                self.peak = max(self.peak, self.total - self.torch.cuda.mem_get_info(0)[0])
                time.sleep(0.002)

        self.th = threading.Thread(target=sample)
        self.th.start()
        return self

    def __exit__(self, *exc):
        self.done.set()
        self.th.join()


def _state(a):
    """The context's encoded genome (the used part of binRef), concat length and k-mer index."""
    import ctypes as C
    a.lib.ngmlr_b200_cs_get_reference.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                                  C.POINTER(C.c_uint64)]
    nb, cl = C.c_uint64(0), C.c_uint64(0)
    a._check(a.lib.ngmlr_b200_cs_get_reference(a.h, None, 0, C.byref(nb), C.byref(cl)))
    ref = np.zeros(nb.value, np.uint8)
    a._check(a.lib.ngmlr_b200_cs_get_reference(a.h, ref.ctypes.data_as(C.c_void_p), ref.size, None, None))
    return ref, cl.value, a.get_index()


@pytest.fixture(scope="module")
def layouts(tmp_path_factory):
    """Host side: R, the padding, CsOracle(L), and the gzip FASTA of H."""
    real = _real_contigs()
    pads, d = _padding_lengths()
    orc = CsOracle([c.tobytes() for c in real])
    starts_l = orc.ref_starts()
    assert len(starts_l) == 4 and starts_l[0] == 1000            # tiny is dropped
    lens_l = [CONTIG, CONTIG, CONTIG, 30_001]
    starts_h = [s + d for s in starts_l]
    concat_h = orc.concat_len + d
    # the three properties the relation and the point of the module rest on
    assert d % 64 == 0
    assert starts_h[0] < TWO31 < starts_h[0] + lens_l[0] and TWO31 - starts_h[0] > 400_000
    assert all(s > TWO31 for s in starts_h[1:])
    assert concat_h < 0xFFFF0000 and all(p < TWO31 for p in pads)
    # the maxPrefixFreq cutoff fires: the 29 k-mers of the planted unit that every copy calls back (one in three)
    # have 1100 callbacks and are not indexed; the other 58 occur nowhere else but by chance
    rci = orc.index()[1]
    unit = ((real[3][400_000:400_099] >> 1) & 3).astype(np.int64)   # CS k-mer codes A0 C1 T2 G3
    codes = [int(sum(int(b) << (2 * (12 - t)) for t, b in enumerate(unit[j:j + 13]))) for j in range(87)]
    assert sum(rci[c] == 0 for c in codes) >= 84
    path = str(tmp_path_factory.mktemp("h") / "h.fa.gz")
    _write_fasta(path, real, pads)
    kept = [real[0], real[1], real[3], real[4]]
    yield dict(real=real, kept=kept, genome=np.concatenate(kept[:3]), pads=pads, d=d, orc=orc, starts_l=starts_l,
               starts_h=starts_h, lens=lens_l, concat_h=concat_h, path=path)
    orc.close()


@pytest.fixture(scope="module")
def loaded(layouts):
    """Device side: context `a` loads H from the FASTA file (builds and writes both caches), its arrays are fetched
    and it is closed; the working context `w` then loads the same path from the caches."""
    import torch
    need = BYTES_PER_POSITION * layouts["concat_h"] + (2 << 30)
    free = torch.cuda.mem_get_info(0)[0]
    if free < need:
        pytest.skip(f"loading a {layouts['concat_h'] / 1e9:.2f} G-position reference needs about {need / 1e9:.0f} GB "
                    f"of device memory; {free / 1e9:.0f} GB free")
    t0 = time.perf_counter()
    a = B200Aligner(0)
    try:
        with _Peak() as peak:
            first = a.load_reference(layouts["path"])
        state = _state(a)
    finally:
        a.close()
    load_s = time.perf_counter() - t0
    print(f"\nH: {layouts['concat_h']} positions; load from FASTA {load_s:.1f} s {first.ms}; peak device memory in "
          f"use {peak.peak / 1e9:.1f} GB ({(peak.total - peak.free0) / 1e9:.1f} GB before)")
    w = B200Aligner(0)
    second = w.load_reference(layouts["path"])
    yield dict(first=first, second=second, state=state, w=w)
    w.close()


@pytest.fixture(scope="module")
def l_ctx(layouts):
    """A context holding L (encoded and indexed on the device)."""
    c = B200Aligner(0)
    enc = c.encode_reference([x.tobytes() for x in layouts["real"]], fetch=False)
    assert enc.ref_start == layouts["starts_l"]
    c.build_index(enc)
    yield c
    c.close()


# ---- 1. start-up ----------------------------------------------------------------------------------------------------
def _check_arrays(lay, ref, concat_len, idx, enc_l, tab_l, rci_l, pos_l):
    d = lay["d"]
    assert concat_len == lay["concat_h"]
    assert ref.size == d // 2 + enc_l.size
    assert np.all(ref[:d // 2] == 0x44) and np.array_equal(ref[d // 2:], enc_l)
    assert np.array_equal(idx.tab, tab_l) and np.array_equal(idx.rci, rci_l)
    assert np.array_equal(idx.pos, pos_l.astype(np.uint64) + d)


def test_start_up(layouts, loaded):
    lay = layouts
    enc_l = lay["orc"].encoded()
    tab_l, rci_l, pos_l = lay["orc"].index()
    first, second = loaded["first"], loaded["second"]
    assert (first.reference_read, first.reference_written, first.index_read, first.index_written) == \
        (False, True, False, True)
    assert (second.reference_read, second.reference_written, second.index_read, second.index_written) == \
        (True, False, True, False)
    names = [b"pad%d" % i for i in range(N_PAD)] + [b"r0", b"r1", b"r2", b"odd"]
    for r in (first, second):
        assert r.names == names
        assert r.lens == lay["pads"] + lay["lens"]
        assert r.starts[N_PAD:] == lay["starts_h"] and r.concat_len == lay["concat_h"]
    ref, cl, idx = loaded["state"]
    _check_arrays(lay, ref, cl, idx, enc_l, tab_l, rci_l, pos_l)
    assert idx.pos.min() < TWO31 <= idx.pos.max()
    # the second context installed the same arrays from the caches
    ref2, cl2, idx2 = _state(loaded["w"])
    assert np.array_equal(ref, ref2) and cl == cl2
    for x, y in ((idx.tab, idx2.tab), (idx.rci, idx2.rci), (idx.pos, idx2.pos)):
        assert np.array_equal(x, y)
    del ref2, idx2
    # the numpy and the C readers of the caches
    enc_path, ht_path = lay["path"] + "-enc.2.ngm", lay["path"] + "-ht-13-2.2.ngm"
    for read_ref, read_idx in ((ngmfiles.read_encoded_reference, ngmfiles.read_index),
                               (ngmfiles.c_read_encoded_reference, ngmfiles.c_read_index)):
        er, enames = read_ref(enc_path)
        assert [n.encode() for n in enames] == names and er.ref_start == first.starts and er.ref_len == first.lens
        _check_arrays(lay, er.enc, er.concat_len, read_idx(ht_path)[0], enc_l, tab_l, rci_l, pos_l)
        del er


@need_plain
def test_plain_ngmlr_writes_the_same_caches(layouts, loaded, tmp_path):
    """The plain binary's own CPU build of H: the index cache byte for byte, the encoded cache up to the used part."""
    theirs = str(tmp_path / "h.fa.gz")
    shutil.copyfile(layouts["path"], theirs)
    q = str(tmp_path / "q.fa")
    with open(q, "w") as f:
        f.write(">q\n" + "ACGTTGCA" * 40 + "\n")
    t0 = time.perf_counter()
    r = subprocess.run([PLAIN, "-r", theirs, "-q", q, "-o", str(tmp_path / "o.sam"), "-t", "1", "--no-progress"],
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]
    print(f"\nplain ngmlr: CPU build of H and both caches in {time.perf_counter() - t0:.0f} s")
    _compare_caches(layouts["path"], theirs, 13, 2)


# ---- 2. candidate search and sub-read scoring -----------------------------------------------------------------------
def _subreads(lay):
    """cs_cases-style sub-reads of R, plus sub-reads whose candidate window (loc - 20, 308 characters) straddles 2^31."""
    kept = lay["kept"]
    subs = [s[:256] for s in cs_cases.subreads(300, 71, kept)]
    subs += cs_cases.option_reads(kept, 256, 60, 72)
    subs = [s for r in subs for s in cs_cases.split_read(r, 256)]
    o = TWO31 - lay["starts_h"][0]                    # offset of 2^31 in r0
    rng = np.random.default_rng(73)
    for k, s in enumerate(range(o - 300, o + 40, 17)):
        n = (256, 255, 100, 40)[k % 4]
        sub = kept[0][s:s + n]
        if k % 3 == 1:
            sub = synth.mutate(sub, rng, err=0.08)[0][:n]
        if k % 2:
            sub = synth.revcomp(sub)
        subs.append(np.ascontiguousarray(sub, dtype=np.uint8).tobytes())
    return subs


def _sw_want(lay, oracle, sub, loc_l, rev):
    w = lay["orc"].decode((loc_l - 20) % (1 << 64), 308) or b"N" * 308
    q = synth.revcomp_upper(np.frombuffer(sub, dtype=np.uint8)).tobytes() if rev else sub
    return oracle.ssw_score(w, q)


def test_candidate_search_and_scoring(layouts, loaded, oracle):
    lay, w, d = layouts, loaded["w"], layouts["d"]
    subs = _subreads(lay)
    assert max(len(s) for s in subs) == 256      # one sub-read per read on the resident path below
    want = [lay["orc"].search(s) for s in subs]
    shifted = [[(sc, loc + d, rv) for sc, loc, rv in cands] for cands, _ in want]
    got, mx = w.cs_search(subs)
    assert got == shifted
    assert np.array_equal(mx, np.array([m for _, m in want], dtype=np.float32))
    scored, mx2 = w.cs_score(subs)
    assert [[g[:3] for g in c] for c in scored] == shifted and np.array_equal(mx, mx2)
    n_sw = 0
    straddle = 0
    for sub, (cands, _), c in zip(subs, want, scored):
        for (_sc, loc_l, rev), g in zip(cands, c):
            assert g[3] == _sw_want(lay, oracle, sub, loc_l, rev), (loc_l + d, rev)
            n_sw += 1
            straddle += loc_l + d - 20 < TWO31 < loc_l + d - 20 + 308
    locs = [loc for c in shifted for _, loc, _ in c]
    assert n_sw > 300 and straddle >= 3 and max(locs) > TWO31 + 2 * CONTIG and min(locs) < TWO31
    # the resident path: reads_upload -> cs_run -> cs_fetch
    assert w.reads_upload(subs) == len(subs)
    m, _ = w.cs_run()
    start, sc, lo, rv, sw, mx3 = w.cs_fetch()
    assert m == start[-1] == n_sw and np.array_equal(mx3, mx)
    for i, c in enumerate(scored):
        got_i = [(sc[j], int(lo[j]), int(rv[j]), sw[j]) for j in range(start[i], start[i + 1])]
        assert got_i == c, i


# ---- 3. window decoding ---------------------------------------------------------------------------------------------
def test_window_decoding(layouts, loaded):
    lay, w, d = layouts, loaded["w"], layouts["d"]
    first = lay["starts_h"][0]
    # the spacer before r0 is the padding's last spacer at H and the leading spacer at L: not compared
    wins = [x for x in cs_cases.exact_windows(lay["starts_h"], lay["lens"]) if x[0] >= first]
    wins += [(TWO31 - k, n) for k in (1, 2, 3, 150, 151, 2999) for n in (2, 3, 11, 302, 3001)]
    got = w.decode_windows([x[0] for x in wins], [x[1] for x in wins])
    n_straddle = 0
    for (st, n), text in zip(wins, got):
        assert text == lay["orc"].decode_exact(st - d, n), (st, n)
        n_straddle += st < TWO31 < st + n - 1
    assert n_straddle >= 12 and max(st for st, _ in wins) > TWO31
    # windows wholly inside the padding contigs, away from their ends: seq_len - 1 N characters
    pads = loaded["first"]
    inner = [(pads.starts[i] + off, n) for i in (0, 4, N_PAD - 1) for off in (5000, 100_000_001, pads.lens[i] - 9000)
             for n in (2, 301, 4000)]
    for (st, n), text in zip(inner, w.decode_windows([x[0] for x in inner], [x[1] for x in inner])):
        assert text == b"N" * (n - 1), (st, n)


# ---- 4. compute_alignments ------------------------------------------------------------------------------------------
def _straddling_reads(lay, seed):
    """Plain reads of r0 whose reference window runs across 2^31 at H, on both strands."""
    rng = np.random.default_rng(seed)
    o = TWO31 - lay["starts_h"][0]
    genome = lay["genome"]
    reads, ivs = [], []
    for k, L in enumerate((6000, 3000, 9000, 1200)):
        start = o - int(rng.integers(200, L - 200))
        read, starts = synth.mutate(genome[start:start + L], rng, 0.12, (1, 1, 1))
        ax, ay = synth._anchors(starts, int(read.size), rng)
        rev = bool(k % 2)
        reads.append((synth.revcomp_upper(read) if rev else read).tobytes())
        ivs.append(synth.SimInterval(k, 0, int(read.size), rev, start, L, ax, ay))
    return reads, ivs


def _align_check(lay, w, oracle, reads, ivs, min_valid):
    starts_l, starts_h = lay["starts_l"], lay["starts_h"]
    g2c_h = lambda p: starts_h[p // CONTIG] + p % CONTIG
    g2c_l = lambda p: starts_l[p // CONTIG] + p % CONTIG
    tasks_h = synth.interval_tasks(ivs, reads, g2c_h, by_index=True)
    tasks_l = synth.interval_tasks(ivs, reads, g2c_l, by_index=False)
    # coordinates the module is about: a window across 2^31, anchors above it through the ctypes Anchor
    assert any(t.on_ref_start < TWO31 < t.on_ref_stop for t in tasks_h)
    ib = IntervalBatch(tasks_h)
    assert max(ib.anchors[i].on_ref for i in range(sum(len(t.anchors) for t in tasks_h))) > TWO31 + CONTIG
    assert max(ib.intervals[i].on_ref_start for i in range(ib.n)) > TWO31
    w.reads_upload(reads)
    got, calls = w.compute_alignments(ib)
    got = list(got)
    want, want_calls = compute_alignments(_OracleBackend(lay["orc"], oracle), tasks_l)
    assert list(calls) == want_calls
    n_valid = 0
    for i, (a, g) in enumerate(zip(want, got)):
        assert (a is None) == (g.ret < 0), i
        if a is not None:
            n_valid += 1
            diff = same_alignment(a, dict(g.as_dict(), nm_positions=a["nm_positions"]))
            assert diff == [], (i, diff)
            assert g.nmCount == len(a["nm_positions"])
    assert n_valid >= min_valid, (n_valid, len(ivs))
    return calls


def test_compute_alignments_ont_shape(layouts, loaded, oracle):
    genome = layouts["genome"]
    reads, ivs = synth.simulate_reads(16, genome, CONTIG, 81, median=6000, err=0.12, ratio=(1, 1, 1), hi=16000)
    more_reads, more_ivs = _straddling_reads(layouts, 82)
    for iv in more_ivs:
        iv.read += len(reads)
    _align_check(layouts, loaded["w"], oracle, reads + more_reads, ivs + more_ivs, min_valid=18)


def test_compute_alignments_sv_shape(layouts, loaded, oracle):
    genome = layouts["genome"]
    reads, ivs = synth.simulate_reads(40, genome, CONTIG, 83, median=4000, err=0.15, sv=True, lo=2000, hi=9000)
    more_reads, more_ivs = _straddling_reads(layouts, 84)
    for iv in more_ivs:
        iv.read += len(reads)
    ivs += more_ivs
    assert sum(iv.full_alignment for iv in ivs) >= 1 and sum(iv.reverse for iv in ivs) >= 8
    calls = _align_check(layouts, loaded["w"], oracle, reads + more_reads, ivs, min_valid=int(0.8 * len(ivs)))
    assert len(calls) == len(ivs)


# ---- 5. short-read path and SAM -------------------------------------------------------------------------------------
def _short_reads(lay, seed, n=600):
    rng = np.random.default_rng(seed)
    kept = lay["kept"]
    o = TWO31 - lay["starts_h"][0]
    reads = []
    for i in range(n):
        c = kept[i % len(kept)]
        L = int(rng.integers(5, 257))
        kind = i % 8
        if kind == 0:
            r = synth.random_genome(L, 5000 + i)
        elif kind == 1:                                   # across 2^31 at H
            s = o - int(rng.integers(0, L))
            r = kept[0][s:s + L].copy()
        elif kind == 2:                                   # contig ends
            r = c[:L].copy() if i % 16 == 2 else c[c.size - L:].copy()
        else:
            s = int(rng.integers(0, c.size - L))
            r, _ = synth.mutate(c[s:s + L].copy(), rng, err=(0.0, 0.05, 0.15)[i % 3])
            r = np.ascontiguousarray(r[:256], dtype=np.uint8)
        if r.size == 0:
            r = np.frombuffer(b"ACGTA", dtype=np.uint8).copy()
        if rng.integers(0, 2):
            r = synth.revcomp(r)
        reads.append(np.ascontiguousarray(r, dtype=np.uint8).tobytes())
    return reads


def test_short_reads_and_sam(layouts, loaded, l_ctx):
    w = loaded["w"]
    reads = _short_reads(layouts, 91)
    names = [b"s%d" % i for i in range(len(reads))]
    quals = [b"I" * len(r) for r in reads]
    out = {}
    for key, ctx, ref_names in (("H", w, loaded["first"].sam_ref_names()),
                                ("L", l_ctx, [n for n in (b"r0", b"r1", b"r2", b"odd") for _ in (0, 1)])):
        ctx.reads_upload(reads)
        ctx.cs_run()
        res = ctx.map_short_reads()
        assert all(r is not None for r in res)
        recs = [(m, [(ref_names[a.ref_id], a.ref_pos, a.reverse, a.score, a.mq, a.nm, a.identity, a.qstart, a.qend,
                      a.cigar, a.md, a.sv_type, a.primary, a.skip, a.cigar_ops) for a in al]) for m, al in res]
        text = samtext.sam_format([samtext.Read(n, s, q, al, m) for n, s, q, (m, al) in zip(names, reads, quals, res)],
                                  ref_names, threads=1)
        out[key] = recs, text
    assert out["H"][0] == out["L"][0]
    assert out["H"][1] == out["L"][1]
    mapped = [(al[0], len(r)) for (m, al), r in zip(out["H"][0], reads) if m and al]
    assert len(mapped) > len(reads) // 2
    o = TWO31 - layouts["starts_h"][0]
    assert sum(1 for a, _ in mapped if a[0] != b"r0" or a[1] > o) >= 100                # wholly above 2^31
    assert sum(1 for a, n in mapped if a[0] == b"r0" and a[1] <= o < a[1] + n) >= 20    # across it


@need_plain
def test_plain_ngmlr_from_gpu_caches_at_h(layouts, loaded, tmp_path):
    """The plain binary started from the caches the GPU wrote for H writes the SAM body it writes on L."""
    lay = layouts
    short = _short_reads(lay, 95, n=24)
    long_reads, _ = synth.simulate_reads(12, lay["genome"], CONTIG, 96, median=3000, err=0.1, lo=1000, hi=8000)
    s_reads, _ = _straddling_reads(lay, 97)
    reads = short + long_reads + s_reads
    fq = str(tmp_path / "reads.fq")
    with open(fq, "wb") as f:
        for i, r in enumerate(reads):
            f.write(b"@q%d\n%s\n+\n%s\n" % (i, r, b"I" * len(r)))
    l_fa = str(tmp_path / "l.fa")
    _write_plain_fasta(l_fa, REAL_NAMES, [c.tobytes() for c in lay["real"]])
    caches = [lay["path"] + "-enc.2.ngm", lay["path"] + "-ht-13-2.2.ngm"]
    mtimes = [os.stat(f).st_mtime_ns for f in caches]
    sams = {}
    for key, ref, extra in (("H", lay["path"], []), ("L", l_fa, ["--skip-write"])):
        sam = str(tmp_path / f"{key}.sam")
        r = subprocess.run([PLAIN, "-r", ref, "-q", fq, "-o", sam, "-t", "1", "--no-progress", *extra],
                           capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-2000:]
        sams[key] = [l for l in open(sam, "rb") if not l.startswith(b"@")]
    assert [os.stat(f).st_mtime_ns for f in caches] == mtimes         # read, not rebuilt
    assert sams["H"] == sams["L"] and len(sams["L"]) >= len(reads)
    o = TWO31 - lay["starts_h"][0]
    fields = [l.split(b"\t") for l in sams["L"]]
    assert sum(1 for f in fields if f[2] in (b"r1", b"r2")) >= 5                                   # above 2^31
    assert sum(1 for f in fields if f[2] == b"r0" and int(f[3]) <= o < int(f[3]) + 1000) >= 3     # across it


# ---- 6. a context sharing H -----------------------------------------------------------------------------------------
def test_shared_context(layouts, loaded):
    w = loaded["w"]
    subs = _subreads(layouts)[-60:] + [s[:256] for s in cs_cases.subreads(60, 99, layouts["kept"])]
    w.reads_upload(subs)
    w.cs_run()
    want = w.cs_fetch()
    assert int(want[0][-1]) > 0 and int(want[2].max()) > TWO31
    c = B200Aligner(0)
    try:
        c.share_reference(w)
        c.reads_upload(subs)
        c.cs_run()
        for x, y in zip(want, c.cs_fetch()):
            assert np.array_equal(x, y)
    finally:
        c.close()
