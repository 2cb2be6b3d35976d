"""ngmlr's short-read path and sub-read scorer at --subread-length above 256.

  - map_short_reads + sam_format print the plain ngmlr binary's records for every read of at most --subread-length
    bases, at 300, 510, 511, 512 and 1000 (reads of rpl - 1, rpl and rpl + 1 bases, both strands);
  - score_short_reads on reads of 257-1500 bases, cs_score / cs_run at --subread-length 400-510 and BatchScore with
    queries of 321-1500 characters equal the C restatement of StrippedSW;
  - the scorer's branch counters: queries of at most 510 bases never reach the general affine path, the wide ungapped
    instantiation takes them; longer ones take the general path with several passes."""
import os

import numpy as np
import pytest

from ngmlr_b200 import B200Aligner, samtext, synth
from oracle_lib import CsOracle
from test_gpu_options import _plain_records
from test_gpu_short_reads import PLAIN, _write

pytestmark = pytest.mark.gpu
need_plain = pytest.mark.skipif(not os.path.exists(PLAIN),
                                reason="oracle/_ref/ngmlr not built (needs the reference sources at build time)")

UNGAPPED_MAX_BASES = 510   # queries of <= 511 characters (NUL included) are provably ungapped
PASS_ROWS = 288            # query characters per pass of the general path
CORRIDOR = 40              # --subread-corridor default


def _contigs(seed):
    c1 = synth.random_genome(150_000, seed + 1)
    c2 = synth.random_genome(90_001, seed + 2)
    seg = synth.random_genome(1_200, seed + 3)
    # one segment planted 3 and 1 times: tied scores, MQ 0 and the alignIndex < 2 continuation
    for c, where in ((c1, (20_000, 60_000, 110_000)), (c2, (40_000,))):
        for w in where:
            c[w:w + seg.size] = seg
    c1[80_000:80_040] = ord("N")
    return [c1, c2], seg


def _reads(contigs, seg, rpl, n, seed):
    """Reads of 5 .. rpl + 1 bases, most of them longer than 256; the first twelve of rpl - 1, rpl and rpl + 1."""
    rng = np.random.default_rng(seed)
    reads = []
    for i in range(n):
        kind = i % 8
        c = contigs[i % 2]
        if i < 12:
            L = rpl - 1 + i % 3
            kind = 3
        elif i % 5 == 0:
            L = int(rng.integers(5, rpl + 2))
        else:
            L = int(rng.integers(min(257, rpl), rpl + 2))
        if kind == 0:                      # random, unmappable
            r = synth.random_genome(L, 5000 + i)
        elif kind == 1 and L <= seg.size:  # the planted segment
            a = int(rng.integers(0, seg.size - L + 1))
            r = seg[a:a + L].copy()
        elif kind == 2:                    # contig ends: the window runs into the spacer
            r = c[:L].copy() if i % 4 == 2 else c[c.size - L:].copy()
        else:
            s = int(rng.integers(0, c.size - L))
            r = c[s:s + L].copy()
            if kind in (3, 4, 5):          # sequencing errors (substitutions only keep the length)
                r, _ = synth.mutate(r, rng, err=0.08 if kind != 5 else 0.2, ratio=(0, 0, 1))
            if kind == 6 and r.size > 40:  # an N run in the read
                a = int(rng.integers(0, r.size - 20))
                r[a:a + 15] = ord("N")
        reverse = i % 2 if i < 12 else rng.integers(0, 2)
        if reverse:
            r = synth.revcomp(r)
        reads.append(np.ascontiguousarray(r, dtype=np.uint8).tobytes())
    return reads


@need_plain
@pytest.mark.parametrize("rpl", [300, 510, 511, 512, 1000])
def test_short_reads_at_subread_length_identical_to_plain_binary(rpl, tmp_path):
    contigs, seg = _contigs(71)
    reads = _reads(contigs, seg, rpl, 400, rpl)
    assert sorted(len(r) for r in reads[:12]) == [rpl - 1] * 4 + [rpl] * 4 + [rpl + 1] * 4
    ref, fq, quals = _write(str(tmp_path), contigs, reads)
    names = [f"r{i}".encode() for i in range(len(reads))]
    o = dict(k=13, skip=2, bin=4, s=0.8, rpl=rpl, corridor=CORRIDOR)
    want = _plain_records(ref, fq, str(tmp_path), o)
    a = B200Aligner(0)
    try:
        enc = a.encode_reference([c.tobytes() for c in contigs], fetch=False)
        a.build_index(enc)
        a.reads_upload(reads, rpl)
        a.cs_run(0.8, 0.0, CORRIDOR, rpl)
        res = a.map_short_reads(rpl, 0.25)
        counts = a.debug_short_read_pairs()
    finally:
        a.close()
    ref_names = [b"chr1", b"chr1", b"chr2", b"chr2"]
    n_mapped = n_long = n_rev = n_edge = 0
    for i, r in enumerate(reads):
        if len(r) > rpl:
            assert res[i] is None, f"read {i} ({len(r)} bp) must be reported as not handled"
            n_long += 1
            continue
        mapped, al = res[i]
        text = samtext.sam_format([samtext.Read(names[i], r, quals[i], al, mapped)], ref_names, threads=1)
        w = want.get(names[i], [])
        assert text.splitlines(keepends=True) == w, f"read {i} ({len(r)} bp) differs:\nngmlr: {w}\nlib  : {text}"
        if w and not int(w[0].split(b"\t")[1]) & 4:
            n_mapped += 1
            n_rev += bool(int(w[0].split(b"\t")[1]) & 16)
            n_edge += len(r) >= rpl - 1
    assert n_mapped > 150 and n_rev > 50 and n_edge >= 4 and n_long >= 4, (n_mapped, n_rev, n_edge, n_long)
    # the scorer's branches
    if rpl <= UNGAPPED_MAX_BASES:
        assert counts["general"] == 0 and counts["wide"] > 10, counts
    else:
        assert counts["general"] > 0 and counts["wide"] > 10, counts
    if rpl == 1000:
        assert counts["general"] > 10, counts   # every general pair has >= 512 > PASS_ROWS query characters


def _short_window(cso, L, loc):
    corridor = int(L * 0.3 + 256)
    start = (int(loc) - (corridor >> 1)) % (1 << 64)
    return start, cso.decode(start, L + corridor) or b"N" * (L + corridor)


def test_short_read_scores_above_256_match_oracle(oracle):
    rng = np.random.default_rng(17)
    contigs = [synth.random_genome(40_000, 81), synth.random_genome(30_001, 82)]
    cso = CsOracle([c.tobytes() for c in contigs])
    a = B200Aligner(0)
    try:
        enc = a.encode_reference([c.tobytes() for c in contigs], fetch=False)
        lens = [257, 296, 297, 320, 321, 509, 510, 511, 512, 1000, 1500] + [int(x) for x in rng.integers(257, 1501, 109)]
        reads, origin = [], []
        for i, L in enumerate(lens):
            if i % 3 == 0:
                reads.append(synth.random_genome(L, 900 + i).tobytes())
                origin.append(None)
                continue
            c = i % 2
            s = int(rng.integers(0, contigs[c].size - L))
            # indels: long reads gain from a gap (both halves > 255 bases), so the general path's result differs from
            # the best ungapped piece
            r, _ = synth.mutate(contigs[c][s:s + L].copy(), rng, err=0.03)
            r = np.ascontiguousarray(r, dtype=np.uint8)
            if i % 7 == 1:
                r[10:30] = ord("N")
            reads.append(r.tobytes())
            origin.append(enc.ref_start[c] + s)
        a.reads_upload(reads)
        cl = cso.concat_len
        n = 1600
        ri = rng.integers(0, len(reads), n).astype(np.int32)
        loc = rng.integers(0, cl, n).astype(np.uint64)
        ends = [enc.ref_start[c] + enc.ref_len[c] for c in range(2)]
        loc[:150] = [ends[j % 2] - int(rng.integers(0, 900)) for j in range(150)]          # window runs into the spacer
        loc[150:200] = [enc.ref_start[1] - int(rng.integers(0, 400)) for _ in range(50)]  # starts in the spacer
        loc[200:260] = cl + rng.integers(0, 1000, 60).astype(np.uint64)                    # decoding fails: 'N' window
        loc[260:300] = rng.integers(0, 300, 40).astype(np.uint64)                          # loc - corridor/2 wraps
        for j in range(300, 900):                                                          # the read's own location
            if origin[ri[j]] is not None:
                loc[j] = origin[ri[j]] + int(rng.integers(-5, 6))
        rv = rng.integers(0, 2, n).astype(np.uint8)
        rv[300:900] = 0
        got = a.score_short_reads(ri, loc, rv)
        counts_all = a.debug_short_read_pairs()
        # the pairs of reads of <= 510 bases alone: the wide ungapped instantiation takes every one
        sel = np.array([len(reads[r]) <= UNGAPPED_MAX_BASES for r in ri])
        got_short = a.score_short_reads(ri[sel], loc[sel], rv[sel])
        counts_short = a.debug_short_read_pairs()
    finally:
        a.close()
    reach = dict(odd_start=0, padding=0, past_end=0, n_window=0, reverse=0, high=0)
    for j in range(n):
        q = reads[ri[j]]
        L = len(q)
        start, w = _short_window(cso, L, loc[j])
        qq = synth.revcomp_upper(np.frombuffer(q, dtype=np.uint8)).tobytes() if rv[j] else q
        want = oracle.ssw_score(w, qq)
        assert float(got[j]) == want, (j, L, int(loc[j]), int(rv[j]))
        reach["odd_start"] += start % 2 == 1 and start < cl
        reach["padding"] += start < cl and b"N" * 20 in w          # the spacer between the contigs
        reach["past_end"] += start < cl and w.count(b"x") > 1      # 'x' fill past the concatenated genome
        reach["n_window"] += start >= cl
        reach["reverse"] += int(rv[j])
        reach["high"] += want > 255
    assert np.array_equal(got_short, got[sel])
    assert min(reach.values()) > 10, reach
    assert counts_all["general"] == int((~sel).sum()) and counts_all["wide"] == int(sel.sum()), counts_all
    assert counts_short == {"general": 0, "wide": int(sel.sum())}, counts_short
    assert int(sel.sum()) > 100 and int((~sel).sum()) > 100
    cso.close()


def test_batch_score_queries_above_320_match_oracle(oracle):
    """The drop-in BatchScore with queries of 321-1500 characters and references of up to 1500."""
    rng = np.random.default_rng(23)
    genome = synth.random_genome(50_000, 91)
    refs, qrys = [], []
    for i in range(600):
        L = int(rng.integers(321, 511)) if i % 3 else int(rng.integers(511, 1501))
        W = int(rng.integers(L, max(L + 1, 1024))) if i % 4 else int(rng.integers(max(L, 1025), 1600))
        s = int(rng.integers(0, genome.size - W))
        ref = genome[s:s + W].copy()
        a0 = int(rng.integers(0, max(1, W - L)))
        q, _ = synth.mutate(ref[a0:a0 + L].copy(), rng, err=0.04)
        refs.append(ref.tobytes())
        qrys.append(np.ascontiguousarray(q, dtype=np.uint8).tobytes())
    a = B200Aligner(0)
    try:
        got = a.BatchScore(refs, qrys)
        # pairs that fit the default instantiation, in a batch whose longest query does not
        refs2 = [genome[100:400].tobytes(), genome[2000:2380].tobytes(), genome[100:400].tobytes()]
        qrys2 = [genome[130:380].tobytes(), genome[2020:2340].tobytes(), qrys[0]]
        got2 = a.BatchScore(refs2, qrys2)
    finally:
        a.close()
    want = np.array([oracle.ssw_score(r, q) for r, q in zip(refs, qrys)], dtype=np.float32)
    assert np.array_equal(got, want)
    want2 = np.array([oracle.ssw_score(r, q) for r, q in zip(refs2, qrys2)], dtype=np.float32)
    assert np.array_equal(got2, want2) and want2[0] == 250 and want2[1] == 320


def _split(read, rpl):
    parts = len(read) // rpl
    return [read[k * rpl:(k + 1) * rpl] for k in range(parts)] if parts else [read]


@pytest.mark.parametrize("rpl", [400, 480, 510])
def test_subreads_at_subread_length_ungapped(rpl, oracle):
    """cs_score and cs_run at --subread-length 400-510: scores equal the oracle on ScoreBuffer's windows, and no
    sub-read reaches the general path."""
    rng = np.random.default_rng(rpl)
    genome = synth.random_genome(300_000, 95)
    contigs = [genome[:150_000], genome[150_000:]]
    cso = CsOracle([c.tobytes() for c in contigs])
    reads = []
    for i in range(40):
        L = int(rng.integers(rpl, 4 * rpl)) if i % 4 else int(rng.integers(100, rpl))
        c = contigs[i % 2]
        s = int(rng.integers(0, c.size - L - 100))
        r, _ = synth.mutate(c[s:s + L].copy(), rng, err=0.05)
        r = np.ascontiguousarray(r, dtype=np.uint8)
        reads.append((synth.revcomp(r) if i % 3 == 0 else r).tobytes())
    subs = [s for r in reads for s in _split(r, rpl)]
    win_len = ((rpl + 10 + CORRIDOR) | 1) + 1   # ScoreBuffer's refMaxLen
    a = B200Aligner(0)
    try:
        enc = a.encode_reference([c.tobytes() for c in contigs], fetch=False)
        a.build_index(enc)
        scored, _mx = a.cs_score(subs, 0.8, 0.0, CORRIDOR, rpl)
        counts_score = a.debug_subread_pairs()
        a.reads_upload(reads, rpl)
        m, _ms = a.cs_run(0.8, 0.0, CORRIDOR, rpl)
        counts_run = a.debug_subread_pairs()
        start, _sc, lo, rv, sw, _mx2 = a.cs_fetch()
    finally:
        a.close()
    n_pairs = n_long = 0
    for i, s in enumerate(subs):
        assert [(int(lo[x]), int(rv[x]), sw[x]) for x in range(start[i], start[i + 1])] == \
            [(g[1], g[2], g[3]) for g in scored[i]], i
        for (_cs, loc, rev, score) in scored[i]:
            w = cso.decode((loc - (CORRIDOR >> 1)) % (1 << 64), win_len) or b"N" * win_len
            q = synth.revcomp_upper(np.frombuffer(s, dtype=np.uint8)).tobytes() if rev else s
            assert score == oracle.ssw_score(w, q), (i, loc, rev)
            n_pairs += 1
            n_long += len(s) > 320
    cso.close()
    assert n_long > 10 and m == n_pairs, (n_long, m, n_pairs)
    assert counts_score == {"general": 0, "wide": n_pairs}, counts_score
    assert counts_run == {"general": 0, "wide": n_pairs}, counts_run
