"""The fill at production batch size: the real call streams of plain ngmlr on an SV and a long-read workload, replayed as
one batch of more than one problem per SM, so that all three concurrent fill launches are non-empty:
  * 16-warp teams (stream 2): problems of >= 8 Mi cells in corridors >= 768 columns wide;
  * ramped 4-warp teams (stream 3, beside the ramp-free schedule): the other problems of >= 8 Mi cells;
  * the one-warp kernel (two rows per lane, skewed, by default): everything else.
They share one direction bump allocator, one boundary-strip arena and the overflow -> grow -> re-run loop, and a
corridor row wider than 32 767 switches all three to the RAW instantiation.

The streams are recorded at test time by oracle/_ref/ngmlr_rec (the unmodified reference with recording decorators,
scripts/record_workload.py); every SingleAlign call is compared bit for bit with what the reference returned (ret,
Score bits, CIGAR, MD, NM, PositionOffset, QStart, QEnd), through both text stages. Every test also checks the fill's
routing counters (B200Aligner.debug_fill_counts) against a restatement of the host's routing rules (_route).

The stream-composition test needs no GPU: it checks that the recordings really hold such a batch."""
import os
import subprocess
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

from ngmlr_b200 import corridor, synth
from oracle_lib import Oracle, same_alignment

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REC = os.path.join(ROOT, "oracle", "_ref", "ngmlr_rec")
sys.path.insert(0, os.path.join(ROOT, "scripts"))

needs_rec = pytest.mark.skipif(not os.path.exists(REC), reason="oracle/_ref/ngmlr_rec not built")

# an SV workload (anchor-widened corridors up to a few thousand columns, full matrices, retries) and a long-read one
# (reads of more than 32 767 bases in corridors a few hundred columns wide)
RECIPES = (
    ["--reads", "120", "--genome-mb", "2", "--contigs", "2", "--median", "6000", "--sv", "--seed", "7"],
    ["--reads", "60", "--genome-mb", "4", "--contigs", "2", "--median", "20000", "--seed", "8"],
)
H100_SMS = 132
TEAM_CELLS = 8 << 20     # RF_TEAM_CELLS
BIG_CELLS, BIG_WIDTH = 8 << 20, 768
RF_MIN_WIDTH = 128       # kernels.h
TEAM_WIDTH = 352         # corridors from which the ramped schedule picks 4-warp teams
COUNTS = ("big_team", "rf_team", "rampfree", "ramped_warp", "ramped_team", "raw", "fill_launches", "multi_launch",
          "three_way")


# ---- the recorded batch ---------------------------------------------------------------------------------------------
def _record(d, recipe):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "record_workload.py"), *recipe,
                        "--threads", "16", "--out", d], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    from replay_workload import parse
    aligns, _pairs = parse(os.path.join(d, "calls.bin"))
    return aligns


def _shape(ref_len, offsets, lengths):
    """What the host's routing sees of a problem: estimated cells (sum of the row lengths), width (widest row, clipped
    to the reference), rows, reference length, and whether the corridor is monotone with non-empty rows."""
    off, ln = np.asarray(offsets, np.int64), np.asarray(lengths, np.int64)
    orderly = ln.size > 0 and bool((ln > 0).all()) and bool((np.diff(off) >= 0).all())
    return dict(est=int(np.maximum(ln, 0).sum()), width=min(int(ln.max()) if ln.size else 0, ref_len),
                rows=int(ln.size), ref_len=ref_len, orderly=orderly)


def _shapes(aligns):
    return [_shape(len(a["ref"]), a["off"], a["len"]) for a in aligns]


def _composition(shapes):
    big = sum(s["est"] >= BIG_CELLS and s["width"] >= BIG_WIDTH for s in shapes)
    team = sum(s["est"] >= TEAM_CELLS and s["width"] < BIG_WIDTH for s in shapes)
    return dict(n=len(shapes), big=big, team=team, longest=max(s["rows"] for s in shapes),
                orderly=all(s["orderly"] for s in shapes))


@pytest.fixture(scope="module")
def stream(tmp_path_factory):
    """Both recorded streams as one batch (SV calls first), with the composition this module relies on."""
    aligns = []
    for k, recipe in enumerate(RECIPES):
        aligns += _record(str(tmp_path_factory.mktemp(f"rec{k}")), recipe)
    c = _composition(_shapes(aligns))
    assert c["n"] > H100_SMS and c["big"] >= 8 and c["team"] >= 8 and c["longest"] > 32767 and c["orderly"], c
    return aligns


# ---- the host's routing, restated -----------------------------------------------------------------------------------
def _route(shapes, num_sms, schedule="rampfree", force_team=-1, no_big_teams=False, small_batch_big_teams=True,
           big_cells=BIG_CELLS, big_width=BIG_WIDTH):
    """Problems per launch of one convex_run (convex_host.cu), as the counters report them, from the host's estimates."""
    n = len(shapes)
    team_safe = all(s["orderly"] for s in shapes)
    big = [s["est"] >= big_cells and s["width"] >= big_width for s in shapes]
    big_ok = team_safe and force_team != 0 and not no_big_teams
    n_big = sum(big)
    if not big_ok or (n_big > 2 * num_sms and 2 * n_big > n):
        big, n_big = [False] * n, 0
    rf_team = sum(not b and s["est"] >= TEAM_CELLS for b, s in zip(big, shapes))
    team = sum(s["width"] >= TEAM_WIDTH for s in shapes) * 2 > n
    if force_team >= 0:
        team = force_team != 0
    team = team and team_safe
    rf_fits = all(((s["rows"] + 31) // 32) * (s["ref_len"] + 400) < (1 << 30) for s in shapes)
    rampfree = (schedule != "ramped" and force_team != 1 and rf_fits
                and sum(s["width"] >= RF_MIN_WIDTH for s in shapes) * 2 > n)
    if rampfree:
        team = False
    if big_ok and n <= num_sms and small_batch_big_teams:
        n_big = n
    n_team = min(rf_team, n - n_big) if rampfree and team_safe and force_team != 0 else 0
    rest = n - n_big - n_team
    launches = (n_big > 0) + (n_team > 0) + (rest > 0)
    return dict(big_team=n_big, rf_team=n_team, rampfree=rest if rampfree else 0,
                ramped_warp=rest if not rampfree and not team else 0, ramped_team=rest if not rampfree and team else 0,
                raw=n if max(s["width"] for s in shapes) > 32767 else 0, fill_launches=1,
                multi_launch=int(launches > 1), three_way=int(launches == 3))


def _plus(a, b):
    return {k: a[k] + b[k] for k in COUNTS}


@needs_rec
def test_recorded_streams_fill_all_three_launches(stream):
    """No GPU: the two recordings hold a batch of more than one problem per SM of an H100 with >= 8 problems for each
    team launch and a read longer than 32 767 bases, and the host's rules route it to all three launches."""
    shapes = _shapes(stream)
    c = _composition(shapes)
    assert c["n"] > H100_SMS and c["big"] >= 8 and c["team"] >= 8 and c["longest"] > 32767 and c["orderly"], c
    r = _route(shapes, H100_SMS)
    assert r["big_team"] == c["big"] and r["rf_team"] == c["team"], (r, c)
    assert r["rampfree"] == c["n"] - c["big"] - c["team"] and r["three_way"] == 1 and r["raw"] == 0, r
    # without the 16-warp launch every problem of >= 8 Mi cells belongs to the 4-warp launch
    assert _route(shapes, H100_SMS, no_big_teams=True)["rf_team"] == c["big"] + c["team"]


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _diff(a, r):
    """Fields in which the library's record r differs from the recorded call a ([] if none); a call the reference
    failed must fail."""
    if a["threw"] or a["ret"] < 0:
        return [] if r["ret"] < 0 else ["ret"]
    pairs = (("ret", "ret"), ("score_bits", "score_bits"), ("cigar", "cigar"), ("md", "md"), ("nm", "nm"),
             ("po", "position_offset"), ("qstart", "qstart"), ("qend", "qend"))
    return [k for k, kr in pairs if a[k] != r[kr]]


def _batch(aligns, extra=()):
    from ngmlr_b200 import PackedBatch
    refs = [a["ref"] for a in aligns] + [p.ref for p in extra]
    qrys = [a["qry"] for a in aligns] + [p.qry for p in extra]
    offs = [a["off"] for a in aligns] + [p.offsets for p in extra]
    lens = [a["len"] for a in aligns] + [p.lengths for p in extra]
    qs = [a["qs"] for a in aligns] + [p.ext_qstart for p in extra]
    qe = [a["qe"] for a in aligns] + [p.ext_qend for p in extra]
    return PackedBatch(refs, qrys, offs, lens, qs, qe)


def _align(al, aligns, want_counts, extra=(), check=None):
    """BatchAlign of the recorded calls (plus `extra` problems) through both text stages: every recorded call equal to
    the reference, the counters of each batch equal to `want_counts`; `check(results, on_device)` sees the rest."""
    for on_device in (True, False):
        al.set_text_stage(on_device, False)
        before = al.debug_fill_counts()
        res = al.BatchAlign(_batch(aligns, extra))
        got = {k: v - before[k] for k, v in al.debug_fill_counts().items()}
        assert got == want_counts, (on_device, got, want_counts)
        bad = [(i, d) for i, (a, g) in enumerate(zip(aligns, res)) if (d := _diff(a, g.as_dict()))]
        assert not bad, (on_device, len(bad), bad[:5])
        if check:
            check(res, on_device)


@pytest.fixture
def make_aligner(monkeypatch):
    """B200Aligner created under the given environment (fill knobs are read when a context is created)."""
    from ngmlr_b200 import B200Aligner
    made = []

    def make(env=None):
        for k, v in (env or {}).items():
            monkeypatch.setenv(k, v)
        made.append(B200Aligner(0))
        return made[-1]

    yield make
    for a in made:
        a.close()


# ---- 1. default routing, the whole stream as one batch --------------------------------------------------------------
@needs_rec
@pytest.mark.gpu
def test_default_routing_fills_all_three_launches(stream, make_aligner, oracle):
    """No overrides: 16-warp teams, ramped 4-warp teams and the skewed two-row one-warp kernel in one fill launch, every
    call as the reference returned it, and every direction code and the best cell of two problems per launch equal to
    the oracle's."""
    shapes = _shapes(stream)
    want = _route(shapes, _num_sms())
    c = _composition(shapes)
    assert (want["big_team"], want["rf_team"], want["rampfree"]) == (c["big"], c["team"], c["n"] - c["big"] - c["team"])
    assert want["three_way"] == 1
    al = make_aligner()
    skew0 = al.debug_rampfree2_skew_problems()
    _align(al, stream, want)
    assert al.debug_rampfree2_skew_problems() - skew0 == 2 * want["rampfree"]
    assert al.stats()["fill_launches"] == 1
    # the two smallest problems of each team launch; of the one-warp launch the largest and the one with most rows
    big =[i for i, s in enumerate(shapes) if s["est"] >= BIG_CELLS and s["width"] >= BIG_WIDTH]
    team = [i for i, s in enumerate(shapes) if s["est"] >= TEAM_CELLS and s["width"] < BIG_WIDTH]
    rest = [i for i, s in enumerate(shapes) if s["est"] < TEAM_CELLS]
    by_est = lambda ix: sorted(ix, key=lambda i: shapes[i]["est"])
    longest = max(rest, key=lambda i: shapes[i]["rows"])
    picks = by_est(big)[:2] + by_est(team)[:2] + [by_est(rest)[-1], longest]
    assert len(set(picks)) == 6
    for i in picks:
        a = stream[i]
        wd, wbs, wbx, wby = oracle.fill(a["ref"], a["qry"], a["off"], a["len"])
        gd, gbs, gbx, gby = al.debug_directions(i, int(wd.size))
        assert (gbs, gbx, gby) == (wbs, wbx, wby), i
        bad = np.flatnonzero(gd != wd)
        assert bad.size == 0, (i, bad.size, bad[:8])


# ---- 2. the same batch under each knob ------------------------------------------------------------------------------
KNOBS = {
    "rows1": dict(env={"NGMLR_B200_FILL_ROWS_PER_LANE": "1"}),
    "unskewed": dict(env={"NGMLR_B200_FILL_RF2_SKEW": "0"}),
    "ramped-team0": dict(env={"NGMLR_B200_FILL_SCHEDULE": "ramped", "NGMLR_B200_FILL_TEAM": "0"},
                         route=dict(schedule="ramped", force_team=0)),
    "ramped-team1": dict(env={"NGMLR_B200_FILL_SCHEDULE": "ramped", "NGMLR_B200_FILL_TEAM": "1"},
                         route=dict(schedule="ramped", force_team=1)),
    "ramped-auto": dict(env={"NGMLR_B200_FILL_SCHEDULE": "ramped"}, route=dict(schedule="ramped")),
    "no-big-teams": dict(env={"NGMLR_B200_NO_BIG_TEAMS": "1"}, route=dict(no_big_teams=True)),
    "persistent": dict(env={"NGMLR_B200_FILL_PERSISTENT": "1"}, ctas_per_sm=1),
    "chunks100": dict(chunk=100),
    "chunks256": dict(chunk=256),   # the plugin batcher's NGMLR_B200_BATCH_MAX
}


@needs_rec
@pytest.mark.gpu
@pytest.mark.parametrize("knob", list(KNOBS))
def test_production_batch_under_each_knob(stream, make_aligner, knob):
    """Every fill knob, the persistent launch and the batch sizes the plugin sends: results as the reference returned
    them, and each launch filled what the host's estimates route to it."""
    k = KNOBS[knob]
    al = make_aligner(k.get("env"))
    if k.get("ctas_per_sm"):
        al.set_fill_ctas_per_sm(k["ctas_per_sm"])
    num_sms = _num_sms()
    chunk = k.get("chunk", len(stream))
    rows = int(k.get("env", {}).get("NGMLR_B200_FILL_ROWS_PER_LANE", "2"))
    skew = int(k.get("env", {}).get("NGMLR_B200_FILL_RF2_SKEW", "1"))
    rf0 = (al.debug_rampfree2_problems(), al.debug_rampfree2_skew_problems())
    total = dict.fromkeys(COUNTS, 0)
    for c0 in range(0, len(stream), chunk):
        part = stream[c0:c0 + chunk]
        want = _route(_shapes(part), num_sms, **k.get("route", {}))
        _align(al, part, want)
        total = _plus(total, want)
    rf2 = al.debug_rampfree2_problems() - rf0[0], al.debug_rampfree2_skew_problems() - rf0[1]
    assert rf2 == (2 * total["rampfree"] * (rows == 2), 2 * total["rampfree"] * (rows == 2 and skew == 1)), rf2
    if knob == "chunks100":      # batches of at most one problem per SM: 16-warp teams throughout
        assert total["big_team"] == len(stream) and total["multi_launch"] == 0
    elif knob in ("rows1", "unskewed", "no-big-teams", "persistent", "chunks256"):
        assert total["multi_launch"] >= 1 and total["rampfree"] > 0


# ---- 3. the RAW switch across all three launches --------------------------------------------------------------------
def _wide_rows_problems():
    """Two full-matrix problems over a 40 kb window (rows of 40 000 cells): 1.6 M cells (one-warp launch) and 8.8 M
    cells (16-warp launch)."""
    rng = np.random.default_rng(11)
    g = synth.random_genome(41000, 78)
    probs = []
    for h in (40, 220):
        q = g[20000:20000 + h].copy()
        q[rng.integers(0, h, 4)] = ord("A")
        o, l = corridor.corridor_full(h, 40000)
        probs.append(synth.AlignProblem(g[:40000].tobytes(), q.tobytes(), o, l))
    return probs


@needs_rec
@pytest.mark.gpu
def test_rows_wider_than_int16_switch_all_three_launches_to_raw(stream, make_aligner, oracle):
    """Rows wider than 32 767 cells (indelRun is a C `short` in the reference) route the whole batch to the RAW
    instantiation, in all three concurrent launches: the planted problems equal the oracle, the rest the reference."""
    planted = _wide_rows_problems()
    shapes = _shapes(stream) + [_shape(len(p.ref), p.offsets, p.lengths) for p in planted]
    assert shapes[-2]["est"] < TEAM_CELLS and shapes[-1]["est"] >= BIG_CELLS
    want = _route(shapes, _num_sms())
    assert want["raw"] == len(shapes) and want["three_way"] == 1, want
    assert want["big_team"] == _composition(shapes)["big"]
    want_planted = [oracle.single_align(p.ref, p.qry, p.offsets, p.lengths) for p in planted]

    def check(res, on_device):
        for k, w in enumerate(want_planted):
            g = res[len(stream) + k].as_dict()
            if on_device:      # nmPerPosition is not requested from the device text stage
                g["nm_positions"] = w["nm_positions"]
            assert same_alignment(w, g) == [], (on_device, k, same_alignment(w, g))

    _align(make_aligner(), stream, want, extra=planted, check=check)


# ---- 4. direction-arena overflow while three launches bump one allocator ---------------------------------------------
@needs_rec
@pytest.mark.gpu
def test_direction_arena_overflow_with_three_launches(stream, make_aligner):
    """A direction arena of 5 000 words overflows in all three launches at once: the batch is grown and re-run, every
    fill launch again three-way, and the results are unchanged."""
    al = make_aligner()
    al.debug_set_arena_words(5000)
    want = _route(_shapes(stream), _num_sms())
    for on_device in (True, False):
        al.set_text_stage(on_device, False)
        before = al.debug_fill_counts()
        res = al.BatchAlign(_batch(stream))
        got = {k: v - before[k] for k, v in al.debug_fill_counts().items()}
        launches = al.stats()["fill_launches"]
        assert launches >= 2 and got["fill_launches"] == launches, (launches, got)
        assert got["three_way"] == launches and got["multi_launch"] == launches, got
        assert {k: got[k] for k in COUNTS[:6]} == {k: want[k] for k in COUNTS[:6]}, (got, want)
        bad = [(i, d) for i, (a, g) in enumerate(zip(stream, res)) if (d := _diff(a, g.as_dict()))]
        assert not bad, (on_device, len(bad), bad[:5])


# ---- 5. routing with the 16-warp launch off --------------------------------------------------------------------------
@needs_rec
@pytest.mark.gpu
@pytest.mark.parametrize("how", ["env", "mostly-big"])
def test_team_launch_takes_every_large_problem_without_big_teams(stream, make_aligner, how):
    """With no 16-warp launch -- NGMLR_B200_NO_BIG_TEAMS, or a big-team threshold so low that most of the batch (more
    than two problems per SM) qualifies -- every problem of >= RF_TEAM_CELLS estimated cells is filled by the 4-warp
    team launch (DESIGN.md section 4.1), none by the one-warp kernel."""
    shapes = _shapes(stream)
    num_sms = _num_sms()
    n_large = sum(s["est"] >= TEAM_CELLS for s in shapes)
    if how == "env":
        al = make_aligner({"NGMLR_B200_NO_BIG_TEAMS": "1"})
        want = _route(shapes, num_sms, no_big_teams=True)
    else:
        al = make_aligner()
        # the smallest estimate among the 2 * num_sms + 20 largest problems: that many problems, most of the batch
        cells = sorted((s["est"] for s in shapes), reverse=True)[2 * num_sms + 19]
        n_big = sum(s["est"] >= cells for s in shapes)
        assert n_big > 2 * num_sms and 2 * n_big > len(shapes) and cells < TEAM_CELLS
        al.debug_set_big_team(cells, 0)
        want = _route(shapes, num_sms, big_cells=cells, big_width=0)
    assert want["big_team"] == 0 and want["rf_team"] == n_large and want["rampfree"] == len(shapes) - n_large
    _align(al, stream, want)


# ---- 6. the resident pipeline at production size ----------------------------------------------------------------------
CONTIG = 2_000_000


def _align_one(args):
    return Oracle().single_align(*args)


class _PoolBackend:
    """ngmlr_b200.intervals' backend on the CPU oracle, each attempt's problems spread over a process pool (the oracle
    fills ~33 M cells/s on one core)."""

    def __init__(self, cs_oracle, pool):
        self.cs, self.pool = cs_oracle, pool

    def decode(self, starts, seq_lens):
        return [self.cs.decode_exact(int(s), int(n)) for s, n in zip(starts, seq_lens)]

    def align(self, tasks, refs, offsets, lengths):
        args = [(r, t.read_seq, np.asarray(o, np.int32), np.asarray(l, np.int32), t.ext_qstart, t.ext_qend)
                for t, r, o, l in zip(tasks, refs, offsets, lengths)]
        return list(self.pool.map(_align_one, args, chunksize=1))


@pytest.mark.gpu
def test_resident_pipeline_at_production_size(make_aligner):
    """reads_upload -> compute_alignments on 120 SV reads and 30 long reads, a first attempt of more than one interval
    per SM that fills all three launches, against the Python mirror of computeAlignment over the oracle."""
    from ngmlr_b200 import refindex
    from ngmlr_b200.intervals import compute_alignments
    from oracle_lib import CsOracle
    genome = synth.random_genome(2 * CONTIG, 2026)
    sv_reads, sv_ivs = synth.simulate_reads(120, genome, CONTIG, 41, median=6000, sv=True)
    long_reads, long_ivs = synth.simulate_reads(30, genome, CONTIG, 42, median=20000, err=0.12, ratio=(1, 1, 1),
                                                hi=45000)
    for iv in long_ivs:
        iv.read += len(sv_reads)
    reads, ivs = sv_reads + long_reads, sv_ivs + long_ivs
    c = _composition([_shape(len(p.ref), p.offsets, p.lengths) for p in (iv.problem(genome, reads) for iv in ivs)])
    assert c["n"] > _num_sms() and c["big"] >= 8 and c["team"] >= 8, c
    enc = refindex.encode_reference([genome[:CONTIG], genome[CONTIG:]])
    g2c = lambda pos: enc.ref_start[pos // CONTIG] + pos % CONTIG
    cso = CsOracle([genome[:CONTIG].tobytes(), genome[CONTIG:].tobytes()])
    al = make_aligner()
    try:
        al.set_reference(enc)
        al.set_text_stage(True, False)
        al.reads_upload(reads)
        # the first attempt on its own: all three launches, in one fill launch
        before = al.debug_fill_counts()
        al.intervals_upload(synth.interval_tasks(ivs, reads, g2c, by_index=True))
        al.run()
        first = [r.as_dict() for r in al.fetch()]
        got1 = {k: v - before[k] for k, v in al.debug_fill_counts().items()}
        assert got1["three_way"] == 1 and got1["fill_launches"] == 1, got1
        assert got1["big_team"] >= 8 and got1["rf_team"] >= 8 and got1["rampfree"] > 0, got1
        assert got1["big_team"] + got1["rf_team"] + got1["rampfree"] == len(ivs), got1
        # every attempt, retries included
        got, calls = al.compute_alignments(synth.interval_tasks(ivs, reads, g2c, by_index=True))
        got = [g.as_dict() for g in got]
        with ProcessPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as pool:
            want, want_calls = compute_alignments(_PoolBackend(cso, pool),
                                                  synth.interval_tasks(ivs, reads, g2c, by_index=False))
        assert list(calls) == want_calls
        n_valid = 0
        for i, (w, g) in enumerate(zip(want, got)):
            assert (w is None) == (g["ret"] < 0), i
            if w is not None:
                n_valid += 1
                d = same_alignment(w, dict(g, nm_positions=w["nm_positions"]))   # nmPerPosition not requested
                assert d == [], (i, d)
            if calls[i] == 1:      # decided on the first attempt: the staged first attempt agrees
                assert (first[i]["ret"], first[i]["cigar"], first[i]["score_bits"]) == \
                    (g["ret"], g["cigar"], g["score_bits"]), i
        assert n_valid >= 0.8 * len(ivs), n_valid
    finally:
        cso.close()
