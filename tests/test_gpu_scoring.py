"""GPU: the convex path at ngmlr's scoring options (tests/scoring_cases.py), against the oracle's as-coded rule 0 and
the reference's vectors in scoring_golden.json.

- every scoring, automatic kernel choice: results, cell counts, every direction code and the best cell of random,
  edge and stress problems; the golden records; and which kernel the batch got (the RAW routing counter against
  scoring_cases.needs_raw);
- every scoring with the RAW kernel forced, and every in-class scoring at ordinary magnitude with the scalar-rule
  kernel forced (the class claim, checked on the device);
- every fill instantiation (ramped, ramp-free with its team launch, one and two rows per lane, skewed or not, the
  persistent grid, 4-warp and 16-warp teams) at two in-class scorings and one outside the class, each checked by the
  routing counters to have filled the problems;
- large magnitudes: long problems whose scores reach millions at a scoring on the class boundary go to the RAW kernel
  and match; forced onto the scalar-rule kernel they give the scalar rule, which is not ngmlr's result; short problems
  at the same scoring, margin 2 on the long ones, and default-scoring pacbio batches stay on the scalar-rule kernel;
- the resident path (compute_alignments with its retries) against ngmlr_b200.intervals over the oracle;
- whole ngmlr runs with the scoring flags: the plain binary and the plugin-linked one write identical SAM records."""
import os
import subprocess
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

import cases
import cs_cases
import e2e_data
import golden_util as gu
import scoring_cases as S
from ngmlr_b200 import B200Aligner, PackedBatch, _lib, synth
from oracle_lib import Oracle, same_alignment
from test_gpu_fill_rows import _stress_problems

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDS = [c.name for c in S.SCORINGS]


# ---- oracle results, computed once per (scoring, problem set) on a process pool -------------------------------------
def _oracle_one(args):
    p, sc, rule = args
    o = Oracle()
    w = o.single_align(p.ref, p.qry, p.offsets, p.lengths, p.ext_qstart, p.ext_qend, scoring=sc, rule=rule)
    if (np.asarray(p.lengths) < 0).any():
        return w, None   # negative lengths: the direction layout is not comparable cell by cell
    d, bs, bx, by = o.fill(p.ref, p.qry, p.offsets, p.lengths, sc, rule)
    return w, (d, int(np.float32(bs).view(np.uint32)), bx, by)


_WANT = {}


def _want(key, probs, sc, rule=0):
    if (key, sc, rule) not in _WANT:
        with ProcessPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:
            _WANT[key, sc, rule] = list(ex.map(_oracle_one, [(p, sc, rule) for p in probs], chunksize=1))
    return _WANT[key, sc, rule]


def _mixed(case):
    """Random problems (anchored, narrow, full and linear corridors, N runs), the edge problems, ragged stress shapes."""
    s = sum(case.name.encode())
    return (cases.random_problems(16, 60 + s, max_len=900) + cases.edge_problems()
            + _stress_problems(70 + s, True)[::4])


def _orderly(case):
    """Monotone corridors with no empty row (the team kernels' precondition), most of them >= 128 columns wide."""
    s = sum(case.name.encode())
    return (cases.random_problems(24, 80 + s, max_len=1800, modes=(0, 2, 3))
            + synth.pacbio_problems(4, genome_len=300_000, seed=13, median=4000))


class _Counts:
    """Routing counters of the problems a block of code filled (B200Aligner.debug_fill_counts, rampfree2, skew)."""

    def __init__(self, a):
        self.a = a

    def _now(self):
        c = self.a.debug_fill_counts()
        c["rf2"], c["skew"] = self.a.debug_rampfree2_problems(), self.a.debug_rampfree2_skew_problems()
        return c

    def __enter__(self):
        self.before = self._now()
        return self

    def __exit__(self, *exc):
        after = self._now()
        self.d = {k: after[k] - self.before[k] for k in after}
        return False


def _check(a, probs, want, what, dirs=True):
    """One BatchAlign of `probs` against the oracle's results: every ALIGN_KEYS field, nmPerPosition, status, cells,
    and (dirs) every direction code and the best cell."""
    res = list(a.BatchAlign(PackedBatch.from_problems(probs)))
    assert len(res) == len(probs)
    bad = []
    for i, (p, r, (w, wf)) in enumerate(zip(probs, res, want)):
        got = r.as_dict()
        d = same_alignment(w, got)
        if w["status"] != got["status"]:
            d.append("status")
        if r.cells != p.cells:
            d.append("cells")
        if dirs and wf is not None:
            dg, bs, bx, by = a.debug_directions(i, int(wf[0].size))
            if not np.array_equal(dg, wf[0]):
                k = np.flatnonzero(dg != wf[0])
                d.append(f"dirs ({k.size} cells, first {int(k[0])}: gpu {dg[k[0]]} oracle {wf[0][k[0]]})")
            if (int(np.float32(bs).view(np.uint32)), bx, by) != wf[1:]:
                d.append(f"best gpu {(bs, bx, by)} oracle {wf[1:]}")
        if d:
            bad.append((i, d, w["ret"], got["ret"]))
    assert not bad, f"{what}: {len(bad)} of {len(probs)} problems differ: {bad[:5]}"
    return res


def _raw_expected(sc, probs):
    return len(probs) if S.needs_raw(sc, probs) else 0


# ---- 1. automatic kernel choice, every scoring ----------------------------------------------------------------------
@pytest.mark.parametrize("case", S.SCORINGS, ids=IDS)
def test_automatic_routing(case):
    probs = _mixed(case)
    want = _want(("mixed", case.name), probs, case.sc)
    (_c, gprobs, grecs), = [s for s in S.golden_sets() if s[0] is case]
    a = B200Aligner(0, scoring=case.sc)
    try:
        with _Counts(a) as c:
            _check(a, probs, want, case.name)
        assert c.d["raw"] == _raw_expected(case.sc, probs)
        with _Counts(a) as c:
            res = list(a.BatchAlign(PackedBatch.from_problems(gprobs)))
            for i, (p, r, rec) in enumerate(zip(gprobs, res, grecs)):
                gu.check_against_record(r.as_dict(), rec, f"{case.name} golden[{i}]")
                if not (np.asarray(p.lengths) < 0).any():
                    dg, bs, bx, by = a.debug_directions(i, int(np.maximum(p.lengths, 0).sum()))
                    assert gu.digest(np.asarray(dg, np.uint8)) == rec["dirs_sha"], (case.name, i)
                    assert [int(np.float32(bs).view(np.uint32)), bx, by] == rec["best"], (case.name, i)
        assert c.d["raw"] == _raw_expected(case.sc, gprobs)
    finally:
        a.close()


# ---- 2. forced kernels ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", S.SCORINGS, ids=IDS)
def test_forced_kernels(case):
    """The RAW kernel equals rule 0 at every scoring; the scalar-rule kernel does at every in-class scoring at
    ordinary magnitude (these problems)."""
    probs = _mixed(case)
    want = _want(("mixed", case.name), probs, case.sc)
    a = B200Aligner(0, scoring=case.sc)
    try:
        a.force_raw(1)
        with _Counts(a) as c:
            _check(a, probs, want, f"{case.name} RAW")
        assert c.d["raw"] == len(probs)
        if case.in_class:
            assert not S.needs_raw(case.sc, probs)
            a.force_raw(0)
            with _Counts(a) as c:
                _check(a, probs, want, f"{case.name} scalar")
            assert c.d["raw"] == 0
    finally:
        a.close()


# ---- 3. every fill instantiation at non-default scorings ------------------------------------------------------------
BASE_ENV = {"NGMLR_B200_SMALL_BATCH_BIG_TEAMS": "0"}
RF_ALL = dict(BASE_ENV, NGMLR_B200_FILL_SCHEDULE="rampfree-all", NGMLR_B200_FILL_TEAM="0")
RF_TEAM_CELLS = 1_000_000
CONFIGS = {
    # name: (environment, problem set, aligner set-up, expected counters as a function of the problem set)
    "ramped": (dict(BASE_ENV, NGMLR_B200_FILL_SCHEDULE="ramped", NGMLR_B200_FILL_TEAM="0"), _mixed, None,
               lambda ps: {"ramped_warp": len(ps), "rampfree": 0}),
    "rampfree-teams": (dict(BASE_ENV, NGMLR_B200_FILL_SCHEDULE="rampfree", NGMLR_B200_RF_TEAM_CELLS=str(RF_TEAM_CELLS)),
                       _orderly, None,
                       lambda ps: {"rf_team": sum(_est(p) >= RF_TEAM_CELLS for p in ps),
                                   "rampfree": sum(_est(p) < RF_TEAM_CELLS for p in ps)}),
    "rows1": (dict(RF_ALL, NGMLR_B200_FILL_ROWS_PER_LANE="1"), _mixed, None,
              lambda ps: {"rampfree": len(ps), "rf2": 0}),
    "rows2-skew0": (dict(RF_ALL, NGMLR_B200_FILL_ROWS_PER_LANE="2", NGMLR_B200_FILL_RF2_SKEW="0"), _mixed, None,
                    lambda ps: {"rampfree": len(ps), "rf2": len(ps), "skew": 0}),
    "rows2-skew1": (dict(RF_ALL, NGMLR_B200_FILL_ROWS_PER_LANE="2", NGMLR_B200_FILL_RF2_SKEW="1"), _mixed, None,
                    lambda ps: {"rampfree": len(ps), "rf2": len(ps), "skew": len(ps)}),
    "persistent": (dict(RF_ALL, NGMLR_B200_FILL_PERSISTENT="1"), _mixed, None,
                   lambda ps: {"rampfree": len(ps), "skew": len(ps)}),
    "team4": (BASE_ENV, _orderly, lambda a: a.force_team(1),
              lambda ps: {"ramped_team": len(ps), "rampfree": 0, "big_team": 0}),
    "team16": (BASE_ENV, _orderly, lambda a: a.debug_set_big_team(150_000, 100),
               lambda ps: {"big_team": sum(_est(p) >= 150_000 and _width(p) >= 100 for p in ps)}),
}
INSTANCE_SCORINGS = [S.BY_NAME["ont_like"], S.BY_NAME["fractional"], S.BY_NAME["mild"]]


def _est(p):
    return int(np.maximum(np.asarray(p.lengths, np.int64), 0).sum())


def _width(p):
    return min(int(np.max(p.lengths)), len(p.ref))


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("case", INSTANCE_SCORINGS, ids=[c.name for c in INSTANCE_SCORINGS])
def test_fill_instantiations(monkeypatch, case, config):
    env, make, setup, expect = CONFIGS[config]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    probs = make(case)
    want = _want((make.__name__, case.name), probs, case.sc)
    exp = expect(probs)
    assert sum(exp.values()) > 0
    a = B200Aligner(0, scoring=case.sc)
    try:
        if setup:
            setup(a)
        with _Counts(a) as c:
            _check(a, probs, want, f"{case.name} {config}")
        got = {k: c.d[k] for k in exp}
        assert got == exp, (config, got, exp)
        assert c.d["raw"] == (0 if case.in_class else len(probs))
    finally:
        a.close()


# ---- 4. large magnitudes --------------------------------------------------------------------------------------------
def test_large_magnitude_boundary_scoring():
    """(512,-64,-32.125,-32.125,-32.125,0.5): the long problems (scores 3.3 M - 8.4 M) go to the RAW kernel and equal
    rule 0; forced onto the scalar-rule kernel they give rule 1 cell for cell -- which differs from rule 0 in tens of
    thousands of direction codes and in every alignment. Short problems stay on the scalar-rule kernel; one long problem
    moves its whole batch."""
    sc = S.LARGE.sc
    rep = S.reproducer()
    short = cases.random_problems(16, 31, max_len=1500)
    want_rep = _want("reproducer", rep, sc)
    want_rep1 = _want("reproducer", rep, sc, rule=1)
    want_short = _want("short", short, sc)
    a = B200Aligner(0, scoring=sc)
    try:
        with _Counts(a) as c:
            _check(a, rep, want_rep, "reproducer")
        assert c.d["raw"] == len(rep)
        a.force_raw(0)
        with _Counts(a) as c:
            _check(a, rep, want_rep1, "reproducer, scalar-rule kernel forced")
        assert c.d["raw"] == 0
        for (w0, f0), (w1, f1) in zip(want_rep, want_rep1):
            assert same_alignment(w0, w1) != [] and int((f0[0] != f1[0]).sum()) > 10_000
        a.force_raw(-1)
        with _Counts(a) as c:
            _check(a, short, want_short, "short problems")
        assert c.d["raw"] == 0
        with _Counts(a) as c:
            _check(a, short + rep[:1], want_short + want_rep[:1], "short problems + one long")
        assert c.d["raw"] == len(short) + 1
    finally:
        a.close()


def test_large_magnitude_margin2_stays_scalar():
    sc = S.BY_NAME["large_margin2"].sc
    rep = S.reproducer()
    a = B200Aligner(0, scoring=sc)
    try:
        with _Counts(a) as c:
            _check(a, rep, _want("reproducer", rep, sc), "reproducer at margin 2")
        assert c.d["raw"] == 0
    finally:
        a.close()


def test_default_scoring_pacbio_batch_stays_scalar():
    """Production-shaped work at the default scoring keeps the scalar-rule kernel."""
    probs = synth.pacbio_problems(24, genome_len=2_000_000, seed=9, median=8000)
    a = B200Aligner(0)
    try:
        with _Counts(a) as c:
            _check(a, probs, _want("pacbio24", probs, S.BY_NAME["default"].sc), "pacbio", dirs=False)
        assert c.d["raw"] == 0
    finally:
        a.close()


# ---- 5. the resident path -------------------------------------------------------------------------------------------
class _ScoredOracleBackend:
    """test_cs_oracle._OracleBackend at a given scoring."""

    def __init__(self, cs_oracle, oracle, scoring):
        self.cs, self.o, self.sc = cs_oracle, oracle, scoring

    def decode(self, starts, seq_lens):
        return [self.cs.decode_exact(int(s), int(n)) for s, n in zip(starts, seq_lens)]

    def align(self, tasks, refs, offsets, lengths):
        return [self.o.single_align(r, t.read_seq, o, l, t.ext_qstart, t.ext_qend, scoring=self.sc)
                for t, r, o, l in zip(tasks, refs, offsets, lengths)]


@pytest.mark.parametrize("case", [S.BY_NAME["ont_like"], S.BY_NAME["mild"]], ids=["ont_like", "mild"])
def test_resident_path(oracle, case):
    """compute_alignments (windows decoded on the device, corridors per attempt, retries inside the call) against the
    same host logic over the oracle: results and the number of SingleAlign calls per interval."""
    from ngmlr_b200 import refindex
    from ngmlr_b200.intervals import compute_alignments
    from oracle_lib import CsOracle
    from test_cs_oracle import _interval_tasks
    contigs = cs_cases.genome_contigs()
    orc = CsOracle([c.tobytes() for c in contigs])
    enc = refindex.encode_reference(contigs)
    a = B200Aligner(0, scoring=case.sc)
    try:
        a.set_reference(enc)
        a.set_text_stage(True, want_nm_positions=True)
        with _Counts(a) as c:
            got, calls = a.compute_alignments(_interval_tasks(contigs, enc))
        assert (c.d["raw"] == 0) == case.in_class
        want, want_calls = compute_alignments(_ScoredOracleBackend(orc, oracle, case.sc), _interval_tasks(contigs, enc))
        assert list(calls) == list(want_calls)
        assert max(want_calls) > 1   # some intervals were retried
        n_valid = 0
        for i, (w, g) in enumerate(zip(want, got)):
            assert (w is None) == (g.ret < 0), i
            if w is not None:
                n_valid += 1
                assert same_alignment(w, g.as_dict()) == [], i
        assert n_valid >= len(want) // 2
    finally:
        a.close()
        orc.close()


# ---- 6. whole ngmlr runs with the scoring flags ---------------------------------------------------------------------
PLAIN = os.path.join(ROOT, "oracle", "_ref", "ngmlr")
SWAPPED = os.path.join(ROOT, "oracle", "_ref", "ngmlr_b200")
needs_bins = pytest.mark.skipif(not (os.path.exists(PLAIN) and os.path.exists(SWAPPED)),
                                reason="oracle/_ref/ngmlr{,_b200} not built (needs the reference sources at build time)")


def _ngmlr(tmp_path, name, exe, sc, threads="1", extra=None):
    ref, fq = e2e_data.write_dataset(str(tmp_path))
    sam = str(tmp_path / f"{name}.sam")
    env = dict(os.environ, NGMLR_B200_LIB=_lib.LIB_PATH, **(extra or {}))
    r = subprocess.run([exe, "-r", ref, "-q", fq, "-o", sam, "-t", threads, "--skip-write", "--no-progress"]
                       + S.cli_flags(sc), capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    return e2e_data.sam_records(sam)


def _max_as(records):
    return max((int(f[5:]) for rec in records for f in rec.split("\t") if f.startswith("AS:i:")), default=0)


@needs_bins
@pytest.mark.parametrize("case", [S.BY_NAME["ont_like"], S.BY_NAME["mild"], S.LARGE],
                         ids=["ont_like", "mild", "large_margin_quarter"])
def test_ngmlr_sam_identical_at_scoring(tmp_path, case):
    cpu = _ngmlr(tmp_path, "cpu", PLAIN, case.sc)
    gpu = _ngmlr(tmp_path, "b200", SWAPPED, case.sc)
    assert len(cpu) >= 24 and len(cpu) == len(gpu)
    for a, b in zip(cpu, gpu):
        assert a == b, f"SAM record differs:\nCPU : {a[:300]}\nB200: {b[:300]}"
    if case.large:
        assert _max_as(cpu) >= 2 ** 21   # the run reaches the magnitudes where the kernel choice matters


@needs_bins
def test_ngmlr_cross_thread_batcher_at_large_scoring(tmp_path):
    """8 worker threads whose SingleAlign calls the plugin batches (the batcher's context takes the scoring of its
    first client) at the boundary scoring: the records of the single-threaded CPU run, compared sorted."""
    sc = S.LARGE.sc
    cpu = sorted(_ngmlr(tmp_path, "cpu", PLAIN, sc))
    gpu = sorted(_ngmlr(tmp_path, "b200", SWAPPED, sc, threads="8", extra={"NGMLR_B200_BATCH_WINDOW_US": "300"}))
    assert len(cpu) >= 24 and cpu == gpu
    assert _max_as(cpu) >= 2 ** 21
