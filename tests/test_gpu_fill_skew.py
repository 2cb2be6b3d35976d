"""GPU: the two-row ramp-free fill with the second row of each lane one column behind its first
(NGMLR_B200_FILL_RF2_SKEW=1, direction layout dir_shift 2) and with both rows in the same column (=0, dir_shift 1) give
the oracle's matrices and alignments. Every case of test_gpu_convex, the golden and property tests, both non-default
scorings (the RAW kernel), the persistent grid and the stress set of odd heights, 1-row problems, narrow, empty and
clipped corridors run under NGMLR_B200_FILL_SCHEDULE=rampfree-all with one warp per problem at both settings; each
test checks which of the two schedules filled its batches (counters of the context). The stress set also runs through
both settings side by side: score bits, best cell, cell counts, every direction code and the alignment text agree."""
import numpy as np
import pytest

import cases
import test_gpu_convex as tg
from ngmlr_b200 import PackedBatch
from test_gpu_fill_rows import _stress_problems
from test_gpu_fill_schedule import CONVEX_CASES

pytestmark = pytest.mark.gpu

SKEW = [0, 1]


def _env(monkeypatch, skew):
    monkeypatch.setenv("NGMLR_B200_FILL_SCHEDULE", "rampfree-all")
    monkeypatch.setenv("NGMLR_B200_FILL_ROWS_PER_LANE", "2")
    monkeypatch.setenv("NGMLR_B200_FILL_RF2_SKEW", str(skew))
    monkeypatch.setenv("NGMLR_B200_FILL_TEAM", "0")
    monkeypatch.setenv("NGMLR_B200_SMALL_BATCH_BIG_TEAMS", "0")


@pytest.fixture(params=SKEW, ids=[f"skew{s}" for s in SKEW])
def skew(request, monkeypatch):
    _env(monkeypatch, request.param)
    return request.param


@pytest.fixture
def aligner_skew(skew):
    from ngmlr_b200 import B200Aligner
    a = B200Aligner(0)
    yield a, skew
    a.close()


class _Filled:
    """Checks that the problems run while the context is in use went to the two-row kernel in the schedule `skew`."""

    def __init__(self, aligner, skew):
        self.a, self.skew = aligner, skew

    def _counts(self):
        return (self.a.debug_rampfree_problems(), self.a.debug_rampfree2_problems(),
                self.a.debug_rampfree2_skew_problems())

    def __enter__(self):
        self.before = self._counts()
        return self

    def __exit__(self, *exc):
        if exc[0] is not None:
            return False
        rf, rf2, sk = (b - a for a, b in zip(self.before, self._counts()))
        assert rf > 0
        assert rf2 == rf
        assert sk == (rf if self.skew else 0)
        return False


@pytest.mark.parametrize("case", CONVEX_CASES)
def test_convex_cases(aligner_skew, oracle, case):
    aligner, skew = aligner_skew
    with _Filled(aligner, skew):
        getattr(tg, case)(aligner, oracle)


def test_convex_properties_and_golden(aligner_skew):
    aligner, skew = aligner_skew
    with _Filled(aligner, skew):
        tg.test_golden_vectors_from_reference(aligner)
        tg.test_properties_at_scale(aligner)
        tg.test_empty_batch(aligner)


@pytest.mark.parametrize("sc", [cases.WEIRD_SCORING, cases.MILD_SCORING])
def test_convex_non_default_scoring(skew, oracle, sc):
    """The as-coded (RAW) kernel variant: its tail rule runs per row, on the skewed rows too."""
    from ngmlr_b200 import B200Aligner
    a = B200Aligner(0, scoring=sc)
    try:
        with _Filled(a, skew):
            tg._compare_batch(a, oracle, cases.random_problems(32, 303, max_len=900), scoring=sc, rule=0,
                              check_dirs=True)
            tg._compare_batch(a, oracle, _stress_problems(82, True)[::3], scoring=sc, rule=0, check_dirs=True)
    finally:
        a.close()


def test_grid_cap(aligner_skew, oracle):
    """The persistent form: a grid of 1 CTA per SM, every warp walks many problems."""
    aligner, skew = aligner_skew
    with _Filled(aligner, skew):
        tg.test_fill_grid_cap_does_not_change_results(aligner, oracle, 0)


@pytest.mark.parametrize("ragged", [False, True], ids=["orderly", "ragged"])
def test_stress_corridors(aligner_skew, oracle, ragged):
    aligner, skew = aligner_skew
    probs = _stress_problems(83 if ragged else 84, ragged)
    with _Filled(aligner, skew):
        tg._compare_batch(aligner, oracle, probs, check_dirs=True)
        for p in probs[::5]:
            tg._compare_batch(aligner, oracle, [p], check_dirs=True)


def _run(monkeypatch, skew, probs, persistent, scoring=None):
    """Everything a batch computes, per problem: Score bits, best cell, cells, raw directions, alignment text."""
    from ngmlr_b200 import B200Aligner
    _env(monkeypatch, skew)
    a = B200Aligner(0) if scoring is None else B200Aligner(0, scoring=scoring)
    try:
        if persistent:
            a.set_fill_ctas_per_sm(1)
        with _Filled(a, skew):
            res = a.BatchAlign(PackedBatch.from_problems(probs))
        out = []
        for i, (p, r) in enumerate(zip(probs, res)):
            d = r.as_dict()
            dirs = None
            if not (np.asarray(p.lengths) < 0).any():
                dg, bs, bx, by = a.debug_directions(i, int(np.maximum(p.lengths, 0).sum()))
                dirs = (dg.tobytes(), np.float32(bs).view(np.uint32).item(), bx, by)
            text = sorted((k, v.tobytes() if isinstance(v, np.ndarray) else repr(v)) for k, v in d.items())
            out.append((r.cells, dirs, text))
        return out
    finally:
        a.close()


@pytest.mark.parametrize("persistent", [False, True], ids=["short-lived", "persistent"])
@pytest.mark.parametrize("raw", [False, True], ids=["scalar", "raw"])
def test_skew_equals_unskewed(monkeypatch, persistent, raw):
    """Old and new schedule side by side on the same batch: identical results, cell for cell."""
    probs = _stress_problems(85, True) + _stress_problems(86, False)[::2] + cases.edge_problems()
    sc = cases.WEIRD_SCORING if raw else None
    old = _run(monkeypatch, 0, probs, persistent, sc)
    new = _run(monkeypatch, 1, probs, persistent, sc)
    bad = [i for i, (o, n) in enumerate(zip(old, new)) if o != n]
    assert not bad, f"{len(bad)} of {len(probs)} problems differ, first {bad[:5]}"
