"""GPU: the ramp-free fill with two rows per lane (64-row blocks) and with one (32-row blocks) give the oracle's
matrices and alignments. Every case of test_gpu_convex, the golden and property tests and the non-default scorings
run under NGMLR_B200_FILL_SCHEDULE=rampfree-all with one warp per problem and NGMLR_B200_FILL_ROWS_PER_LANE=1 and =2;
each test checks which of the two kernels filled its batches (counters of the context). A stress set of odd and even
heights around the 64-row block, every slope from -3 to 3, clipped and ragged rows compares every direction code, so
the traceback's and the debug reader's view of the two-row direction layout is checked cell by cell."""
import numpy as np
import pytest

import cases
import test_gpu_convex as tg
from ngmlr_b200 import synth
from test_gpu_fill_schedule import CONVEX_CASES

pytestmark = pytest.mark.gpu

ROWS = [1, 2]


def _env(monkeypatch, rows):
    monkeypatch.setenv("NGMLR_B200_FILL_SCHEDULE", "rampfree-all")
    monkeypatch.setenv("NGMLR_B200_FILL_ROWS_PER_LANE", str(rows))
    monkeypatch.setenv("NGMLR_B200_FILL_TEAM", "0")
    monkeypatch.setenv("NGMLR_B200_SMALL_BATCH_BIG_TEAMS", "0")


@pytest.fixture(params=ROWS, ids=[f"rows{r}" for r in ROWS])
def rows(request, monkeypatch):
    _env(monkeypatch, request.param)
    return request.param


@pytest.fixture
def aligner_rows(rows):
    from ngmlr_b200 import B200Aligner
    a = B200Aligner(0)
    yield a, rows
    a.close()


class _Filled:
    """Checks that the problems run while the context is in use went to the kernel with `rows` rows per lane."""

    def __init__(self, aligner, rows):
        self.a, self.rows = aligner, rows

    def __enter__(self):
        self.rf, self.rf2 = self.a.debug_rampfree_problems(), self.a.debug_rampfree2_problems()
        return self

    def __exit__(self, *exc):
        if exc[0] is not None:
            return False
        rf = self.a.debug_rampfree_problems() - self.rf
        rf2 = self.a.debug_rampfree2_problems() - self.rf2
        assert rf > 0
        assert rf2 == (rf if self.rows == 2 else 0)
        return False


# test_direction_arena_overflow_is_recovered among them: a too-small arena, ST_DIR_OVERFLOW, grown and re-run
@pytest.mark.parametrize("case", CONVEX_CASES)
def test_convex_cases(aligner_rows, oracle, case):
    aligner, rows = aligner_rows
    with _Filled(aligner, rows):
        getattr(tg, case)(aligner, oracle)


def test_convex_properties_and_golden(aligner_rows):
    aligner, rows = aligner_rows
    with _Filled(aligner, rows):
        tg.test_golden_vectors_from_reference(aligner)
        tg.test_properties_at_scale(aligner)
        tg.test_empty_batch(aligner)


@pytest.mark.parametrize("sc", [cases.WEIRD_SCORING, cases.MILD_SCORING])
def test_convex_non_default_scoring(rows, oracle, sc):
    """The as-coded (RAW) kernel variant: its tail rule runs per row."""
    from ngmlr_b200 import B200Aligner
    a = B200Aligner(0, scoring=sc)
    try:
        with _Filled(a, rows):
            tg._compare_batch(a, oracle, cases.random_problems(32, 303, max_len=900), scoring=sc, rule=0,
                              check_dirs=True)
    finally:
        a.close()


def test_grid_cap(aligner_rows, oracle):
    """The persistent form: a grid of 1 CTA per SM, every warp walks many problems."""
    aligner, rows = aligner_rows
    with _Filled(aligner, rows):
        tg.test_fill_grid_cap_does_not_change_results(aligner, oracle, 0)


def _noisy_copy(rng, ref, start, n, slope):
    """A read of n bases that follows ref from `start` at `slope` reference columns per read base, 10 % substituted."""
    idx = np.clip((start + slope * np.arange(n)).astype(np.int64), 0, len(ref) - 1)
    q = np.frombuffer(ref, dtype=np.uint8)[idx].copy()
    sub = rng.random(n) < 0.1
    q[sub] = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=int(sub.sum()))
    return q.tobytes()


def _stress_problems(seed, ragged):
    """Heights around the 64-row block (odd ones leave the last lane's second row outside the matrix), widths 1 ..
    500, slopes -3 .. 3 columns per row, rows clipped at 0 and at refLen; ragged: row lengths vary too."""
    rng = np.random.default_rng(seed)
    probs = []
    slopes = [-3.0, -2.0, -1.0, -0.5, 0.0, 0.5, 0.93, 1.0, 1.07, 2.0, 3.0]
    for H in (1, 2, 63, 64, 65, 127, 128, 129, 200, 701):
        for W in (1, 7, 30, 61, 90, 200, 500):
            slope = float(rng.choice(slopes))
            ref_len = int(max(W, abs(slope) * H) + rng.integers(1, 400))
            ref = synth.random_genome(ref_len, int(rng.integers(1 << 30))).tobytes()
            start = int(rng.integers(-W - 20, ref_len // 2 + 1))  # negative: rows clipped at 0
            if slope < 0:
                start = int(rng.integers(ref_len // 2, ref_len + 20))  # beyond refLen: rows clipped there
            offs = (start + slope * np.arange(H)).astype(np.int32)
            lens = np.full(H, W, dtype=np.int32)
            if ragged:
                lens = np.maximum(1, W + rng.integers(-W // 2, W // 2 + 1, size=H)).astype(np.int32)
            qry = _noisy_copy(rng, ref, max(start + W // 2, 0), H, max(slope, 0.0))
            probs.append(synth.AlignProblem(ref, qry, offs, lens))
    return probs


@pytest.mark.parametrize("ragged", [False, True], ids=["orderly", "ragged"])
def test_stress_corridors(aligner_rows, oracle, ragged):
    aligner, rows = aligner_rows
    probs = _stress_problems(81 if ragged else 80, ragged)
    with _Filled(aligner, rows):
        tg._compare_batch(aligner, oracle, probs, check_dirs=True)
        # the same problems alone: a batch smaller than one CTA, single problems
        for p in probs[::7]:
            tg._compare_batch(aligner, oracle, [p], check_dirs=True)
