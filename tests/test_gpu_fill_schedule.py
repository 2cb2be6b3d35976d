"""GPU: the ramp-free fill schedule and the ramped one give the oracle's matrices and alignments. Every case of
test_gpu_convex runs under
- NGMLR_B200_FILL_SCHEDULE=ramped with one warp per problem (NGMLR_B200_FILL_TEAM=0), 4-warp teams (=1) and the
  automatic choice;
- =rampfree (the default: the ramp-free kernel for batches whose corridors are mostly >= 128 columns wide), automatic;
- =rampfree-all (the ramp-free kernel for every batch, whatever its widths) with one warp per problem, and automatic
  with the ramp-free schedule's team threshold lowered to 1.5 M cells (its largest problems then go to the concurrent
  4-warp team launch, the rest to the ramp-free kernel).
In the rampfree-all modes the tests check that the ramp-free kernel filled the batches (a counter of the context).
The regular kernels fill every batch (small batches are not handed to the 16-warp teams here). New corridors stress
the ramp-free placement rules."""
import numpy as np
import pytest

import cases
import test_gpu_convex as tg
from ngmlr_b200 import synth

pytestmark = pytest.mark.gpu

MODES = [("ramped", "warp"), ("ramped", "team"), ("ramped", "auto"), ("rampfree", "auto"),
         ("rampfree-all", "warp"), ("rampfree-all", "auto")]


@pytest.fixture(params=MODES, ids=[f"{s}-{m}" for s, m in MODES])
def sched(request, monkeypatch):
    """(aligner, team, forced): the environment every aligner of the test is created under, one such aligner,
    its NGMLR_B200_FILL_TEAM value (-1: automatic) and whether the ramp-free kernel is forced."""
    from ngmlr_b200 import B200Aligner
    schedule, mode = request.param
    monkeypatch.setenv("NGMLR_B200_FILL_SCHEDULE", schedule)
    monkeypatch.setenv("NGMLR_B200_SMALL_BATCH_BIG_TEAMS", "0")
    if mode == "auto":
        monkeypatch.delenv("NGMLR_B200_FILL_TEAM", raising=False)
        monkeypatch.setenv("NGMLR_B200_RF_TEAM_CELLS", "1500000")
        team = -1
    else:
        team = 1 if mode == "team" else 0
        monkeypatch.setenv("NGMLR_B200_FILL_TEAM", str(team))
    a = B200Aligner(0)
    yield a, team, schedule == "rampfree-all"
    a.close()


# the cases of test_gpu_convex that take (aligner, oracle) or (aligner)
CONVEX_CASES = [
    "test_small_random_with_direction_matrix",
    "test_edge_cases",
    "test_random_default_scoring",
    "test_single_align_matches_batch",
    "test_raw_kernel_equals_scalar_kernel_on_default_scoring",
    "test_pacbio_shaped_reads",
    "test_direction_arena_overflow_is_recovered",
    "test_rows_wider_than_int16_use_the_as_coded_kernel",
    "test_big_team_fill_is_bit_exact",
]


@pytest.mark.parametrize("case", CONVEX_CASES)
def test_convex_cases(sched, oracle, case):
    aligner, team, forced = sched
    before = aligner.debug_rampfree_problems()
    getattr(tg, case)(aligner, oracle)
    if forced and team == 0:  # one warp per problem: every problem outside the 16-warp teams is ramp-free
        assert aligner.debug_rampfree_problems() > before


def test_convex_properties_and_golden(sched):
    aligner, team, forced = sched
    before = aligner.debug_rampfree_problems()
    tg.test_golden_vectors_from_reference(aligner)
    tg.test_properties_at_scale(aligner)
    tg.test_empty_batch(aligner)
    if forced:
        assert aligner.debug_rampfree_problems() > before


@pytest.mark.parametrize("sc", [cases.WEIRD_SCORING, cases.MILD_SCORING])
def test_convex_non_default_scoring(sched, oracle, sc):
    tg.test_non_default_scoring_uses_as_coded_sse_semantics(oracle, sc)


def test_convex_team_and_grid_cap(sched, oracle):
    aligner, team, forced = sched
    for t in ([0, 1] if team < 0 else [team]):
        tg.test_both_fill_schedules_are_bit_exact(aligner, oracle, t)
        before = aligner.debug_rampfree_problems()
        # a persistent grid of 1 CTA per SM: every warp of the ramp-free kernel walks many problems
        tg.test_fill_grid_cap_does_not_change_results(aligner, oracle, t)
        if forced and t == 0:
            assert aligner.debug_rampfree_problems() - before >= 300


def _noisy_copy(rng, ref, start, n, slope):
    """A read of n bases that follows ref from `start` at `slope` reference columns per read base, 10 % substituted."""
    idx = np.clip((start + slope * np.arange(n)).astype(np.int64), 0, len(ref) - 1)
    q = np.frombuffer(ref, dtype=np.uint8)[idx].copy()
    sub = rng.random(n) < 0.1
    q[sub] = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=int(sub.sum()))
    return q.tobytes()


def _stress_problems(seed, orderly):
    """Corridors for the ramp-free rules: rows clipped at 0 and at refLen, widths below 32 * (1 + slope), slopes
    0 .. 3 columns per row, single-row and single-block problems; not orderly: decreasing offsets and rows of
    varying length too (one warp per problem)."""
    rng = np.random.default_rng(seed)
    probs = []
    for H in (1, 2, 31, 32, 33, 63, 65, 200, 700):
        for W in (1, 7, 30, 61, 90, 200, 500):
            slope = float(rng.choice([0.0, 0.5, 0.93, 1.0, 1.07, 2.0, 3.0]))
            if not orderly and rng.random() < 0.5:
                slope = -slope
            ref_len = int(max(W, abs(slope) * H) + rng.integers(1, 400))
            ref = synth.random_genome(ref_len, int(rng.integers(1 << 30))).tobytes()
            start = int(rng.integers(-W - 20, ref_len // 2 + 1))   # negative: rows clipped at 0
            offs = (start + slope * np.arange(H)).astype(np.int32)
            lens = np.full(H, W, dtype=np.int32)
            if not orderly:
                lens = np.maximum(1, W + rng.integers(-W // 2, W // 2 + 1, size=H)).astype(np.int32)
            qry = _noisy_copy(rng, ref, max(start + W // 2, 0), H, max(slope, 0.0))
            probs.append(synth.AlignProblem(ref, qry, offs, lens))
    return probs


@pytest.mark.parametrize("orderly", [True, False], ids=["orderly", "ragged"])
def test_stress_corridors(sched, oracle, orderly):
    aligner, _team, forced = sched
    probs = _stress_problems(71 if orderly else 72, orderly)
    before = aligner.debug_rampfree_problems()
    tg._compare_batch(aligner, oracle, probs, check_dirs=True)
    # the same problems alone: a batch smaller than one CTA, single problems
    for p in probs[::9]:
        tg._compare_batch(aligner, oracle, [p], check_dirs=True)
    if forced:  # every problem here is far below the team threshold
        assert aligner.debug_rampfree_problems() - before == len(probs) + len(probs[::9])
