"""GPU: the corners of the skewed two-row fill's cell update (cell_update<TRIM>: the left deletion test read from the
run length, the saturating [S != 0] factor) and of its best-cell tracker. Problems built to put best-score ties inside
one unrolled 4-step block, between the two rows of a lane and across a block switch, deletion and insertion runs that
start in a lane's first column or cross a 16-step group, odd heights and 1-row problems, run under
NGMLR_B200_FILL_SCHEDULE=rampfree-all with the skewed two-row kernel, scalar and RAW scorings, short-lived and
persistent forms, against the oracle with every direction code checked."""
import numpy as np
import pytest

import cases
import test_gpu_convex as tg
from ngmlr_b200 import synth

pytestmark = pytest.mark.gpu

_BASES = np.frombuffer(b"ACGT", dtype=np.uint8)


def _seq(rng, n):
    return _BASES[rng.integers(0, 4, size=n)].tobytes()


def _band(H, W, shift=0, slope=1.0):
    offs = (np.arange(H) * slope - W // 2 + shift).astype(np.int32)
    return offs, np.full(H, W, dtype=np.int32)


def _tie_problems():
    """Many cells share the best score: periodic and single-letter sequences, and a lone match in a mismatch sea."""
    probs = []
    for H in (1, 3, 4, 5, 8, 33, 63, 64, 65, 129):
        for ref, qry in ((b"AC" * 200, b"AC" * 100), (b"A" * 300, b"A" * 150), (b"ACGT" * 80, b"ACG" * 60),
                         (b"C" * 300, b"A" * 150), (b"AAAC" * 80, b"A" * 150)):
            q = qry[:H]
            for W, sl in ((9, 1.0), (64, 1.0), (200, 1.0), (40, 0.0)):
                offs, lens = _band(H, W, shift=W // 4, slope=sl)
                probs.append(synth.AlignProblem(ref, q, offs, lens))
    return probs


def _run_problems(seed):
    """A deletion or insertion of d in 1 .. 40 characters placed at rows / columns around lane and group boundaries
    (16-step groups, 2 rows per lane, 64-row blocks)."""
    rng = np.random.default_rng(seed)
    probs = []
    for k in (0, 1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 66):
        for d in (1, 2, 3, 15, 16, 17, 40):
            ref = _seq(rng, 400)
            if (k + d) % 2:
                qry = ref[:k] + ref[k + d:k + d + 150]          # deletion: the path moves d columns right
                offs, lens = _band(min(len(qry), 150), 2 * d + 48, shift=d)
            else:
                qry = ref[:k] + _seq(rng, d) + ref[k:k + 150]   # insertion: d rows in one column
                offs, lens = _band(min(len(qry), 150), 2 * d + 48, shift=-d)
            H = min(int(rng.choice([1, 3, 17, 63, 65, 101, len(qry)])), len(qry), len(offs))
            probs.append(synth.AlignProblem(ref, qry[:H], offs[:H], lens[:H]))
    return probs


def _filled(a, n_before):
    rf, sk = a.debug_rampfree_problems() - n_before[0], a.debug_rampfree2_skew_problems() - n_before[1]
    assert rf > 0 and sk == rf


@pytest.mark.parametrize("persistent", [False, True], ids=["short-lived", "persistent"])
@pytest.mark.parametrize("raw", [False, True], ids=["scalar", "raw"])
@pytest.mark.parametrize("kind", ["ties", "runs"])
def test_fill_corners(monkeypatch, oracle, kind, raw, persistent):
    from ngmlr_b200 import B200Aligner
    monkeypatch.setenv("NGMLR_B200_FILL_SCHEDULE", "rampfree-all")
    monkeypatch.setenv("NGMLR_B200_FILL_ROWS_PER_LANE", "2")
    monkeypatch.setenv("NGMLR_B200_FILL_RF2_SKEW", "1")
    monkeypatch.setenv("NGMLR_B200_FILL_TEAM", "0")
    monkeypatch.setenv("NGMLR_B200_SMALL_BATCH_BIG_TEAMS", "0")
    sc = cases.WEIRD_SCORING if raw else tg.DEFAULT_SCORING
    a = B200Aligner(0, scoring=sc) if raw else B200Aligner(0)
    try:
        if persistent:
            a.set_fill_ctas_per_sm(1)
        probs = _tie_problems() if kind == "ties" else _run_problems(91)
        before = (a.debug_rampfree_problems(), a.debug_rampfree2_skew_problems())
        tg._compare_batch(a, oracle, probs, scoring=sc, rule=0, check_dirs=True)
        for p in probs[::17]:  # alone: a batch smaller than one CTA
            tg._compare_batch(a, oracle, [p], scoring=sc, rule=0, check_dirs=True)
        _filled(a, before)
    finally:
        a.close()
