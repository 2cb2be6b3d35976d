"""Scorings the convex path is tested at, and a restatement of how the library picks its fill kernel for them.

ngmlr passes six options to the aligner (--match, --mismatch, --gap-open, --gap-extend-max, --gap-extend-min,
--gap-decay); its argument parser flips signs so that match >= 0, decay >= 0 and the other four are <= 0. The C ABI
takes any floats. From the scoring and the size of a batch's problems the library picks the scalar-rule fill kernel
or the as-coded (RAW) one (ngmlr_b200/csrc/capi.cu scoring_needs_raw); `needs_raw` below is the same rule."""
import math
from dataclasses import dataclass

import numpy as np

import cases
from oracle_lib import DEFAULT_SCORING


@dataclass(frozen=True)
class ScoringCase:
    name: str
    sc: tuple          # match, mismatch, gap open, gap extend (max), gap extend min, decay
    in_class: bool     # the scalar-rule kernel equals the SSE fill at ordinary score magnitudes
    cli: bool          # reachable from ngmlr's command line
    large: bool = False  # scores of a few kb reads reach millions


SCORINGS = [
    ScoringCase("default", DEFAULT_SCORING, True, True),
    ScoringCase("margin3", (3.0, -4.0, -6.0, -4.0, -1.0, 0.1), True, True),
    ScoringCase("ont_like", (3.0, -3.0, -4.0, -2.0, -0.5, 0.3), True, True),
    ScoringCase("fractional", (1.5, -2.75, -3.125, -2.5, -0.375, 0.0625), True, True),
    ScoringCase("decay0", (2.0, -5.0, -5.0, -5.0, -1.0, 0.0), True, True),
    ScoringCase("extmin_below_ext", (2.0, -4.0, -5.0, -1.0, -3.0, 0.2), True, True),
    ScoringCase("match0", (0.0, -4.0, -5.0, -3.0, -1.0, 0.1), True, True),
    ScoringCase("mismatch0", (2.0, 0.0, -3.0, -2.0, -1.0, 0.1), True, True),
    ScoringCase("margin_quarter", (2.0, -5.0, -2.625, -2.625, -2.625, 0.15), True, True),
    ScoringCase("negative_decay", (2.0, -5.0, -5.0, -5.0, -1.0, -0.05), True, False),
    ScoringCase("margin_0.2", (2.0, -5.0, -2.6, -2.6, -2.6, 0.15), False, True),
    ScoringCase("weird", cases.WEIRD_SCORING, False, True),
    ScoringCase("mild", cases.MILD_SCORING, False, True),
    ScoringCase("large_margin_quarter", (512.0, -64.0, -32.125, -32.125, -32.125, 0.5), True, True, True),
    ScoringCase("large_margin2", (512.0, -64.0, -33.0, -33.0, -33.0, 0.5), True, True, True),
]
BY_NAME = {c.name: c for c in SCORINGS}
LARGE = BY_NAME["large_margin_quarter"]


def reproducer():
    """Three pacbio-shaped problems whose scores reach 3.3 M, 4.0 M and 8.4 M at LARGE's scoring: there the scalar
    rule differs from the reference's fill, so the library must route them to the RAW kernel."""
    from ngmlr_b200 import synth
    return synth.pacbio_problems(3, genome_len=200_000, seed=4, median=9000)


def golden_problems(case):
    """The problems of tests/golden/scoring_golden.json for one scoring: seeded random problems, every second edge
    problem, and for the large-magnitude scorings the reproducer."""
    seed = 900 + sum(case.name.encode())
    probs = cases.random_problems(6, seed, max_len=900) + cases.edge_problems()[::2]
    return probs + (reproducer() if case.large else [])


def golden_sets():
    """[(ScoringCase, problems, records)] of tests/golden/scoring_golden.json, inputs regenerated and checked."""
    import golden_util as gu
    g = gu.load("scoring_golden.json")
    assert sorted(g) == sorted(BY_NAME), "scoring table and golden file differ"
    out = []
    for case in SCORINGS:
        blob = g[case.name]
        assert tuple(blob["scoring"]) == tuple(case.sc)
        probs = golden_problems(case)
        assert len(probs) == len(blob["records"])
        for p, r in zip(probs, blob["records"]):
            assert gu.digest(p.ref, p.qry, p.offsets, p.lengths) == r["input_sha"], "generator drifted"
        out.append((case, probs, blob["records"]))
    return out


def cli_flags(sc):
    """ngmlr's command-line options for a scoring (sign-exact: the parser keeps values of the right sign as given)."""
    mat, mis, go, ge, gemin, decay = sc
    return ["--match", repr(mat), "--mismatch", repr(mis), "--gap-open", repr(go), "--gap-extend-max", repr(ge),
            "--gap-extend-min", repr(gemin), "--gap-decay", repr(decay)]


def in_class(sc):
    """The scoring class test in float32, as the library evaluates it."""
    f = np.float32
    mat, mis, go, _ge, gemin, _decay = (f(v) for v in sc)
    sub_min = min(mat, mis)
    lim = f(sub_min - f(0.25))
    return bool(go < 0 and f(max(go, gemin) + go) <= lim)


def margin(sc):
    """min(match, mismatch) - (max(open, ext_min) + open), exact (in double, from the float32 values)."""
    mat, mis, go, _ge, gemin, _decay = (float(np.float32(v)) for v in sc)
    return min(mat, mis) - (max(go, gemin) + go)


def magnitude_bound(sc, qry_len, ref_len):
    """score_magnitude_bound of capi.cu: bound on |S| (+ one gap or substitution score) in one problem."""
    mat, mis, go, _ge, gemin, _decay = (float(np.float32(v)) for v in sc)
    gain = max(mat, mis, 0.0)
    gap = max(go, gemin, 0.0)
    steps = float(qry_len + ref_len)
    smax = (gain * float(min(qry_len, ref_len)) + gap * steps) * math.exp(steps * 2.0 ** -24)
    return smax + gap + max(abs(mat), abs(mis))


def batch_magnitude(sc, problems):
    return max((magnitude_bound(sc, len(p.qry), len(p.ref)) for p in problems), default=0.0)


def needs_raw(sc, problems=None):
    """Which kernel a batch of `problems` gets under `sc` (the scoring class alone when `problems` is None)."""
    if not in_class(sc):
        return True
    m = batch_magnitude(sc, problems) if problems is not None else 0.0
    ulp = math.ldexp(1.0, math.frexp(m)[1] - 24) if m > 0 else 0.0
    if any(min(int(np.max(p.lengths, initial=0)), len(p.ref)) > 32767 for p in problems or []):
        return True   # rows wider than a C short: always RAW
    return not (margin(sc) > 1.5 * ulp)
