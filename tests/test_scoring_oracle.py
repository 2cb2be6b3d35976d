"""CPU tests: the oracle's three fill rules against the compiled reference at every scoring of scoring_cases, the
kernel choice at large score magnitudes, and the oracle against the reference's vectors in scoring_golden.json.

Rule 0 (as coded) and rule 2 (the RAW kernel's single-pass form) must equal the reference at every scoring. Rule 1
(the scalar rule, what the scalar-rule kernel computes) must equal it wherever the library's kernel choice sends a
problem to that kernel -- and at the large-magnitude boundary scoring it must not, on the long problems: that is the
corner the choice avoids."""
import numpy as np
import pytest

import cases
import golden_util as gu
import scoring_cases as S
from oracle_lib import Reference, same_alignment

needs_ref = pytest.mark.skipif(not Reference.available(), reason="oracle/_ref not built (no reference sources here)")
IDS = [c.name for c in S.SCORINGS]


def _same_fill(a, b):
    return np.array_equal(a[0], b[0]) and tuple(a[1:]) == tuple(b[1:])


def _oracle_align(oracle, p, sc, rule):
    return oracle.single_align(p.ref, p.qry, p.offsets, p.lengths, p.ext_qstart, p.ext_qend, scoring=sc, rule=rule)


def test_table_and_routing_rule():
    """The table's class column is what the library's float32 class test gives; the CLI-reachable scorings have the
    signs ngmlr's parser enforces; the kernel each size of problem gets."""
    for c in S.SCORINGS:
        assert S.in_class(c.sc) == c.in_class, c.name
        assert S.needs_raw(c.sc) == (not c.in_class), c.name
        mat, mis, go, ge, gemin, decay = c.sc
        if c.cli:
            assert mat >= 0 and decay >= 0 and max(mis, go, ge, gemin) <= 0, c.name
        if c.in_class:
            assert S.margin(c.sc) >= 0.25, c.name
    assert 0.0 < S.margin(S.BY_NAME["margin_0.2"].sc) < 0.25
    assert S.margin(S.LARGE.sc) == 0.25 and S.margin(S.BY_NAME["large_margin2"].sc) == 2.0
    assert not S.BY_NAME["negative_decay"].cli and S.BY_NAME["negative_decay"].sc[5] < 0
    rep = S.reproducer()
    short = cases.random_problems(16, 31, max_len=1500)
    # the long problems at the boundary scoring reach 2^21 and go to RAW; short ones and margin 2 stay scalar
    assert S.batch_magnitude(S.LARGE.sc, rep) > 2 ** 21 and S.needs_raw(S.LARGE.sc, rep)
    assert S.batch_magnitude(S.LARGE.sc, short) < 2 ** 21 and not S.needs_raw(S.LARGE.sc, short)
    assert not S.needs_raw(S.BY_NAME["large_margin2"].sc, rep)
    assert S.needs_raw(S.LARGE.sc, short + rep[:1])   # one long problem moves its whole batch
    # default scoring (margin 1): scalar until the magnitude reaches 2^23 -- reads and windows of about 2.9 M bases
    from ngmlr_b200 import synth
    d = S.BY_NAME["default"].sc
    assert not S.needs_raw(d, synth.pacbio_problems(8, genome_len=400_000, seed=2, median=8000))
    assert S.magnitude_bound(d, 2_800_000, 2_800_000) < 2 ** 23 < S.magnitude_bound(d, 3_000_000, 3_000_000)


@needs_ref
@pytest.mark.parametrize("case", S.SCORINGS, ids=IDS)
def test_rules_vs_compiled_reference(oracle, case):
    """Rules 0 and 2 equal the reference everywhere; rule 1 wherever the kernel choice routes the problem to the
    scalar-rule kernel: direction codes, best cell, and SingleAlign's outputs."""
    sc = case.sc
    ref = Reference(sc)
    try:
        probs = cases.random_problems(10, 40 + sum(case.name.encode()), max_len=900) + cases.edge_problems()
        n_rule1 = 0
        for i, p in enumerate(probs):
            want = ref.single_align(p.ref, p.qry, p.offsets, p.lengths, p.ext_qstart, p.ext_qend)
            want_fill = ref.fill(p.ref, p.qry, p.offsets, p.lengths, 0)
            layout = not (np.asarray(p.lengths) < 0).any()   # negative lengths: direction layout differs by design
            rules = (0, 2) + ((1,) if not S.needs_raw(sc, [p]) else ())
            n_rule1 += 1 in rules
            for rule in rules:
                got = _oracle_align(oracle, p, sc, rule)
                assert same_alignment(want, got) == [] and got["status"] == want["status"], (case.name, i, rule)
                f = oracle.fill(p.ref, p.qry, p.offsets, p.lengths, sc, rule)
                assert tuple(f[1:]) == tuple(want_fill[1:]), (case.name, i, rule, "best cell")
                if layout:
                    assert np.array_equal(f[0], want_fill[0]), (case.name, i, rule, "directions")
        assert n_rule1 == (len(probs) if case.in_class else 0)
    finally:
        ref.close()


@needs_ref
def test_scalar_rule_diverges_at_large_magnitude(oracle):
    """At (512,-64,-32.125,-32.125,-32.125,0.5), margin 0.25, the long problems score millions: the scalar rule
    differs from the reference in tens of thousands of direction codes and in every SingleAlign result, while rules 0
    and 2 equal it. With open and extension -33 (margin 2) the scalar rule holds on the same problems."""
    rep = S.reproducer()
    for case, diverges in ((S.LARGE, True), (S.BY_NAME["large_margin2"], False)):
        ref = Reference(case.sc)
        try:
            for i, p in enumerate(rep):
                want = ref.single_align(p.ref, p.qry, p.offsets, p.lengths, p.ext_qstart, p.ext_qend)
                want_fill = ref.fill(p.ref, p.qry, p.offsets, p.lengths, 0)
                assert want["ret"] == len(p.qry) and want["score"] > 2 ** 21, (case.name, i)
                for rule in (0, 2):
                    assert same_alignment(want, _oracle_align(oracle, p, case.sc, rule)) == [], (case.name, i, rule)
                    assert _same_fill(want_fill, oracle.fill(p.ref, p.qry, p.offsets, p.lengths, case.sc, rule))
                f1 = oracle.fill(p.ref, p.qry, p.offsets, p.lengths, case.sc, 1)
                d1 = same_alignment(want, _oracle_align(oracle, p, case.sc, 1))
                if diverges:
                    assert int((f1[0] != want_fill[0]).sum()) > 10_000 and d1 != [], (case.name, i)
                else:
                    assert _same_fill(want_fill, f1) and d1 == [], (case.name, i)
        finally:
            ref.close()


@pytest.mark.parametrize("case", S.SCORINGS, ids=IDS)
def test_oracle_matches_scoring_golden(oracle, case):
    """The oracle against the reference's vectors (no reference needed): rule 0 everywhere, rule 1 on the problems
    the kernel choice gives the scalar-rule kernel, and rule 1's divergence on the long problems at the boundary."""
    (_c, probs, recs), = [s for s in S.golden_sets() if s[0] is case]
    for i, (p, rec) in enumerate(zip(probs, recs)):
        layout = not (np.asarray(p.lengths) < 0).any()
        scalar = not S.needs_raw(case.sc, [p])
        for rule in (0, 1) if scalar else (0,):
            gu.check_against_record(_oracle_align(oracle, p, case.sc, rule), rec, f"{case.name}[{i}] rule {rule}")
            dirs, bs, bx, by = oracle.fill(p.ref, p.qry, p.offsets, p.lengths, case.sc, rule)
            assert [int(np.float32(bs).view(np.uint32)), bx, by] == rec["best"], (case.name, i, rule)
            if layout:
                assert gu.digest(dirs) == rec["dirs_sha"], (case.name, i, rule)
        if case is S.LARGE and len(p.qry) > 5000:
            dirs, *_ = oracle.fill(p.ref, p.qry, p.offsets, p.lengths, case.sc, 1)
            assert gu.digest(dirs) != rec["dirs_sha"], (case.name, i)
    assert sum(len(p.qry) > 5000 for p in probs) == (3 if case.large else 0)
