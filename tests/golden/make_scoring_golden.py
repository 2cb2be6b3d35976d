"""Generates tests/golden/scoring_golden.json from the UNMODIFIED reference (oracle/_ref/libngmlr_ref.so, built by
oracle/Makefile from the reference sources). Run where those sources are:

    python tests/golden/make_scoring_golden.py

For every scoring of tests/scoring_cases.py: ConvexAlignFast::SingleAlign outputs, the direction-matrix checksum and
the best cell of scoring_cases.golden_problems() (seeded random problems and edge problems; for the large-magnitude
scorings also the three long problems whose scores reach millions). Inputs are regenerated from the seeds, so only
outputs are stored, with an input checksum per problem to detect generator drift."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import scoring_cases  # noqa: E402
from make_golden import record  # noqa: E402
from oracle_lib import Reference, build_ref  # noqa: E402


def main():
    build_ref()
    out = {}
    for case in scoring_cases.SCORINGS:
        ref = Reference(case.sc)
        try:
            recs = [record(ref, p) for p in scoring_cases.golden_problems(case)]
        finally:
            ref.close()
        for r in recs:
            r.pop("cigar")   # the checksums pin it
        out[case.name] = {"scoring": list(case.sc), "records": recs}
    with open(os.path.join(HERE, "scoring_golden.json"), "w") as f:
        json.dump(out, f, indent=0)
    print("wrote scoring golden vectors:", {k: len(v["records"]) for k, v in out.items()})


if __name__ == "__main__":
    main()
