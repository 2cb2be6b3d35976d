"""Time the sub-read scorer at --subread-length above 256, for one or more builds of the package, alternating them.

Workloads on a seeded synthetic genome (random ACGT, default 20 Mb in 2 contigs), reads mutated from it:
  cs_run_480        reads_upload + cs_run at --subread-length 480 (sub-reads of 480 bases against windows of 532
                    characters); cs_run's own CUDA-event time and the host time of the call
  cs_run_256        the same reads at the default --subread-length 256
  short_256         score_short_reads on reads of 100-256 bases (every build accepts them)
  short_257_510     score_short_reads on reads of 257-510 bases
  batch_257_510     BatchScore on the same queries and their short-read windows (copied to the host), timed with the
                    library's CUDA events around the kernel (ngmlr_b200_sw_last_kernel_ms); a build that refuses
                    reads of more than 256 bases in score_short_reads still scores these pairs here
Each workload is warmed up, then timed --reps times (host clocks around calls that end in a device synchronise); the
median is reported. Scores of every build are compared with the first build's.

    python scripts/subread_length_timing.py [--variant NAME=DIR ...] [--rounds 2] [--reps 7] [--out DIR]

A variant's DIR holds an importable ngmlr_b200 package with its built library (default: this tree). Each round runs
every variant once, in its own process, in turn. The card's name, power limit and maximum SM clock are read in the
same run and written next to the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def _timed(fn, reps, warmup=2):
    for _ in range(warmup):
        out = fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return out, ts


def worker(args):
    import numpy as np
    from ngmlr_b200 import B200Aligner, synth

    rng = np.random.default_rng(args.seed)
    half = args.mbp * 500_000
    genome = synth.random_genome(2 * half, args.seed)
    contigs = [genome[:half], genome[half:]]
    res = {"variant": args.name, "package": os.path.dirname(os.path.dirname(os.path.abspath(
        sys.modules["ngmlr_b200"].__file__)))}
    a = B200Aligner(0)
    try:
        enc = a.encode_reference([c.tobytes() for c in contigs], fetch=False)
        a.build_index(enc)

        def mutated(L):
            c = int(rng.integers(0, 2))
            s = int(rng.integers(0, half - L - 1))
            r, _ = synth.mutate(contigs[c][s:s + L].copy(), rng, err=0.08)
            r = np.ascontiguousarray(r, dtype=np.uint8)
            return (synth.revcomp(r) if rng.integers(0, 2) else r).tobytes(), enc.ref_start[c] + s

        # ---- cs_run at --subread-length 480, and at the default 256 (the default instantiation) ----
        long_reads = [mutated(int(rng.integers(2_000, 10_000)))[0] for _ in range(args.long_reads)]
        for rpl in (480, 256):
            n_sub = a.reads_upload(long_reads, rpl)
            (m, kms), ts = _timed(lambda: a.cs_run(0.8, 0.0, 40, rpl), args.reps)
            kms_all = []
            for _ in range(args.reps):
                kms_all.append(a.cs_run(0.8, 0.0, 40, rpl)[1])
            sw = a.cs_fetch()[4]
            res[f"cs_run_{rpl}"] = dict(sub_reads=n_sub, candidates=int(m), host_ms=_median(ts),
                                        kernel_ms=_median(kms_all), score_sum=float(np.sum(sw, dtype=np.float64)))

        # ---- short reads ----
        for name, lo, hi in (("short_256", 100, 257), ("short_257_510", 257, 511)):
            reads, origin = [], []
            while len(reads) < args.short_reads:
                r, o = mutated(int(rng.integers(lo, hi)))
                if lo <= len(r) < hi:
                    reads.append(r)
                    origin.append(o)
            a.reads_upload(reads)
            n = args.short_reads * args.pairs_per_read
            ri = np.repeat(np.arange(len(reads), dtype=np.int32), args.pairs_per_read)
            loc = rng.integers(0, enc.concat_len, n).astype(np.uint64)
            loc[::args.pairs_per_read] = np.array(origin, dtype=np.uint64)   # one candidate at the read's origin
            rv = rng.integers(0, 2, n).astype(np.uint8)
            entry = dict(pairs=n)
            try:
                got, ts = _timed(lambda: a.score_short_reads(ri, loc, rv), args.reps)
                entry.update(host_ms=_median(ts), score_sum=float(np.sum(got, dtype=np.float64)))
            except RuntimeError as e:
                entry["refused"] = str(e)[:200]
            res[name] = entry
            if name == "short_257_510":
                # the same pairs through the drop-in BatchScore: windows cut from the genome like scoreShortRead's
                # (the encoded genome's spacer aside), the reverse candidates as reverse-complemented queries
                m2 = min(n, args.batch_pairs)
                refs, qrys = [], []
                for j in range(m2):
                    q = reads[ri[j]]
                    L = len(q)
                    corr = int(L * 0.3 + 256)
                    start = max(0, min(int(loc[j]) - (corr >> 1), 2 * half - L - corr))
                    refs.append(genome[start:start + L + corr].tobytes())
                    qrys.append(synth.revcomp_upper(np.frombuffer(q, dtype=np.uint8)).tobytes() if rv[j] else q)
                kms = []
                for k in range(args.reps + 2):
                    out = a.BatchScore(refs, qrys)
                    if k >= 2:
                        kms.append(float(a.lib.ngmlr_b200_sw_last_kernel_ms(a.h)))
                res["batch_257_510"] = dict(pairs=m2, kernel_ms=_median(kms),
                                            score_sum=float(np.sum(out, dtype=np.float64)))
    finally:
        a.close()
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--variant", action="append", default=[], help="NAME=DIR with an ngmlr_b200 package")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--mbp", type=int, default=20)
    ap.add_argument("--long-reads", type=int, default=6_000)
    ap.add_argument("--short-reads", type=int, default=20_000)
    ap.add_argument("--pairs-per-read", type=int, default=10)
    ap.add_argument("--batch-pairs", type=int, default=100_000)
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--name", default="", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        worker(args)
        return
    variants = [v.split("=", 1) for v in args.variant] or [["this_tree", ROOT]]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card}), flush=True)
    results = []
    for rnd in range(args.rounds):
        for name, d in variants:
            env = dict(os.environ, PYTHONPATH=os.path.abspath(d))
            env.pop("NGMLR_B200_LIBRARY", None)
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--name", name]
            for k in ("reps", "mbp", "long_reads", "short_reads", "pairs_per_read", "batch_pairs", "seed"):
                cmd += ["--" + k.replace("_", "-"), str(getattr(args, k))]
            r = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=os.path.abspath(d))
            if r.returncode != 0:
                sys.exit(f"{name}: worker failed\n{r.stderr[-3000:]}")
            line = json.loads(r.stdout.strip().splitlines()[-1])
            line["round"] = rnd
            print(json.dumps(line), flush=True)
            results.append(line)
    first = results[0]
    for r in results[1:]:
        for key in ("cs_run_480", "cs_run_256", "short_256", "short_257_510", "batch_257_510"):
            a, b = first.get(key, {}), r.get(key, {})
            if "score_sum" in a and "score_sum" in b and a["score_sum"] != b["score_sum"]:
                print(json.dumps({"score_mismatch": key, "variant": r["variant"], "want": a["score_sum"],
                                  "got": b["score_sum"]}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "subread_length_timing.json"), "w") as f:
            json.dump({"gpu": card, "runs": results}, f, indent=1)


if __name__ == "__main__":
    main()
