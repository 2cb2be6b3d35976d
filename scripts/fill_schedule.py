"""Ramped vs ramp-free row schedule of the convex fill (csrc/convex_fill.cu), the latter with one or two rows per lane.

--cpu (the default) counts, from the bench workload's own corridors, the lane-steps each schedule issues per DP
cell: the ramped kernel's block_geom arithmetic, and the ramp-free kernels' placement rule restated here (entry at
a 16-step group boundary, no overlap within a lane, one chunk between a block's last entry and the next block's
first, the hand-off spacing O_b >= O_{b-1} + RF_RING), for 32-row blocks and for 64-row blocks with two rows per lane,
the latter with both rows in the same column and with the second one column behind (lane stagger 2, RF2S_RING).
A lane-step of the two-row kernels evaluates two cells; "rampfree2" and "rampfree2-skew" count cell slots (2 per
lane-step) per cell, so the figures compare idle work. No GPU is needed.

--gpu runs `bench.py --profile-only` and the full `bench.py` under each of --settings (default: all of them),
alternating, and prints the medians and spreads of the fill kernel time and of the headline value, with the card name,
power limit and SM clock read in the same run. --dump-outputs also writes each setting's bench outputs once.
--libraries NAME=PATH,... compares builds of the library instead (NGMLR_B200_LIBRARY, default fill settings), e.g. the
parent commit's build against the working tree's.

    python scripts/fill_schedule.py --cpu [--reads 300]
    python scripts/fill_schedule.py --gpu --runs 3 --out DIR [--settings rampfree-rows2,rampfree-rows2-skew]
    python scripts/fill_schedule.py --gpu --runs 3 --out DIR --libraries old=/path/libngmlr_b200.so,new=ngmlr_b200/libngmlr_b200.so
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

INT_MAX = 2**31 - 1
RF_CHUNK = 64                  # steps staged per chunk (RF_CHUNK)
RF_RING = 32 + 2 * RF_CHUNK    # hand-off spacing of consecutive origins (RF_RING)
RF2S_RING = 64 + 2 * RF_CHUNK  # the same for the skewed two-row schedule (RF2S_RING)


def spans(offs, lens, ref_len, b, H):
    """row_span of the 32 rows of block b -> xlo, xhi, rlen (rows >= H are empty)."""
    y = 32 * b + np.arange(32)
    ok = y < H
    off = np.where(ok, offs[np.minimum(y, H - 1)], 0).astype(np.int64)
    ln = np.where(ok, lens[np.minimum(y, H - 1)], 0).astype(np.int64)
    xlo = np.maximum(off, 0)
    xhi = np.minimum(off + ln, ref_len)
    rlen = np.maximum(xhi - xlo, 0)
    return xlo, xhi, rlen


def ramped_steps(offs, lens, ref_len):
    """block_geom: a block runs ngroups * 16 steps, base = min xlo, end = max(xhi + lane)."""
    H = len(offs)
    steps = 0
    for b in range((H + 31) // 32):
        xlo, xhi, rlen = spans(offs, lens, ref_len, b, H)
        if not rlen.any():
            continue
        n = int((xhi + np.arange(32))[rlen > 0].max() - xlo[rlen > 0].min())
        steps += (n + 15) // 16 * 16
    return steps


def rf_cols(xlo, xhi, rlen):
    a = np.where(rlen > 0, xlo, INT_MAX)
    e = np.where(rlen > 0, xhi, -INT_MAX)
    a1 = np.append(a[1:], INT_MAX)
    e1 = np.append(e[1:], e.max())
    amin = np.minimum(a, a1)
    A = np.where(amin == INT_MAX, INT_MAX, amin - 1)
    E = np.maximum(e, e1)
    return A, E


def rf2_cols(offs, lens, ref_len, b, H):
    """Lane t's columns of 64-row block b: its rows 64b + 2t, 64b + 2t + 1 and lane t+1's first row."""
    xlo0, xhi0, rl0 = spans(offs, lens, ref_len, 2 * b, H)
    xlo1, xhi1, rl1 = spans(offs, lens, ref_len, 2 * b + 1, H)
    xlo, xhi, rl = np.concatenate([xlo0, xlo1]), np.concatenate([xhi0, xhi1]), np.concatenate([rl0, rl1])
    a = np.where(rl > 0, xlo, INT_MAX)
    e = np.where(rl > 0, xhi, -INT_MAX)
    aA, aB, eA, eB = a[0::2], a[1::2], e[0::2], e[1::2]
    a1 = np.append(aA[1:], INT_MAX)
    e1 = np.append(eA[1:], e.max())
    amin = np.minimum(np.minimum(aA, aB), a1)
    A = np.where(amin == INT_MAX, INT_MAX, amin - 1)
    E = np.maximum(np.maximum(eA, eB), e1)
    return A, E


def rampfree_steps(offs, lens, ref_len, rows=1, skew=False):
    """Steps of the warp under the ramp-free placement (pass 1 of convex_fill_rf_kernel / convex_fill_rf2_kernel).
    skew: lane t's first row is at column x at step O + 2t + x and its second row one column behind, so its range
    ends one step later."""
    H = len(offs)
    lane = np.arange(32) * (2 if skew else 1)
    tail, ring = (1, RF2S_RING) if skew else (0, RF_RING)
    L = np.full(32, -INT_MAX, dtype=np.int64)
    R, O_last = 0, None
    per = 32 * rows
    for b in range((H + per - 1) // per):
        if rows == 1:
            A, E = rf_cols(*spans(offs, lens, ref_len, b, H))
        else:
            A, E = rf2_cols(offs, lens, ref_len, b, H)
        has = A != INT_MAX
        frm = np.maximum(L, R)
        need = np.where(has, ((frm + 15) // 16) * 16 - lane - A, -INT_MAX)
        O = int(need.max())
        if O_last is not None:
            O = max(O, O_last + ring)
        sw = np.where(has, ((O + lane + A) // 16) * 16, -INT_MAX)
        assert (sw[has] >= L[has]).all() and (sw[has] <= (O + lane + A)[has]).all()
        if has.any():
            O_last = O
        L = np.where(has, O + lane + E + tail, L)
        swmax = int(sw[has].max()) if has.any() else R - 1
        R = ((swmax + RF_CHUNK) // RF_CHUNK + 1) * RF_CHUNK
    return (max(0, int(L.max())) + 15) // 16 * 16


def cpu(args):
    from ngmlr_b200 import synth
    cfg = dict(median=8000, err=0.15, ratio=(9, 4, 2), hi=40000)   # bench.py CONFIGS["pacbio50"]
    contig = 10_000_000
    genome = synth.random_genome(5 * contig, 1)
    reads, ivs = synth.simulate_reads(args.reads, genome, contig, 3, **cfg)
    cells = ramp = rf = rf2 = rf2s = 0
    widths = []
    for iv in ivs:
        p = iv.problem(genome, reads)
        offs, lens = np.asarray(p.offsets), np.asarray(p.lengths)
        ref_len = len(p.ref)
        c = int(np.maximum(np.minimum(offs.astype(np.int64) + lens, ref_len) - np.maximum(offs, 0), 0).sum())
        cells += c
        widths.append(int(lens.max()))
        ramp += 32 * ramped_steps(offs, lens, ref_len)
        rf += 32 * rampfree_steps(offs, lens, ref_len)
        rf2 += 64 * rampfree_steps(offs, lens, ref_len, rows=2)
        rf2s += 64 * rampfree_steps(offs, lens, ref_len, rows=2, skew=True)
    w = np.array(widths)
    out = {
        "problems": len(ivs),
        "width_p10_p50_p90": [int(np.percentile(w, q)) for q in (10, 50, 90)],
        "lane_steps_per_cell": {
            "ramped": round(ramp / cells, 4),
            "rampfree": round(rf / cells, 4),
            "rampfree2": round(rf2 / cells, 4),
            "rampfree2-skew": round(rf2s / cells, 4),
        },
    }
    print(json.dumps(out, indent=1))


def smi():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


# schedule, rows per lane, skew of the two-row kernel
SETTINGS = {"ramped": ("ramped", "1", "0"), "rampfree-rows1": ("rampfree", "1", "0"),
            "rampfree-rows2": ("rampfree", "2", "0"), "rampfree-rows2-skew": ("rampfree", "2", "1")}


def bench(setting, extra, steps, warmup, config, libraries=None):
    if libraries:
        env = dict(os.environ, NGMLR_B200_LIBRARY=os.path.abspath(libraries[setting]))
    else:
        schedule, rows, skew = SETTINGS[setting]
        env = dict(os.environ, NGMLR_B200_FILL_SCHEDULE=schedule, NGMLR_B200_FILL_ROWS_PER_LANE=rows,
                   NGMLR_B200_FILL_RF2_SKEW=skew)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps),
           "--warmup", str(warmup), "--config", config] + extra
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        raise SystemExit(f"bench.py failed ({setting} {extra}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
    return json.loads(lines[-1])


def gpu(args):
    print("card:", smi())
    libraries = dict(kv.split("=", 1) for kv in args.libraries.split(",")) if args.libraries else None
    settings = list(libraries) if libraries else (args.settings.split(",") if args.settings else list(SETTINGS))
    res = {k: {"prof": [], "full": []} for k in settings}
    for i in range(args.runs):
        for sched in settings:
            dump = ["--dump-outputs", os.path.join(args.out, "dump", sched)] if args.dump_outputs and i == 0 else []
            prof = (bench(sched, ["--profile-only"], args.steps, args.warmup, args.config, libraries)
                    if not args.full_only else None)
            full = bench(sched, dump, args.steps, args.warmup, args.config, libraries)
            res[sched]["prof"].append(prof)
            res[sched]["full"].append(full)
            print(f"run {i} {sched}: fill {full['kernel_ms_per_step']['fill']:.2f} ms/step, value {full['value']:.4f}, "
                  f"parity {full.get('parity_checked')}", flush=True)
    summary = {"card": smi(), "config": args.config}
    for sched, r in res.items():
        fill = np.array([x["kernel_ms_per_step"]["fill"] for x in r["full"]])
        val = np.array([x["value"] for x in r["full"]])
        summary[sched] = {"fill_ms_median": float(np.median(fill)), "fill_ms_spread": float(fill.max() - fill.min()),
                          "value_median": float(np.median(val)), "value_spread": float(val.max() - val.min()),
                          "fill_ms": fill.tolist(), "value": val.tolist()}
        if not args.full_only:
            pfill = np.array([x["fill_ms"] for x in r["prof"]])
            summary[sched].update(solo_fill_ms_median=float(np.median(pfill)),
                                  solo_fill_ms_spread=float(pfill.max() - pfill.min()), solo_fill_ms=pfill.tolist())
    pairs = (("ramped", "rampfree-rows1"), ("rampfree-rows1", "rampfree-rows2"), ("rampfree-rows2", "rampfree-rows2-skew"))
    if libraries:
        pairs = tuple(zip(settings, settings[1:]))
    for a, b in (ab for ab in pairs if ab[0] in res and ab[1] in res):
        summary[f"fill_change {a} -> {b}"] = summary[b]["fill_ms_median"] / summary[a]["fill_ms_median"] - 1.0
        summary[f"value_change {a} -> {b}"] = summary[b]["value_median"] / summary[a]["value_median"] - 1.0
    print(json.dumps(summary, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fill_schedule.json"), "w") as f:
            json.dump({"summary": summary, "runs": res}, f, indent=1)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--cpu", action="store_true", help="lane-steps per cell from the workload geometry (default)")
    ap.add_argument("--gpu", action="store_true", help="A/B of the schedules with bench.py")
    ap.add_argument("--reads", type=int, default=300)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--settings", default=None, help="comma-separated subset of " + ", ".join(SETTINGS))
    ap.add_argument("--config", default="pacbio50", help="bench.py --config")
    ap.add_argument("--full-only", action="store_true", help="skip the --profile-only runs")
    ap.add_argument("--dump-outputs", action="store_true", help="bench.py --dump-outputs OUT/dump/SETTING, first run")
    ap.add_argument("--libraries", default=None, help="NAME=PATH,...: A/B of library builds (NGMLR_B200_LIBRARY)")
    args = ap.parse_args()
    if args.dump_outputs and not args.out:
        ap.error("--dump-outputs needs --out")
    if args.gpu:
        gpu(args)
    if args.cpu or not args.gpu:
        cpu(args)


if __name__ == "__main__":
    main()
