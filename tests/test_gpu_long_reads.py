"""GPU: convex alignment at ONT scale through every SingleAlign surface, against the oracle.

The problems are ONT-shaped (synth.simulate_reads: median 20 kb, 12 % errors 1:1:1, up to 100 kb) on a 4 Mb genome.
Every problem set holds both strands, read parts longer than 32 767 and 65 535 bases (one is planted) and at least
8 problems of >= 8 Mi cells, the size from which the ramp-free schedule hands a problem to its concurrent launch of
ramped 4-warp teams. Comparisons are bit-exact on every ALIGN_KEYS field and on nmPerPosition.

- the default fill configuration (ramp-free, one and two rows per lane, with the team launch) via BatchAlign, with
  the counters showing which launch filled what, and every direction code of two team-filled problems;
- the resident path (reads_upload -> compute_alignments, intervals_upload -> run -> fetch) with nmPerPosition;
- the IAlignment object (tests/cpp/plugin_driver.cpp): SingleAlign, BatchAlign, and SingleAlign served by the
  cross-thread batcher, nmPerPosition included;
- bench.py's cross-check at test size: IAlignment::BatchAlign against the resident pipeline, GPU against GPU;
- a batch that runs out of device memory (NGMLR_B200_DEBUG_ARENA_CAP, a host-side cap on the arenas): the plugin
  splits it instead of failing every problem, and only a problem that does not fit alone fails."""
import os
import subprocess
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

from ngmlr_b200 import B200Aligner, PackedBatch, _lib, refindex, synth
from ngmlr_b200.intervals import compute_alignments
from oracle_lib import CsOracle, Oracle, same_alignment
from test_cs_oracle import _OracleBackend

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONTIG = 2_000_000
TEAM_CELLS = 8 << 20          # RF_TEAM_CELLS: problems of at least this many cells (width x height) go to the team launch
MINUS_ONE = int(np.float32(-1.0).view(np.uint32))


def _est(p):
    """The host's cell estimate of a problem: sum of the corridor row lengths (width x height), not clipped."""
    return int(np.maximum(np.asarray(p.lengths, np.int64), 0).sum())


def _oracle_one(p):
    return Oracle().single_align(p.ref, p.qry, p.offsets, p.lengths, p.ext_qstart, p.ext_qend)


def _oracle_all(probs):
    """single_align of every problem, spread over a process pool (the oracle fills ~33 M cells/s on one core)."""
    with ProcessPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:
        return list(ex.map(_oracle_one, probs, chunksize=1))


def _assert_same(want, got, what):
    d = same_alignment(want, got)
    assert d == [], (what, d, {k: (want[k], got[k]) for k in d if k != "nm_positions"})


@pytest.fixture(scope="module")
def world():
    return _make_world()


def _make_world():
    """4 Mb genome, ONT-shaped reads, and the intervals every test draws its problems from."""
    genome = synth.random_genome(2 * CONTIG, 2024)
    reads, ivs = synth.simulate_reads(300, genome, CONTIG, 17, median=20000, err=0.12, ratio=(1, 1, 1), hi=100000)
    # the seed draws nothing above 65 535 bases: plant two long reads, one per strand
    long_reads, long_ivs = synth.simulate_reads(6, genome, CONTIG, 99, median=70000, err=0.12, ratio=(1, 1, 1),
                                                lo=66000, hi=72000)
    fwd = next(iv for iv in long_ivs if not iv.reverse)
    rev = next(iv for iv in long_ivs if iv.reverse)
    base = len(reads)
    for k, iv in enumerate((fwd, rev)):
        reads.append(long_reads[iv.read])
        iv.read = base + k
        ivs.append(iv)
    enc = refindex.encode_reference([genome[:CONTIG], genome[CONTIG:]])
    probs = [iv.problem(genome, reads) for iv in ivs]
    return genome, enc, reads, ivs, probs


def _pick(world, n_team, n_small):
    """Indices of a problem set: the planted > 65 535-base parts, n_team problems of >= 8 Mi cells (a > 32 767-base
    one among them), n_small smaller ones; then checks what the set provably contains."""
    _g, _e, _r, ivs, probs = world
    planted = [len(probs) - 2, len(probs) - 1]
    big = [i for i in range(len(probs) - 2) if _est(probs[i]) >= TEAM_CELLS]
    over32k = [i for i in big if len(probs[i].qry) > 32767][:1]
    team = over32k + [i for i in big if i not in over32k][:n_team - 1]
    small = [i for i in range(len(probs) - 2) if _est(probs[i]) < TEAM_CELLS][:n_small]
    sel = sorted(planted + team + small)
    ps = [probs[i] for i in sel]
    assert any(ivs[i].reverse for i in sel) and not all(ivs[i].reverse for i in sel)
    assert sum(len(p.qry) > 32767 for p in ps) >= 3 and sum(len(p.qry) > 65535 for p in ps) >= 2
    assert sum(_est(p) >= TEAM_CELLS for p in ps) >= 8
    return sel


@pytest.fixture(scope="module")
def set_a(world):
    """The problem set of the BatchAlign, plugin and allocation tests, with the oracle's results."""
    sel = _pick(world, 10, 10)
    probs = [world[4][i] for i in sel]
    return probs, _oracle_all(probs)


# ---- 1. the default fill configuration at real size ---------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 2], ids=["rows1", "rows2"])
def test_default_fill_at_ont_scale(set_a, monkeypatch, rows):
    """No overrides but the row count: the ramp-free launch fills the problems below 8 Mi cells and the concurrent
    launch of ramped 4-warp teams the others, in one fill launch (the host's arena estimate held)."""
    probs, want = set_a
    monkeypatch.setenv("NGMLR_B200_FILL_ROWS_PER_LANE", str(rows))
    a = B200Aligner(0)
    try:
        a.set_small_batch_teams(0)   # a batch of at most one problem per SM would take 16-warp teams throughout
        rf0, rf20 = a.debug_rampfree_problems(), a.debug_rampfree2_problems()
        got = list(a.BatchAlign(PackedBatch.from_problems(probs)))
        rf, rf2 = a.debug_rampfree_problems() - rf0, a.debug_rampfree2_problems() - rf20
        n_team = sum(_est(p) >= TEAM_CELLS for p in probs)
        assert n_team >= 8
        assert rf == len(probs) - n_team, (rf, len(probs), n_team)
        assert rf2 == (rf if rows == 2 else 0)
        assert a.stats()["fill_launches"] == 1
        for i, (w, g) in enumerate(zip(want, got)):
            _assert_same(w, g.as_dict(), i)
        # every direction code of two team-filled problems (the largest and a > 32 767-row one)
        orc = Oracle()
        team = [i for i, p in enumerate(probs) if _est(p) >= TEAM_CELLS]
        for i in (max(team, key=lambda j: _est(probs[j])),
                  next(j for j in team if 32767 < len(probs[j].qry) <= 65535)):
            p = probs[i]
            wd, wbs, wbx, wby = orc.fill(p.ref, p.qry, p.offsets, p.lengths)
            gd, gbs, gbx, gby = a.debug_directions(i, int(wd.size))
            assert (gbs, gbx, gby) == (wbs, wbx, wby), i
            bad = np.flatnonzero(gd != wd)
            assert bad.size == 0, (i, bad.size, bad[:8])
    finally:
        a.close()


# ---- 2. the resident path on long intervals -------------------------------------------------------------------------
def test_resident_path_on_long_intervals(world, oracle):
    """reads_upload -> compute_alignments (windows decoded on the device, closed-form corridors, read parts gathered
    by index; retries inside the call) against the Python mirror over the oracle, and intervals_upload -> run ->
    fetch against the oracle on each interval's first attempt -- nmPerPosition requested and compared."""
    genome, enc, reads, ivs, probs = world
    sel = _pick(world, 8, 6)
    read_ids = sorted({ivs[i].read for i in sel})
    rmap = {r: k for k, r in enumerate(read_ids)}
    sub_reads = [reads[r] for r in read_ids]
    sub_ivs = []
    for i in sel:
        iv = ivs[i]
        sub_ivs.append(synth.SimInterval(rmap[iv.read], iv.on_read_start, iv.read_len, iv.reverse, iv.ref_start,
                                         iv.ref_len, iv.ax, iv.ay, iv.full_alignment, iv.corridor))
    g2c = lambda pos: enc.ref_start[pos // CONTIG] + pos % CONTIG
    cso = CsOracle([genome[:CONTIG].tobytes(), genome[CONTIG:].tobytes()])
    a = B200Aligner(0)
    try:
        a.set_reference(enc)
        a.set_text_stage(True, want_nm_positions=True)   # compute_alignments runs the device text stage
        a.reads_upload(sub_reads)
        got, calls = a.compute_alignments(synth.interval_tasks(sub_ivs, sub_reads, g2c, by_index=True))
        got = list(got)
        want, want_calls = compute_alignments(_OracleBackend(cso, oracle),
                                              synth.interval_tasks(sub_ivs, sub_reads, g2c, by_index=False))
        assert list(calls) == want_calls
        n_valid = 0
        for i, (w, g) in enumerate(zip(want, got)):
            assert (w is None) == (g.ret < 0), i
            if w is not None:
                n_valid += 1
                _assert_same(w, g.as_dict(), ("compute_alignments", i))
        assert n_valid >= len(sub_ivs) - 1
        # first attempts, inputs resident
        a.intervals_upload(synth.interval_tasks(sub_ivs, sub_reads, g2c, by_index=True))
        a.run()
        first = list(a.fetch())
        want1 = _oracle_all([iv.problem(genome, sub_reads) for iv in sub_ivs])
        for i, (w, g) in enumerate(zip(want1, first)):
            _assert_same(w, g.as_dict(), ("intervals_upload", i))
    finally:
        a.close()
        cso.close()


# ---- 3. the IAlignment object at ONT scale ---------------------------------------------------------------------------
def _write_problems(path, probs):
    with open(path, "w") as f:
        f.write(f"{len(probs)}\n")
        for p in probs:
            f.write(f"{len(p.ref)} {len(p.qry)} {p.ext_qstart} {p.ext_qend}\n{p.ref.decode()}\n{p.qry.decode()}\n")
            f.write(" ".join(f"{o} {l}" for o, l in zip(p.offsets, p.lengths)) + "\n")


def _nm_digest(nm):
    """FNV-1a over the (refPosition, readPosition, nm) triples as little-endian int32s, as plugin_driver prints it."""
    h = 2166136261
    for b in np.ascontiguousarray(nm, dtype="<i4").tobytes():
        h = ((h ^ b) * 16777619) & 0xffffffff
    return h


def _run_driver(tmp_path, probs, env=None, threads=1):
    exe = str(tmp_path / "plugin_driver")
    if not os.path.exists(exe):
        subprocess.run(["g++", "-O1", "-std=c++11", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "cpp", "plugin_driver.cpp"), "-o", exe, "-ldl", "-lpthread"],
                       check=True)
    path = tmp_path / "problems.txt"
    if not path.exists():
        _write_problems(path, probs)
    out = subprocess.run([exe, _lib.LIB_PATH, str(path), str(threads)], capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, **(env or {})))
    assert out.returncode == 0, out.stderr[-2000:]
    lines = out.stdout.splitlines()
    kv = lambda l, k: dict(x.split("=", 1) for x in l.split()[k:])
    res = {}
    for tag in ("single", "batch"):
        rows = {int(l.split()[1]): kv(l, 2) for l in lines if l.startswith(tag + " ")}
        nms = {int(l.split()[2]): kv(l, 3) for l in lines if l.startswith(f"nm {tag} ")}
        res[tag] = (rows, nms)
    assert f"batchalign rc={len(probs)}" in lines
    return res


def _check_driver(res, want, failing=()):
    """Every problem of both surfaces against the oracle; `failing` ones must report ret -1 / Score -1."""
    for tag, (rows, nms) in res.items():
        for i, w in enumerate(want):
            got = rows[i]
            if i in failing:
                assert int(got["ret"]) == -1 and int(got["score_bits"]) == MINUS_ONE, (tag, i, got.get("ret"))
                continue
            assert w["ret"] >= 0, i
            assert int(got["ret"]) >= 0 and int(got["score_bits"]) == w["score_bits"], (tag, i, got["score_bits"])
            if tag == "single":
                assert int(got["ret"]) == w["ret"], (tag, i)
            assert got["cigar"] == w["cigar"] and got["md"] == w["md"], (tag, i)
            assert int(got["identity_bits"]) == w["identity_bits"], (tag, i)
            for k, wk in (("pos", "position_offset"), ("qstart", "qstart"), ("qend", "qend"), ("nm", "nm"),
                          ("alen", "alignment_length"), ("ops", "cigar_op_count"), ("sv", "sv_type")):
                assert int(got[k]) == w[wk], (tag, i, k)
            assert got["first"] == f"{w['first_ref']},{w['first_read']}" and got["last"] == f"{w['last_ref']},{w['last_read']}"
            assert int(nms[i]["count"]) == w["nm_count"], (tag, i, nms[i]["count"], w["nm_count"])
            assert int(nms[i]["fnv"]) == _nm_digest(w["nm_positions"]), (tag, i, "nmPerPosition")


def test_ialignment_object_at_ont_scale(set_a, tmp_path):
    probs, want = set_a
    _check_driver(_run_driver(tmp_path, probs), want)


def test_ialignment_batcher_at_ont_scale(set_a, tmp_path):
    """SingleAlign from 8 threads, served by the cross-thread batcher (several problems per launch)."""
    probs, want = set_a
    _check_driver(_run_driver(tmp_path, probs, env={"NGMLR_B200_BATCH_WINDOW_US": "20000"}, threads=8), want)


# ---- 4. bench.py's cross-check at test size --------------------------------------------------------------------------
def test_ialignment_batch_align_equals_resident_pipeline(world):
    """A few hundred ONT intervals through CreateAlignment -> IAlignment::BatchAlign (ngmlr_b200_plugin_time_batch_align,
    what bench.py times) against intervals_upload -> run -> fetch: Score bits, CIGAR and MD of every interval; a
    sample of both against the oracle."""
    import ctypes as C
    genome, enc, reads, ivs, probs = world
    n = len(ivs)
    assert n >= 250
    lib = _lib.load()
    lib.CreateAlignment.restype = C.c_void_p
    lib.CreateAlignment.argtypes = [C.c_int]
    lib.DeleteAlignment.argtypes = [C.c_void_p]
    i32p, i64p, u32p = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_uint32)
    lib.ngmlr_b200_plugin_time_batch_align.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p),
                                                       C.POINTER(C.c_char_p), i32p, i32p, i64p, i32p, i32p, C.c_int,
                                                       C.POINTER(C.c_double), i32p, u32p, u32p]
    g2c = lambda pos: enc.ref_start[pos // CONTIG] + pos % CONTIG
    a = B200Aligner(0)
    try:
        a.set_reference(enc)
        a.reads_upload(reads)
        a.intervals_upload(synth.interval_tasks(ivs, reads, g2c, by_index=True))
        a.run()
        res = [r.as_dict() for r in a.fetch()]
    finally:
        a.close()
    pb = PackedBatch.from_problems(probs)
    rets = np.zeros(n, np.int32)
    bits = np.zeros(n, np.uint32)
    crc = np.zeros(n, np.uint32)
    sec = C.c_double(0)
    args = pb.c_args()
    obj = lib.CreateAlignment(0)
    assert obj
    try:
        for _ in range(2):   # the second call on grown arenas, as bench.py's timed repeats
            rc = lib.ngmlr_b200_plugin_time_batch_align(obj, n, args[1], args[3], args[5], args[6], args[7], args[8],
                                                        args[9], 1, C.byref(sec), rets.ctypes.data_as(i32p),
                                                        bits.ctypes.data_as(u32p), crc.ctypes.data_as(u32p))
            assert rc == 0
            for i, d in enumerate(res):
                if d["ret"] < 0:
                    assert rets[i] < 0, i
                    continue
                h = 2166136261
                for ch in (d["cigar"] + d["md"]).encode():
                    h = ((h ^ ch) * 16777619) & 0xffffffff
                assert (int(bits[i]), int(crc[i])) == (d["score_bits"], h), i
    finally:
        lib.DeleteAlignment(obj)
    assert sum(d["ret"] >= 0 for d in res) >= n - 2
    sample = [0, 1, 2, n // 2, n - 2, n - 1]        # the planted > 65 535-base parts are the last two
    for i, w in zip(sample, _oracle_all([probs[i] for i in sample])):
        _assert_same(w, dict(res[i], nm_positions=w["nm_positions"]), i)   # nmPerPosition not requested here
        assert res[i]["nm_count"] == w["nm_count"]


# ---- 5. a batch that runs out of memory -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def arena_needs(set_a):
    """Bytes the device arenas of a context with the plugin's defaults hold after the whole batch, and after each
    problem alone (from released arenas)."""
    probs, _want = set_a
    a = B200Aligner(0)
    try:
        a.BatchAlign(PackedBatch.from_problems(probs))
        whole = a.debug_arena_bytes()
        alone = []
        for p in probs:
            a.release_arenas()
            a.BatchAlign(PackedBatch.from_problems([p]))
            alone.append(a.debug_arena_bytes())
    finally:
        a.close()
    return whole, alone


def test_out_of_memory_batch_is_split(set_a, arena_needs, tmp_path):
    """Arenas capped below what the batch needs, above what any problem needs alone: BatchAlign and the batcher's
    SingleAlign rounds give every problem the oracle's result, nmPerPosition included."""
    probs, want = set_a
    whole, alone = arena_needs
    assert max(alone) < whole
    cap = (max(alone) + whole) // 2
    env = {"NGMLR_B200_DEBUG_ARENA_CAP": str(cap)}
    _check_driver(_run_driver(tmp_path, probs, env=env), want)
    _check_driver(_run_driver(tmp_path, probs, env=dict(env, NGMLR_B200_BATCH_WINDOW_US="20000"), threads=8), want)


def test_out_of_memory_alone_fails_only_that_problem(set_a, arena_needs, tmp_path):
    """Arenas capped below what the largest problem needs alone: that problem gets ret -1 / Score -1 on every surface,
    its neighbours in the same batches match the oracle."""
    probs, want = set_a
    _whole, alone = arena_needs
    order = sorted(range(len(alone)), key=lambda i: alone[i])
    biggest, second = order[-1], order[-2]
    assert alone[second] < alone[biggest]
    env = {"NGMLR_B200_DEBUG_ARENA_CAP": str((alone[second] + alone[biggest]) // 2)}
    _check_driver(_run_driver(tmp_path, probs, env=env), want, failing=(biggest,))
    _check_driver(_run_driver(tmp_path, probs, env=dict(env, NGMLR_B200_BATCH_WINDOW_US="20000"), threads=8), want,
                  failing=(biggest,))
