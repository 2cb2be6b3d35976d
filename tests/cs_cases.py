"""Seeded genomes / sub-reads for the candidate-search tests (shared by CPU and GPU tests)."""
import numpy as np

from ngmlr_b200 import synth


def genome_contigs():
    g1 = synth.random_genome(60000, 1)
    g2 = synth.random_genome(30001, 2)          # odd length: nibble padding
    g1[5000:5010] = ord("N")
    g1[7000:7400] = ord("A")                    # homopolymer: same-bin de-duplication
    g1[0:3] = ord("N")
    g1[20:25] = ord("N")
    g1[59990:59995] = ord("N")
    g2[100:160] = np.tile(np.frombuffer(b"ACGTAC", dtype=np.uint8), 10)   # tandem repeat
    g3 = np.tile(synth.random_genome(300, 5), 50)                          # repeats: frequencies
    g4 = np.frombuffer(b"N" * 30 + b"ACGTACGTAGCTAGCTAGCATCGATCGATCAGCTACGATCAGCTACGACT" + b"N" * 5 +
                       b"ACGATCGATCGAC", dtype=np.uint8)
    return [g1, g2, g3, np.frombuffer(b"ACGTACGT", dtype=np.uint8), g4]


def subreads(n, seed, contigs=None):
    contigs = contigs or genome_contigs()
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        g = contigs[int(rng.integers(0, 3))]
        s = int(rng.integers(0, g.size - 400))
        sub, _m = synth.mutate(g[s:s + 320], rng, err=float(rng.choice([0, 0.1, 0.2])))
        sub = sub[:int(rng.choice([256, 256, 256, 100, 30, 13, 12, 1]))]
        if rng.random() < 0.3:
            sub = synth.revcomp(sub)
        if rng.random() < 0.2 and sub.size:
            sub = sub.copy()
            sub[rng.integers(0, sub.size, 3)] = ord("N")
        out.append(sub.tobytes())
    out += [b"", b"N" * 40, b"ACGT" * 64, b"A" * 256]
    return out


# ngmlr's options that the k-mer index, the candidate search and the sub-read scorer take: -k, --kmer-skip,
# --bin-size, -s, --subread-length and --subread-corridor (min_hits is IConfig's minKmerHits, which has no
# command-line flag). D holds ngmlr's defaults; each other set reaches branches the defaults never take.
OPTION_SETS = {
    "D": dict(k=13, skip=2, bin=4, s=0.8, min_hits=0, rpl=256, corridor=40),   # control
    "A": dict(k=10, skip=0, bin=4, s=0.8, min_hits=0, rpl=256, corridor=40),   # vote tables above CS_SMEM_CAP
    "B": dict(k=12, skip=1, bin=0, s=0.5, min_hits=0, rpl=128, corridor=42),   # odd window starts, half = 0
    "C": dict(k=14, skip=3, bin=6, s=1.0, min_hits=3, rpl=300, corridor=40),   # sw_ungapped<5>, ties at s = 1
    "E": dict(k=11, skip=2, bin=4, s=0.0, min_hits=0, rpl=512, corridor=120),  # gapped path, one and two passes
    "F": dict(k=15, skip=2, bin=4, s=0.8, min_hits=0, rpl=256, corridor=40),   # 4^15 + 1 index entries
}


def ref_max_len(o):
    """ScoreBuffer's refMaxLen: the decoded window of a sub-read candidate."""
    return ((o["rpl"] + 10 + o["corridor"]) | 1) + 1


def repeat_contigs():
    """A repeat-rich genome: 24 diverged copies of one 1.5 kb unit, so that a sub-read of the unit hits
    thousands of index positions; N runs inside and between the copies."""
    rng = np.random.default_rng(9)
    unit = synth.random_genome(1500, 8)
    g1 = np.concatenate([synth.mutate(unit, rng, err=0.03)[0] for _ in range(24)] + [synth.random_genome(9000, 10)])
    g1[2000:2003] = ord("N")
    g1[15000:15040] = ord("N")
    g2 = synth.random_genome(7001, 11)
    g3 = np.concatenate([unit, synth.random_genome(3000, 12), unit])
    return [g1, g2, g3]


def split_read(read, rpl):
    """ReadProvider::splitRead: a read of at least rpl bases -> its whole rpl-base parts, else the read itself."""
    if len(read) < rpl:
        return [read]
    return [read[k * rpl:(k + 1) * rpl] for k in range(len(read) // rpl)]


def option_reads(contigs, rpl, n, seed):
    """Reads for an option set: lengths around rpl - 1, rpl, rpl + 1 and 2 rpl + 1, plus short ones; both strands,
    sequencing errors, N runs, and reads that start or end at a contig end."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        c = contigs[i % len(contigs)]
        L = (rpl - 1, rpl, rpl + 1, 2 * rpl + 1, int(rng.integers(20, rpl)))[i % 5]
        L = min(L, c.size)
        if i % 7 == 3:
            r = c[:L].copy()
        elif i % 7 == 4:
            r = c[c.size - L:].copy()
        else:
            s = int(rng.integers(0, c.size - L + 1))
            r, _ = synth.mutate(c[s:s + L].copy(), rng, err=float(rng.choice([0.0, 0.05, 0.12])))
            r = np.ascontiguousarray(r[:L], dtype=np.uint8)
        if i % 6 == 5 and r.size > 40:
            a = int(rng.integers(0, r.size - 20))
            r[a:a + int(rng.integers(1, 12))] = ord("N")
        if rng.integers(0, 2):
            r = synth.revcomp(r)
        out.append(np.ascontiguousarray(r, dtype=np.uint8).tobytes())
    return out


def option_subreads(contigs, o, seed, n_reads=60):
    """The sub-reads stage 0 sees at option set o: cs_cases.subreads cut at rpl, then the parts of option_reads."""
    rpl = o["rpl"]
    subs = [s[:rpl] for s in subreads(120, seed, contigs)]
    for r in option_reads(contigs, rpl, n_reads, seed + 1):
        subs += split_read(r, rpl)
    return subs


def exact_windows(ref_starts, ref_lens, seed=3, n_random=300):
    """(start, sequence_len) pairs for DecodeRefSequenceExact(seq, start, sequence_len, 0): inside
    contigs (odd/even starts and lengths), running over a contig end ('x' padding), starting in the
    1000-N spacer before a contig. Starts behind a contig end but not within 1000 of the next contig
    make the reference decode a negative length (it crashes), so they are not part of the contract."""
    rng = np.random.default_rng(seed)
    out = []
    for s0, L in zip(ref_starts, ref_lens):
        end = s0 + L
        for st in (s0, s0 + 1, s0 + 2, s0 + 7, max(s0, end - 50), max(s0, end - 51), max(s0 + 1, end - 2), end - 1):
            for ln in (2, 3, 10, 11, 64, 301):
                out.append((int(st), int(ln)))
        for back in (1, 2, 17, 500, 998, 999):      # inside the spacer before the contig
            for ln in (5, 18, 700, 1301):
                out.append((int(s0 - back), int(ln)))
        for _ in range(n_random // len(ref_starts)):
            st = int(rng.integers(s0, end))
            out.append((st, int(rng.integers(2, 3000))))
    return out
