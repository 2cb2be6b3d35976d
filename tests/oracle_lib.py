"""ctypes bindings for the TEST-ONLY oracles: oracle/liboracle.so (C restatement) and, when it
was built in this container, oracle/_ref/libngmlr_ref.so (the unmodified reference)."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")

DEFAULT_SCORING = (2.0, -5.0, -5.0, -5.0, -1.0, 0.15)  # match mismatch gapopen gapext(max) gapext_min decay


class AlignOut(C.Structure):
    _fields_ = [("ret", C.c_int), ("score", C.c_float), ("position_offset", C.c_int),
                ("qstart", C.c_int), ("qend", C.c_int), ("nm", C.c_int),
                ("alignment_length", C.c_int), ("cigar_op_count", C.c_int), ("sv_type", C.c_int),
                ("identity", C.c_float), ("first_ref", C.c_int), ("first_read", C.c_int),
                ("last_ref", C.c_int), ("last_read", C.c_int), ("nm_count", C.c_int)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["score_bits"] = int(np.float32(d["score"]).view(np.uint32))
        d["identity_bits"] = int(np.float32(d["identity"]).view(np.uint32))
        return d


class Scoring(C.Structure):
    _fields_ = [(k, C.c_float) for k in ("mat", "mis", "gap_open_read", "gap_open_ref", "gap_ext",
                                          "gap_ext_min", "gap_decay")]


def scoring_struct(sc=DEFAULT_SCORING):
    mat, mis, go, ge, gemin, decay = sc
    return Scoring(mat, mis, go, go, ge, gemin, decay)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _p(a, t=C.c_int):
    return a.ctypes.data_as(C.POINTER(t))


def build_oracle():
    subprocess.run(["make", "-s", "-C", ORACLE_DIR, "liboracle.so"], check=True)


def build_ref():
    subprocess.run(["make", "-s", "-C", ORACLE_DIR, "ref"], check=True)


class Oracle:
    """The C restatement (always available)."""

    def __init__(self):
        path = os.path.join(ORACLE_DIR, "liboracle.so")
        if not os.path.exists(path):
            build_oracle()
        self.lib = C.CDLL(path)
        self.lib.or_ssw_score.restype = C.c_float
        self.lib.or_ssw_score_striped.restype = C.c_float
        self.lib.or_convex_cells.restype = C.c_int64

    def single_align(self, ref, qry, offsets, lengths, ext_qstart=0, ext_qend=0,
                     scoring=DEFAULT_SCORING, rule=0):
        offsets, lengths = _i32(offsets), _i32(lengths)
        H = len(offsets)
        out = AlignOut()
        cap = 8 * (len(qry) + len(ref)) + 64
        cig = C.create_string_buffer(cap)
        md = C.create_string_buffer(cap)
        nm = np.zeros(3 * (2 * (len(qry) + 1) + len(ref)), dtype=np.int32)
        sc = scoring_struct(scoring)
        st = self.lib.or_convex_single_align(C.byref(sc), ref, qry, _p(offsets), _p(lengths), H,
                                             ext_qstart, ext_qend, rule, C.byref(out), cig, cap, md,
                                             cap, _p(nm), len(nm) // 3)
        d = out.as_dict()
        d.update(status=st, cigar=cig.value.decode(), md=md.value.decode(),
                 nm_positions=nm[:3 * d["nm_count"]].reshape(-1, 3).copy())
        return d

    def fill(self, ref, qry, offsets, lengths, scoring=DEFAULT_SCORING, rule=0):
        offsets, lengths = _i32(offsets), _i32(lengths)
        dirs = np.zeros(int(np.maximum(lengths, 0).sum()) + 1, dtype=np.uint8)
        bs, bx, by = C.c_float(), C.c_int(), C.c_int()
        sc = scoring_struct(scoring)
        self.lib.or_convex_fill(C.byref(sc), ref, len(ref), qry, len(offsets), _p(offsets), _p(lengths),
                                rule, _p(dirs, C.c_ubyte), C.byref(bs), C.byref(bx), C.byref(by))
        return dirs[:-1], bs.value, bx.value, by.value

    def cells(self, ref_len, offsets, lengths):
        offsets, lengths = _i32(offsets), _i32(lengths)
        return int(self.lib.or_convex_cells(ref_len, len(offsets), _p(offsets), _p(lengths)))

    def score_select(self, scores):
        """ScoreBuffer::topNSE restatement -> (order, kept, mq)."""
        s = np.ascontiguousarray(scores, dtype=np.float32)
        order = np.zeros(max(s.size, 1), dtype=np.int32)
        mq = C.c_int()
        kept = self.lib.or_score_select(s.ctypes.data_as(C.c_void_p), int(s.size),
                                        order.ctypes.data_as(C.c_void_p), C.byref(mq))
        return order[:s.size].copy(), int(kept), mq.value

    def ssw_score(self, ref, qry, striped=False):
        f = self.lib.or_ssw_score_striped if striped else self.lib.or_ssw_score
        return float(f(ref, qry))


def score_select_cases(seed, count):
    """Seeded score lists for ScoreBuffer::topNSE parity: small integer scores (ties everywhere),
    lengths around the 16-element insertion-sort threshold of std::sort and beyond."""
    rng = np.random.default_rng(seed)
    out = []
    for t in range(count):
        n = int(rng.choice([0, 1, 2, 3, 5, 16, 17, 18, 33, 64, 65, 100, 300])) if t % 3 else int(rng.integers(0, 40))
        kind = t % 5
        if kind == 0:
            s = rng.integers(0, 8, n)
        elif kind == 1:
            s = rng.integers(100, 257, n)
        elif kind == 2:
            s = np.sort(rng.integers(0, 50, n))
        elif kind == 3:
            s = np.full(n, 7)
        else:
            s = np.sort(rng.integers(0, 300, n))[::-1]
        out.append(np.ascontiguousarray(s, dtype=np.float32))
    return out


class Reference:
    """The unmodified reference (only where oracle/_ref was built, i.e. /root/reference exists)."""

    PATH = os.path.join(ORACLE_DIR, "_ref", "libngmlr_ref.so")

    @classmethod
    def available(cls):
        return os.path.exists(cls.PATH)

    def __init__(self, scoring=DEFAULT_SCORING):
        self.lib = C.CDLL(self.PATH)
        self.lib.ref_convex_create.restype = C.c_void_p
        self.lib.ref_convex_create.argtypes = [C.c_float] * 6
        self.lib.ref_ssw_create.restype = C.c_void_p
        self.h = C.c_void_p(self.lib.ref_convex_create(*scoring))
        self.ssw = C.c_void_p(self.lib.ref_ssw_create())

    def close(self):
        if self.h:
            self.lib.ref_convex_destroy(self.h)
            self.lib.ref_ssw_destroy(self.ssw)
            self.h = None

    def single_align(self, ref, qry, offsets, lengths, ext_qstart=0, ext_qend=0):
        offsets, lengths = _i32(offsets), _i32(lengths)
        out = AlignOut()
        cap = 8 * (len(qry) + len(ref)) + 64
        cig = C.create_string_buffer(cap)
        md = C.create_string_buffer(cap)
        nm = np.zeros(3 * (2 * (len(qry) + 1) + len(ref)), dtype=np.int32)
        threw = self.lib.ref_convex_single_align(self.h, ref, qry, _p(offsets), _p(lengths),
                                                 len(offsets), ext_qstart, ext_qend, C.byref(out),
                                                 cig, cap, md, cap, _p(nm), len(nm) // 3)
        d = out.as_dict()
        d.update(status=threw, cigar=cig.value.decode(), md=md.value.decode(),
                 nm_positions=nm[:3 * d["nm_count"]].reshape(-1, 3).copy())
        return d

    def fill(self, ref, qry, offsets, lengths, which=0):
        offsets, lengths = _i32(offsets), _i32(lengths)
        dirs = np.zeros(int(np.maximum(lengths, 0).sum()) + 1, dtype=np.uint8)
        bs, bx, by = C.c_float(), C.c_int(), C.c_int()
        self.lib.ref_convex_fill(self.h, ref, qry, _p(offsets), _p(lengths), len(offsets), which,
                                 _p(dirs, C.c_ubyte), C.byref(bs), C.byref(bx), C.byref(by))
        return dirs[:-1], bs.value, bx.value, by.value

    def ssw_score(self, ref, qry):
        r = C.c_float(0)
        self.lib.ref_ssw_single_score(self.ssw, ref, qry, C.byref(r))
        return r.value


ALIGN_KEYS = ("ret", "score_bits", "position_offset", "qstart", "qend", "nm", "alignment_length",
              "cigar_op_count", "sv_type", "identity_bits", "first_ref", "first_read", "last_ref",
              "last_read", "nm_count", "cigar", "md")


def same_alignment(a, b):
    """Bit-exact comparison of two single_align results; returns list of differing keys."""
    bad = []
    if a["ret"] < 0 and b["ret"] < 0:
        return [] if a["score_bits"] == b["score_bits"] else ["score_bits"]
    for k in ALIGN_KEYS:
        if a[k] != b[k]:
            bad.append(k)
    if not bad and not np.array_equal(a["nm_positions"], b["nm_positions"]):
        bad.append("nm_positions")
    return bad


# ---------------------------------------------------------------------------------------------
# candidate search (stage 0)
# ---------------------------------------------------------------------------------------------
class CsOracle:
    """C restatement of the reference layout, k-mer index and vote (oracle/cs_oracle.c)."""

    def __init__(self, contigs, k=13, skip=2, bin_shift=4, max_freq=1000):
        path = os.path.join(ORACLE_DIR, "liboracle.so")
        if not os.path.exists(path):
            build_oracle()
        lib = C.CDLL(path)
        lib.or_cs_create.restype = C.c_void_p
        lib.or_cs_concat_len.restype = C.c_uint64
        lib.or_cs_ref_start.restype = C.c_uint64
        for f in ("or_cs_tab", "or_cs_rci", "or_cs_pos", "or_cs_encoded"):
            getattr(lib, f).restype = C.c_void_p
        lib.or_cs_index_len.restype = C.c_uint32
        lib.or_cs_npos.restype = C.c_uint32
        self.lib = lib
        self.contigs = [bytes(c) for c in contigs]
        arr = (C.c_char_p * len(contigs))(*self.contigs)
        lens = (C.c_int64 * len(contigs))(*[len(c) for c in self.contigs])
        self.h = C.c_void_p(lib.or_cs_create(len(contigs), arr, lens))
        lib.or_cs_build_index(self.h, k, skip, bin_shift, max_freq)

    def close(self):
        if self.h:
            self.lib.or_cs_destroy(self.h)
            self.h = None

    @property
    def concat_len(self):
        return int(self.lib.or_cs_concat_len(self.h))

    def ref_starts(self):
        return [int(self.lib.or_cs_ref_start(self.h, i)) for i in range(self.lib.or_cs_ref_count(self.h))]

    def encoded(self):
        n = C.c_uint64()
        p = self.lib.or_cs_encoded(self.h, C.byref(n))
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n.value,)).copy()

    def index(self):
        n = int(self.lib.or_cs_index_len(self.h))
        npos = int(self.lib.or_cs_npos(self.h))
        tab = np.ctypeslib.as_array(C.cast(self.lib.or_cs_tab(self.h), C.POINTER(C.c_uint32)), shape=(n,)).copy()
        rci = np.ctypeslib.as_array(C.cast(self.lib.or_cs_rci(self.h), C.POINTER(C.c_int8)), shape=(n,)).copy()
        pos = np.ctypeslib.as_array(C.cast(self.lib.or_cs_pos(self.h), C.POINTER(C.c_uint32)), shape=(npos + 1,)).copy()
        return tab, rci, pos[:npos]

    def decode(self, position, buffer_len=308):
        buf = C.create_string_buffer(buffer_len + 4)
        ok = self.lib.or_cs_decode(self.h, C.c_uint64(position), C.c_uint64(buffer_len), buf)
        return buf.value if ok else None

    def decode_exact(self, start, seq_len, corridor=0):
        """DecodeRefSequenceExact -> bytes before the terminating NUL, or None for an invalid start."""
        buf = C.create_string_buffer(seq_len + 8)
        ok = self.lib.or_cs_decode_exact(self.h, C.c_uint64(start), C.c_uint64(seq_len), int(corridor), buf)
        return buf.raw[:seq_len].split(b"\0")[0] if ok else None

    def search(self, seq, sensitivity=0.8, min_kmer_hits=0.0, cap=4096):
        sc = (C.c_float * cap)()
        lo = (C.c_uint64 * cap)()
        rv = (C.c_int * cap)()
        mh = C.c_float()
        n = self.lib.or_cs_search(self.h, bytes(seq), len(seq), C.c_float(sensitivity),
                                  C.c_float(min_kmer_hits), sc, lo, rv, cap, C.byref(mh))
        return [(sc[i], int(lo[i]), rv[i]) for i in range(min(n, cap))], mh.value


class CsReference:
    """The unmodified reference's candidate search (oracle/_ref/libngmlr_full.so). One instance per
    process: the reference keeps its state in singletons."""

    PATH = os.path.join(ORACLE_DIR, "_ref", "libngmlr_full.so")
    _inited = None

    @classmethod
    def available(cls):
        return os.path.exists(cls.PATH)

    def __init__(self, fasta_path, options=None):
        """options: one of cs_cases.OPTION_SETS (ngmlr's defaults when None)."""
        assert CsReference._inited in (None, fasta_path), "reference singletons already initialised"
        self.lib = C.CDLL(self.PATH)
        lib = self.lib
        lib.ref_cs_concat_len.restype = C.c_ulonglong
        lib.ref_cs_ref_start.restype = C.c_ulonglong
        lib.ref_cs_ref_len.restype = C.c_ulonglong
        lib.ref_cs_index.restype = C.c_void_p
        if CsReference._inited is None:
            if options is None:
                lib.ref_cs_init(fasta_path.encode())
            else:
                o = options
                lib.ref_cs_init_opts(fasta_path.encode(), o["k"], o["skip"], o["bin"], C.c_float(o["s"]),
                                     o["min_hits"], o["rpl"], o["corridor"], 0)
            CsReference._inited = fasta_path

    @property
    def concat_len(self):
        return int(self.lib.ref_cs_concat_len())

    def ref_starts(self):
        return [int(self.lib.ref_cs_ref_start(i)) for i in range(0, self.lib.ref_cs_ref_count(), 2)]

    def index(self):
        il, rl, uo, uc = C.c_uint(), C.c_uint(), C.c_ulonglong(), C.c_uint()
        rt = C.POINTER(C.c_uint)()
        ip = self.lib.ref_cs_index(C.byref(il), C.byref(rt), C.byref(rl), C.byref(uo), C.byref(uc))
        raw = np.ctypeslib.as_array(C.cast(ip, C.POINTER(C.c_uint8)), shape=(il.value * 5,)).reshape(-1, 5)
        tab = np.empty(il.value, dtype=np.uint32)
        tab.view(np.uint8).reshape(-1, 4)[:] = raw[:, :4]   # no intermediate copy: a 15-mer index has 4^15 + 1 rows
        rci = raw[:, 4].copy().view(np.int8)
        pos = np.ctypeslib.as_array(rt, shape=(rl.value + 1,))[:rl.value].copy()
        assert uo.value == 0 and uc.value == 1
        return tab, rci, pos

    @classmethod
    def score_select(cls, scores):
        """The unmodified ScoreBuffer::topNSE on one (sub-)read's scores -> (order, kept, mq).
        Needs no reference genome (usable before/without __init__)."""
        lib = C.CDLL(cls.PATH)
        s = np.ascontiguousarray(scores, dtype=np.float32).copy()
        tags = np.arange(s.size, dtype=np.uint64)
        mq = C.c_int()
        kept = lib.ref_score_select(s.ctypes.data_as(C.c_void_p), tags.ctypes.data_as(C.c_void_p), int(s.size),
                                    C.byref(mq))
        return tags.astype(np.int32), int(kept), mq.value

    def decode(self, position, buffer_len=308):
        buf = C.create_string_buffer(buffer_len + 4)
        ok = self.lib.ref_cs_decode(C.c_ulonglong(position), C.c_ulonglong(buffer_len), buf)
        return buf.value if ok else None

    def decode_exact(self, start, seq_len, corridor=0):
        buf = C.create_string_buffer(seq_len + 128)
        ok = self.lib.ref_cs_decode_exact(C.c_ulonglong(start), C.c_ulonglong(seq_len), int(corridor), buf)
        return buf.raw[:seq_len].split(b"\0")[0] if ok else None

    def search(self, seq, table_bits=16, cap=4096):
        sc = (C.c_float * cap)()
        lo = (C.c_ulonglong * cap)()
        rv = (C.c_int * cap)()
        mh = C.c_float()
        n = self.lib.ref_cs_search(bytes(seq), len(seq), table_bits, sc, lo, rv, cap, C.byref(mh))
        return [(sc[i], int(lo[i]), rv[i]) for i in range(max(0, min(n, cap)))], mh.value


class _RefSamAln(C.Structure):
    _fields_ = [("ref_pos", C.c_ulonglong), ("ref_id", C.c_int), ("reverse", C.c_int), ("score", C.c_float),
                ("mq", C.c_int), ("nm", C.c_int), ("identity", C.c_float), ("qstart", C.c_int), ("qend", C.c_int),
                ("sv_type", C.c_int), ("primary", C.c_int), ("skip", C.c_int), ("cigar_ops", C.c_int),
                ("cigar", C.c_char_p), ("md", C.c_char_p)]


class _RefSamRead(C.Structure):
    _fields_ = [("name", C.c_char_p), ("seq", C.c_char_p), ("qual", C.c_char_p), ("length", C.c_int),
                ("n_aln", C.c_int), ("first_aln", C.c_longlong), ("mapped", C.c_int), ("empty", C.c_int)]


class SamReference:
    """The unmodified SAMWriter + GenericReadWriter::WriteRead (src/SAMWriter.cpp, src/GenericReadWriter.h)
    through ref_sam_write of oracle/ref_cs_shim.cpp. `lib` = libngmlr_full.so AFTER ref_cs_init (the writer takes
    the contig names from the reference's SequenceProvider singleton). Reads are ngmlr_b200.samtext.Read."""

    def __init__(self, lib):
        self.lib = lib
        lib.ref_sam_write.restype = C.c_longlong
        lib.ref_cs_ref_len.restype = C.c_ulonglong
        self.names, self.lens = [], []
        for i in range(0, lib.ref_cs_ref_count(), 2):   # every contig is listed twice (src/SAMWriter.cpp:30-35)
            buf = C.create_string_buffer(1024)
            k = lib.ref_cs_ref_name(i, buf, 1024)
            self.names.append(buf.raw[:k])
            self.lens.append(int(lib.ref_cs_ref_len(i)))

    def pack(self, reads):
        n_aln = sum(len(r.alignments) for r in reads)
        rr = (_RefSamRead * max(len(reads), 1))()
        aa = (_RefSamAln * max(n_aln, 1))()
        k = 0
        for i, r in enumerate(reads):
            rr[i] = _RefSamRead(r.name, r.seq, r.qual, len(r.seq), len(r.alignments), k, int(r.mapped), int(r.empty))
            for a in r.alignments:
                # the reference's ref ids count forward / reverse slots: contig j is id 2 * j
                aa[k] = _RefSamAln(a.ref_pos, 2 * a.ref_id, int(a.reverse), a.score, a.mq, a.nm, a.identity, a.qstart,
                                   a.qend, a.sv_type, int(a.primary), int(a.skip), a.cigar_ops, a.cigar, a.md)
                k += 1
        return rr, aa, len(reads), reads

    def write(self, what, packed, write_unmapped=True, bam_cigar_fix=False, rg_id=None, rg_fields=None,
              cmdline=b"ngmlr", cap=None):
        rr, aa, n, _keep = packed
        fields = (C.c_char_p * 11)(*rg_fields) if rg_fields else None
        args = (what, rr, n, aa, int(bam_cigar_fix), int(write_unmapped), rg_id, fields, cmdline)
        if cap is None:
            cap = self.lib.ref_sam_write(*args, None, 0)
        buf = C.create_string_buffer(cap + 1)
        got = self.lib.ref_sam_write(*args, buf, cap)
        assert got <= cap
        return buf.raw[:got]

    def records(self, reads, **kw):
        return self.write(1, self.pack(reads), **kw)

    def header(self, **kw):
        return self.write(0, self.pack([]), **kw)
