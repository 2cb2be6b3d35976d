"""Host-side mirror of ngmlr's aligner interface over the C ABI (include/ngmlr_b200.h).

`B200Aligner` plays the role of the reference's two IAlignment implementations on the hot path:
  convex alignment  <- Convex::ConvexAlignFast::SingleAlign  (src/ConvexAlignFast.cpp:452-559)
  sub-read scoring  <- StrippedSW::BatchScore / SingleScore   (src/StrippedSW.cpp:118-202)
Method names and argument meaning follow `class IAlignment` (src/IAlignment.h:211-247); the
batched convex entry point is what the reference's BatchAlign would be had it been implemented
(src/ConvexAlignFast.cpp:441-450 throws "Not implemented").

All compute happens in the CUDA library; nothing here (or anywhere in the package) computes an
alignment on the CPU.
"""
import ctypes as C
import os
from dataclasses import dataclass, field

import numpy as np

from . import _lib

DEFAULT_SCORING = (2.0, -5.0, -5.0, -5.0, -1.0, 0.15)


@dataclass
class LoadedReference:
    """What B200Aligner.load_reference installed: the contig table of SequenceProvider (kept contigs, names cut to
    100 characters; SAM writers list every contig twice), which cache files were read or written, and the phase times
    in milliseconds (host clock around work that ends in a device synchronise)."""
    PHASES = ("read", "install", "reference_write", "index", "index_write", "total")
    names: list
    starts: list
    lens: list
    concat_len: int
    reference_read: bool
    reference_written: bool
    index_read: bool
    index_written: bool
    ms: dict
    # the FASTA file's inflate (0 when the caches were read): bytes read from the file, BGZF members inflated on the
    # device, bytes returned by the host continuation, device inflate milliseconds
    compressed_bytes: int = 0
    device_members: int = 0
    host_bytes: int = 0
    inflate_ms: float = 0.0
    # the plain gzip path (a gzip file whose first member is not BGZF): bytes it returned from the device, chunks
    # placed, chunks decoded again after a chain mismatch, kernel milliseconds
    gzip_bytes: int = 0
    gzip_chunks: int = 0
    gzip_redecoded: int = 0
    gzip_ms: float = 0.0

    def sam_ref_names(self):
        """The reference list SAM records index (ids count both strands): every name twice."""
        return [n for n in self.names for _ in (0, 1)]


@dataclass
class Align:
    """The fields of the reference's `Align` that SingleAlign fills (src/IAlignment.h:112-191)."""
    ret: int = -1
    threw: bool = False
    Score: float = -1.0
    Identity: float = 0.0
    PositionOffset: int = 0
    QStart: int = 0
    QEnd: int = 0
    NM: int = 0
    alignmentLength: int = 0
    cigarOpCount: int = 0
    svType: int = 0
    firstPosition: tuple = (0, 0)
    lastPosition: tuple = (0, 0)
    pBuffer1: str = ""   # CIGAR
    pBuffer2: str = ""   # MD
    nmPerPosition: np.ndarray = field(default_factory=lambda: np.zeros((0, 3), np.int32))
    cells: int = 0
    nmCount: int = 0          # entries convertCigar records (nmPerPosition may be absent: device text stage)
    nSvRegions: int = 0       # low-identity regions the peak scan of detectMisalignment closes
    svRegions: np.ndarray = field(default_factory=lambda: np.zeros((0, 4), np.int32))

    def as_dict(self):
        """Same keys as tests/oracle_lib.py results, for bit-exact comparison."""
        return dict(ret=self.ret, status=int(self.threw),
                    score_bits=int(np.float32(self.Score).view(np.uint32)),
                    identity_bits=int(np.float32(self.Identity).view(np.uint32)),
                    position_offset=self.PositionOffset, qstart=self.QStart, qend=self.QEnd,
                    nm=self.NM, alignment_length=self.alignmentLength,
                    cigar_op_count=self.cigarOpCount, sv_type=self.svType,
                    first_ref=self.firstPosition[0], first_read=self.firstPosition[1],
                    last_ref=self.lastPosition[0], last_read=self.lastPosition[1],
                    nm_count=self.nmCount, cigar=self.pBuffer1, md=self.pBuffer2,
                    nm_positions=self.nmPerPosition, score=self.Score)


class PackedBatch:
    """A batch of SingleAlign problems laid out for the C ABI (host buffers)."""

    def __init__(self, refs, qrys, offsets, lengths, ext_qstart=None, ext_qend=None):
        n = len(refs)
        self.n = n
        self.refs = [bytes(r) for r in refs]
        self.qrys = [bytes(q) for q in qrys]
        self.ref_arr = (C.c_char_p * n)(*self.refs)
        self.qry_arr = (C.c_char_p * n)(*self.qrys)
        self.ref_lens = np.array([len(r) for r in self.refs], dtype=np.int32)
        self.qry_lens = np.array([len(q) for q in self.qrys], dtype=np.int32)
        self.row_start = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(self.qry_lens, out=self.row_start[1:])
        self.offsets = (np.ascontiguousarray(np.concatenate([np.asarray(o, np.int32) for o in offsets]))
                        if n else np.zeros(0, np.int32))
        self.lengths = (np.ascontiguousarray(np.concatenate([np.asarray(l, np.int32) for l in lengths]))
                        if n else np.zeros(0, np.int32))
        assert self.offsets.size == self.row_start[-1] == self.lengths.size, \
            "corridorHeight must equal the read length of every problem"
        self.ext_qstart = np.zeros(n, np.int32) if ext_qstart is None else np.asarray(ext_qstart, np.int32)
        self.ext_qend = np.zeros(n, np.int32) if ext_qend is None else np.asarray(ext_qend, np.int32)
        self.read_bases = int(self.qry_lens.sum())

    @classmethod
    def from_problems(cls, problems):
        return cls([p.ref for p in problems], [p.qry for p in problems], [p.offsets for p in problems],
                   [p.lengths for p in problems], [p.ext_qstart for p in problems],
                   [p.ext_qend for p in problems])

    def c_args(self):
        i32p, i64p = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
        return (self.n, self.ref_arr, self.ref_lens.ctypes.data_as(i32p), self.qry_arr,
                self.qry_lens.ctypes.data_as(i32p), self.offsets.ctypes.data_as(i32p),
                self.lengths.ctypes.data_as(i32p), self.row_start.ctypes.data_as(i64p),
                self.ext_qstart.ctypes.data_as(i32p), self.ext_qend.ctypes.data_as(i32p))


class PackedReads:
    """(Sub-)reads laid out for the C ABI once, reusable across calls."""

    def __init__(self, seqs):
        self.seqs = [bytes(s) for s in seqs]
        self.n = len(self.seqs)
        self.arr = (C.c_char_p * max(self.n, 1))(*self.seqs)
        self.lens = np.array([len(s) for s in self.seqs], dtype=np.int32)
        self.bases = int(self.lens.sum())


def split_read(seq, part_length=256):
    """ReadProvider::splitRead's sub-reads (src/ReadProvider.cpp:57-134): floor(len / part_length)
    consecutive pieces of part_length bases (the tail shorter than a part is not searched); a read
    shorter than one part is its own single sub-read (:76-104)."""
    n = len(seq) // part_length
    if n == 0:
        return [seq]
    return [seq[i * part_length:(i + 1) * part_length] for i in range(n)]


def select_candidates(cand_start, sw_scores):
    """ScoreBuffer::topNSE + computeMQ (src/ScoreBuffer.cpp:170-192, 33-45) for every (sub-)read of a
    scored batch (the arrays cs_score/cs_fetch return). Returns (order, kept, mq): `order` lists the
    candidate indices of each (sub-)read by descending score in the reference's std::sort order,
    kept[i] candidates of (sub-)read i go on to alignment, mq[i] is its mapping quality."""
    lib = _lib.load()
    cand_start = np.ascontiguousarray(cand_start, dtype=np.int64)
    sw_scores = np.ascontiguousarray(sw_scores, dtype=np.float32)
    n = int(cand_start.size) - 1
    if n < 0 or (n >= 0 and int(cand_start[-1]) != sw_scores.size):
        raise ValueError("cand_start must have n+1 entries ending at len(sw_scores)")
    order = np.zeros(max(sw_scores.size, 1), dtype=np.int32)
    kept = np.zeros(max(n, 1), dtype=np.int32)
    mq = np.zeros(max(n, 1), dtype=np.int32)
    rc = lib.ngmlr_b200_select_candidates(
        n, cand_start.ctypes.data_as(C.POINTER(C.c_int64)), sw_scores.ctypes.data_as(C.POINTER(C.c_float)),
        order.ctypes.data_as(C.POINTER(C.c_int32)), kept.ctypes.data_as(C.POINTER(C.c_int32)),
        mq.ctypes.data_as(C.POINTER(C.c_int32)))
    if rc != n:
        raise RuntimeError("ngmlr_b200_select_candidates failed")
    return order[:sw_scores.size], kept[:n], mq[:n]


class IntervalBatch:
    """computeAlignment calls laid out for the C ABI (ngmlr_b200_interval / ngmlr_b200_anchor arrays),
    built once from IntervalTask-like objects: attributes on_ref_start, on_ref_stop, corridor, ext_qstart,
    ext_qend, full_read_length, anchors [(onRead, onRef, isReverse)], realign, full_alignment, short_read,
    and either read_index / on_read_start / read_seq_len / reverse (resident read set) or read_seq (text)."""

    def __init__(self, tasks):
        n = len(tasks)
        self.n = n
        self.intervals = (_lib.Interval * max(n, 1))()
        n_anchor = sum(len(t.anchors) for t in tasks)
        self.anchors = (_lib.Anchor * max(n_anchor, 1))()
        self._keep = []
        a = 0
        for i, t in enumerate(tasks):
            iv = self.intervals[i]
            ridx = getattr(t, "read_index", -1)
            iv.read_index = ridx
            if ridx >= 0:
                iv.on_read_start = t.on_read_start
                iv.read_seq_len = t.read_seq_len
                iv.reverse = int(bool(t.reverse))
                iv.read_seq = None
            else:
                seq = None if t.read_seq is None else bytes(t.read_seq)
                self._keep.append(seq)
                iv.on_read_start = 0
                iv.read_seq_len = 0 if seq is None else len(seq)
                iv.reverse = 0
                iv.read_seq = seq
            iv.on_ref_start = t.on_ref_start
            iv.on_ref_stop = t.on_ref_stop
            iv.corridor = t.corridor
            iv.ext_qstart = t.ext_qstart
            iv.ext_qend = t.ext_qend
            iv.full_read_length = t.full_read_length
            iv.realign = int(bool(t.realign))
            iv.full_alignment = int(bool(t.full_alignment))
            iv.short_read = int(bool(t.short_read))
            iv.anchor_begin = a
            iv.n_anchors = len(t.anchors)
            for (on_read, on_ref, is_rev) in t.anchors:
                self.anchors[a].on_read = int(on_read)
                self.anchors[a].on_ref = int(on_ref)
                self.anchors[a].is_reverse = int(bool(is_rev))
                a += 1


@dataclass
class ReadBatch:
    """One ngmlr_b200_reads_load call: samtext.Read records, the number of sub-reads of the resident set, and the name
    of a read ngmlr would have dropped (quality length differs from the sequence length; it ends the file). The inflate
    counters are the handle's so far: bytes read from the file, BGZF members inflated on the device, bytes returned by
    the host continuation, device inflate milliseconds. So are the chunk counters: records resolved, the most device
    memory the handle held, chunks resolved, chunks cut short at a full line table, chunk doublings and the chunk
    capacity in bytes now. So are the plain gzip counters: bytes returned from the device, chunks placed, chunks
    decoded again after a chain mismatch, kernel milliseconds. `format` is the file's (_lib.READ_FORMAT_FASTX or
    READ_FORMAT_BAM), and the BAM counters are the handle's so far: header bytes, records walked, of them skipped
    (flag 0x100 / 0x800), reverse-complemented back (0x10) and without qualities."""
    reads: list
    n_sub: int
    dropped: list
    compressed_bytes: int = 0
    device_members: int = 0
    host_bytes: int = 0
    inflate_ms: float = 0.0
    records: int = 0
    device_bytes: int = 0
    chunks: int = 0
    line_limited: int = 0
    grows: int = 0
    chunk_cap: int = 0
    gzip_bytes: int = 0
    gzip_chunks: int = 0
    gzip_redecoded: int = 0
    gzip_ms: float = 0.0
    format: int = -1
    bam_header_bytes: int = 0
    bam_records: int = 0
    bam_skipped: int = 0
    bam_reversed: int = 0
    bam_no_quality: int = 0


class BgzfWriter:
    """A BGZF file written through a context's device (ngmlr_b200_bgzf_*): write() any bytes, flush() to end the
    current block and put everything written so far into the file, close() to add the EOF block. Usable as a context
    manager. stats(): bytes in, bytes of members out (the EOF block not counted), members, stored members, device
    milliseconds, device bytes held."""

    def __init__(self, lib, ctx, path, chunk_bytes=0):
        self.lib = lib
        self.h = C.c_void_p()
        opts = _lib.BgzfOptions(int(chunk_bytes))
        if lib.ngmlr_b200_bgzf_open(ctx, os.fsencode(path), C.byref(opts), C.byref(self.h)) != 0:
            self.h = None
            raise RuntimeError(lib.ngmlr_b200_last_error(None).decode())
        self._final = None

    def _check(self, rc):
        if rc < 0:
            raise RuntimeError(self.lib.ngmlr_b200_bgzf_last_error(self.h).decode())

    def write(self, data):
        data = bytes(data)
        self._check(self.lib.ngmlr_b200_bgzf_write(self.h, data, len(data)))

    def flush(self):
        self._check(self.lib.ngmlr_b200_bgzf_flush(self.h))

    def stats(self):
        if self.h is None:
            return self._final
        v = [C.c_int64(0) for _ in range(4)] + [C.c_float(0), C.c_int64(0)]
        self.lib.ngmlr_b200_bgzf_stats(self.h, *[C.byref(x) for x in v])
        keys = ("bytes_in", "bytes_out", "blocks", "stored_blocks", "device_ms", "device_bytes")
        return dict(zip(keys, [x.value for x in v]))

    def close(self):
        h = self.h
        if h is None:
            return
        if self.lib.ngmlr_b200_bgzf_flush(h) == 0:
            self._final = self.stats()
        self.h = None
        if self.lib.ngmlr_b200_bgzf_close(h) != 0:
            raise RuntimeError(self.lib.ngmlr_b200_last_error(None).decode())

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        # a handle dropped without close() still frees its buffers; an error it met has nobody left to report to
        try:
            self.close()
        except RuntimeError:
            pass


class B200Aligner:
    def __init__(self, gpu_id=0, scoring=DEFAULT_SCORING, stream=None):
        self.lib = _lib.load()
        sc = _lib.Scoring(*scoring)
        h = C.c_void_p()
        if self.lib.ngmlr_b200_create(gpu_id, C.byref(sc), C.byref(h)) != 0:
            raise RuntimeError(self.lib.ngmlr_b200_last_error(None).decode())
        self.h = h
        if stream is not None:
            self.lib.ngmlr_b200_set_stream(self.h, C.c_void_p(stream))

    def close(self):
        if getattr(self, "h", None):
            self.lib.ngmlr_b200_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc < 0:
            raise RuntimeError(self.lib.ngmlr_b200_last_error(self.h).decode())
        return rc

    # ---- IAlignment surface -------------------------------------------------------------
    def GetScoreBatchSize(self):
        return 1024

    def GetAlignBatchSize(self):
        return 1024

    def BatchScore(self, refSeqList, qrySeqList):
        n = len(refSeqList)
        refs = (C.c_char_p * n)(*[bytes(r) for r in refSeqList])
        qrys = (C.c_char_p * n)(*[bytes(q) for q in qrySeqList])
        out = np.full(n, -1.0, dtype=np.float32)
        self._check(self.lib.ngmlr_b200_sw_score_batch(self.h, n, refs, qrys,
                                                       out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def SingleScore(self, refSeq, qrySeq):
        return float(self.BatchScore([refSeq], [qrySeq])[0])

    def SingleAlign(self, refSeq, qrySeq, corridor_offsets, corridor_lengths, externalQStart=0,
                    externalQEnd=0):
        b = PackedBatch([refSeq], [qrySeq], [corridor_offsets], [corridor_lengths], [externalQStart],
                        [externalQEnd])
        return self.BatchAlign(b)[0]

    def BatchAlign(self, batch):
        """Returns an AlignBatchResult: records are decoded on access and, like the C ABI's result
        array, are valid until the next batch call on this aligner (`list(result)` copies them)."""
        res = (_lib.AlignResult * max(batch.n, 1))()
        self._check(self.lib.ngmlr_b200_convex_align_batch(self.h, *batch.c_args(), res))
        return self._collect(res, batch.n)

    # ---- candidate search (CS::RunRead's search) --------------------------------------------
    def set_index(self, index):
        """index: ngmlr_b200.refindex.KmerIndex (the reference's CompactPrefixTable arrays)."""
        packed = np.ascontiguousarray(index.packed_index())
        pos = np.ascontiguousarray(index.pos, dtype=np.uint32)
        self._check(self.lib.ngmlr_b200_cs_set_index(
            self.h, packed.ctypes.data_as(C.c_void_p), index.tab.size, pos.ctypes.data_as(C.c_void_p),
            pos.size, 0, index.k, index.bin_shift))

    def build_index(self, ref, k=13, kmer_skip=2, bin_shift=4, max_prefix_freq=1000, fetch=False):
        """CompactPrefixTable::CreateTable on the device, from the encoded reference set with set_reference
        (`ref`: its EncodedReference, for the contig table). Installs the index in this context; with
        fetch=True also returns it as a refindex.KmerIndex (host arrays in the reference's format)."""
        starts = np.asarray(ref.ref_start, dtype=np.uint64)
        lens = np.asarray(ref.ref_len, dtype=np.uint64)
        npos = C.c_uint32(0)
        u64p = C.POINTER(C.c_uint64)
        self._check(self.lib.ngmlr_b200_cs_build_index(self.h, starts.ctypes.data_as(u64p), lens.ctypes.data_as(u64p),
                                                       int(starts.size), k, kmer_skip, bin_shift, max_prefix_freq,
                                                       C.byref(npos)))
        self.index_build_ms = float(self.lib.ngmlr_b200_cs_last_build_ms(self.h))
        if not fetch:
            return npos.value
        return self.get_index(k, bin_shift)

    def share_reference(self, owner):
        """Use the encoded reference and k-mer index resident in `owner` (another B200Aligner on this GPU)."""
        self._check(self.lib.ngmlr_b200_cs_share_reference(self.h, owner.h))

    def get_index(self, k=13, bin_shift=4):
        from .refindex import KmerIndex
        n_idx, n_pos = C.c_uint32(0), C.c_uint32(0)
        self._check(self.lib.ngmlr_b200_cs_get_index(self.h, C.byref(n_idx), C.byref(n_pos), None, None))
        packed = np.zeros(n_idx.value * 5, dtype=np.uint8)
        pos = np.zeros(max(n_pos.value, 1), dtype=np.uint32)
        self._check(self.lib.ngmlr_b200_cs_get_index(self.h, None, None, packed.ctypes.data_as(C.c_void_p),
                                                     pos.ctypes.data_as(C.c_void_p)))
        rec = packed.reshape(-1, 5)
        tab = np.ascontiguousarray(rec[:, :4]).view(np.uint32).reshape(-1)
        rci = np.ascontiguousarray(rec[:, 4]).view(np.int8)
        return KmerIndex(k, bin_shift, tab, rci, pos[:n_pos.value])

    def cs_search(self, seqs, sensitivity=0.8, min_kmer_hits=0.0):
        """Candidates of each (sub-)read, in the reference's emission order:
        list of [(score, location, reverse)], plus maxHitNumber per read."""
        n = len(seqs)
        arr = (C.c_char_p * n)(*[bytes(s) for s in seqs])
        lens = np.array([len(s) for s in seqs], dtype=np.int32)
        start = np.zeros(n + 1, dtype=np.int64)
        mx = np.zeros(max(n, 1), dtype=np.float32)
        sc, lo, rv = C.POINTER(C.c_float)(), C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint8)()
        self._check(self.lib.ngmlr_b200_cs_search_batch(
            self.h, n, arr, lens.ctypes.data_as(C.POINTER(C.c_int32)), sensitivity, min_kmer_hits,
            start.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(sc), C.byref(lo), C.byref(rv),
            mx.ctypes.data_as(C.POINTER(C.c_float))))
        out = []
        for i in range(n):
            out.append([(sc[j], int(lo[j]), int(rv[j])) for j in range(start[i], start[i + 1])])
        return out, mx[:n]

    def encode_reference(self, contigs, fetch=True):
        """_SequenceProvider::Init's encoding of the contigs (bytes / uint8 arrays) on the device; installs the encoded
        genome and refStartPos in this context. Returns the EncodedReference (with its bytes when fetch=True)."""
        from .refindex import EncodedReference
        seqs = [bytes(c) if not isinstance(c, (bytes, bytearray)) else c for c in contigs]
        n = len(seqs)
        arr = (C.c_char_p * max(n, 1))(*seqs)
        lens = (C.c_uint64 * max(n, 1))(*[len(s) for s in seqs])
        kept = C.c_int32(0)
        ks = (C.c_uint64 * max(n, 1))()
        kl = (C.c_uint64 * max(n, 1))()
        nb, cl = C.c_uint64(0), C.c_uint64(0)
        self.lib.ngmlr_b200_cs_encode_reference.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p),
                                                            C.POINTER(C.c_uint64), C.POINTER(C.c_int32),
                                                            C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                                            C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        self.lib.ngmlr_b200_cs_get_reference.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                                         C.POINTER(C.c_uint64)]
        self._check(self.lib.ngmlr_b200_cs_encode_reference(self.h, n, arr, lens, C.byref(kept), ks, kl, C.byref(nb),
                                                            C.byref(cl)))
        enc = np.zeros(nb.value if fetch else 0, dtype=np.uint8)
        if fetch:
            self._check(self.lib.ngmlr_b200_cs_get_reference(self.h, enc.ctypes.data_as(C.c_void_p), enc.size, None,
                                                             None))
        return EncodedReference(enc, int(cl.value), [int(ks[i]) for i in range(kept.value)],
                                [int(kl[i]) for i in range(kept.value)])

    def load_reference(self, path, k=13, kmer_skip=2, bin_shift=4, skip_write=False, rebuild=False, max_prefix_freq=1000):
        """ngmlr's start-up (ngmlr_b200_load_reference): the reference and its k-mer index from <path>-enc.2.ngm and
        <path>-ht-<k>-<kmer_skip>.2.ngm where they exist, else from the FASTA / FASTQ file (plain, gzip or BGZF) with the
        encoding and the index built on the device and both caches written next to it (unless skip_write). Installs
        the reference, refStartPos and the index in this context. Returns a LoadedReference: the contig table (names
        cut to 100 characters, SeqStart, SeqLen), which cache files were read / written, and the phase times."""
        opts = _lib.ReferenceOptions(k, kmer_skip, bin_shift, max_prefix_freq, int(bool(skip_write)), int(bool(rebuild)))
        n, cl, fl = C.c_int32(0), C.c_uint64(0), C.c_int32(0)
        self._check(self.lib.ngmlr_b200_load_reference(self.h, os.fsencode(path), C.byref(opts), C.byref(n),
                                                       C.byref(cl), C.byref(fl)))
        names = (C.c_char_p * n.value)()
        nlen = np.zeros(n.value, dtype=np.int32)
        starts = np.zeros(n.value, dtype=np.uint64)
        lens = np.zeros(n.value, dtype=np.uint64)
        u64p = C.POINTER(C.c_uint64)
        self._check(self.lib.ngmlr_b200_reference_contigs(self.h, names, nlen.ctypes.data_as(C.POINTER(C.c_int32)),
                                                          starts.ctypes.data_as(u64p), lens.ctypes.data_as(u64p)))
        ms = (C.c_float * 6)()
        self._check(self.lib.ngmlr_b200_load_reference_ms(self.h, ms))
        f = fl.value
        cb, dm, hb, ims = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_float(0)
        self._check(self.lib.ngmlr_b200_load_reference_inflate_stats(self.h, C.byref(cb), C.byref(dm), C.byref(hb),
                                                                      C.byref(ims)))
        gb, gc, gr, gms = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_float(0)
        self._check(self.lib.ngmlr_b200_load_reference_gzip_stats(self.h, C.byref(gb), C.byref(gc), C.byref(gr),
                                                                   C.byref(gms)))
        return LoadedReference([names[i][:int(nlen[i])] for i in range(n.value)], [int(x) for x in starts],
                               [int(x) for x in lens], int(cl.value),
                               bool(f & _lib.LOAD_REFERENCE_READ), bool(f & _lib.LOAD_REFERENCE_WRITTEN),
                               bool(f & _lib.LOAD_INDEX_READ), bool(f & _lib.LOAD_INDEX_WRITTEN),
                               dict(zip(LoadedReference.PHASES, [float(x) for x in ms])),
                               cb.value, dm.value, hb.value, float(ims.value), gb.value, gc.value, gr.value,
                               float(gms.value))

    def set_reference(self, ref):
        """ref: ngmlr_b200.refindex.EncodedReference (the reference's 4-bit `binRef`)."""
        enc = np.ascontiguousarray(ref.enc, dtype=np.uint8)
        self._check(self.lib.ngmlr_b200_cs_set_reference(self.h, enc.ctypes.data_as(C.c_void_p), enc.size,
                                                         ref.concat_len))
        if ref.ref_start:
            # refStartPos: contig starts + one artificial end entry (src/SequenceProvider.cpp:416-424)
            starts = np.array(list(ref.ref_start) + [ref.ref_start[-1] + ref.ref_len[-1] + 1000], dtype=np.uint64)
            self._check(self.lib.ngmlr_b200_set_ref_starts(self.h, starts.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                           int(starts.size)))

    def decode_windows(self, starts, seq_lens):
        """DecodeRefSequenceExact(buf, start, seq_len, 0) for every window -> list of bytes (the C
        strings, i.e. seq_len - 1 characters unless the reference data holds a NUL)."""
        starts = np.ascontiguousarray(starts, dtype=np.uint64)
        seq_lens = np.ascontiguousarray(seq_lens, dtype=np.int32)
        n = int(starts.size)
        off = np.zeros(n + 1, dtype=np.int64)
        off[1:] = np.cumsum(seq_lens.astype(np.int64))
        buf = C.create_string_buffer(int(off[-1]) + 1)
        self._check(self.lib.ngmlr_b200_decode_windows(
            self.h, n, starts.ctypes.data_as(C.POINTER(C.c_uint64)), seq_lens.ctypes.data_as(C.POINTER(C.c_int32)),
            buf, off.ctypes.data_as(C.POINTER(C.c_int64))))
        raw = buf.raw
        return [raw[off[i]:off[i + 1]].split(b"\0")[0] for i in range(n)]

    def upload_windows(self, batch, on_ref_start, on_ref_stop):
        """upload() with the reference windows of `batch` named by concatenated-genome positions
        (extractReferenceSequenceForAlignment(onRefStart, onRefStop)) and decoded on the device;
        batch.refs / ref_lens are ignored."""
        a = np.ascontiguousarray(on_ref_start, dtype=np.uint64)
        b = np.ascontiguousarray(on_ref_stop, dtype=np.uint64)
        assert a.size == batch.n and b.size == batch.n
        args = batch.c_args()
        u64p = C.POINTER(C.c_uint64)
        self._n = batch.n
        self._check(self.lib.ngmlr_b200_convex_upload_windows(self.h, batch.n, a.ctypes.data_as(u64p),
                                                             b.ctypes.data_as(u64p), *args[3:]))

    def cs_score(self, seqs, sensitivity=0.8, min_kmer_hits=0.0, corridor=40, read_part_length=256):
        """CS::RunRead + ScoreBuffer::DoRun for sub-reads: per read [(cs_score, location, reverse,
        sw_score)] in the reference's emission order."""
        n = len(seqs)
        arr = (C.c_char_p * n)(*[bytes(s) for s in seqs])
        lens = np.array([len(s) for s in seqs], dtype=np.int32)
        start = np.zeros(n + 1, dtype=np.int64)
        mx = np.zeros(max(n, 1), dtype=np.float32)
        sc, lo, rv, sw = (C.POINTER(C.c_float)(), C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint8)(),
                          C.POINTER(C.c_float)())
        self._check(self.lib.ngmlr_b200_cs_score_batch(
            self.h, n, arr, lens.ctypes.data_as(C.POINTER(C.c_int32)), sensitivity, min_kmer_hits, corridor,
            read_part_length, start.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(sc), C.byref(lo),
            C.byref(rv), C.byref(sw), mx.ctypes.data_as(C.POINTER(C.c_float))))
        return [[(sc[j], int(lo[j]), int(rv[j]), sw[j]) for j in range(start[i], start[i + 1])]
                for i in range(n)], mx[:n]

    def cs_upload(self, seqs):
        """seqs: list of bytes, or a PackedReads (pre-built C arrays, no per-call Python work)."""
        reads = seqs if isinstance(seqs, PackedReads) else PackedReads(seqs)
        self._cs_n = reads.n
        self._check(self.lib.ngmlr_b200_cs_upload(self.h, reads.n, reads.arr,
                                                  reads.lens.ctypes.data_as(C.POINTER(C.c_int32))))

    def cs_run(self, sensitivity=0.8, min_kmer_hits=0.0, corridor=40, read_part_length=256):
        """Resident stage 0/2 pass; returns (number of candidates, kernel milliseconds)."""
        m, ms = C.c_int64(0), C.c_float(0)
        self._check(self.lib.ngmlr_b200_cs_run(self.h, sensitivity, min_kmer_hits, corridor, read_part_length,
                                               C.byref(m), C.byref(ms)))
        return m.value, ms.value

    def cs_fetch(self):
        n = self._cs_n
        start = np.zeros(n + 1, dtype=np.int64)
        mx = np.zeros(max(n, 1), dtype=np.float32)
        sc, lo, rv, sw = (C.POINTER(C.c_float)(), C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint8)(),
                          C.POINTER(C.c_float)())
        self._check(self.lib.ngmlr_b200_cs_fetch(self.h, start.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(sc),
                                                 C.byref(lo), C.byref(rv), C.byref(sw),
                                                 mx.ctypes.data_as(C.POINTER(C.c_float))))
        m = int(start[-1])
        as_np = lambda p, dt: (np.ctypeslib.as_array(p, shape=(m,)).copy() if m else np.zeros(0, dt))
        return start, as_np(sc, np.float32), as_np(lo, np.uint64), as_np(rv, np.uint8), as_np(sw, np.float32), mx[:n]

    # ---- resident read set + computeAlignment for a batch of intervals -------------------------
    def set_text_stage(self, on_device, want_nm_positions=False):
        """Where convertCigar + the peak scan of detectMisalignment run (see ngmlr_b200_set_text_stage)."""
        self._check(self.lib.ngmlr_b200_set_text_stage(self.h, int(bool(on_device)), int(bool(want_nm_positions))))

    def reads_upload(self, reads, read_part_length=256):
        """The reads of a batch -> HBM, once. Stage 0/2 (cs_run / cs_fetch) then runs on their sub-reads
        (ReadProvider::splitRead, in read order), compute_alignments names read parts by index.
        Returns the number of sub-reads."""
        reads = reads if isinstance(reads, PackedReads) else PackedReads(reads)
        n_sub = self._check(self.lib.ngmlr_b200_reads_upload(
            self.h, reads.n, reads.arr, reads.lens.ctypes.data_as(C.POINTER(C.c_int32)), int(read_part_length)))
        self._cs_n = n_sub
        self._cs_reads = reads.n
        return n_sub

    def load_reads(self, path, read_part_length=256, max_reads=100_000, max_bases=0, chunk_bytes=0):
        """Reads a FASTA / FASTQ file (plain, gzip or BGZF) as ngmlr's ReadProvider reads its query file, parsed on the device
        (ngmlr_b200_reads_load). Yields one ReadBatch per call: its reads -- at most max_reads, and after the first no
        more than max_bases bases (0: no limit) -- are this context's resident read set while the batch is current,
        exactly as reads_upload would make them (cs_run / map_short_reads follow), and its `reads` are samtext.Read
        records (name, normalised bases, quality) for sam_format. A read ngmlr would drop for a quality string of
        another length ends the file; its name is in the last batch's `dropped`. A BAM file (any stream that starts
        with "BAM\\1" once inflated) gives the reads ReadProvider makes from `samtools fastq -n` of it, decoded on the
        device."""
        from .samtext import Read, SamRead
        f = C.c_void_p()
        opts = _lib.ReadFileOptions(int(chunk_bytes))
        if self.lib.ngmlr_b200_read_file_open(os.fsencode(path), C.byref(opts), C.byref(f)) != 0:
            raise RuntimeError(self.lib.ngmlr_b200_last_error(None).decode())
        try:
            recs = (SamRead * max(int(max_reads), 1))()
            n, nd = C.c_int32(0), C.c_int32(0)
            while True:
                n_sub = self._check(self.lib.ngmlr_b200_reads_load(self.h, f, int(max_reads), int(max_bases),
                                                                   int(read_part_length), recs, C.byref(n),
                                                                   C.byref(nd)))
                self._cs_n = n_sub
                self._cs_reads = n.value
                reads = []
                base, size = C.addressof(recs), C.sizeof(SamRead)
                ptr = lambda i, fld: C.c_void_p.from_address(base + i * size + getattr(SamRead, fld).offset).value
                for i in range(n.value):
                    r = recs[i]
                    seq = C.string_at(ptr(i, "seq"), r.length)
                    qual = C.string_at(ptr(i, "qual"), 2)  # "*" (FASTA, or no qualities) is NUL terminated
                    qual = b"*" if qual == b"*\0" else C.string_at(ptr(i, "qual"), r.length)
                    reads.append(Read(C.string_at(ptr(i, "name")), seq, qual, empty=bool(r.empty)))
                dropped = [self.lib.ngmlr_b200_reads_load_dropped(f)] if nd.value else []
                if reads or dropped:
                    cb, dm, hb, ims = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_float(0)
                    self.lib.ngmlr_b200_read_file_inflate_stats(f, C.byref(cb), C.byref(dm), C.byref(hb), C.byref(ims))
                    recs_n, dev = C.c_int64(0), C.c_int64(0)
                    self.lib.ngmlr_b200_read_file_stats(f, None, C.byref(recs_n), None, None, None, C.byref(dev))
                    ch = [C.c_int64(0) for _ in range(4)]
                    self.lib.ngmlr_b200_debug_read_file_chunks(f, *[C.byref(x) for x in ch])
                    gz = [C.c_int64(0) for _ in range(3)] + [C.c_float(0)]
                    self.lib.ngmlr_b200_read_file_gzip_stats(f, *[C.byref(x) for x in gz])
                    bam = [C.c_int64(0) for _ in range(5)]
                    self.lib.ngmlr_b200_read_file_bam_stats(f, *[C.byref(x) for x in bam])
                    yield ReadBatch(reads, n_sub, dropped, cb.value, dm.value, hb.value, float(ims.value), recs_n.value,
                                    dev.value, *[x.value for x in ch], *[x.value for x in gz],
                                    self.lib.ngmlr_b200_read_file_format(f), *[x.value for x in bam])
                if n.value == 0:
                    break
        finally:
            self.lib.ngmlr_b200_read_file_close(f)

    def bgzf_writer(self, path, chunk_bytes=0):
        """A BgzfWriter on this context's device: BAM (samtext.bam_header, then flush(), then samtext.bam_format
        batches) or BGZF-compressed SAM. chunk_bytes: page-locked staging per batch (0: 64 MiB)."""
        return BgzfWriter(self.lib, self.h, path, chunk_bytes)

    def resident_reads(self):
        """Test aid: the resident read set as the device holds it -- (read offsets, read lengths, sub-read offsets,
        sub-read lengths, arena bytes)."""
        n, m, nb = C.c_int32(0), C.c_int32(0), C.c_int64(0)
        self._check(self.lib.ngmlr_b200_debug_resident_reads(self.h, C.byref(n), C.byref(m), C.byref(nb), *[None] * 5))
        off = np.zeros(n.value + 1, dtype=np.uint64)
        ln = np.zeros(max(n.value, 1), dtype=np.int32)
        soff = np.zeros(max(m.value, 1), dtype=np.uint64)
        slen = np.zeros(max(m.value, 1), dtype=np.int32)
        arena = np.zeros(max(nb.value, 1), dtype=np.uint8)
        self._check(self.lib.ngmlr_b200_debug_resident_reads(self.h, None, None, None, off.ctypes.data, ln.ctypes.data,
                                                             soff.ctypes.data, slen.ctypes.data, arena.ctypes.data))
        return off if n.value else off[:1], ln[:n.value], soff[:m.value], slen[:m.value], arena[:nb.value]

    def reads_h2d_bytes(self):
        return int(self.lib.ngmlr_b200_reads_h2d_bytes(self.h))

    def score_short_reads(self, read_index, locs, reverse):
        """ScoreBuffer::scoreShortRead's score of every (resident read, location, strand) pair -> float32[n]."""
        ri = np.ascontiguousarray(read_index, dtype=np.int32)
        lo = np.ascontiguousarray(locs, dtype=np.uint64)
        rv = np.ascontiguousarray(reverse, dtype=np.uint8)
        out = np.zeros(max(ri.size, 1), dtype=np.float32)
        self._check(self.lib.ngmlr_b200_score_short_reads(
            self.h, int(ri.size), ri.ctypes.data_as(C.POINTER(C.c_int32)), lo.ctypes.data_as(C.POINTER(C.c_uint64)),
            rv.ctypes.data_as(C.POINTER(C.c_uint8)), out.ctypes.data_as(C.POINTER(C.c_float))))
        return out[:ri.size]

    def map_short_reads(self, read_part_length=256, min_residues=0.25):
        """ngmlr's short-read path (scoreShortRead -> processShortRead -> WriteRead) for every resident read of at most
        read_part_length bases, after reads_upload + cs_run. Returns one entry per resident read: None for a longer
        read (it takes the chaining path), else (mapped, [samtext.Alignment]) -- with the caller's name, bases and
        qualities a samtext.Read. ref_id indexes the reference list that names every contig twice."""
        from .samtext import Alignment, SamAln
        n = self._cs_reads
        n_aln = np.zeros(max(n, 1), dtype=np.int32)
        first = np.zeros(max(n, 1), dtype=np.int64)
        mapped = np.zeros(max(n, 1), dtype=np.int32)
        alns = C.c_void_p()
        total = C.c_int64(0)
        self._check(self.lib.ngmlr_b200_map_short_reads(
            self.h, int(read_part_length), float(min_residues), n_aln.ctypes.data_as(C.POINTER(C.c_int32)),
            first.ctypes.data_as(C.POINTER(C.c_int64)), mapped.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(alns),
            C.byref(total)))
        recs = C.cast(alns, C.POINTER(SamAln))
        out = []
        for i in range(n):
            if n_aln[i] < 0:
                out.append(None)
                continue
            al = []
            for k in range(int(first[i]), int(first[i]) + int(n_aln[i])):
                a = recs[k]
                al.append(Alignment(int(a.ref_pos), int(a.ref_id), bool(a.reverse), a.score, a.mq, a.nm, a.identity,
                                    a.qstart, a.qend, bytes(a.cigar), bytes(a.md), a.sv_type, bool(a.primary),
                                    bool(a.skip), a.cigar_ops))
            out.append((bool(mapped[i]), al))
        return out

    def compute_alignments(self, tasks, read_part_length=256):
        """AlignmentBuffer::computeAlignment for every task (ngmlr_b200.intervals.IntervalTask or a
        prepared IntervalBatch): -> (AlignBatchResult, attempts int32[n]); a record with ret < 0 means the
        reference's computeAlignment returns 0."""
        ib = tasks if isinstance(tasks, IntervalBatch) else IntervalBatch(tasks)
        res = (_lib.AlignResult * max(ib.n, 1))()
        attempts = np.zeros(max(ib.n, 1), dtype=np.int32)
        self._check(self.lib.ngmlr_b200_compute_alignments(
            self.h, ib.n, ib.intervals, ib.anchors, int(read_part_length), res,
            attempts.ctypes.data_as(C.POINTER(C.c_int32))))
        return AlignBatchResult(res, ib.n), attempts[:ib.n]

    def intervals_upload(self, tasks, read_part_length=256):
        """Stage the first attempt of compute_alignments for run() / fetch() (inputs resident in HBM)."""
        ib = tasks if isinstance(tasks, IntervalBatch) else IntervalBatch(tasks)
        self._n = ib.n
        self._check(self.lib.ngmlr_b200_intervals_upload(self.h, ib.n, ib.intervals, ib.anchors, int(read_part_length)))

    def compute_alignments_stats(self):
        s = _lib.BatchStats()
        self._check(self.lib.ngmlr_b200_compute_alignments_stats(self.h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in s._fields_}

    # ---- phased interface (bench: inputs resident in HBM) ---------------------------------
    def upload(self, batch):
        self._n = batch.n
        self._check(self.lib.ngmlr_b200_convex_upload(self.h, *batch.c_args()))

    def run(self):
        self._check(self.lib.ngmlr_b200_convex_run(self.h))

    def fetch(self):
        res = (_lib.AlignResult * max(self._n, 1))()
        self._check(self.lib.ngmlr_b200_convex_fetch(self.h, res))
        return self._collect(res, self._n)

    def stats(self):
        s = _lib.BatchStats()
        self._check(self.lib.ngmlr_b200_convex_stats(self.h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in s._fields_}

    def force_raw(self, v):
        self.lib.ngmlr_b200_set_force_raw(self.h, int(v))

    def debug_set_arena_words(self, words):
        """Test hook: initial size of the direction arena (-1 = the host's estimate)."""
        self.lib.ngmlr_b200_debug_set_arena_words(self.h, int(words))

    def debug_set_arena_cap(self, nbytes):
        """Test hook: the device arenas of convex batches may hold at most `nbytes` bytes (-1 = no cap); a batch that
        needs more fails with "out of memory" as on a full device."""
        self.lib.ngmlr_b200_debug_set_arena_cap(self.h, int(nbytes))

    def debug_arena_bytes(self):
        """Test hook: bytes the device arenas of convex batches hold now."""
        return int(self.lib.ngmlr_b200_debug_arena_bytes(self.h))

    def release_arenas(self):
        """Free the arenas the convex batches grew (see ngmlr_b200_release_arenas)."""
        self._check(self.lib.ngmlr_b200_release_arenas(self.h))

    def debug_rampfree_problems(self):
        """Test hook: problems filled by the ramp-free fill kernels since the context was created."""
        return int(self.lib.ngmlr_b200_debug_rampfree_problems(self.h))

    def debug_rampfree2_problems(self):
        """Test hook: of those, problems filled by the kernel with two rows per lane."""
        return int(self.lib.ngmlr_b200_debug_rampfree2_problems(self.h))

    def debug_rampfree2_skew_problems(self):
        """Test hook: of those, problems filled with the second row of each lane one column behind its first."""
        return int(self.lib.ngmlr_b200_debug_rampfree2_skew_problems(self.h))

    def debug_short_read_pairs(self):
        """Test hook: pairs of the last short-read scoring (score_short_reads, map_short_reads) by scorer branch --
        the general affine path (general) and the ungapped path of the wide instantiation (wide)."""
        return {"general": int(self.lib.ngmlr_b200_debug_short_read_general_pairs(self.h)),
                "wide": int(self.lib.ngmlr_b200_debug_short_read_wide_pairs(self.h))}

    def debug_subread_pairs(self):
        """Test hook: the same counters for the last sub-read scoring (cs_run, cs_score)."""
        return {"general": int(self.lib.ngmlr_b200_debug_subread_general_pairs(self.h)),
                "wide": int(self.lib.ngmlr_b200_debug_subread_wide_pairs(self.h))}

    FILL_COUNTS = ("big_team", "rf_team", "rampfree", "ramped_warp", "ramped_team", "raw",
                   "fill_launches", "multi_launch", "three_way")

    def debug_fill_counts(self):
        """Test hook: the fill's routing counters since the aligner was created -- problems filled by the 16-warp launch
        (big_team), the ramp-free schedule's concurrent 4-warp team launch (rf_team), the ramp-free kernels (rampfree),
        the ramped one-warp and 4-warp team kernels of the ordinary launch (ramped_warp, ramped_team) and the RAW
        instantiation in any launch (raw); fill launches, those with more than one of the three concurrent launches
        non-empty (multi_launch) and those with all three (three_way)."""
        out = (C.c_longlong * len(self.FILL_COUNTS))()
        self._check(self.lib.ngmlr_b200_debug_fill_counts(self.h, out, len(out)))
        return dict(zip(self.FILL_COUNTS, (int(v) for v in out)))

    def set_small_batch_teams(self, on):
        """16-warp teams for batches of at most one problem per SM (default on); see ngmlr_b200_set_small_batch_teams."""
        self.lib.ngmlr_b200_set_small_batch_teams(self.h, int(bool(on)))

    def set_fill_ctas_per_sm(self, v):
        """Cap the persistent fill grid (0 = full occupancy); see ngmlr_b200_set_fill_ctas_per_sm."""
        self.lib.ngmlr_b200_set_fill_ctas_per_sm(self.h, int(v))

    def debug_set_big_team(self, cells, width):
        """Test hook: matrices of at least `cells` cells in corridors at least `width` wide get 16-warp teams."""
        self.lib.ngmlr_b200_debug_set_big_team(self.h, int(cells), int(width))

    def force_team(self, v):
        """-1 auto, 0 one warp per problem, 1 four-warp teams (fill kernel scheduling)."""
        self.lib.ngmlr_b200_set_force_team(self.h, int(v))

    def debug_directions(self, i, total_cells):
        dirs = np.zeros(total_cells + 1, dtype=np.uint8)
        bs, bx, by = C.c_float(), C.c_int32(), C.c_int32()
        self._check(self.lib.ngmlr_b200_convex_debug_directions(
            self.h, i, dirs.ctypes.data_as(C.POINTER(C.c_uint8)), total_cells, C.byref(bs),
            C.byref(bx), C.byref(by)))
        return dirs[:total_cells], bs.value, bx.value, by.value

    def sw_kernel_ms(self):
        return float(self.lib.ngmlr_b200_sw_last_kernel_ms(self.h))

    @staticmethod
    def _collect(res, n):
        return AlignBatchResult(res, n)


class AlignBatchResult:
    """Sequence of `Align` records of one batch. Records are materialised on access from the
    C result array (whose text/position buffers are owned by the aligner context and stay valid
    until its next batch call) -- copy what must outlive that."""

    def __init__(self, res, n):
        self._res = res
        self._n = n

    def __len__(self):
        return self._n

    def __eq__(self, other):
        return list(self) == other

    def __iter__(self):
        return (self[i] for i in range(self._n))

    def ret(self, i):
        return self._res[i].ret

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self[j] for j in range(*i.indices(self._n))]
        if i < 0:
            i += self._n
        if not 0 <= i < self._n:
            raise IndexError(i)
        r = self._res[i]
        nm = (np.ctypeslib.as_array(r.nm_positions, shape=(r.nm_count * 3,)).reshape(-1, 3).copy()
              if r.nm_count > 0 and r.nm_positions else np.zeros((0, 3), np.int32))
        sv = (np.ctypeslib.as_array(r.sv_regions, shape=(r.n_sv_regions_stored * 4,)).reshape(-1, 4).copy()
              if r.n_sv_regions_stored > 0 and r.sv_regions else np.zeros((0, 4), np.int32))
        return Align(ret=r.ret, threw=bool(r.threw), Score=float(r.score),
                     Identity=float(r.identity), PositionOffset=r.position_offset,
                     QStart=r.qstart, QEnd=r.qend, NM=r.nm,
                     alignmentLength=r.alignment_length, cigarOpCount=r.cigar_op_count,
                     svType=r.sv_type, firstPosition=(r.first_ref, r.first_read),
                     lastPosition=(r.last_ref, r.last_read),
                     pBuffer1=(r.cigar or b"").decode(), pBuffer2=(r.md or b"").decode(),
                     nmPerPosition=nm, cells=r.cells, nmCount=r.nm_count, nSvRegions=r.n_sv_regions,
                     svRegions=sv)
