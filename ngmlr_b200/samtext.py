"""ctypes mirror of the SAM text entry points (include/ngmlr_b200.h, csrc/sam_text.cpp): the records
SAMWriter / GenericReadWriter::WriteRead (src/SAMWriter.cpp, src/GenericReadWriter.h:78-108) would print for a
batch of reads, formatted by host threads of the library. Used by the tests and bench.py."""
import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional

from . import _lib


class SamAln(C.Structure):
    _fields_ = [("ref_pos", C.c_uint64), ("ref_id", C.c_int32), ("reverse", C.c_int32), ("score", C.c_float),
                ("mq", C.c_int32), ("nm", C.c_int32), ("identity", C.c_float), ("qstart", C.c_int32),
                ("qend", C.c_int32), ("sv_type", C.c_int32), ("primary", C.c_int32), ("skip", C.c_int32),
                ("cigar_ops", C.c_int32), ("cigar", C.c_char_p), ("md", C.c_char_p)]


class SamRead(C.Structure):
    _fields_ = [("name", C.c_char_p), ("seq", C.c_char_p), ("qual", C.c_char_p), ("length", C.c_int32),
                ("n_aln", C.c_int32), ("first_aln", C.c_int64), ("mapped", C.c_int32), ("empty", C.c_int32)]


class SamOptions(C.Structure):
    _fields_ = [("write_unmapped", C.c_int32), ("bam_cigar_fix", C.c_int32),
                ("fix_quality_orientation", C.c_int32), ("threads", C.c_int32), ("rg_id", C.c_char_p)]


@dataclass
class Alignment:
    """MappedRead::Scores[i] + MappedRead::Alignments[i] as the writer reads them."""
    ref_pos: int
    ref_id: int
    reverse: bool
    score: float
    mq: int
    nm: int
    identity: float
    qstart: int
    qend: int
    cigar: bytes
    md: bytes
    sv_type: int = -1
    primary: bool = True
    skip: bool = False
    cigar_ops: int = 0


@dataclass
class Read:
    name: bytes
    seq: bytes
    qual: Optional[bytes]          # None: no quality array; b"*": FASTA input
    alignments: List[Alignment] = field(default_factory=list)
    mapped: bool = True
    empty: bool = False


def _bind(lib):
    if getattr(lib, "_sam_bound", False):
        return
    lib.ngmlr_b200_sam_header.restype = C.c_size_t
    lib.ngmlr_b200_sam_header.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_uint64), C.c_char_p,
                                          C.c_char_p, C.POINTER(SamOptions), C.POINTER(C.c_char_p), C.c_void_p,
                                          C.c_size_t]
    lib.ngmlr_b200_sam_format.restype = C.c_int
    lib.ngmlr_b200_sam_format.argtypes = [C.POINTER(SamOptions), C.c_int64, C.POINTER(SamRead), C.POINTER(SamAln),
                                          C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int32), C.c_void_p,
                                          C.c_size_t, C.POINTER(C.c_size_t)]
    lib.ngmlr_b200_bam_header.restype = C.c_int
    lib.ngmlr_b200_bam_header.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_uint64), C.c_char_p,
                                          C.c_char_p, C.POINTER(SamOptions), C.POINTER(C.c_char_p), C.c_void_p,
                                          C.c_size_t, C.POINTER(C.c_size_t)]
    lib.ngmlr_b200_bam_format.restype = C.c_int
    lib.ngmlr_b200_bam_format.argtypes = [C.POINTER(SamOptions), C.c_int64, C.POINTER(SamRead), C.POINTER(SamAln),
                                          C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int32), C.c_int,
                                          C.POINTER(C.c_char_p), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib._sam_bound = True


def _options(write_unmapped, bam_cigar_fix, fix_quality_orientation, threads, rg_id):
    return SamOptions(int(write_unmapped), int(bam_cigar_fix), int(fix_quality_orientation), int(threads), rg_id)


def sam_header(ref_names, ref_lens, version=b"0.2.8", command_line=b"ngmlr", rg_id=None, rg_fields=None):
    """@HD / @SQ / @PG / @RG lines (SAMWriter::DoWriteProlog, src/SAMWriter.cpp:22-85)."""
    lib = _lib.load()
    _bind(lib)
    n = len(ref_names)
    names = (C.c_char_p * max(n, 1))(*ref_names)
    lens = (C.c_uint64 * max(n, 1))(*ref_lens)
    opts = _options(1, 0, 0, 1, rg_id)
    fields = None
    if rg_fields is not None:
        assert len(rg_fields) == 11
        fields = (C.c_char_p * 11)(*rg_fields)
    need = lib.ngmlr_b200_sam_header(n, names, lens, version, command_line, C.byref(opts), fields, None, 0)
    buf = C.create_string_buffer(need + 1)
    got = lib.ngmlr_b200_sam_header(n, names, lens, version, command_line, C.byref(opts), fields, buf, need)
    assert got == need
    return buf.raw[:need]


class PackedReads:
    """The C arrays of a batch (kept alive together with the byte strings they point to)."""

    def __init__(self, reads: List[Read]):
        self.n = len(reads)
        n_aln = sum(len(r.alignments) for r in reads)
        self.reads = (SamRead * max(self.n, 1))()
        self.alns = (SamAln * max(n_aln, 1))()
        self._keep = reads
        k = 0
        for i, r in enumerate(reads):
            self.reads[i] = SamRead(r.name, r.seq, r.qual, len(r.seq), len(r.alignments), k, int(r.mapped),
                                    int(r.empty))
            for a in r.alignments:
                self.alns[k] = SamAln(a.ref_pos, a.ref_id, int(a.reverse), a.score, a.mq, a.nm, a.identity, a.qstart,
                                      a.qend, a.sv_type, int(a.primary), int(a.skip), a.cigar_ops, a.cigar, a.md)
                k += 1


def sam_format(reads, ref_names, write_unmapped=True, bam_cigar_fix=False, fix_quality_orientation=False,
               threads=0, rg_id=None, cap=None):
    """SAM records of `reads` (list of Read or a PackedReads) in read order. With cap: (rc, bytes needed, text)."""
    lib = _lib.load()
    _bind(lib)
    packed = reads if isinstance(reads, PackedReads) else PackedReads(reads)
    n = len(ref_names)
    names = (C.c_char_p * max(n, 1))(*ref_names)
    name_lens = (C.c_int32 * max(n, 1))(*[len(x) for x in ref_names])
    opts = _options(write_unmapped, bam_cigar_fix, fix_quality_orientation, threads, rg_id)
    written = C.c_size_t(0)
    if cap is None:
        rc = lib.ngmlr_b200_sam_format(C.byref(opts), packed.n, packed.reads, packed.alns, n, names, name_lens, None,
                                       0, C.byref(written))
        assert rc in (0, -2), rc
        cap_ = written.value
    else:
        cap_ = cap
    buf = C.create_string_buffer(cap_ + 1)
    rc = lib.ngmlr_b200_sam_format(C.byref(opts), packed.n, packed.reads, packed.alns, n, names, name_lens, buf, cap_,
                                   C.byref(written))
    if cap is not None:
        return rc, written.value, buf.raw[:written.value] if rc == 0 else b""
    assert rc == 0, rc
    return buf.raw[:written.value]


def _bam_error(lib):
    return RuntimeError(lib.ngmlr_b200_last_error(None).decode())


def bam_header(ref_names, ref_lens, version=b"0.2.8", command_line=b"ngmlr", rg_id=None, rg_fields=None):
    """The BAM header whose text is sam_header's for the same arguments (ngmlr_b200_bam_header). Raises
    RuntimeError for an LN above 2^31 - 1."""
    lib = _lib.load()
    _bind(lib)
    n = len(ref_names)
    names = (C.c_char_p * max(n, 1))(*ref_names)
    lens = (C.c_uint64 * max(n, 1))(*ref_lens)
    opts = _options(1, 0, 0, 1, rg_id)
    fields = None
    if rg_fields is not None:
        assert len(rg_fields) == 11
        fields = (C.c_char_p * 11)(*rg_fields)
    need = C.c_size_t(0)
    rc = lib.ngmlr_b200_bam_header(n, names, lens, version, command_line, C.byref(opts), fields, None, 0,
                                   C.byref(need))
    if rc == -1:
        raise _bam_error(lib)
    buf = C.create_string_buffer(need.value)
    rc = lib.ngmlr_b200_bam_header(n, names, lens, version, command_line, C.byref(opts), fields, buf, need.value,
                                   C.byref(need))
    assert rc == 0, rc
    return buf.raw[:need.value]


def bam_format(reads, ref_names, target_names=None, write_unmapped=True, bam_cigar_fix=False,
               fix_quality_orientation=False, threads=0, rg_id=None, cap=None):
    """BAM records of `reads` (list of Read or a PackedReads) in read order: what samtools makes of sam_format's text
    for the same arguments (ngmlr_b200_bam_format). target_names: the header's contig names (default: ref_names
    without repeats, in order). Raises RuntimeError for a record BAM cannot hold. With cap: (rc, bytes needed,
    records)."""
    lib = _lib.load()
    _bind(lib)
    packed = reads if isinstance(reads, PackedReads) else PackedReads(reads)
    if target_names is None:
        target_names = list(dict.fromkeys(ref_names))
    n, nt = len(ref_names), len(target_names)
    names = (C.c_char_p * max(n, 1))(*ref_names)
    name_lens = (C.c_int32 * max(n, 1))(*[len(x) for x in ref_names])
    targets = (C.c_char_p * max(nt, 1))(*target_names)
    opts = _options(write_unmapped, bam_cigar_fix, fix_quality_orientation, threads, rg_id)
    written = C.c_size_t(0)

    def call(buf, size):
        rc = lib.ngmlr_b200_bam_format(C.byref(opts), packed.n, packed.reads, packed.alns, n, names, name_lens, nt,
                                       targets, buf, size, C.byref(written))
        if rc == -1:
            raise _bam_error(lib)
        return rc

    if cap is None:
        call(None, 0)
        cap_ = written.value
    else:
        cap_ = cap
    buf = C.create_string_buffer(cap_ + 1)
    rc = call(buf, cap_)
    if cap is not None:
        return rc, written.value, buf.raw[:written.value] if rc == 0 else b""
    assert rc == 0, rc
    return buf.raw[:written.value]
