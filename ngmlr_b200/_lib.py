"""Loader for the in-tree CUDA library (ngmlr_b200/libngmlr_b200.so).

The product has no CPU compute path: if the library is missing, or no CUDA device is present when
a context is created, this fails loudly instead of falling back."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# NGMLR_B200_LIBRARY: developer override to A/B-test another build of the same library (still CUDA only)
LIB_PATH = os.environ.get("NGMLR_B200_LIBRARY") or os.path.join(_HERE, "libngmlr_b200.so")


class Scoring(C.Structure):
    _fields_ = [(k, C.c_float) for k in ("match", "mismatch", "gap_open", "gap_extend",
                                          "gap_extend_min", "gap_decay")]


class AlignResult(C.Structure):
    _fields_ = [("ret", C.c_int32), ("threw", C.c_int32), ("score", C.c_float),
                ("identity", C.c_float), ("position_offset", C.c_int32), ("qstart", C.c_int32),
                ("qend", C.c_int32), ("nm", C.c_int32), ("alignment_length", C.c_int32),
                ("cigar_op_count", C.c_int32), ("sv_type", C.c_int32), ("first_ref", C.c_int32),
                ("first_read", C.c_int32), ("last_ref", C.c_int32), ("last_read", C.c_int32),
                ("nm_count", C.c_int32), ("cigar_len", C.c_int32), ("md_len", C.c_int32),
                ("cigar", C.c_char_p), ("md", C.c_char_p), ("nm_positions", C.POINTER(C.c_int32)),
                ("cells", C.c_int64), ("n_sv_regions", C.c_int32), ("n_sv_regions_stored", C.c_int32),
                ("sv_regions", C.POINTER(C.c_int32))]


class BatchStats(C.Structure):
    _fields_ = [("cells", C.c_int64), ("dir_bytes", C.c_int64), ("seq_bytes", C.c_int64),
                ("path_steps", C.c_int64), ("cigar_runs", C.c_int64), ("fill_ms", C.c_float),
                ("traceback_ms", C.c_float), ("compact_ms", C.c_float),
                ("fill_launches", C.c_int32), ("traceback_launches", C.c_int32),
                ("compact_launches", C.c_int32), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
                ("host_pack_ms", C.c_float), ("host_h2d_ms", C.c_float), ("host_run_ms", C.c_float),
                ("host_d2h_ms", C.c_float), ("host_text_ms", C.c_float), ("host_threads", C.c_int32),
                ("text_ms", C.c_float), ("text_launches", C.c_int32), ("text_bytes", C.c_int64)]


class Anchor(C.Structure):
    _fields_ = [("on_read", C.c_int32), ("is_reverse", C.c_int32), ("on_ref", C.c_int64)]


class Interval(C.Structure):
    _fields_ = [("read_index", C.c_int32), ("on_read_start", C.c_int32), ("read_seq_len", C.c_int32),
                ("reverse", C.c_int32), ("on_ref_start", C.c_uint64), ("on_ref_stop", C.c_uint64),
                ("corridor", C.c_int32), ("ext_qstart", C.c_int32), ("ext_qend", C.c_int32),
                ("full_read_length", C.c_int32), ("realign", C.c_int32), ("full_alignment", C.c_int32),
                ("short_read", C.c_int32), ("anchor_begin", C.c_int32), ("n_anchors", C.c_int32),
                ("read_seq", C.c_char_p)]


# every symbol include/ngmlr_b200.h declares (tests/test_abi.py checks the list against the header)
C_API_SYMBOLS = (
    "ngmlr_b200_abi_version", "ngmlr_b200_device_count", "ngmlr_b200_create", "ngmlr_b200_destroy",
    "ngmlr_b200_last_error", "ngmlr_b200_set_stream", "ngmlr_b200_get_stream",
    "ngmlr_b200_set_fill_ctas_per_sm", "ngmlr_b200_set_small_batch_teams",
    "ngmlr_b200_convex_align_batch", "ngmlr_b200_convex_upload", "ngmlr_b200_convex_run",
    "ngmlr_b200_convex_fetch", "ngmlr_b200_convex_stats", "ngmlr_b200_convex_debug_directions",
    "ngmlr_b200_sw_score_batch", "ngmlr_b200_cs_set_index", "ngmlr_b200_cs_search_batch",
    "ngmlr_b200_cs_set_reference", "ngmlr_b200_cs_score_batch", "ngmlr_b200_cs_upload",
    "ngmlr_b200_cs_run", "ngmlr_b200_cs_fetch", "ngmlr_b200_select_candidates",
    "ngmlr_b200_set_ref_starts", "ngmlr_b200_decode_windows", "ngmlr_b200_convex_upload_windows",
    "ngmlr_b200_cs_build_index", "ngmlr_b200_cs_get_index", "ngmlr_b200_cs_share_reference",
    "ngmlr_b200_set_text_stage", "ngmlr_b200_reads_upload", "ngmlr_b200_reads_h2d_bytes",
    "ngmlr_b200_compute_alignments", "ngmlr_b200_compute_alignments_stats", "ngmlr_b200_intervals_upload",
    "ngmlr_b200_sam_header", "ngmlr_b200_sam_format", "ngmlr_b200_ngm_write_index", "ngmlr_b200_ngm_read_index",
    "ngmlr_b200_ngm_write_reference", "ngmlr_b200_ngm_read_reference", "ngmlr_b200_cs_encode_reference",
    "ngmlr_b200_cs_get_reference", "ngmlr_b200_dedupe_short_read_candidates", "ngmlr_b200_score_short_reads",
    "ngmlr_b200_map_short_reads", "ngmlr_b200_load_reference", "ngmlr_b200_reference_contigs",
)

# flags of ngmlr_b200_load_reference (include/ngmlr_b200.h)
LOAD_REFERENCE_READ, LOAD_REFERENCE_WRITTEN, LOAD_INDEX_READ, LOAD_INDEX_WRITTEN = 1, 2, 4, 8


class ReferenceOptions(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("k", "kmer_skip", "bin_shift", "max_prefix_freq", "skip_write", "rebuild")]
PLUGIN_SYMBOLS = ("CreateAlignment", "DeleteAlignment", "SetAlignmentScoring")

_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(make -C ngmlr_b200/csrc). ngmlr_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i32p, i64p = C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    cpp = C.POINTER(C.c_char_p)
    lib.ngmlr_b200_create.argtypes = [C.c_int, C.POINTER(Scoring), C.POINTER(vp)]
    lib.ngmlr_b200_destroy.argtypes = [vp]
    lib.ngmlr_b200_destroy.restype = None
    lib.ngmlr_b200_last_error.argtypes = [vp]
    lib.ngmlr_b200_last_error.restype = C.c_char_p
    lib.ngmlr_b200_set_stream.argtypes = [vp, vp]
    lib.ngmlr_b200_get_stream.argtypes = [vp]
    lib.ngmlr_b200_get_stream.restype = vp
    lib.ngmlr_b200_set_force_raw.argtypes = [vp, C.c_int]
    lib.ngmlr_b200_set_force_team.argtypes = [vp, C.c_int]
    lib.ngmlr_b200_set_fill_ctas_per_sm.argtypes = [vp, C.c_int]
    lib.ngmlr_b200_set_small_batch_teams.argtypes = [vp, C.c_int]
    lib.ngmlr_b200_debug_set_arena_words.argtypes = [vp, C.c_longlong]
    lib.ngmlr_b200_debug_rampfree_problems.argtypes = [vp]
    lib.ngmlr_b200_debug_rampfree_problems.restype = C.c_longlong
    lib.ngmlr_b200_debug_set_big_team.argtypes = [vp, C.c_longlong, C.c_int]
    batch = [vp, C.c_int, cpp, i32p, cpp, i32p, i32p, i32p, i64p, i32p, i32p]
    lib.ngmlr_b200_convex_upload.argtypes = batch
    lib.ngmlr_b200_convex_align_batch.argtypes = batch + [C.POINTER(AlignResult)]
    lib.ngmlr_b200_convex_run.argtypes = [vp]
    lib.ngmlr_b200_convex_fetch.argtypes = [vp, C.POINTER(AlignResult)]
    lib.ngmlr_b200_convex_stats.argtypes = [vp, C.POINTER(BatchStats)]
    lib.ngmlr_b200_convex_debug_directions.argtypes = [vp, C.c_int, C.POINTER(C.c_uint8), C.c_size_t,
                                                       C.POINTER(C.c_float), i32p, i32p]
    lib.ngmlr_b200_sw_score_batch.argtypes = [vp, C.c_int, cpp, cpp, C.POINTER(C.c_float)]
    lib.ngmlr_b200_cs_set_index.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, C.c_uint64, C.c_int, C.c_int]
    lib.ngmlr_b200_cs_search_batch.argtypes = [vp, C.c_int, cpp, i32p, C.c_float, C.c_float, i64p,
                                               C.POINTER(C.POINTER(C.c_float)),
                                               C.POINTER(C.POINTER(C.c_uint64)),
                                               C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_float)]
    lib.ngmlr_b200_cs_set_reference.argtypes = [vp, vp, C.c_uint64, C.c_uint64]
    lib.ngmlr_b200_cs_score_batch.argtypes = [vp, C.c_int, cpp, i32p, C.c_float, C.c_float, C.c_int, C.c_int,
                                              i64p, C.POINTER(C.POINTER(C.c_float)),
                                              C.POINTER(C.POINTER(C.c_uint64)),
                                              C.POINTER(C.POINTER(C.c_uint8)),
                                              C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_float)]
    lib.ngmlr_b200_cs_upload.argtypes = [vp, C.c_int, cpp, i32p]
    lib.ngmlr_b200_cs_run.argtypes = [vp, C.c_float, C.c_float, C.c_int, C.c_int, i64p, C.POINTER(C.c_float)]
    lib.ngmlr_b200_cs_fetch.argtypes = [vp, i64p, C.POINTER(C.POINTER(C.c_float)),
                                        C.POINTER(C.POINTER(C.c_uint64)), C.POINTER(C.POINTER(C.c_uint8)),
                                        C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_float)]
    u64p = C.POINTER(C.c_uint64)
    lib.ngmlr_b200_set_ref_starts.argtypes = [vp, u64p, C.c_int]
    lib.ngmlr_b200_decode_windows.argtypes = [vp, C.c_int, u64p, i32p, C.c_char_p, i64p]
    lib.ngmlr_b200_convex_upload_windows.argtypes = [vp, C.c_int, u64p, u64p, cpp, i32p, i32p, i32p, i64p, i32p, i32p]
    lib.ngmlr_b200_select_candidates.argtypes = [C.c_int, i64p, C.POINTER(C.c_float), i32p, i32p, i32p]
    lib.ngmlr_b200_cs_build_index.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_int, C.c_int, C.c_int,
                                              C.c_int, C.c_int, C.POINTER(C.c_uint32)]
    lib.ngmlr_b200_cs_get_index.argtypes = [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), vp, vp]
    lib.ngmlr_b200_cs_share_reference.argtypes = [vp, vp]
    lib.ngmlr_b200_cs_last_build_ms.argtypes = [vp]
    lib.ngmlr_b200_cs_last_build_ms.restype = C.c_float
    lib.ngmlr_b200_set_text_stage.argtypes = [vp, C.c_int, C.c_int]
    lib.ngmlr_b200_reads_upload.argtypes = [vp, C.c_int, cpp, i32p, C.c_int]
    lib.ngmlr_b200_reads_h2d_bytes.argtypes = [vp]
    lib.ngmlr_b200_reads_h2d_bytes.restype = C.c_int64
    lib.ngmlr_b200_compute_alignments.argtypes = [vp, C.c_int, C.POINTER(Interval), C.POINTER(Anchor), C.c_int,
                                                  C.POINTER(AlignResult), i32p]
    lib.ngmlr_b200_intervals_upload.argtypes = [vp, C.c_int, C.POINTER(Interval), C.POINTER(Anchor), C.c_int]
    lib.ngmlr_b200_compute_alignments_stats.argtypes = [vp, C.POINTER(BatchStats)]
    lib.ngmlr_b200_dedupe_short_read_candidates.argtypes = [C.c_int, i64p, C.POINTER(C.c_uint64), C.c_int, i32p, i64p]
    lib.ngmlr_b200_score_short_reads.argtypes = [vp, C.c_int, i32p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint8),
                                                 C.POINTER(C.c_float)]
    lib.ngmlr_b200_debug_short_read_general_pairs.argtypes = [vp]
    lib.ngmlr_b200_debug_short_read_general_pairs.restype = C.c_uint
    # the records' type is samtext.SamAln (passed as an untyped pointer here: samtext imports this module)
    lib.ngmlr_b200_map_short_reads.argtypes = [vp, C.c_int, C.c_float, i32p, i64p, i32p, C.POINTER(vp), i64p]
    lib.ngmlr_b200_load_reference.argtypes = [vp, C.c_char_p, C.POINTER(ReferenceOptions), i32p, u64p, i32p]
    lib.ngmlr_b200_reference_contigs.argtypes = [vp, cpp, i32p, u64p, u64p]
    lib.ngmlr_b200_load_reference_ms.argtypes = [vp, C.POINTER(C.c_float)]
    lib.ngmlr_b200_debug_read_fasta.argtypes = [C.c_char_p, C.c_uint64, i64p, u64p, u64p, u64p, i64p, u64p, C.c_char_p,
                                                C.c_char_p, C.c_char_p, C.c_int]
    lib.ngmlr_b200_sw_last_kernel_ms.argtypes = [vp]
    lib.ngmlr_b200_sw_last_kernel_ms.restype = C.c_float
    _lib = lib
    return lib
