/* include/ngmlr_b200.h -- C ABI of the H100-native ngmlr alignment hot path.
 *
 * libngmlr_b200.so exports two surfaces:
 *
 *  (1) The reference's dormant plugin contract, src/IAlignment.h:249-250:
 *          typedef IAlignment* (*pfCreateAlignment)(int const gpu_id);
 *          typedef void        (*pfDeleteAlignment)(IAlignment*);
 *      as  extern "C" IAlignment* CreateAlignment(int gpu_id) / void DeleteAlignment(IAlignment*).
 *      The object implements every virtual of `class IAlignment` (src/IAlignment.h:211-247)
 *      with the reference's argument meaning and error behaviour; the ABI-compatible C++
 *      declarations are in include/ngmlr_b200_ialignment.h. See INTEGRATION.md for the two
 *      construction sites a maintainer switches (src/AlignmentBuffer.h:345-363, src/NGM.cpp:350-362).
 *
 *  (2) The plain-C batch interface below (pointers + sizes only), which the C++ plugin object,
 *      the Python host layer (ctypes) and any other FFI bind. Each entry point names the reference
 *      interface it replaces.
 *
 * All calls on one context must come from one thread at a time (the reference uses one aligner
 * object per worker thread, SURVEY.md section 1). Functions return 0 on success, <0 on error;
 * ngmlr_b200_last_error() describes the failure. There is NO CPU fallback: without a CUDA device
 * ngmlr_b200_create() fails. The entry points that take no context (ngmlr_b200_select_candidates,
 * ngmlr_b200_sam_*, ngmlr_b200_ngm_*) are host code by design -- they touch only host-resident data
 * (sort order of the reference's std::sort, SAM text, cache files) -- and run without a device.
 */
#ifndef NGMLR_B200_H
#define NGMLR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NGMLR_B200_ABI_VERSION 3

/* Convex scoring parameters = ConvexAlignFast's constructor arguments
 * (src/ConvexAlignFast.h:20-27, src/ConvexAlignFast.cpp:29-43; CLI defaults src/IConfig.h:23-71):
 * --match 2 --mismatch -5 --gap-open -5 --gap-extend-max -5 --gap-extend-min -1 --gap-decay 0.15 */
typedef struct {
  float match, mismatch, gap_open, gap_extend, gap_extend_min, gap_decay;
} ngmlr_b200_scoring;

typedef struct ngmlr_b200_ctx ngmlr_b200_ctx;

/* Result of one convex alignment = the fields ConvexAlignFast::SingleAlign fills in `Align`
 * (src/IAlignment.h:112-191) plus its return value. Text and position buffers are owned by the
 * context and stay valid until the next *_align_batch / *_fetch call on it. */
typedef struct {
  int32_t ret;              /* SingleAlign return value: read bases covered by CIGAR incl. clips, or -1 */
  int32_t threw;            /* 1 where the reference would `throw` (caller maps to "unmapped") */
  float score;              /* Align::Score (-1.0f when ret < 0) */
  float identity;           /* Align::Identity */
  int32_t position_offset;  /* Align::PositionOffset */
  int32_t qstart, qend;     /* Align::QStart / QEnd (incl. externalQStart/End) */
  int32_t nm;               /* Align::NM */
  int32_t alignment_length; /* Align::alignmentLength */
  int32_t cigar_op_count;   /* Align::cigarOpCount */
  int32_t sv_type;          /* Align::svType */
  int32_t first_ref, first_read, last_ref, last_read; /* Align::firstPosition / lastPosition */
  int32_t nm_count;         /* entries written to Align::nmPerPosition */
  int32_t cigar_len, md_len;
  const char* cigar;        /* Align::pBuffer1, NUL-terminated */
  const char* md;           /* Align::pBuffer2, NUL-terminated */
  const int32_t* nm_positions; /* nm_count x {refPosition, readPosition, nm}; NULL in the device text
                               * stage unless requested (ngmlr_b200_set_text_stage) */
  int64_t cells;            /* DP cells evaluated (SURVEY.md section 8d unit of work) */
  /* The peak scan of AlignmentBuffer::detectMisalignment over nmPerPosition
   * (src/AlignmentBuffer.cpp:1319-1388): closed low-identity regions, each {startInv, stopInv,
   * startInvRead, stopInvRead} = the arguments from which the reference calls checkForSV.
   * n_sv_regions counts all of them (the reference's checkCount), the first n_sv_regions_stored
   * (at most 32) are listed. */
  int32_t n_sv_regions, n_sv_regions_stored;
  const int32_t* sv_regions;
} ngmlr_b200_align_result;

/* Aggregate device-side statistics of the last convex batch (for roofline accounting). */
typedef struct {
  int64_t cells;            /* DP cells evaluated by the fill kernel */
  int64_t dir_bytes;        /* direction bytes written to HBM (2 bit/cell, blocked layout incl. padding) */
  int64_t seq_bytes;        /* sequence bytes staged */
  int64_t path_steps;       /* traceback steps */
  int64_t cigar_runs;       /* binary CIGAR runs emitted */
  float fill_ms, traceback_ms, compact_ms; /* CUDA-event durations on the context's stream; compact_ms
                                            * is 0 (compaction is part of the traceback kernel) */
  int32_t fill_launches, traceback_launches, compact_launches;
  int64_t h2d_bytes, d2h_bytes;
  /* host wall-clock of the last upload / run / fetch phases (ms) */
  float host_pack_ms, host_h2d_ms, host_run_ms, host_d2h_ms, host_text_ms;
  int32_t host_threads;
  /* device text stage (convex_text.cu): kernel time, launches, bytes of CIGAR + MD text produced */
  float text_ms;
  int32_t text_launches;
  int64_t text_bytes;
} ngmlr_b200_batch_stats;

int ngmlr_b200_abi_version(void);
int ngmlr_b200_device_count(void);

/* Creates a context on CUDA device gpu_id. Replaces `new ConvexAlignFast(...)` + `new StrippedSW()`
 * (src/AlignmentBuffer.h:355-368) / `_NGM::CreateAlignment` (src/NGM.cpp:350-362). */
int ngmlr_b200_create(int gpu_id, const ngmlr_b200_scoring* scoring, ngmlr_b200_ctx** out);
void ngmlr_b200_destroy(ngmlr_b200_ctx* ctx);
const char* ngmlr_b200_last_error(const ngmlr_b200_ctx* ctx); /* ctx may be NULL: last create error */

/* Use an externally owned CUDA stream (e.g. torch's current stream) for all work; 0 = own stream. */
int ngmlr_b200_set_stream(ngmlr_b200_ctx* ctx, void* cuda_stream);
void* ngmlr_b200_get_stream(ngmlr_b200_ctx* ctx);

/* Tuning: cap the persistent grid of the fill kernel at `ctas_per_sm` CTAs per SM (0 = full occupancy,
 * the default; also NGMLR_B200_FILL_CTAS_PER_SM). A process that drives several contexts on one GPU
 * gets more overlap between their launches with a smaller grid per launch (bench.py uses 4). No
 * reference counterpart. Results do not depend on it. */
int ngmlr_b200_set_fill_ctas_per_sm(ngmlr_b200_ctx* ctx, int ctas_per_sm);

/* Tuning: a batch of at most one problem per SM (the plugin's SingleAlign batches -- a handful of blocking
 * callers) is filled by 16-warp teams, one SM per problem, because such a batch is about latency; `on` = 0
 * keeps the 4-warp teams / one-warp-per-problem kernels for every batch size (also
 * NGMLR_B200_SMALL_BATCH_BIG_TEAMS=0). Default on. No reference counterpart. Results do not depend on it. */
int ngmlr_b200_set_small_batch_teams(ngmlr_b200_ctx* ctx, int on);

/* Frees the device and pinned host arenas the context's convex batches grew (they grow again on the next batch).
 * The results of the last batch become invalid. The C++ plugin calls it when a batch ran out of memory, before it
 * splits the batch and retries the halves. No reference counterpart. */
int ngmlr_b200_release_arenas(ngmlr_b200_ctx* ctx);

/* ---- convex banded alignment: IAlignment::SingleAlign(mode, CorridorLine*, ...) batched -------
 * Replaces ConvexAlignFast::SingleAlign (src/ConvexAlignFast.cpp:452-559) for n independent
 * problems. Problem i: refs[i]/qrys[i] are the reference window and read part (need not be
 * NUL-terminated; lengths given), corridor rows i are offsets[row_start[i] .. row_start[i+1]) and
 * the matching lengths (CorridorLine::offset / ::length); row count must equal qry_lens[i].
 * ext_qstart/ext_qend may be NULL (zeros). Host buffers; H2D/D2H happen inside the call. */
int ngmlr_b200_convex_align_batch(ngmlr_b200_ctx* ctx, int n, const char* const* refs,
                                  const int32_t* ref_lens, const char* const* qrys,
                                  const int32_t* qry_lens, const int32_t* corridor_offsets,
                                  const int32_t* corridor_lengths, const int64_t* row_start,
                                  const int32_t* ext_qstart, const int32_t* ext_qend,
                                  ngmlr_b200_align_result* results);

/* The same work split into its three phases, so that benchmarks can time the kernels with the
 * inputs already resident in HBM:
 *   upload : pack + H2D (no kernels)
 *   run    : fill -> traceback (+ CIGAR compaction) kernels on resident inputs (no host<->device copies
 *            except the 16-byte allocation counters); may be called repeatedly on one upload
 *   fetch  : D2H of the binary CIGARs + host CIGAR/MD text, fills results[n] */
int ngmlr_b200_convex_upload(ngmlr_b200_ctx* ctx, int n, const char* const* refs,
                             const int32_t* ref_lens, const char* const* qrys,
                             const int32_t* qry_lens, const int32_t* corridor_offsets,
                             const int32_t* corridor_lengths, const int64_t* row_start,
                             const int32_t* ext_qstart, const int32_t* ext_qend);
int ngmlr_b200_convex_run(ngmlr_b200_ctx* ctx);
int ngmlr_b200_convex_fetch(ngmlr_b200_ctx* ctx, ngmlr_b200_align_result* results);
int ngmlr_b200_convex_stats(ngmlr_b200_ctx* ctx, ngmlr_b200_batch_stats* out);

/* Where ConvexAlignFast::convertCigar (src/ConvexAlignFast.cpp:112-333) and the peak scan of its
 * consumer AlignmentBuffer::detectMisalignment (src/AlignmentBuffer.cpp:1319-1388) run:
 *   on_device = 0 (default)  host threads; results carry the full nmPerPosition array -- what the
 *                            IAlignment plugin object needs to fill the caller's `Align`;
 *   on_device = 1            one more kernel after the traceback: CIGAR / MD text, NM, identity,
 *                            positions and the low-identity regions are produced on the GPU; only
 *                            strings and 96 bytes per alignment cross PCIe. nmPerPosition (12 bytes
 *                            per alignment column) is materialised only if want_nm_positions != 0.
 * Results are identical either way (tests/test_gpu_text.py). Takes effect at the next upload. */
int ngmlr_b200_set_text_stage(ngmlr_b200_ctx* ctx, int on_device, int want_nm_positions);

/* Debug/parity aid: after convex_run, decode problem i's direction matrix into the reference's
 * row-major layout (AlignmentMatrixFast::directionMatrix, src/AlignmentMatrixFast.h:261): one
 * byte per corridor cell, values CIGAR_EQ 7 / X 8 / I 1 / D 2 / STOP 10, 0xFF = never written.
 * dirs must hold sum(lengths) bytes. Also returns the forward-fill best cell. */
int ngmlr_b200_convex_debug_directions(ngmlr_b200_ctx* ctx, int i, uint8_t* dirs, size_t dirs_cap,
                                       float* best_score, int32_t* best_ref, int32_t* best_read);

/* ---- sub-read scoring: IAlignment::BatchScore / SingleScore -----------------------------------
 * Replaces StrippedSW::BatchScore (src/StrippedSW.cpp:118-160). Strings must be NUL-terminated
 * (the reference scores strlen+1 characters). results[i] = best local score as float, or -1.0f
 * when a length is >= 100000. Returns n. */
int ngmlr_b200_sw_score_batch(ngmlr_b200_ctx* ctx, int n, const char* const* refs,
                              const char* const* qrys, float* results);

/* ---- k-mer candidate search: CS::RunRead's search --------------------------------------------
 * ngmlr_b200_cs_set_index takes the reference's in-memory k-mer index of one table unit exactly as
 * CompactPrefixTable holds it (src/PrefixTable.h:17-75): `packed_index` = Index records, 5 bytes
 * each ({uint m_TabIndex; char m_RevCompIndex}, #pragma pack(1)), index_len = 4^k + 1 of them;
 * `positions` = Location{uint} lists (cRefTableLen entries); unit_offset = TableUnit::Offset;
 * k = CS::prefixBasecount (--kmer-length, <= 16), bin_shift = Config.getBinSize() (--bin-size).
 * The arrays are copied to the device; host buffers may be released afterwards. */
int ngmlr_b200_cs_set_index(ngmlr_b200_ctx* ctx, const void* packed_index, uint32_t index_len,
                            const uint32_t* positions, uint32_t n_positions, uint64_t unit_offset,
                            int k, int bin_shift);

/* The same index BUILT ON THE DEVICE from the encoded reference that ngmlr_b200_cs_set_reference made
 * resident: replaces CompactPrefixTable::CreateTable for one table unit (src/PrefixTable.cpp:323-370:
 * CountKmerFreq + createRefTableIndex + Generate/BuildPrefixTable, driven by CS::PrefixIteration with
 * prefixskip = kmer_skip) and installs the result as the context's index. contig_start / contig_len =
 * SequenceProvider.GetRefStart / GetRefLen of the forward-strand entries (sorted); k = --kmer-length (13),
 * kmer_skip = --kmer-skip (2), bin_shift = --bin-size (4), max_prefix_freq = 1000
 * (src/PrefixTable.cpp:28). Bit-identical to the reference's arrays (tests/test_gpu_index.py). */
int ngmlr_b200_cs_build_index(ngmlr_b200_ctx* ctx, const uint64_t* contig_start, const uint64_t* contig_len,
                              int n_contigs, int k, int kmer_skip, int bin_shift, int max_prefix_freq,
                              uint32_t* n_positions);
/* Several contexts on one GPU (one per host thread -- the reference has one aligner object per worker
 * thread) share ONE copy of the encoded reference and k-mer index: ctx uses owner's device arrays. owner
 * must outlive ctx and must not replace its reference / index meanwhile. */
int ngmlr_b200_cs_share_reference(ngmlr_b200_ctx* ctx, ngmlr_b200_ctx* owner);
/* The context's index back in the reference's in-memory format (for the byte-compatible
 * -ht-<k>-<skip>.2.ngm writer): sizes, and -- where the pointers are not NULL -- index_len x 5 packed
 * Index bytes and n_positions Location words. */
int ngmlr_b200_cs_get_index(ngmlr_b200_ctx* ctx, uint32_t* index_len, uint32_t* n_positions, void* packed_index,
                            uint32_t* positions);

/* Candidate search for n (sub-)reads: replaces CS::PrefixIteration + PrefixSearch + AddLocationStd +
 * CollectResultsStd (src/CSstatic.cpp:23-73, src/CS.cpp:57-149, 217-269) as driven by
 * CS::RunRead (src/CS.cpp:324-398). sensitivity = Config.getSensitivity() (0.8),
 * min_kmer_hits = Config.getMinKmerHits() (0). On return cand_start[i] .. cand_start[i+1] index the
 * candidates of read i in the context-owned arrays *scores / *locs / *reverse
 * (LocationScore::Score.f, Location.m_Location, isReverse()), in the reference's emission order;
 * max_hits[i] = maxHitNumber (MappedRead::s). Arrays stay valid until the next cs call. */
int ngmlr_b200_cs_search_batch(ngmlr_b200_ctx* ctx, int n, const char* const* seqs,
                               const int32_t* lens, float sensitivity, float min_kmer_hits,
                               int64_t* cand_start, const float** scores, const uint64_t** locs,
                               const uint8_t** reverse, float* max_hits);

/* The 4-bit encoded, spacer-padded concatenated genome exactly as _SequenceProvider holds it
 * (`binRef`, src/SequenceProvider.cpp:76-105, 292-400): 2 bases per byte, A0 T1 G2 C3 N4;
 * concat_len = GetConcatRefLen(). Needed by ngmlr_b200_cs_score_batch. Copied to the device. */
int ngmlr_b200_cs_set_reference(ngmlr_b200_ctx* ctx, const uint8_t* bin_ref, uint64_t n_bytes,
                                uint64_t concat_len);

/* Candidate search + candidate scoring in one call: what CS::RunRead followed by
 * ScoreBuffer::DoRun computes for (sub-)reads (src/ScoreBuffer.cpp:87-168): every candidate of
 * ngmlr_b200_cs_search_batch is scored with the StrippedSW kernel against the window
 * DecodeRefSequence(buf, 0, loc - (corridor >> 1), ((read_part_length + 10 + corridor) | 1) + 1)
 * decoded on the device (src/SequenceProvider.cpp:567-625), using the read or, for reverse
 * candidates, MappedRead::computeReverseSeq (src/MappedRead.cpp:35-73). *sw_scores[j] is the float
 * ScoreBuffer writes to Scores[j].Score.f. corridor = Config.getReadPartCorridor() (40),
 * read_part_length = Config.getReadPartLength() (256). Other outputs as in cs_search_batch. */
int ngmlr_b200_cs_score_batch(ngmlr_b200_ctx* ctx, int n, const char* const* seqs,
                              const int32_t* lens, float sensitivity, float min_kmer_hits,
                              int corridor, int read_part_length, int64_t* cand_start,
                              const float** cs_scores, const uint64_t** locs, const uint8_t** reverse,
                              const float** sw_scores, float* max_hits);

/* The same stage-0/2 work in phases, so that benchmarks can time it with the reads resident in HBM:
 *   cs_upload : (sub-)reads -> device (no kernels)
 *   cs_run    : count -> size (device prefix sums) -> vote -> compact -> decode + score; results stay
 *               on the device; *n_candidates and the CUDA-event kernel time are returned. Needs
 *               cs_set_index and cs_set_reference. May be called repeatedly on one upload.
 *   cs_fetch  : D2H of the candidate arrays (same meaning as ngmlr_b200_cs_score_batch). */
int ngmlr_b200_cs_upload(ngmlr_b200_ctx* ctx, int n, const char* const* seqs, const int32_t* lens);
int ngmlr_b200_cs_run(ngmlr_b200_ctx* ctx, float sensitivity, float min_kmer_hits, int corridor,
                      int read_part_length, int64_t* n_candidates, float* kernel_ms);
int ngmlr_b200_cs_fetch(ngmlr_b200_ctx* ctx, int64_t* cand_start, const float** cs_scores,
                        const uint64_t** locs, const uint8_t** reverse, const float** sw_scores,
                        float* max_hits);

/* The same encoded genome BUILT ON THE DEVICE from the contigs' text: replaces the encoding loop of
 * _SequenceProvider::Init (src/SequenceProvider.cpp:292-400): A0 T1 G2 C3 in either case, everything else N;
 * 1000-N spacers before, between and after the contigs; contigs of <= 10 characters are skipped. Installs the
 * result as the context's reference AND its refStartPos (= ngmlr_b200_cs_set_reference + ngmlr_b200_set_ref_starts).
 * kept_start / kept_len (n_contigs entries of room) receive SeqStart / SeqLen of the *n_kept contigs that were kept:
 * the arguments of ngmlr_b200_cs_build_index and of the -enc.2.ngm writer. */
int ngmlr_b200_cs_encode_reference(ngmlr_b200_ctx* ctx, int n_contigs, const char* const* seqs, const uint64_t* lens,
                                   int32_t* n_kept, uint64_t* kept_start, uint64_t* kept_len, uint64_t* n_bytes,
                                   uint64_t* concat_len);
/* The context's encoded genome back in host memory: sizes always, the bytes where bin_ref is not NULL. */
int ngmlr_b200_cs_get_reference(ngmlr_b200_ctx* ctx, uint8_t* bin_ref, uint64_t cap, uint64_t* n_bytes,
                                uint64_t* concat_len);

/* ---- reference windows for alignment, decoded on the device -------------------------------------
 * refStartPos as _SequenceProvider holds it (src/SequenceProvider.cpp:416-424): the concatenated
 * start position of every contig (forward strand entries only) followed by one artificial entry
 * last_start + last_len + 1000. Needs ngmlr_b200_cs_set_reference (the encoded genome). */
int ngmlr_b200_set_ref_starts(ngmlr_b200_ctx* ctx, const uint64_t* ref_start_pos, int n_entries);

/* Replaces _SequenceProvider::DecodeRefSequenceExact(sequence, start, seq_len, 0)
 * (src/SequenceProvider.cpp:493-565) for n windows: window i is written to out + out_off[i],
 * seq_len[i] bytes with the NUL at seq_len[i] - 1; 'x' where the window runs past its contig or
 * starts in the spacer in front of it. Contract (as far as the reference itself is well defined):
 * 0 < start < GetConcatRefLen(), and start lies inside a contig or inside the 1000-N spacer in front
 * of one; otherwise -1. Returns n. */
int ngmlr_b200_decode_windows(ngmlr_b200_ctx* ctx, int n, const uint64_t* start, const int32_t* seq_len,
                              char* out, const int64_t* out_off);

/* ngmlr_b200_convex_upload with the reference windows named by position instead of shipped as text:
 * problem i aligns qrys[i] against extractReferenceSequenceForAlignment(on_ref_start[i], on_ref_stop[i])
 * (src/AlignmentBuffer.cpp:203-223: DecodeRefSequenceExact of stop - start + 1 characters incl. NUL),
 * decoded on the device straight into the sequence arena; run/fetch as usual. Same contract for the
 * start positions as ngmlr_b200_decode_windows, and start < stop. */
int ngmlr_b200_convex_upload_windows(ngmlr_b200_ctx* ctx, int n, const uint64_t* on_ref_start,
                                     const uint64_t* on_ref_stop, const char* const* qrys,
                                     const int32_t* qry_lens, const int32_t* corridor_offsets,
                                     const int32_t* corridor_lengths, const int64_t* row_start,
                                     const int32_t* ext_qstart, const int32_t* ext_qend);

/* ---- the read set resident in HBM + AlignmentBuffer::computeAlignment for a batch of intervals -----
 * ngmlr_b200_reads_upload: the reads of a batch cross PCIe once. Stage 0/2 then runs on their
 * sub-reads -- ReadProvider::splitRead (src/ReadProvider.cpp:57-134): floor(len / read_part_length)
 * consecutive pieces, a read shorter than one piece is its own sub-read -- through
 * ngmlr_b200_cs_run / ngmlr_b200_cs_fetch (sub-reads in read order), and stage 4 names read parts by
 * index. Returns the number of sub-reads, or < 0.
 * A read of at most read_part_length bases takes ngmlr's short-read path, whose candidate windows differ from the
 * sub-reads': cs_run's scores for it are the sub-read window's; ngmlr_b200_map_short_reads computes the real ones. */
int ngmlr_b200_reads_upload(ngmlr_b200_ctx* ctx, int n_reads, const char* const* seqs, const int32_t* lens,
                            int read_part_length);
int64_t ngmlr_b200_reads_h2d_bytes(const ngmlr_b200_ctx* ctx);

/* Anchor (src/Types.h: Anchor::onRead / onRef / isReverse) of an interval. */
typedef struct {
  int32_t on_read;
  int32_t is_reverse;
  int64_t on_ref;
} ngmlr_b200_anchor;

/* One call of AlignmentBuffer::computeAlignment(interval, corridor, readSeq, readLength,
 * externalQStart, externalQEnd, fullReadLength, read, realign, fullAlignment, shortRead)
 * (src/AlignmentBuffer.cpp:226-465). readSeq is named, not shipped: the part
 * [on_read_start, on_read_start + read_seq_len) of resident read `read_index`, reverse-complemented
 * when `reverse` (AlignmentBuffer::extractReadSeq, :1514-1545) -- or, with read_index < 0, the text
 * read_seq of read_seq_len characters (all intervals of a call must use the same form). */
typedef struct {
  int32_t read_index;
  int32_t on_read_start;
  int32_t read_seq_len;      /* readLength = strlen(readSeq) */
  int32_t reverse;
  uint64_t on_ref_start, on_ref_stop;   /* Interval::onRefStart / onRefStop */
  int32_t corridor;          /* the corridor argument (estimateCorridor(interval), :1454-1467) */
  int32_t ext_qstart, ext_qend;
  int32_t full_read_length;
  int32_t realign, full_alignment, short_read;
  int32_t anchor_begin, n_anchors;      /* Interval::anchors as a range of the anchors array */
  const char* read_seq;      /* only with read_index < 0 */
} ngmlr_b200_interval;

/* computeAlignment for n intervals: reference windows are decoded on the device
 * (extractReferenceSequenceForAlignment), the corridor of every attempt -- getCorridorFull /
 * getCorridorLinear / getCorridorEndpointsWithAnchors (multiplier < 3, not realigning, anchors
 * present) / getCorridorEndpoints, :333-352 -- is sent in closed form and its rows are generated on
 * the device, and while an alignment does not cover the read (cigarLength != fullReadLength) it is
 * repeated with corridorMultiplier + 1, at most 5 times and while corridor * multiplier <=
 * 2 * refSeqLen (:303-305). Attempt k of all intervals that are still invalid is ONE device batch.
 * results[i].ret == full_read_length for a valid alignment; ret = -1 where computeAlignment returns 0
 * (no reference window, every attempt invalid, or SingleAlign threw). attempts[i] (optional) = number
 * of SingleAlign calls the reference would have made. Uses the device text stage; result strings stay
 * valid until the next fetch / compute call on the context. Needs ngmlr_b200_cs_set_reference and
 * ngmlr_b200_set_ref_starts. read_part_length = Config.getReadPartLength() (256). Returns n or < 0. */
int ngmlr_b200_compute_alignments(ngmlr_b200_ctx* ctx, int n, const ngmlr_b200_interval* intervals,
                                  const ngmlr_b200_anchor* anchors, int read_part_length,
                                  ngmlr_b200_align_result* results, int32_t* attempts);
/* The first attempt of ngmlr_b200_compute_alignments only, staged for the phased calls:
 * ngmlr_b200_convex_run / ngmlr_b200_convex_fetch then operate on it (benchmarks time the kernels with
 * the batch resident in HBM). Every interval must reach SingleAlign. Switches the context to the device
 * text stage. */
int ngmlr_b200_intervals_upload(ngmlr_b200_ctx* ctx, int n, const ngmlr_b200_interval* intervals,
                                const ngmlr_b200_anchor* anchors, int read_part_length);
/* Totals over the device batches of the last ngmlr_b200_compute_alignments call. */
int ngmlr_b200_compute_alignments_stats(ngmlr_b200_ctx* ctx, ngmlr_b200_batch_stats* out);

/* Candidate selection once a (sub-)read's candidates are scored. Replaces ScoreBuffer::topNSE and
 * ScoreBuffer::computeMQ (src/ScoreBuffer.cpp:170-192, 33-45). Host code (the reference's is too): for
 * (sub-)read i the candidates [cand_start[i], cand_start[i+1]) are ordered by descending sw_scores with
 * the reference's std::sort call (same order among equal scores); order[] receives the candidate
 * indices in that order, kept[i] = how many exceed 0.75 x the best (MappedRead::Calculated: the
 * candidates that go on to alignment), mq[i] = ceil(60 * (s0 - s1) / s0), 60 with fewer than two
 * candidates (MappedRead::mappingQlty). No context: nothing runs on the device. Returns n or -1. */
int ngmlr_b200_select_candidates(int n, const int64_t* cand_start, const float* sw_scores, int32_t* order,
                                 int32_t* kept, int32_t* mq);

/* ---- ngmlr's on-disk caches, byte-compatible (SURVEY section 8(f)3) --------------------------------
 * <ref>-ht-<k>-<skip>.2.ngm: CompactPrefixTable::saveToFile / readFromFile (src/PrefixTable.cpp:534-630), one table
 * unit. packed_index / positions are the arrays of ngmlr_b200_cs_set_index / ngmlr_b200_cs_get_index, so an index
 * built on the device becomes the cache an unmodified ngmlr starts from. 0 on success; -2 cannot open, -3 short or
 * foreign file, -4 more than one table unit, -5 signature mismatch (the reference would rebuild the table). */
int ngmlr_b200_ngm_write_index(const char* path, int k, int kmer_skip, const void* packed_index, uint32_t index_len,
                               const uint32_t* positions, uint32_t n_positions, uint64_t unit_offset);
/* Sizes and header fields always; the arrays where the pointers are not NULL (index_len x 5 bytes, n_positions words). */
int ngmlr_b200_ngm_read_index(const char* path, int32_t* k, int32_t* kmer_skip, uint32_t* index_len,
                              uint32_t* n_positions, uint64_t* unit_offset, void* packed_index, uint32_t* positions);
/* <ref>-enc.2.ngm: _SequenceProvider::writeEncRefToFile / readEncRefFromFile (src/SequenceProvider.cpp:207-272).
 * bin_ref = the encoded genome of ngmlr_b200_cs_set_reference (used_bytes of it); alloc_bytes = the size the
 * reference allocates and writes, ((getSize() / 2) | 1) + 1 (src/SequenceProvider.cpp:274-290, 318) -- the tail
 * behind the used part is written as zeros (uninitialised memory in the reference's own file); seq_start / seq_len
 * = RefIdx::SeqStart / SeqLen per contig, names[i] (NULL: "c<i>") cut at 100 characters. */
int ngmlr_b200_ngm_write_reference(const char* path, const uint8_t* bin_ref, uint64_t used_bytes, uint64_t alloc_bytes,
                                   int n_refs, const uint64_t* seq_start, const uint32_t* seq_len,
                                   const char* const* names);
/* Counts always; arrays where not NULL: seq_start / seq_len[n_refs], names = n_refs x 101 bytes (NUL terminated),
 * bin_ref = used_bytes. */
int ngmlr_b200_ngm_read_reference(const char* path, uint32_t* n_refs, uint64_t* used_bytes, uint64_t* alloc_bytes,
                                  uint64_t* seq_start, uint32_t* seq_len, char* names, uint8_t* bin_ref);

/* ---- ngmlr's start-up in one call: _SequenceProvider::Init + the CompactPrefixTable constructor ------------------
 * (src/SequenceProvider.cpp:246-424, src/PrefixTable.cpp:97-128), with the encoding and the k-mer index built on the
 * device. In ngmlr's order:
 *   - <fasta>-enc.2.ngm exists: it is read and installed (ngmlr_b200_ngm_read_reference -> cs_set_reference +
 *     set_ref_starts); an invalid one is an error, as in ngmlr. Otherwise the FASTA / FASTQ file (plain or gzip) is
 *     read as ngmlr's kseq_read loop reads it, encoded on the device (cs_encode_reference) and the file is written
 *     unless skip_write.
 *   - <fasta>-ht-<k>-<kmer_skip>.2.ngm exists and is a valid single-unit table for k / kmer_skip: it is read and
 *     installed (cs_set_index). Otherwise the index is built on the device (cs_build_index) and written unless
 *     skip_write. A table ngmlr would reject (wrong cookie, k or skip; ngmlr stops there) is rebuilt as well.
 *   - rebuild = 1 ignores both files.
 * Caches are written under a temporary name and renamed; a cache that cannot be written is skipped (ngmlr warns and
 * goes on) and its flag stays clear. Genomes of more than 0xffff0000 - 1 positions (more than one table unit of the
 * reference's index) or with more k-mer callbacks than 2^31 are refused. On success the context holds the reference,
 * refStartPos and the index, ready for reads_upload -> cs_run; on failure it keeps what it held when the failure is
 * found before anything reaches the device (missing / unreadable / empty / oversized input) and holds no reference
 * and no index otherwise. opts NULL: k 13, kmer_skip 2, bin_shift 4, max_prefix_freq 1000, write, no rebuild.
 * *n_contigs = contigs kept (more than 10 bases), *concat_len = GetConcatRefLen(), *flags = NGMLR_B200_LOAD_* bits.
 * Returns 0 or < 0 (ngmlr_b200_last_error). */
typedef struct {
  int32_t k, kmer_skip, bin_shift, max_prefix_freq;
  int32_t skip_write;
  int32_t rebuild;
} ngmlr_b200_reference_options;
#define NGMLR_B200_LOAD_REFERENCE_READ 1    /* <fasta>-enc.2.ngm was read */
#define NGMLR_B200_LOAD_REFERENCE_WRITTEN 2 /* <fasta>-enc.2.ngm was written */
#define NGMLR_B200_LOAD_INDEX_READ 4        /* <fasta>-ht-<k>-<skip>.2.ngm was read */
#define NGMLR_B200_LOAD_INDEX_WRITTEN 8     /* <fasta>-ht-<k>-<skip>.2.ngm was written */
int ngmlr_b200_load_reference(ngmlr_b200_ctx* ctx, const char* fasta_path, const ngmlr_b200_reference_options* opts,
                              int32_t* n_contigs, uint64_t* concat_len, int32_t* flags);
/* The contig table of the last load_reference: per kept contig its name (cut to 100 characters as RefIdx::name,
 * name_lens[i] characters, NUL terminated; valid until the context's reference changes), SeqStart and SeqLen.
 * SAM writers name contig i twice (SequenceProvider's ids count both strands). Arrays may be NULL. Returns the number
 * of contigs, or < 0 when the context's reference did not come from load_reference. */
int ngmlr_b200_reference_contigs(ngmlr_b200_ctx* ctx, const char** names, int32_t* name_lens, uint64_t* starts,
                                 uint64_t* lens);

/* ---- SAM text (SURVEY section 8(f)4) ----------------------------------------------------------
 * Replaces SAMWriter::DoWriteProlog / DoWriteRead -> DoWriteReadGeneric / DoWriteUnmappedRead
 * (src/SAMWriter.cpp:22-85, 87-224, 301-363) and the per-read loop of GenericReadWriter::WriteRead
 * (src/GenericReadWriter.h:78-108) for batches of reads: the records of a batch are sized and then
 * written by host threads straight into the caller's buffer, in read order. Host code on purpose:
 * every byte of a SAM record that is not already host resident (CIGAR / MD from the device text
 * stage) is a few per cent of the record; names, bases and qualities never leave host memory.
 * Byte-identical with the reference's writer on the same records (tests/test_sam_text.py drives the
 * unmodified SAMWriter through oracle/_ref/libngmlr_full.so). Paired-end records (DoWritePair) are
 * not produced by ngmlr's long-read pipeline and are not built. */

/* One alignment of a read = MappedRead::Scores[i] + MappedRead::Alignments[i] as SAMWriter reads them. */
typedef struct {
  uint64_t ref_pos;     /* Scores[i].Location.m_Location (0-based on the contig; printed + 1) */
  int32_t ref_id;       /* index into ref_names (SequenceProvider.GetRefName(getrefId())) */
  int32_t reverse;      /* Location.isReverse() */
  float score;          /* Scores[i].Score.f -> AS:i / XE:i as (int) */
  int32_t mq;           /* Alignments[i].MQ */
  int32_t nm;           /* Alignments[i].NM */
  float identity;       /* Alignments[i].Identity -> XI:f as round(x * 10000) / 10000 with %g */
  int32_t qstart, qend; /* Alignments[i].QStart / QEnd */
  int32_t sv_type;      /* Alignments[i].svType, printed as SV:i when > -1 */
  int32_t primary;      /* Alignments[i].primary (flag 0x800 when 0) */
  int32_t skip;         /* Alignments[i].skip: no record, and left out of the other records' SA:Z */
  int32_t cigar_ops;    /* Alignments[i].cigarOpCount (only read with bam_cigar_fix) */
  const char* cigar;    /* Alignments[i].pBuffer1, NUL terminated */
  const char* md;       /* Alignments[i].pBuffer2, NUL terminated */
} ngmlr_b200_sam_aln;

/* One read = the MappedRead handed to GenericReadWriter::WriteRead. */
typedef struct {
  const char* name;      /* MappedRead::name */
  const char* seq;       /* MappedRead::Seq, `length` characters; the reverse complement (MappedRead::RevSeq,
                            src/MappedRead.cpp:37-69: A<->T, C<->G, everything else unchanged) is derived here */
  const char* qual;      /* MappedRead::qlty: `length` characters; "*" for FASTA input (src/IParser.h:93-95);
                            NULL = no quality array */
  int32_t length;        /* MappedRead::length */
  int32_t n_aln;         /* MappedRead::Calculated (<= 0: unmapped) */
  int64_t first_aln;     /* alignments [first_aln, first_aln + n_aln) of the alns array */
  int32_t mapped;        /* the `mapped` argument of WriteRead (0: written as unmapped whatever it holds) */
  int32_t empty;         /* read->HasFlag(NGMNames::Empty): an unmapped empty read is dropped */
} ngmlr_b200_sam_read;

typedef struct {
  int32_t write_unmapped;   /* Config.getWriteUnampped() (default 1) */
  int32_t bam_cigar_fix;    /* Config.getBamCigarFix(): >= 65536 CIGAR operations -> "<len>S" + CG:B:I tag */
  /* 0 (default): as coded -- every reverse-strand record of a read reverses the read's quality string in
   * place (src/SAMWriter.cpp:104-108), so the 2nd, 4th, ... reverse record of a read carries it forward
   * again. 1: the quality string follows the record's strand. A "*" quality (FASTA) is never reversed in
   * either mode; the reference reverses `length` bytes of its 2-byte buffer there (heap overflow). */
  int32_t fix_quality_orientation;
  int32_t threads;          /* host threads (<= 0: NGMLR_B200_HOST_THREADS / hardware default) */
  const char* rg_id;        /* Config.getRgId(): RG:Z tag on every record when not NULL */
} ngmlr_b200_sam_options;

/* @HD / @SQ / @PG / @RG lines (DoWriteProlog). rg_fields: the 11 optional @RG values in the reference's
 * order SM LB PL DS DT PU PI PG CN FO KS (NULL entries are left out; the line is written only with
 * opts->rg_id). Returns the number of bytes the header needs; it is written (without NUL) only when that
 * fits cap. */
size_t ngmlr_b200_sam_header(int n_refs, const char* const* ref_names, const uint64_t* ref_lens,
                             const char* version, const char* command_line, const ngmlr_b200_sam_options* opts,
                             const char* const* rg_fields, char* out, size_t cap);

/* The records of n_reads reads in read order (for each read: its non-skipped alignments in index order,
 * or one unmapped record). ref_names[i] has ref_name_lens[i] characters (the reference prints "%.*s").
 * Returns 0 and sets *written; -2 with *written = the bytes needed when cap is too small (nothing is
 * written then); -1 on invalid arguments. No context: nothing runs on the device. */
int ngmlr_b200_sam_format(const ngmlr_b200_sam_options* opts, int64_t n_reads, const ngmlr_b200_sam_read* reads,
                          const ngmlr_b200_sam_aln* alns, int n_refs, const char* const* ref_names,
                          const int32_t* ref_name_lens, char* out, size_t cap, size_t* written);

/* ---- reads of at most read_part_length bases: ScoreBuffer::scoreShortRead + AlignmentBuffer::processShortRead --
 * ngmlr does not split such a read (src/ReadProvider.cpp:152-156); CS::SendToBuffer (src/CS.cpp:307-316) sends it to
 * scoreShortRead instead of the sub-read scorer and the chaining code. cs_run scores its candidates with the sub-read
 * window of ScoreBuffer::DoRun; the calls below compute what the short-read path computes instead.
 *
 * The duplicate removal of scoreShortRead (src/ScoreBuffer.cpp:225-239): the candidates [cand_start[i],
 * cand_start[i+1]) of read i are sorted by location with the reference's std::sort call (equal locations -- the
 * forward and reverse candidate of one bin -- keep libstdc++'s order, which decides the surviving strand), and one is
 * kept iff lastLocation - location > read_part_length in unsigned 64-bit arithmetic (lastLocation starts at 0): after
 * the sort, exact repeats of the previous location and a first candidate at 0 are dropped. kept[] (room for
 * cand_start[n] entries) receives the candidate indices of the survivors in location order, read i's from
 * kept_start[i] to kept_start[i+1]. No context: host code. Returns n or -1. */
int ngmlr_b200_dedupe_short_read_candidates(int n, const int64_t* cand_start, const uint64_t* locs,
                                            int read_part_length, int32_t* kept, int64_t* kept_start);

/* scoreShortRead's scores (src/ScoreBuffer.cpp:245-272) for n (resident read, location, strand) pairs: read
 * read_index[i] of ngmlr_b200_reads_upload (any resident read), or its MappedRead::computeReverseSeq when
 * reverse[i], against DecodeRefSequence(buf, 0, loc - (corridor >> 1), len + corridor) with
 * corridor = (int)(len * 0.3 + 256) ('N' x (len + corridor) where decoding fails), StrippedSW::SingleScore semantics
 * (-1 for a read or window of >= 100000 characters). Windows decoded straight from the resident genome on the
 * device. Reads of at most 510 bases are scored by the packed ungapped path (exact for them: a gap costs 255); longer
 * ones by the general affine path. Returns n or < 0. */
int ngmlr_b200_score_short_reads(ngmlr_b200_ctx* ctx, int n, const int32_t* read_index, const uint64_t* locs,
                                 const uint8_t* reverse, float* scores);

/* The whole short-read path for every read of the resident batch of at most read_part_length (>= 1, no upper limit)
 * bases, after
 * ngmlr_b200_reads_upload (same read_part_length) + ngmlr_b200_cs_run: duplicate removal, scoring as
 * ngmlr_b200_score_short_reads, order + MQ as ngmlr_b200_select_candidates (without the 0.75 cut), the alignment loop
 * of processShortRead (src/AlignmentBuffer.cpp:2564-2639; each candidate aligned as computeAlignment(..., shortRead =
 * true) through ngmlr_b200_compute_alignments, kept if Score > 0 and the --min-residues test passes) and
 * SequenceProvider::convert of every kept location (src/SequenceProvider.cpp:180-205). Per resident read i:
 * n_aln[i] = -1 for a read longer than read_part_length (not handled here: it takes the chaining path), else the
 * number of alignments (MappedRead::Calculated), records (*alns)[first_aln[i] .. + n_aln[i]) and mapped[i] = the
 * `mapped` argument of WriteRead (the result of the LAST convert, as coded). The records carry everything
 * ngmlr_b200_sam_format needs except name, bases and qualities; ref_id indexes SequenceProvider's reference list,
 * which names every contig twice (ids count both strands: pass ref_names = {c0, c0, c1, c1, ...}). Records and
 * strings are owned by the context and stay valid until the next map_short_reads call. Returns the number of
 * resident reads or < 0. */
int ngmlr_b200_map_short_reads(ngmlr_b200_ctx* ctx, int read_part_length, float min_residues, int32_t* n_aln,
                               int64_t* first_aln, int32_t* mapped, const ngmlr_b200_sam_aln** alns,
                               int64_t* n_alns_total);

/* ---- reads from a FASTA / FASTQ file (plain or gzip): ReadProvider::NextRead -> FastXParser -> kseq_read ->
 * IParser::copyToRead (src/ReadProvider.cpp:136-187, src/IParser.h:51-117), parsed on the device ------------------
 * The file is read in chunks of chunk_bytes (0: 256 MiB) into page-locked memory (gzip inflated by zlib on the calling
 * thread); a chunk too small for one record grows. Each chunk goes to the device once: its line table, the record
 * structure (kseq's rules, multi-line FASTQ and quality lines starting with '@' / '>' included) and the normalised
 * bases are computed there. Device memory of a handle stays below 9 x chunk_bytes. No reference counterpart for
 * the handle itself. */
typedef struct ngmlr_b200_read_file ngmlr_b200_read_file;
typedef struct {
  int64_t chunk_bytes; /* page-locked staging per chunk; 0 = 256 MiB; grows for a larger record */
} ngmlr_b200_read_file_options;
/* opts may be NULL. Returns 0, or < 0 (ngmlr_b200_last_error(NULL) describes it). */
int ngmlr_b200_read_file_open(const char* path, const ngmlr_b200_read_file_options* opts, ngmlr_b200_read_file** out);
void ngmlr_b200_read_file_close(ngmlr_b200_read_file* f);
/* The next reads of the file -- at most max_reads (>= 1) and, after the first, no more than max_bases (<= 0: no
 * limit) bases in all -- become ctx's resident read set exactly as ngmlr_b200_reads_upload(ctx, *n_reads, seqs, lens,
 * read_part_length) with the strings ngmlr's ReadProvider makes: the name cut to 249 characters, bases upper-cased
 * with everything but A / C / G / T as N, the quality string as it is ("*" for FASTA). reads (room for max_reads)
 * receive name / seq / qual / length / empty with n_aln = 0, first_aln = 0, mapped = 0: ready for ngmlr_b200_sam_format once
 * ngmlr_b200_map_short_reads has filled those three. An empty record gets length 0 and empty = 1 (ngmlr writes
 * read_part_length + 16 N's and flags it Empty; no candidate and no SAM record can come of either). The strings
 * are owned by f until its next load. A FASTQ record whose qualities are missing or of another length is dropped
 * and ends the file, as ngmlr's "Length of read not equal length of quality values" error ends ngmlr: *n_dropped = 1
 * and ngmlr_b200_reads_load_dropped names it. Returns the number of sub-reads (as reads_upload), or < 0;
 * *n_reads == 0 at the end of the file. A record of 2^31 or more bases, a read error and a corrupt or truncated
 * gzip stream are errors. */
int ngmlr_b200_reads_load(ngmlr_b200_ctx* ctx, ngmlr_b200_read_file* f, int max_reads, int64_t max_bases,
                          int read_part_length, ngmlr_b200_sam_read* reads, int* n_reads, int* n_dropped);
/* Name of the read the last ngmlr_b200_reads_load dropped (cut as ngmlr cuts it), or NULL. */
const char* ngmlr_b200_reads_load_dropped(const ngmlr_b200_read_file* f);
/* Timings and sizes of the handle so far: bytes of stream read, records, milliseconds reading / inflating on the host,
 * in the device parse, gathering + copying back, and the most device memory the handle held. Any pointer may be NULL. */
int ngmlr_b200_read_file_stats(const ngmlr_b200_read_file* f, int64_t* stream_bytes, int64_t* records, float* read_ms,
                               float* parse_ms, float* gather_ms, int64_t* device_bytes);

#ifdef __cplusplus
}
#endif
#endif /* NGMLR_B200_H */
