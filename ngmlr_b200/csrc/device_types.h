// ngmlr_b200/csrc/device_types.h -- records shared between host runtime and sm_90a kernels.
#pragma once
#include <stdint.h>
#include <vector_types.h>  // int4

namespace nb {

// Direction codes as stored in HBM: 2 bits per DP cell. EQ and X share code 0; the traceback
// re-derives which one by comparing the two bases (raw byte equality, exactly the test the
// reference's fill uses, src/ConvexAlignFast.cpp:657).
enum : uint32_t { DIR_DIAG = 0, DIR_I = 1, DIR_D = 2, DIR_STOP = 3 };

// Reference op codes (src/AlignmentMatrixFast.h:15-24) used in the binary CIGAR.
enum : int { OP_I = 1, OP_D = 2, OP_S = 4, OP_EQ = 7, OP_X = 8, OP_STOP = 10 };

enum : int {
  ST_OK = 0,          // valid alignment
  ST_INVALID = 1,     // reference returns -1 (path left corridor core / best row 0 / length mismatch)
  ST_THROW = 2,       // reference would throw (binary CIGAR buffer exhausted)
  ST_DIR_OVERFLOW = 3 // direction arena exhausted: host grows the arena and re-runs
};

struct Scoring {
  float mat, mis, open_read, open_ref, gap_ext, ext_min, decay;
};

// One alignment problem (SingleAlign call). Offsets index the batch-wide arrays.
struct alignas(16) AlnDesc {
  uint64_t ref_off;   // byte offset of refSeq in the sequence arena (16-byte aligned)
  uint64_t qry_off;   // byte offset of qrySeq
  uint64_t row_off;   // first row in corridor_off[] / corridor_len[]
  uint64_t blk_off;   // first BlockRec of this problem
  uint64_t tb_off;    // first int of this problem's traceback scratch
  int32_t ref_len;
  int32_t height;     // rows = qryLen = corridorHeight
  int32_t tb_cap;     // ints of traceback scratch
  int32_t ref_cap;    // reference's binaryCigar capacity: max(200000, qryLen+1)  (:480-485)
  int32_t max_len;    // max corridor row length
  int32_t const_len;  // packed / closed-form corridor: the (constant) row length
  int32_t packed;     // 0: raw CorridorLines; 1: int8 offset deltas + one int32 base per 32-row block;
                      // 2: closed form -- no per-row data at all, rows are generated on the device
  // closed-form corridor (packed == 2), the reference's builders (src/AlignmentBuffer.cpp:68-197):
  //   ckind 0: offset[y] = c0 + cstep * y                       getCorridorLinear / getCorridorFull
  //   ckind 1: offset[y] = (int)(((float)y - cd) / ck - cright)  getCorridorEndpoints (cright = 0) /
  //                                                             getCorridorEndpointsWithAnchors (cd = 0)
  // float32, one rounding per operation, truncation toward zero -- as the reference computes them.
  int32_t ckind, c0, cstep;
  float cd, ck, cright;
  int32_t ext_qstart, ext_qend;  // externalQStart / externalQEnd of the call (device text stage)
  int32_t pad2;
};

// One 32-row block of a problem: where its direction words live and how steps map to columns.
// Cell (x, y) of row y = 32*b + t was computed at step s = x - base + (t >> k); its 2-bit code is
//   dir[word_off + (s >> 4) * (32 << k) + t] >> ((s & 15) * 2),
// k = FillOut::dir_shift: 0 for the kernels with one row per lane, 1 for the one with two (a lane's two rows share a
// step; its 16-step group of a 64-row block is one 64-word line, and the second 32-row half starts at word 32).
// k = 2, the two-row kernel with the second row one column behind: 64-word lines as for 1, s = x - base + t.
struct alignas(16) BlockRec {
  uint64_t word_off;
  int32_t base;
  int32_t nsteps;
};

// Boundary row handed from lane 31 of one block to lane 0 of the next (through L2), one record
// per reference column.
struct alignas(16) BndEntry {
  float S;        // score of the cell
  float U;        // what the cell below receives as up_cell
  uint32_t pack;  // run (low 16) | dir << 16
  uint32_t pad;
};

struct alignas(16) FillOut {
  float best_score;
  int32_t best_x, best_y;
  int32_t status;
  unsigned long long cells;
  int32_t dir_shift;  // layout of the problem's direction words (BlockRec), set by the kernel that filled it
};

struct alignas(16) TraceOut {
  int32_t status;
  int32_t n_runs;        // entries in the compact binary CIGAR incl. both clip entries
  int32_t ref_position;  // FwdResults::ref_position
  int32_t qstart, qend;
  int32_t steps;
  unsigned long long run_off;  // offset of the runs in the compact arena
};

// Corridor rows of one problem. Raw: CorridorLine::offset / ::length per row (8 B/row). Packed
// (every builder of the reference produces constant lengths and offsets that advance by < 128 per
// row): offset[32b] per block + int8 delta per row (1.1 B/row) -- the PCIe-dominant input shrinks 7x.
struct CorridorView {
  const int32_t* off;
  const int32_t* len;
  const int32_t* blk_base;
  const int8_t* delta;
  int const_len;
  int packed;
  int ckind, c0, cstep;
  float cd, ck, cright;
#ifdef __CUDACC__
  __device__ __forceinline__ void bind(const int32_t* c_off, const int32_t* c_len, const int32_t* c_blkbase,
                                       const int8_t* c_delta, const AlnDesc& d) {
    off = c_off + d.row_off;
    len = c_len + d.row_off;
    blk_base = c_blkbase + d.blk_off;
    delta = c_delta + d.row_off;
    const_len = d.const_len;
    packed = d.packed;
    ckind = d.ckind; c0 = d.c0; cstep = d.cstep;
    cd = d.cd; ck = d.ck; cright = d.cright;
  }
#endif
};

struct FillParams {
  const uint8_t* seq;
  const int32_t* c_off;
  const int32_t* c_len;
  const int32_t* c_blkbase;  // packed corridors: offset of row 32*b, indexed like BlockRec
  const int8_t* c_delta;     // packed corridors: offset[y] - offset[y-1]
  const AlnDesc* desc;
  const int32_t* order;   // problem indices, largest first
  int n;
  int first, last;        // this launch works on order[first, last)
  int problems_per_cta;   // short-lived CTAs: problems a warp / team takes before it exits (1)
  int sm_slot_count;      // strips per SM (<= FILL_SM_SLOTS) = teams of this launch that run on an SM at a time
  unsigned int* sm_slots; // non-persistent launches: per-SM bitmask of boundary strips in use (nullptr: strip = blockIdx.x)
  BlockRec* blocks;
  uint32_t* dir;                        // direction arena (32-bit words)
  unsigned long long dir_capacity;      // words
  unsigned long long* dir_alloc;        // bump pointer
  int* work_counter;
  BndEntry* bnd;                        // per-warp boundary strip: bnd_stride 16-byte records each
  unsigned long long bnd_stride;
  FillOut* out;
  Scoring sc;
};

struct TraceParams {
  const uint8_t* seq;
  const int32_t* c_off;
  const int32_t* c_len;
  const int32_t* c_blkbase;
  const int8_t* c_delta;
  const AlnDesc* desc;
  const int32_t* order;                // problems by decreasing matrix size (longest walks first)
  int n;
  const BlockRec* blocks;
  const uint32_t* dir;
  const FillOut* fill;
  int32_t* scratch;
  TraceOut* out;
  int32_t* runs;                       // compact arena
  unsigned long long runs_capacity;
  unsigned long long* runs_alloc;
};

// ---- device text stage (convex_text.cu) ---------------------------------------------------
enum : int { TX_OK = 0, TX_THROW = 1, TX_OVERFLOW = 2, TX_SKIP = 3 };
constexpr int TEXT_PEAK_CAP = 32;  // low-identity regions kept per alignment (all are counted)

struct alignas(16) TextOut {
  int32_t status;
  int32_t ret;               // SingleAlign's return value: read bases covered by the CIGAR incl. clips
  int32_t qstart, qend;
  int32_t nm, alignment_length, cigar_op_count, sv_type;
  int32_t first_ref, first_read, last_ref, last_read;
  int32_t nm_count, cigar_len, md_len, n_peaks;
  float identity;
  int32_t n_peaks_stored;
  unsigned long long text_off;  // CIGAR, NUL, MD, NUL
  unsigned long long peak_off;  // first stored region (int4: startInv, stopInv, startInvRead, stopInvRead)
  unsigned long long nm_off;    // first int of the nmPerPosition triples (only when requested)
};

struct TextParams {
  const uint8_t* seq;
  const AlnDesc* desc;
  const int32_t* order;
  int n;
  const TraceOut* trace;
  const int32_t* runs;
  TextOut* out;
  char* text;
  unsigned long long text_capacity;
  unsigned long long* text_alloc;
  int4* peaks;
  unsigned long long peaks_capacity;
  unsigned long long* peaks_alloc;
  int32_t* nm;                      // nullptr: nmPerPosition is not materialised
  unsigned long long nm_capacity;   // ints
  unsigned long long* nm_alloc;
};

// ---- read parts gathered from the resident read set (pipeline.cu) ---------------------------
struct GatherParams {
  const uint8_t* reads;        // resident read arena
  const uint64_t* read_off;    // per read: byte offset in the arena
  int n;
  const int32_t* read_index;   // per problem
  const int32_t* part_start;   // extractReadSeq: read->Seq + onReadStart
  const int32_t* part_len;
  const uint8_t* revcomp;      // 1: computeReverseSeq of the part (cplBase, src/AlignmentBuffer.cpp:1117-1141)
  const uint64_t* out_off;     // byte offset of the part in `out`
  const int32_t* out_span;     // bytes to write: the part + zero padding
  uint8_t* out;
};

// ---- reference windows (DecodeRefSequenceExact) -------------------------------------------
struct RefDecodeParams {
  const uint8_t* enc;                    // binRef
  const unsigned long long* ref_starts;  // refStartPos: contig starts + one artificial end entry
  int n_starts;
  int n;
  const unsigned long long* win_start;   // startPosition
  const int32_t* win_len;                // sequenceLength (incl. the NUL)
  const uint64_t* out_off;               // byte offset of the window in `out`
  const int32_t* out_span;               // bytes to write: text, NUL, zero padding
  uint8_t* out;
};

// ---- k-mer index construction on the device (cs_index_build.cu) ------------------------------
struct IndexBuildParams {
  const uint8_t* enc;                      // binRef: 2 bases per byte, A0 T1 G2 C3 N4, spacer-padded
  unsigned long long concat_len;
  const unsigned long long* contig_start;  // device, sorted (SequenceProvider.GetRefStart)
  const unsigned long long* contig_len;    // device (GetRefLen)
  int n_contigs;
  int k, skip, bin_shift, max_freq;        // --kmer-length 13, --kmer-skip 2, --bin-size 4, maxPrefixFreq 1000
  unsigned long long unit_offset;          // TableUnit::Offset
};

struct IndexBuildScratch {
  uint32_t* lastn;      // [concat_len] last N at or before the base; reused as the callback slot index
  uint32_t* slot;       // (= lastn)
  uint8_t* flag;        // [concat_len] PrefixIteration calls back here
  unsigned long long cb_capacity;
  uint32_t *prefix, *pos, *key, *key_out, *pos_out;  // [cb_capacity]
  uint8_t* keep;        // [cb_capacity]
  uint32_t *freq, *alloc_cnt, *used_cnt, *alloc_start, *used_start;  // [4^k + 1]
  // outputs (the context's index arrays)
  uint32_t* tab;        // [4^k + 1] Index::m_TabIndex
  int8_t* rci;          // [4^k + 1] Index::m_RevCompIndex
  uint32_t* used_bits;
  uint32_t* out_pos;    // Location lists
  unsigned long long out_capacity;
  void* cub_tmp;
  size_t cub_bytes;
  // results
  unsigned long long n_callbacks;
  uint32_t n_positions, n_used;
};

// ---- candidate search -------------------------------------------------------------------
struct alignas(16) CsCandidate {
  unsigned long long loc;  // LocationScore::Location.m_Location = ResolveBin(bin)
  float score;             // LocationScore::Score.f
  uint32_t reverse;        // SequenceLocation::isReverse()
};

struct CsParams {
  // index (one table unit)
  const uint32_t* tab;     // Index::m_TabIndex, 4^k + 1 entries
  const uint32_t* used_bits;  // Index::used() as a bitmap, bit (prefix & 31) of word prefix >> 5
  const uint32_t* pos;     // Location::m_Location lists
  unsigned long long unit_offset;
  int k, bin_shift;
  float sensitivity, min_kmer_hits;
  // reads
  const uint8_t* seq;
  const uint64_t* seq_off;
  const int32_t* seq_len;
  int n;
  // pass 1
  unsigned long long* hits;
  // pass 2
  void* tables;
  const uint64_t* table_off;   // in entries
  const uint32_t* table_cap;   // power of two
  uint32_t* order;
  const uint64_t* order_off;
  CsCandidate* out;
  const uint64_t* out_off;
  int32_t* out_count;
  float* max_hits;
};

#ifdef __CUDACC__
// (offset, length) of row 32*blk + lane for the whole warp; rows >= H read as {0, 0}.
__device__ __forceinline__ void load_corridor_rows(const CorridorView& c, int blk, int lane, int H, int& off,
                                                   int& len) {
  const int y = (blk << 5) + lane;
  if (c.packed == 2) {  // closed form: the reference's own float32 expression, evaluated per row
    int o;
    if (c.ckind == 0) o = c.c0 + c.cstep * y;
    else o = (int)__fsub_rn(__fdiv_rn(__fsub_rn((float)y, c.cd), c.ck), c.cright);
    off = y < H ? o : 0;
    len = y < H ? c.const_len : 0;
    return;
  }
  if (!c.packed) {
    off = y < H ? c.off[y] : 0;
    len = y < H ? c.len[y] : 0;
    return;
  }
  int acc = (lane > 0 && y < H) ? (int)c.delta[y] : 0;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, acc, o);
    if (lane >= o) acc += v;
  }
  off = y < H ? c.blk_base[blk] + acc : 0;
  len = y < H ? c.const_len : 0;
}
#endif

}  // namespace nb
