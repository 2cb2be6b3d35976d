// ngmlr_b200/csrc/kernels.h -- launchers of the sm_90a kernels (host-callable).
#pragma once
#include <cuda_runtime.h>

#include "device_types.h"

namespace nb {

#ifndef FILL_WARPS_OVERRIDE
#define FILL_WARPS_OVERRIDE 4
#endif
#ifndef FILL_CTAS_OVERRIDE
#define FILL_CTAS_OVERRIDE 5
#endif
constexpr int FILL_WARPS_PER_CTA = FILL_WARPS_OVERRIDE;  // warps per CTA = team size of the ordinary team kernel
constexpr int FILL_CTAS_PER_SM = FILL_CTAS_OVERRIDE;
#ifndef FILL_TEAM_CTAS_PER_SM
#define FILL_TEAM_CTAS_PER_SM (FILL_CTAS_OVERRIDE + (FILL_WARPS_OVERRIDE == 4 ? 1 : 0))  // 4-warp teams: 80 registers, 6 CTAs = 24 warps per SM
#endif
constexpr int FILL_SM_SLOTS = 8;   // boundary strips per SM for launches of short-lived CTAs (>= resident CTAs per SM)
constexpr int FILL_BIG_TEAM = 16;  // warps that pipeline one huge matrix (one CTA per SM)

constexpr int RF_MIN_WIDTH = 128;  // one-warp launches take the ramp-free schedule when most corridors are this wide
constexpr int RF_MIN_BLOCK_STEPS = 224;  // steps per 32-row block the ramp-free schedule may spend on a narrow corridor
// with the ramp-free schedule, problems of at least this many cells are filled by FILL_WARPS_PER_CTA-warp teams in a
// launch of their own: one warp would still be busy with them long after the rest of the batch is done
constexpr unsigned long long RF_TEAM_CELLS = 8ull << 20;

// team = all FILL_WARPS_PER_CTA warps of a CTA pipeline one problem; otherwise one warp per problem.
// rampfree: one warp per problem in the ramp-free row schedule (convex_fill.cu; `team` is ignored).
cudaError_t launch_convex_fill(const FillParams& p, bool raw, bool team, bool rampfree, int grid, cudaStream_t stream);
// the same kernel with a FILL_BIG_TEAM-warp team per problem, for the huge matrices of a batch
cudaError_t launch_convex_fill_big(const FillParams& p, bool raw, int grid, cudaStream_t stream);
int fill_max_ctas_per_sm(bool raw, bool team, bool rampfree);
// %nsmid of the current device: every %smid is below it (SM ids need not be dense in 0 .. SM count - 1); -1 on error
int fill_sm_id_bound();

// SMs of the current device (grid caps of the grid-stride kernels)
inline int current_device_sms() {
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 1;
}

cudaError_t launch_convex_traceback(const TraceParams& p, cudaStream_t stream);

// StrippedSW score-only kernel: one warp per (ref, qry) pair.
struct SwParams {
  const uint8_t* seq;          // arena holding all strings, NUL included
  const uint64_t* ref_off;
  const uint64_t* qry_off;
  const int32_t* ref_len;      // strlen + 1 (the NUL is scored, StrippedSW.cpp:130-146)
  const int32_t* qry_len;
  float* out;
  int n;
  int32_t* scratch;            // per-warp H/E rows for queries longer than the register tile
  unsigned long long scratch_stride;
  // gather mode (candidate scoring straight from the 4-bit genome, ScoreBuffer::DoRun semantics):
  // pair i scores sub-read qry (reverse-complemented with MappedRead::computeReverseSeq's cpl()
  // when rev[i]) against DecodeRefSequence(buf, 0, win_pos[i], win_len)
  const uint8_t* enc;          // binRef, 2 bases per byte (A0 T1 G2 C3 N4)
  unsigned long long concat_len;
  const unsigned long long* win_pos;
  const uint8_t* rev;
  int win_len;                 // refMaxLen (308)
  // short-read scoring (ScoreBuffer::scoreShortRead): the window length of pair i is win_lens[i]
  const int32_t* win_lens;
  unsigned int* general_pairs; // optional: counts pairs of the short-read launch that miss the ungapped path
};
cudaError_t launch_sw_score(const SwParams& p, int grid, cudaStream_t stream);
cudaError_t launch_sw_score_gather(const SwParams& p, int grid, cudaStream_t stream);
// gather mode with per-pair windows of up to 640 columns (short reads: len + (int)(len * 0.3 + 256) <= 588)
cudaError_t launch_sw_score_gather_short(const SwParams& p, int grid, cudaStream_t stream);

cudaError_t launch_decode_windows(const RefDecodeParams& p, cudaStream_t stream);
// one contig's characters (device) -> 4-bit codes, two per byte (_SequenceProvider::Init's encoding)
cudaError_t launch_encode_contig(const uint8_t* text, unsigned long long len, uint8_t* out, cudaStream_t stream);

// binary CIGAR -> CIGAR/MD text, NM, identity, positions, low-identity regions (convex_text.cu)
cudaError_t launch_convex_text(const TextParams& p, cudaStream_t stream);

// read parts (optionally reverse-complemented) from the resident read set into the sequence arena
cudaError_t launch_gather_reads(const GatherParams& p, cudaStream_t stream);

constexpr uint32_t CS_SMEM_CAP = 512;  // vote tables up to this many entries live in shared memory (no arena space)
// small_tables: some vote table of the batch has at most CS_SMEM_CAP entries (shared-memory tables compiled in)
cudaError_t launch_cs_search(const CsParams& p, bool count_only, bool small_tables, cudaStream_t stream);
cudaError_t launch_unpack_index(const uint8_t* packed, uint32_t n, uint32_t* tab, uint32_t* used_bits,
                                cudaStream_t stream);

// k-mer index of the resident encoded reference, built on the device (cs_index_build.cu)
cudaError_t build_kmer_index(const IndexBuildParams& p, IndexBuildScratch& s, cudaStream_t stream);
size_t index_build_cub_bytes(unsigned long long concat_len, unsigned long long max_callbacks, int k);
// Positions of the genome (< 0xffff0000: one table unit, 32-bit scans) and k-mer callbacks (the radix sort's int item
// count) that build_kmer_index can handle; it refuses anything larger with cudaErrorInvalidValue.
constexpr unsigned long long INDEX_MAX_CONCAT_LEN = 0xffff0000ull - 1;
inline unsigned long long index_callback_capacity(unsigned long long concat_len, int n_contigs, int kmer_skip) {
  return concat_len / (unsigned long long)(kmer_skip + 1) + (unsigned long long)n_contigs * 64 + 1024;
}
inline bool index_build_fits(unsigned long long concat_len, int n_contigs, int kmer_skip) {
  return concat_len <= INDEX_MAX_CONCAT_LEN && index_callback_capacity(concat_len, n_contigs, kmer_skip) <= 0x7fffffffull;
}

// device-resident candidate pipeline glue (cs_pipeline.cu)
cudaError_t cs_exclusive_scan(void* temp, size_t& temp_bytes, const unsigned long long* in,
                              unsigned long long* out, int n, cudaStream_t stream);
cudaError_t launch_cs_sizes(unsigned long long* hits, int n, uint32_t* cap, unsigned long long* a,
                            unsigned long long* b, unsigned long long* c, cudaStream_t stream);
cudaError_t launch_cs_count_to_u64(const int32_t* cnt, int n, unsigned long long* out, cudaStream_t stream);
cudaError_t launch_cs_compact(const CsCandidate* out, const uint64_t* out_off, const int32_t* out_count,
                              const unsigned long long* cstart, const uint64_t* seq_off, const int32_t* seq_len,
                              int n, int half_corridor, unsigned long long* loc, float* score, uint8_t* rev,
                              unsigned long long* win_pos, uint64_t* qoff, int32_t* qlen, cudaStream_t stream);
// short-read candidate pairs (read index, location) -> the window and query of ScoreBuffer::scoreShortRead
cudaError_t launch_cs_short_geometry(const int32_t* read_idx, const unsigned long long* loc, const uint64_t* read_off,
                                     const int32_t* read_len, int n, unsigned long long* win_pos, int32_t* win_len,
                                     uint64_t* qoff, int32_t* qlen, cudaStream_t stream);

}  // namespace nb
