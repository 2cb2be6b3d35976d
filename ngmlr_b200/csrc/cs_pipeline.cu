// ngmlr_b200/csrc/cs_pipeline.cu -- device-resident stage 0/2 pipeline:
//   count hits -> size tables (device prefix sums) -> vote -> compact candidates -> decode + score.
// Glue kernels only; the work is in cs_search.cu (vote) and sw_score.cu (scoring). The two host
// round trips that remain are the arena totals (24 bytes) needed to size device allocations.
#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "device_types.h"
#include "kernels.h"

namespace nb {

namespace {

// hits[n] doubles as the counter of small tables (zeroed by the host before the launch)
__global__ void cs_sizes_kernel(unsigned long long* __restrict__ hits, int n, uint32_t* __restrict__ cap,
                                unsigned long long* __restrict__ a, unsigned long long* __restrict__ b,
                                unsigned long long* __restrict__ c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) {  // sentinel so that the exclusive scan's last element is the total
    a[i] = 0; b[i] = 0; c[i] = 0;
    return;
  }
  const unsigned long long h = hits[i];
  unsigned long long cp = 16;  // 64-bit: a table of 2^31 entries and more is refused by the host (totals check)
  while (cp < 2 * h + 2) cp <<= 1;
  cap[i] = cp > 0x80000000ull ? 0x80000000u : (uint32_t)cp;
  a[i] = cap[i] > CS_SMEM_CAP ? cp : 0ull;  // vote table entries in the arena (small tables live in shared memory)
  // one atomic per warp, not per sub-read (the guard above only removes threads at the very end of the grid)
  const unsigned small = __ballot_sync(__activemask(), cap[i] <= CS_SMEM_CAP);
  if (small && (threadIdx.x & 31) == (__ffs(__activemask()) - 1)) atomicAdd(hits + n, (unsigned long long)__popc(small));
  b[i] = h;       // order list entries
  c[i] = 2 * h;   // candidate slots (forward + reverse per listed bin)
}

__global__ void cs_count_to_u64_kernel(const int32_t* __restrict__ cnt, int n, unsigned long long* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  out[i] = i < n ? (unsigned long long)cnt[i] : 0ull;
}

// One warp per read: its candidates -> compact arrays, plus everything the scorer needs per pair.
__global__ void cs_compact_kernel(const CsCandidate* __restrict__ out, const uint64_t* __restrict__ out_off,
                                  const int32_t* __restrict__ out_count, const unsigned long long* __restrict__ cstart,
                                  const uint64_t* __restrict__ seq_off, const int32_t* __restrict__ seq_len, int n,
                                  int half_corridor, unsigned long long* __restrict__ loc, float* __restrict__ score,
                                  uint8_t* __restrict__ rev, unsigned long long* __restrict__ win_pos,
                                  uint64_t* __restrict__ qoff, int32_t* __restrict__ qlen) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const CsCandidate* src = out + out_off[i];
  const unsigned long long base = cstart[i];
  const int m = out_count[i];
  for (int j = lane; j < m; j += 32) {
    const CsCandidate c = src[j];
    loc[base + j] = c.loc;
    score[base + j] = c.score;
    rev[base + j] = (uint8_t)c.reverse;
    win_pos[base + j] = c.loc - (unsigned long long)half_corridor;  // uloc arithmetic, src/ScoreBuffer.cpp:110
    qoff[base + j] = seq_off[i];
    qlen[base + j] = seq_len[i] + 1;  // strlen + 1
  }
}

// One thread per short-read candidate pair: ScoreBuffer::scoreShortRead's window (src/ScoreBuffer.cpp:245-265),
// corridor = (int)(len * 0.3 + 256) in double arithmetic (no FMA contraction), window
// DecodeRefSequence(buf, 0, loc - (corridor >> 1), len + corridor), and the whole read as the query.
__global__ void cs_short_geometry_kernel(const int32_t* __restrict__ read_idx, const unsigned long long* __restrict__ loc,
                                         const uint64_t* __restrict__ read_off, const int32_t* __restrict__ read_len,
                                         int n, unsigned long long* __restrict__ win_pos, int32_t* __restrict__ win_len,
                                         uint64_t* __restrict__ qoff, int32_t* __restrict__ qlen) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = read_idx[i];
  const int len = read_len[r];
  const int corridor = (int)__dadd_rn(__dmul_rn((double)len, 0.3), 256.0);
  win_pos[i] = loc[i] - (unsigned long long)(corridor >> 1);  // uloc arithmetic
  win_len[i] = len + corridor;
  qoff[i] = read_off[r];
  qlen[i] = len + 1;  // strlen + 1
}

}  // namespace

cudaError_t cs_exclusive_scan(void* temp, size_t& temp_bytes, const unsigned long long* in,
                              unsigned long long* out, int n, cudaStream_t stream) {
  return cub::DeviceScan::ExclusiveSum(temp, temp_bytes, in, out, n, stream);
}

cudaError_t launch_cs_sizes(unsigned long long* hits, int n, uint32_t* cap, unsigned long long* a,
                            unsigned long long* b, unsigned long long* c, cudaStream_t stream) {
  cs_sizes_kernel<<<(n + 1 + 255) / 256, 256, 0, stream>>>(hits, n, cap, a, b, c);
  return cudaGetLastError();
}

cudaError_t launch_cs_count_to_u64(const int32_t* cnt, int n, unsigned long long* out, cudaStream_t stream) {
  cs_count_to_u64_kernel<<<(n + 1 + 255) / 256, 256, 0, stream>>>(cnt, n, out);
  return cudaGetLastError();
}

cudaError_t launch_cs_compact(const CsCandidate* out, const uint64_t* out_off, const int32_t* out_count,
                              const unsigned long long* cstart, const uint64_t* seq_off, const int32_t* seq_len,
                              int n, int half_corridor, unsigned long long* loc, float* score, uint8_t* rev,
                              unsigned long long* win_pos, uint64_t* qoff, int32_t* qlen, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const int warps_per_cta = 8;
  cs_compact_kernel<<<(n + warps_per_cta - 1) / warps_per_cta, warps_per_cta * 32, 0, stream>>>(
      out, out_off, out_count, cstart, seq_off, seq_len, n, half_corridor, loc, score, rev, win_pos, qoff, qlen);
  return cudaGetLastError();
}

cudaError_t launch_cs_short_geometry(const int32_t* read_idx, const unsigned long long* loc, const uint64_t* read_off,
                                     const int32_t* read_len, int n, unsigned long long* win_pos, int32_t* win_len,
                                     uint64_t* qoff, int32_t* qlen, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  cs_short_geometry_kernel<<<(n + 255) / 256, 256, 0, stream>>>(read_idx, loc, read_off, read_len, n, win_pos, win_len,
                                                                qoff, qlen);
  return cudaGetLastError();
}

}  // namespace nb
