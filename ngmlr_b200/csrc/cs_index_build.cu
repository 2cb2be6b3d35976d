// ngmlr_b200/csrc/cs_index_build.cu -- construction of the k-mer index on the device (sm_90a).
//
// Replaces CompactPrefixTable::CreateTable for one table unit (src/PrefixTable.cpp:323-370):
//   CountKmerFreq / CountKmer        (:199-231, :372-394)  k-mer frequencies of the reference
//   createRefTableIndex              (:269-321)            Index{m_TabIndex, m_RevCompIndex} per k-mer
//   Generate / BuildPrefixTable      (:233-267, :404-437)  Location lists
// driven by CS::PrefixIteration (src/CSstatic.cpp:23-73) over every contig with prefixskip = kmerSkip.
// The result is the reference's in-memory index bit for bit (tests/test_gpu_index.py against the numpy /
// oracle builders, which are pinned to the unmodified reference), so the byte-compatible cache writer
// (ngmlr_b200/ngmfiles.py) and the candidate search consume it unchanged.
//
// What the reference does sequentially, restated as data-parallel passes over the 4-bit encoded,
// spacer-padded genome that is already resident in HBM (one thread per base):
//   1. callbacks: PrefixIteration calls back at every (skip+1)-th position of every N-free run of at
//      least k characters, counted from the start of the run. The start of the run = 1 + the position of
//      the last N at or before the base -> one inclusive max-scan (cub). Contig boundaries need no extra
//      care (the spacers are N), except that Generate() decodes each contig with a buffer length that
//      turns its last two characters into k-mer code 0 ('A'), and that a run of exactly k characters at
//      the very end of a contig is dropped when PrefixIteration reaches it through its N-skipping branch
//      (n_skip >= length - k, :38-41).
//   2. the repeat filter of CountKmer / BuildPrefixTable (same k-mer as the previous callback AND same
//      16-bp bin as the previous callback -> skipped, except that the first repetition always counts)
//      only looks two callbacks back: a 3-element window on the compacted callback sequence.
//   3. frequencies: one atomicAdd per kept callback into 4^k counters (L2-resident for k = 13).
//   4. Index records: per k-mer total = freq + freq[revComp]; slots are allocated where freq > 0 and
//      total < maxPrefixFreq (exclusive scan of the allocated frequencies), m_RevCompIndex is the float
//      expression of :300 truncated to a char, used() <=> m_RevCompIndex != 0.
//   5. Location lists: the kept callbacks of used k-mers in callback order within each k-mer = a stable
//      radix sort by k-mer code (cub), then one scatter (slot = m_TabIndex - 1 + rank within the k-mer).
// HBM-bound streaming passes and one sort of (k-mer, position) pairs.
#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include <algorithm>

#include "device_types.h"
#include "kernels.h"

namespace nb {

namespace {

__device__ __forceinline__ uint32_t code4_at(const uint8_t* __restrict__ enc, unsigned long long g) {
  const uint32_t byte = enc[g >> 1];
  return (g & 1ull) ? (byte & 0xFu) : (byte >> 4);
}

// contig of concatenated position g (contigs sorted by start): index, or -1 outside every contig
__device__ __forceinline__ int contig_of(const IndexBuildParams& p, unsigned long long g) {
  int lo = 0, hi = p.n_contigs;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (p.contig_start[mid] <= g) lo = mid + 1; else hi = mid;
  }
  const int c = lo - 1;
  if (c < 0 || g >= p.contig_start[c] + p.contig_len[c]) return -1;
  return c;
}

// The character PrefixIteration sees at g: k-mer code (A0 C1 T2 G3), or 4 for N. enc4 is A0 T1 G2 C3 N4.
__device__ __forceinline__ uint32_t kcode_at(const IndexBuildParams& p, unsigned long long g) {
  const uint32_t c4 = code4_at(p.enc, g);
  return c4 > 3u ? 4u : ((0x1320u >> (4u * c4)) & 0xFu);  // A0->0, T1->2, G2->3, C3->1
}

// pass 1a: isN flags as "position if N else 0" for the max-scan (position 0 is spacer, i.e. N)
__global__ void index_nmark_kernel(const IndexBuildParams p, uint32_t* __restrict__ mark) {
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; g < p.concat_len; g += stride) {
    bool is_n = code4_at(p.enc, g) > 3u;
    if (is_n) {
      // the last two characters of a contig are code 0 for Generate(), whatever they are
      const int c = contig_of(p, g);
      if (c >= 0 && g + 2 >= p.contig_start[c] + p.contig_len[c] && p.contig_len[c] >= 2) is_n = false;
    }
    mark[g] = is_n ? (uint32_t)g : 0u;
  }
}

// pass 1b: callback flags. lastn[g] = position of the last N at or before g.
__global__ void index_flag_kernel(const IndexBuildParams p, const uint32_t* __restrict__ lastn,
                                  uint8_t* __restrict__ flag) {
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  const int k = p.k;
  for (unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; g < p.concat_len; g += stride) {
    uint8_t f = 0;
    const unsigned long long ln = lastn[g];
    if (ln != g && g + (unsigned long long)k <= p.concat_len) {
      const unsigned long long a = ln + 1;  // start of the N-free run
      if ((g - a) % (unsigned long long)(p.skip + 1) == 0 && lastn[g + k - 1] == ln) {  // no N in [g, g + k)
        const int c = contig_of(p, g);
        if (c >= 0) {
          const unsigned long long cs = p.contig_start[c], ce = cs + p.contig_len[c];
          if (g + (unsigned long long)k <= ce) {
            f = 1;
            // a run of exactly k characters that ends with the contig, reached through the N-skipping branch
            // (the N-run in front of it starts the contig or is at least two long): dropped (:38-41)
            if (a == g && ce - a == (unsigned long long)k && a > cs) {
              const bool n1 = lastn[a - 1] == a - 1;
              const bool n2 = (a - 1 == cs) || (lastn[a - 2] == a - 2);
              if (n1 && n2) f = 0;
            }
          }
        }
      }
    }
    flag[g] = f;
  }
}

// pass 1c: compact callbacks: k-mer code + position
__global__ void index_emit_kernel(const IndexBuildParams p, const uint8_t* __restrict__ flag,
                                  const uint32_t* __restrict__ slot, uint32_t* __restrict__ prefix,
                                  uint32_t* __restrict__ pos) {
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  const int k = p.k;
  for (unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; g < p.concat_len; g += stride) {
    if (!flag[g]) continue;
    const int c = contig_of(p, g);
    const unsigned long long ce = p.contig_start[c] + p.contig_len[c];
    uint32_t pre = 0;
    for (int j = 0; j < k; ++j) {
      const unsigned long long q = g + (unsigned long long)j;
      const uint32_t kc = (q + 2 >= ce) ? 0u : kcode_at(p, q);  // the contig's last two characters read as 'A'
      pre = (pre << 2) | (kc & 3u);
    }
    const uint32_t at = slot[g];
    prefix[at] = pre;
    pos[at] = (uint32_t)g;
  }
}

// pass 2 + 3: repeat filter on the callback sequence, frequencies of the kept callbacks
__global__ void index_keep_kernel(const IndexBuildParams p, const uint32_t* __restrict__ prefix,
                                  const uint32_t* __restrict__ pos, unsigned long long n,
                                  uint8_t* __restrict__ keep, uint32_t* __restrict__ freq) {
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t pi = prefix[i];
    const uint32_t xi = pos[i];
    const int ci = contig_of(p, xi);
    // the callback before this one within the same contig; a contig starts with lastPrefix = 111111, lastBin = -1
    const bool has1 = i >= 1 && contig_of(p, pos[i - 1]) == ci;
    const bool has2 = has1 && i >= 2 && contig_of(p, pos[i - 2]) == ci;
    const uint32_t p1 = has1 ? prefix[i - 1] : 111111u;
    const bool same_i = pi == p1;
    bool same_prev = false;  // was the previous callback itself a repetition of the one before it?
    if (has1) same_prev = prefix[i - 1] == (has2 ? prefix[i - 2] : 111111u);
    bool kp = true;
    if (same_i && same_prev) {  // third or later in a row: counts only in a new bin
      kp = (xi >> p.bin_shift) != (pos[i - 1] >> p.bin_shift);
    }
    keep[i] = kp ? 1 : 0;
    if (kp) atomicAdd(freq + pi, 1u);
  }
}

__device__ __forceinline__ uint32_t rev_comp(uint32_t prefix, int k) {
  // revComp, src/PrefixTable.cpp:70-88 (k-mer code A0 C1 T2 G3: complement = xor 10b)
  const uint32_t mask = (k == 16) ? 0xffffffffu : ((1u << (2 * k)) - 1u);
  uint32_t c = (prefix ^ 0xAAAAAAAAu) & mask;
  c = __brev(c);
  c = ((c >> 1) & 0x55555555u) | ((c & 0x55555555u) << 1);
  return c >> (32 - 2 * k);
}

// pass 4: Index records. alloc_cnt / used_cnt feed the two exclusive scans.
__global__ void index_records_kernel(const uint32_t* __restrict__ freq, uint32_t n_kmers, int k, int max_freq,
                                     int8_t* __restrict__ rci, uint32_t* __restrict__ alloc_cnt,
                                     uint32_t* __restrict__ used_cnt) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_kmers) return;
  if (i == n_kmers) {  // sentinel record
    rci[i] = 0;
    alloc_cnt[i] = 0;
    used_cnt[i] = 0;
    return;
  }
  const int f = (int)freq[i];
  const int total = f + (int)freq[rev_comp(i, k)];
  int8_t r = 0;
  uint32_t a = 0;
  if (f > 0 && total < max_freq) {
    a = (uint32_t)f;
    // (maxPrefixFreq - total_freq) * 100.0f / maxPrefixFreq, assigned to a char (:300)
    const float v = __fdiv_rn(__fmul_rn((float)(max_freq - total), 100.0f), (float)max_freq);
    r = (int8_t)(int)v;
  }
  rci[i] = r;
  alloc_cnt[i] = a;
  used_cnt[i] = r != 0 ? a : 0u;
}

__global__ void index_tab_kernel(const uint32_t* __restrict__ alloc_start, uint32_t n1, uint32_t* __restrict__ tab) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n1) tab[i] = alloc_start[i] + 1u;  // m_TabIndex = next + 1
}

// pass 5a: sort keys: the k-mer of kept callbacks of used k-mers, everything else to the end
__global__ void index_sortkey_kernel(const uint32_t* __restrict__ prefix, const uint8_t* __restrict__ keep,
                                     const int8_t* __restrict__ rci, unsigned long long n, uint32_t* __restrict__ key) {
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t pi = prefix[i];
    key[i] = (keep[i] && rci[pi] != 0) ? pi : 0xffffffffu;
  }
}

// pass 5b: sorted (k-mer, position) -> Location lists
__global__ void index_scatter_kernel(const uint32_t* __restrict__ key, const uint32_t* __restrict__ val,
                                     unsigned long long n_used, const uint32_t* __restrict__ tab,
                                     const uint32_t* __restrict__ used_start, unsigned long long unit_offset,
                                     uint32_t* __restrict__ out) {
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long j = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; j < n_used; j += stride) {
    const uint32_t pi = key[j];
    const uint32_t rank = (uint32_t)(j - (unsigned long long)used_start[pi]);
    out[tab[pi] - 1u + rank] = (uint32_t)((unsigned long long)val[j] - unit_offset);
  }
}

__global__ void index_usedbits_kernel(const int8_t* __restrict__ rci, uint32_t n, uint32_t* __restrict__ used_bits) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;  // blockDim is a multiple of 32
  const bool used = i < n && rci[i] != 0;
  const uint32_t word = __ballot_sync(0xffffffffu, used);
  if ((threadIdx.x & 31) == 0) used_bits[i >> 5] = word;
}

struct MaxOp {
  __device__ __forceinline__ uint32_t operator()(uint32_t a, uint32_t b) const { return a > b ? a : b; }
};

}  // namespace

// Scratch sizes are those of a 3 Gb genome at most: concat_len * (4 + 1 + 4) bytes for the scans plus
// 5 x 4 bytes per callback (~ concat_len / (skip + 1)) -- about 45 GB of the 180 GB for a human genome.
cudaError_t build_kmer_index(const IndexBuildParams& p, IndexBuildScratch& s, cudaStream_t st) {
#define IB(call)                      \
  do {                                \
    cudaError_t e__ = (call);         \
    if (e__ != cudaSuccess) return e__; \
  } while (0)
  const int threads = 256;
  const int grid = current_device_sms() * 16;
  const uint32_t n_kmers = 1u << (2 * p.k);
  const long long cl = (long long)p.concat_len;  // 64-bit item counts: a human genome has > 2^31 bases
  // ---- 1. callbacks ----
  index_nmark_kernel<<<grid, threads, 0, st>>>(p, s.lastn);
  size_t tmp = s.cub_bytes;
  IB(cub::DeviceScan::InclusiveScan(s.cub_tmp, tmp, s.lastn, s.lastn, MaxOp(), cl, st));
  index_flag_kernel<<<grid, threads, 0, st>>>(p, s.lastn, s.flag);
  tmp = s.cub_bytes;
  IB(cub::DeviceScan::ExclusiveSum(s.cub_tmp, tmp, s.flag, s.slot, cl, st));
  // number of callbacks = slot[last] + flag[last]
  uint32_t last_slot = 0;
  uint8_t last_flag = 0;
  IB(cudaMemcpyAsync(&last_slot, s.slot + (p.concat_len - 1), 4, cudaMemcpyDeviceToHost, st));
  IB(cudaMemcpyAsync(&last_flag, s.flag + (p.concat_len - 1), 1, cudaMemcpyDeviceToHost, st));
  IB(cudaStreamSynchronize(st));
  const unsigned long long n_cb = (unsigned long long)last_slot + last_flag;
  s.n_callbacks = n_cb;
  if (n_cb > s.cb_capacity) return cudaErrorMemoryAllocation;
  index_emit_kernel<<<grid, threads, 0, st>>>(p, s.flag, s.slot, s.prefix, s.pos);
  // ---- 2 + 3. repeat filter, frequencies ----
  IB(cudaMemsetAsync(s.freq, 0, (size_t)(n_kmers + 1) * 4, st));
  if (n_cb) index_keep_kernel<<<grid, threads, 0, st>>>(p, s.prefix, s.pos, n_cb, s.keep, s.freq);
  // ---- 4. Index records ----
  index_records_kernel<<<(n_kmers + 1 + threads - 1) / threads, threads, 0, st>>>(s.freq, n_kmers, p.k, p.max_freq, s.rci,
                                                                                 s.alloc_cnt, s.used_cnt);
  tmp = s.cub_bytes;
  IB(cub::DeviceScan::ExclusiveSum(s.cub_tmp, tmp, s.alloc_cnt, s.alloc_start, (int)(n_kmers + 1), st));
  tmp = s.cub_bytes;
  IB(cub::DeviceScan::ExclusiveSum(s.cub_tmp, tmp, s.used_cnt, s.used_start, (int)(n_kmers + 1), st));
  index_tab_kernel<<<(n_kmers + 1 + threads - 1) / threads, threads, 0, st>>>(s.alloc_start, n_kmers + 1, s.tab);
  uint32_t n_alloc = 0, n_used = 0;
  IB(cudaMemcpyAsync(&n_alloc, s.alloc_start + n_kmers, 4, cudaMemcpyDeviceToHost, st));
  IB(cudaMemcpyAsync(&n_used, s.used_start + n_kmers, 4, cudaMemcpyDeviceToHost, st));
  IB(cudaStreamSynchronize(st));
  s.n_positions = n_alloc;
  s.n_used = n_used;
  if ((unsigned long long)n_alloc + 1 > s.out_capacity) return cudaErrorMemoryAllocation;
  // ---- 5. Location lists ----
  IB(cudaMemsetAsync(s.out_pos, 0, ((size_t)n_alloc + 1) * 4, st));
  if (n_cb) {
    index_sortkey_kernel<<<grid, threads, 0, st>>>(s.prefix, s.keep, s.rci, n_cb, s.key);
    tmp = s.cub_bytes;
    IB(cub::DeviceRadixSort::SortPairs(s.cub_tmp, tmp, s.key, s.key_out, s.pos, s.pos_out, (int)n_cb, 0, 32, st));
    if (n_used)
      index_scatter_kernel<<<grid, threads, 0, st>>>(s.key_out, s.pos_out, n_used, s.tab, s.used_start, p.unit_offset,
                                                     s.out_pos);
  }
  index_usedbits_kernel<<<(n_kmers + 1 + 255) / 256, 256, 0, st>>>(s.rci, n_kmers + 1, s.used_bits);
  return cudaGetLastError();
#undef IB
}

size_t index_build_cub_bytes(unsigned long long concat_len, unsigned long long max_callbacks, int k) {
  size_t a = 0, b = 0, c = 0, d = 0;
  cub::DeviceScan::InclusiveScan(nullptr, a, (uint32_t*)nullptr, (uint32_t*)nullptr, MaxOp(), (long long)concat_len);
  cub::DeviceScan::ExclusiveSum(nullptr, b, (uint8_t*)nullptr, (uint32_t*)nullptr, (long long)concat_len);
  cub::DeviceScan::ExclusiveSum(nullptr, c, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)((1u << (2 * k)) + 1));
  cub::DeviceRadixSort::SortPairs(nullptr, d, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int)max_callbacks, 0, 32);
  return std::max(std::max(a, b), std::max(c, d)) + 256;
}

}  // namespace nb
