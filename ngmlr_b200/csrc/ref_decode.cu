// ngmlr_b200/csrc/ref_decode.cu -- reference windows for alignment, decoded on the device (sm_90a).
//
// Replaces _SequenceProvider::DecodeRefSequenceExact(sequence, startPosition, sequenceLength, 0)
// (src/SequenceProvider.cpp:493-565 with decode :475-490 and getChrStart :157-178) as called by
// AlignmentBuffer::extractReferenceSequenceForAlignment (src/AlignmentBuffer.cpp:203-223): the
// window [onRefStart, onRefStop] of the 4-bit encoded concatenated genome as characters, 'x' where
// the window runs past the end of its contig or starts inside the spacer in front of it. decode()
// writes whole byte pairs, so up to two characters beyond the contig end come out as the spacer's
// 'N' before the 'x' padding starts -- kept.
//
// One CTA per window, one thread per character: pure HBM streaming (0.5 B read, 1 B written per
// base).
#include <cuda_runtime.h>

#include <algorithm>

#include "device_types.h"
#include "kernels.h"

namespace nb {

namespace {

__global__ void __launch_bounds__(256) decode_windows_kernel(const RefDecodeParams p) {
  const int w = blockIdx.x;
  const unsigned long long start = p.win_start[w];
  const int len = p.win_len[w];  // sequenceLength: characters incl. the terminating NUL
  uint8_t* __restrict__ out = p.out + p.out_off[w];
  const int padded = p.out_span[w];
  // getChrStart: first refStartPos entry > position; one further if the position lies in the
  // 1000-N spacer in front of that contig
  int u = 0;
  {
    int lo = 0, hi = p.n_starts;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (p.ref_starts[mid] > start) hi = mid; else lo = mid + 1;
    }
    u = max(1, min(lo, p.n_starts - 1));
    if (p.ref_starts[u] - start < 1000ull) u = min(u + 1, p.n_starts - 1);
  }
  const unsigned long long chr_start = p.ref_starts[u - 1], chr_end = p.ref_starts[u] - 1000ull;
  const unsigned long long end = start + (unsigned long long)len;
  const unsigned long long dend = end > chr_end ? chr_end : end;
  // characters [skip, skip + nwritten) are decoded from position dstart on, the rest stays 'x'
  unsigned long long dstart = start, skip = 0, nwritten = 0;
  bool any = true;
  if (start < chr_start) {
    skip = chr_start - start;
    dstart = chr_start;
    any = dend > chr_start;
  }
  if (any) nwritten = (dstart & 1ull) + 2ull * ((dend - dstart + 1ull) / 2ull);
  for (int i = threadIdx.x; i < padded; i += blockDim.x) {
    uint8_t c = 0;
    if (i < len - 1) {
      c = 'x';
      const unsigned long long k = (unsigned long long)i - skip;
      if ((unsigned long long)i >= skip && k < nwritten) {
        const unsigned long long b = dstart + k;
        const uint32_t byte = p.enc[b >> 1];
        const uint32_t c4 = (b & 1ull) ? (byte & 0xFu) : (byte >> 4);
        c = (uint8_t)((0x4E43475441ull >> (8u * min(c4, 4u))) & 0xffu);  // "ATGCN"
      }
    }
    out[i] = c;
  }
}

// Read parts for alignment, taken from the read set that is already resident in HBM (uploaded once for
// stage 0/2): AlignmentBuffer::extractReadSeq (src/AlignmentBuffer.cpp:1514-1545) -- the part
// read->Seq[onReadStart, +len) as it is, or its reverse complement (computeReverseSeq / cplBase,
// :1117-1141: only upper-case A C G T are complemented). One CTA per part.
__global__ void __launch_bounds__(256) gather_reads_kernel(const GatherParams p) {
  const int w = blockIdx.x;
  const uint8_t* __restrict__ src = p.reads + p.read_off[p.read_index[w]] + p.part_start[w];
  const int len = p.part_len[w], span = p.out_span[w];
  const bool rc = p.revcomp[w] != 0;
  uint8_t* __restrict__ out = p.out + p.out_off[w];
  for (int i = threadIdx.x; i < span; i += blockDim.x) {
    uint8_t c = 0;
    if (i < len) {
      if (rc) {
        const uint8_t b = src[len - 1 - i];
        c = b == 'A' ? 'T' : (b == 'T' ? 'A' : (b == 'C' ? 'G' : (b == 'G' ? 'C' : b)));
      } else {
        c = src[i];
      }
    }
    out[i] = c;
  }
}


// _SequenceProvider::Init's encoding of one contig (src/SequenceProvider.cpp:76-105, 342-400): two characters per
// byte, high nibble first, A0 T1 G2 C3 (either case), everything else 4 (N); an odd contig ends with an N nibble.
// One thread per 16 output bytes (32 characters, two 16-byte loads where aligned): pure HBM streaming, 1 B read and
// 0.5 B written per base.
__device__ __forceinline__ uint32_t enc4(uint32_t c) {
  c &= 0xdfu;  // upper case
  return c == 'A' ? 0u : (c == 'T' ? 1u : (c == 'G' ? 2u : (c == 'C' ? 3u : 4u)));
}

__global__ void __launch_bounds__(256) encode_contig_kernel(const uint8_t* __restrict__ text, unsigned long long len,
                                                            uint8_t* __restrict__ out) {
  const unsigned long long n_bytes = (len + 1ull) >> 1;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long j = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; j < n_bytes; j += stride) {
    const uint32_t hi = enc4(text[2 * j]);
    const uint32_t lo = (2 * j + 1 < len) ? enc4(text[2 * j + 1]) : 4u;
    out[j] = (uint8_t)((hi << 4) | lo);
  }
}

}  // namespace

cudaError_t launch_gather_reads(const GatherParams& p, cudaStream_t stream) {
  if (p.n <= 0) return cudaSuccess;
  gather_reads_kernel<<<p.n, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_encode_contig(const uint8_t* text, unsigned long long len, uint8_t* out, cudaStream_t stream) {
  if (!len) return cudaSuccess;
  const unsigned long long n_bytes = (len + 1ull) >> 1;
  const int grid = (int)std::min<unsigned long long>((n_bytes + 255ull) / 256ull, (unsigned long long)current_device_sms() * 32ull);
  encode_contig_kernel<<<grid, 256, 0, stream>>>(text, len, out);
  return cudaGetLastError();
}

cudaError_t launch_decode_windows(const RefDecodeParams& p, cudaStream_t stream) {
  if (p.n <= 0) return cudaSuccess;
  decode_windows_kernel<<<p.n, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace nb
