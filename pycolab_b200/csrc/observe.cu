// observe.cu — observation post-processors as a per-cell table look-up.
//
// ObservationCharacterRepainter (rendering.py:304-406), ObservationToArray
// (:409-542) and ObservationToFeatureArray (:545-661) all compute
//     out[d, r, c] = f_d(board[r, c])
// for a function that depends only on the character: a 256-entry LUT, a value
// (scalar or vector) mapping, or a one-hot over chosen layer characters (in
// occluded mode layers[c] == (board == ord(c)), rendering.py:177-178).  One
// kernel serves all three: the [128, depth] table sits in shared memory, each
// thread converts 4 consecutive cells (one aligned 32-bit board word) and writes
// depth values per cell through caller-chosen strides, so `permute` costs
// nothing.  HBM-bound: reads 1 byte, writes depth * sizeof(T) bytes per cell.
// The kernel only copies bits: an element of 1, 2, 4 or 8 bytes is 1, 2, 1 or 2
// words of T (uint8 for 1 and 2 bytes, uint32 for 4 and 8).  A byte >= 128 lies
// outside every mapping (upstream's are keyed by ASCII characters): its cell gets
// zero elements and the launch flags it as unknown.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pcl.h"
#include "pcl_kernels.cuh"

namespace pcl {

namespace {

constexpr int kThreads = 256;

template <typename T>
__global__ void __launch_bounds__(kThreads)
observe_kernel(const ObserveParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  T* table = reinterpret_cast<T*>(smem_raw);
  __shared__ uint8_t valid[128];
  const T* g_table = static_cast<const T*>(p.table);
  const int row_words = p.depth * p.words;       // 8-byte elements travel as two words
  for (int i = threadIdx.x; i < 128 * row_words; i += kThreads) table[i] = g_table[i];
  if (threadIdx.x < 128) valid[threadIdx.x] = p.valid ? p.valid[threadIdx.x] : 1;
  __syncthreads();

  const int words_per_row = p.pitch >> 2;
  const int64_t total = (int64_t)p.B * p.H * words_per_row;
  T* out = static_cast<T*>(p.out);
  bool unknown = false;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * kThreads) {
    const int wcol = (int)(i % words_per_row);
    const int64_t br = i / words_per_row;
    const int r = (int)(br % p.H);
    const int64_t b = br / p.H;
    const uint32_t cells = reinterpret_cast<const uint32_t*>(p.board)[i];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = wcol * 4 + k;
      if (c >= p.W) break;
      const uint32_t byte = (cells >> (8 * k)) & 0xff;
      const bool ascii = byte < 128;
      unknown |= !ascii || !valid[byte & 0x7f];
      T* dst = out + b * p.stride_b + (int64_t)r * p.stride_r + (int64_t)c * p.stride_c;
      const T* src = table + (byte & 0x7f) * row_words;
      for (int d = 0; d < p.depth; ++d)
        for (int w = 0; w < p.words; ++w)
          dst[d * p.stride_d + w] = ascii ? src[d * p.words + w] : T(0);
    }
  }
  if (unknown && p.unknown) *p.unknown = 1;
}

}  // namespace

cudaError_t launch_observe(const ObserveParams& p, cudaStream_t s) {
  const int64_t total = (int64_t)p.B * p.H * (p.pitch >> 2);
  int blocks = (int)((total + kThreads - 1) / kThreads);
  if (blocks > 132 * 16) blocks = 132 * 16;       // grid-stride over 16 CTAs per SM (H100: 132 SMs)
  if (blocks < 1) blocks = 1;
  const bool bytes = p.dtype == 0 || p.dtype == 5;   // 1- and 2-byte elements
  const size_t smem = 128 * (size_t)p.depth * p.words * (bytes ? 1 : 4);
  if (bytes) observe_kernel<uint8_t><<<blocks, kThreads, smem, s>>>(p);
  else observe_kernel<uint32_t><<<blocks, kThreads, smem, s>>>(p);   // 4- / 8-byte bits
  return cudaGetLastError();
}

namespace {

// One warp per env: the view bytes stream across the lanes, lane 0 appends the
// step outputs (include/pcl.h: PCL_HANDOFF_RECORD_BYTES).
__global__ void __launch_bounds__(128) pack_handoff_kernel(const PackParams p) {
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (env >= p.B) return;
  const uint8_t* src = p.view + (int64_t)env * p.view_bytes;
  const int padded = (p.view_bytes + 3) & ~3;
  // The record as 32-bit words, one per lane per round: view bytes, then
  // reward, discount, done | has_reward << 8.
  const int words = (padded >> 2) + 3;
  const int n_dst = p.n_peers > 0 ? p.n_peers : 1;
  for (int w = lane; w < words; w += 32) {
    uint32_t v;
    const int b = w << 2;
    if (b < padded) {
      v = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (b + k < p.view_bytes) v |= (uint32_t)src[b + k] << (8 * k);
    } else if (b == padded) {
      v = (uint32_t)p.out.d_reward[env];
    } else if (b == padded + 4) {
      v = __float_as_uint(p.out.d_discount[env]);
    } else {
      v = (uint32_t)p.out.d_done[env] | ((uint32_t)p.out.d_has_reward[env] << 8);
    }
    // Local buffer, or the same row of every rank's gather buffer over NVLink.
    for (int d = 0; d < n_dst; ++d) {
      uint8_t* base = p.n_peers > 0 ? p.peers[d] + (p.first_row + env) * p.record_bytes
                                    : p.packed + (int64_t)env * p.record_bytes;
      reinterpret_cast<uint32_t*>(base)[w] = v;
    }
  }
}

}  // namespace

cudaError_t launch_pack_handoff(const PackParams& p, cudaStream_t s) {
  pack_handoff_kernel<<<(p.B + 3) / 4, 128, 0, s>>>(p);
  return cudaGetLastError();
}

}  // namespace pcl
