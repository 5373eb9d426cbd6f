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
#include "pcl_crop.cuh"
#include "pcl_kernels.cuh"

namespace pcl {

namespace {

constexpr int kThreads = 256;

// Element d of a cell holding `byte`: its `words` words in row `byte` of a table staged
// with `row_words` words per row, or zeros for a byte >= 128 (outside every mapping).
template <typename T>
__device__ __forceinline__ void put_element(T* dst, const T* table, int row_words, int words,
                                            uint32_t byte, int d) {
  const bool ascii = byte < 128;
  const T* src = table + (byte & 0x7f) * row_words + d * words;
  for (int w = 0; w < words; ++w) dst[w] = ascii ? src[w] : T(0);
}

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
      for (int d = 0; d < p.depth; ++d)
        put_element(dst + d * p.stride_d, table, row_words, p.words, byte, d);
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

// ---- a cropper's window through a post-processor (pcl_crop_observe) ---------------
// One warp per env, four envs per block, as crop_kernel (render.cu): the warp moves its
// env's window corner once (crop_corner), then writes depth elements per window cell.
// The table is staged in shared memory kCropChunk planes at a time, so any depth is one
// launch and the corner advances exactly once per call.  The lanes walk the output in
// the order of its strides, so that neighbouring lanes store neighbouring elements.
constexpr int kCropChunk = 32;

template <typename T>
__global__ void __launch_bounds__(128) crop_observe_kernel(const CropObserveParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  T* table = reinterpret_cast<T*>(smem_raw);               // [128, planes of this chunk]
  __shared__ int s_hist[4][256];                           // drape medians (crop_corner)
  __shared__ uint8_t valid[128];
  __shared__ int plane_of[kCropChunk];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const CropParams& c = p.crop;
  const int env = blockIdx.x * 4 + warp;
  const bool active = env < c.B;                           // whole warps: every thread syncs
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");       // the step kernel's board and records
  int wr = 0, wc = 0;
  if (active) crop_corner(c, env, lane, s_hist[warp], &wr, &wc);
  valid[threadIdx.x] = p.valid ? p.valid[threadIdx.x] : 1;

  const int rows = c.crop.rows, cells = rows * c.crop.cols;
  const int minor = p.col_major ? rows : c.crop.cols;
  const uint32_t padv = c.crop.pad_char >= 0 ? (uint32_t)c.crop.pad_char : 0u;
  const T* g_table = static_cast<const T*>(p.table);
  T* out = static_cast<T*>(p.out) + (int64_t)env * p.stride_b;
  const uint8_t* board = c.board + (int64_t)env * c.H * c.pitch;
  const uint8_t* planes = p.planes + (int64_t)env * p.plane_stride_b;
  bool unknown = false;
  for (int k0 = 0; k0 < p.depth; k0 += kCropChunk) {
    const int n = min(kCropChunk, p.depth - k0);
    const int row_words = n * p.words;
    __syncthreads();                                       // the last chunk's readers are done
    for (int i = threadIdx.x; i < 128 * row_words; i += 128) {
      const int row = i / row_words;
      table[i] = g_table[((int64_t)row * p.depth + k0) * p.words + (i - row * row_words)];
    }
    if (p.planes && threadIdx.x < n) plane_of[threadIdx.x] = p.plane_of[k0 + threadIdx.x];
    __syncthreads();
    if (!active) continue;
    // This lane's element as (fast, slow) = (plane, cell) or (cell, plane); each round
    // the warp moves on by 32 elements.
    const int nf = p.planes_fast ? n : cells, ns = p.planes_fast ? cells : n;
    const int step_f = 32 % nf, step_s = 32 / nf;
    int f = lane % nf, s = lane / nf;
    while (s < ns) {
      const int d = p.planes_fast ? f : s, i = p.planes_fast ? s : f;
      const int major = minor == 1 ? i : (int)__umulhi((uint32_t)i, p.minor_recip);
      const int jr = p.col_major ? i - major * minor : major;
      const int jc = p.col_major ? major : i - major * minor;
      uint32_t byte;
      if (p.planes) {                                      // un-occluded: the layer's bit
        const int k = plane_of[d];
        byte = k >= 0 && crop_cell(c, planes + k * p.plane_stride_d, p.plane_stride_r, wr, wc,
                                   jr, jc, k == p.pad_plane) != 0;
      } else {
        byte = crop_cell(c, board, c.pitch, wr, wc, jr, jc, padv);
        unknown |= byte >= 128 || !valid[byte & 0x7f];
      }
      put_element(out + (k0 + d) * p.stride_d + jr * p.stride_r + jc * p.stride_c, table,
                  row_words, p.words, byte, d);
      f += step_f;
      s += step_s;
      if (f >= nf) { f -= nf; ++s; }
    }
  }
  if (active && __any_sync(0xffffffffu, unknown) && lane == 0 && p.unknown) *p.unknown = 1;
}

}  // namespace

cudaError_t launch_crop_observe(const CropObserveParams& p, cudaStream_t s) {
  const pcl_crop_spec& c = p.crop.crop;
  if (c.rows < 1 || c.cols < 1 || (int64_t)c.rows * c.cols > PCL_MAX_CROP_CELLS || p.depth < 1)
    return cudaErrorInvalidValue;
  CropObserveParams q = p;
  const int64_t sd = llabs(p.stride_d), sr = llabs(p.stride_r), sc = llabs(p.stride_c);
  q.planes_fast = p.depth > 1 && sd < sr && sd < sc;
  q.col_major = sr < sc;
  const int minor = q.col_major ? c.rows : c.cols;
  // floor(2^32 / minor) + 1: __umulhi(i, recip) == i / minor for every i < 65536.
  q.minor_recip = minor > 1 ? (uint32_t)(0x100000000ull / (uint32_t)minor) + 1u : 0u;
  const bool bytes = p.dtype == 0 || p.dtype == 5;         // 1- and 2-byte elements
  const size_t smem = 128 * (size_t)min(p.depth, kCropChunk) * p.words * (bytes ? 1 : 4);
  const int grid = (p.crop.B + 3) / 4;
  if (bytes) return launch_pdl(crop_observe_kernel<uint8_t>, grid, 128, smem, s, q);
  return launch_pdl(crop_observe_kernel<uint32_t>, grid, 128, smem, s, q);
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
