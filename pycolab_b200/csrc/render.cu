// render.cu — the stand-alone renderer, unoccluded-layers and cropper kernels.
//
// render_kernel is Engine._render() + BaseObservationRenderer (engine.py:737-759,
// rendering.py:98-179) over reference-layout inputs: one byte per cell for the
// backdrop and for every drape curtain.  It is a pure HBM streaming kernel:
// per env it reads (1 + D) * H * pitch bytes and writes H * pitch bytes; the
// occlusion flatten down the z-order is done per 16-byte segment with byte-SIMD
// rank compares so that all (1 + D) loads of a segment are issued up front and
// no register array is indexed dynamically.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"
#include "pcl_crop.cuh"

namespace pcl {

namespace {

constexpr int kRenderThreads = 256;

template <int MAXD, int MAXS>
struct RenderShared {
  uint32_t rank_d[MAXD];          // z rank of each drape, replicated in 4 bytes
  uint32_t rank_s[MAXS];
  int seg[MAXS];                  // 16-byte segment holding each visible sprite, or -1
  int word[MAXS];                 // which 32-bit word of the segment
  uint32_t cover[MAXS];           // 0xff at the sprite's byte
};

// Where `cover` (0x00/0xff per byte) is set and the rank is higher, write
// ch4 / rank4 (later z-order entries paint over earlier ones, engine.py:751).
__device__ __forceinline__ void overlay(uint32_t& px, uint32_t& rk, uint32_t cover,
                                        uint32_t ch4, uint32_t rank4) {
  const uint32_t take = cover & __vcmpltu4(rk, rank4);
  px = (px & ~take) | (ch4 & take);
  rk = (rk & ~take) | (rank4 & take);
}

template <int MAXD, int MAXS>
__global__ void __launch_bounds__(kRenderThreads)
render_kernel(const RenderParams p) {
  __shared__ RenderShared<MAXD, MAXS> sh;
  const int env = blockIdx.x;
  const int n = p.S + p.D;
  const int segs_per_row = p.pitch >> 4;
  const uint8_t* backdrop = p.backdrop + (int64_t)env * p.backdrop_bstride;
  const int64_t plane = (int64_t)p.H * p.pitch;
  const uint8_t* curtains = p.curtains + (int64_t)env * p.D * plane;
  uint8_t* board = p.board + (int64_t)env * plane;
  const int total = p.H * segs_per_row;

  // Issue the tile loads of the first segment before anything else: they do not
  // depend on the z-order / sprite decode below, so both round trips overlap.
  int seg = threadIdx.x;
  uint4 px = make_uint4(0, 0, 0, 0);
  uint4 cur[MAXD];
  if (seg < total) {
    const int64_t off = (int64_t)seg << 4;
    px = __ldg(reinterpret_cast<const uint4*>(backdrop + off));
#pragma unroll
    for (int d = 0; d < MAXD; ++d)
      if (d < p.D) cur[d] = __ldg(reinterpret_cast<const uint4*>(curtains + d * plane + off));
  }

  // Decode this env's z-order and sprite cells once per block.
  if (threadIdx.x < n) {
    const uint8_t ch = p.z_order[(int64_t)env * n + threadIdx.x];
    const uint32_t rank4 = (threadIdx.x + 1) * 0x01010101u;
#pragma unroll
    for (int s = 0; s < MAXS; ++s) if (s < p.S && p.sprite_char[s] == ch) sh.rank_s[s] = rank4;
#pragma unroll
    for (int d = 0; d < MAXD; ++d) if (d < p.D && p.drape_char[d] == ch) sh.rank_d[d] = rank4;
  }
  if (threadIdx.x < p.S) {
    const int32_t* rec = p.sprites + ((int64_t)env * p.S + threadIdx.x) * PCL_SPRITE_WORDS;
    // `board[tuple(position)]` (rendering.py:139): a negative row or column counts from
    // the end once; a position still off the board (a plain Sprite may stand anywhere)
    // paints nothing.
    int row = rec[PCL_S_ROW], col = rec[PCL_S_COL];
    row += row < 0 ? p.H : 0;
    col += col < 0 ? p.W : 0;
    const bool vis = (rec[PCL_S_FLAGS] & 1) &&                 // engine.py:754
                     (unsigned)row < (unsigned)p.H && (unsigned)col < (unsigned)p.W;
    sh.seg[threadIdx.x] = vis ? row * segs_per_row + (col >> 4) : -1;
    sh.word[threadIdx.x] = (col & 15) >> 2;
    sh.cover[threadIdx.x] = 0xffu << ((col & 3) * 8);
  }
  __syncthreads();

  while (seg < total) {
    uint4 rk = make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int d = 0; d < MAXD; ++d) {
      if (d < p.D) {
        const uint32_t ch4 = p.drape_char[d] * 0x01010101u;
        const uint32_t r4 = sh.rank_d[d];
        overlay(px.x, rk.x, __vcmpne4(cur[d].x, 0), ch4, r4);   // rendering.py:160
        overlay(px.y, rk.y, __vcmpne4(cur[d].y, 0), ch4, r4);
        overlay(px.z, rk.z, __vcmpne4(cur[d].z, 0), ch4, r4);
        overlay(px.w, rk.w, __vcmpne4(cur[d].w, 0), ch4, r4);
      }
    }
#pragma unroll
    for (int s = 0; s < MAXS; ++s) {
      if (s < p.S && sh.seg[s] == seg) {                         // rendering.py:139
        const uint32_t ch4 = p.sprite_char[s] * 0x01010101u;
        const uint32_t r4 = sh.rank_s[s], cover = sh.cover[s];
        const int w = sh.word[s];
        if (w == 0) overlay(px.x, rk.x, cover, ch4, r4);
        else if (w == 1) overlay(px.y, rk.y, cover, ch4, r4);
        else if (w == 2) overlay(px.z, rk.z, cover, ch4, r4);
        else overlay(px.w, rk.w, cover, ch4, r4);
      }
    }
    *reinterpret_cast<uint4*>(board + ((int64_t)seg << 4)) = px;
    seg += kRenderThreads;
    if (seg < total) {
      const int64_t off = (int64_t)seg << 4;
      px = __ldg(reinterpret_cast<const uint4*>(backdrop + off));
#pragma unroll
      for (int d = 0; d < MAXD; ++d)
        if (d < p.D) cur[d] = __ldg(reinterpret_cast<const uint4*>(curtains + d * plane + off));
    }
  }
}

// BaseUnoccludedObservationRenderer's layers (rendering.py:187-301): the mask of
// character k shows where its OWNER places it, occluded or not — a backdrop
// character where the backdrop holds it (paint_all_of :222-236), a drape's whole
// curtain (paint_drape :262-282 overwrites the layer), a visible sprite's cell on
// top of the backdrop term (paint_sprite :238-260).  One block per env streams
// n_chars planes of H * pitch bytes (0 / 1), 16 cells per thread per store.  A
// drape's plane is its Drape.curtain as bytes (things.py:213-217): pcl_export_curtain
// is a one-plane launch.
__global__ void __launch_bounds__(256) layers_kernel(const LayersParams p) {
  const int env = blockIdx.x;
  const int segs_per_row = p.pitch >> 4;
  const int plane_segs = p.H * segs_per_row;
  const int64_t lvl = p.level ? p.level[env] : env;
  const uint8_t* backdrop = p.backdrop + (p.backdrop_per_env ? env : lvl) * p.backdrop_bstride;
  uint8_t* out = p.out + (int64_t)env * p.n_chars * p.H * p.pitch;
  for (int i = threadIdx.x; i < p.n_chars * plane_segs; i += blockDim.x) {
    const int k = i / plane_segs, seg = i - k * plane_segs;
    const int r = seg / segs_per_row, c0 = (seg - r * segs_per_row) << 4;
    const int ncols = min(16, p.W - c0);
    uint4 px = make_uint4(0, 0, 0, 0);
    const int d = p.drape_of[k];
    if (ncols <= 0) {
      // A segment wholly past the board (pitch > ceil16(W)) is pad: zeros, and nothing is
      // read.  (1u << ncols) would not mask it: the shift of a negative count gives 0, so
      // the mask would be all ones and copy the bits past the window or the row.
    } else if (d >= 0) {
      const int32_t* drec = p.drapes + ((int64_t)env * p.D + d) * PCL_DRAPE_WORDS;
      const int cr = p.scrolly[d] ? drec[PCL_D_CORNER_R] : 0;
      const int cc = p.scrolly[d] ? drec[PCL_D_CORNER_C] : 0;
      const uint32_t* bits = p.bits[d] + (p.per_level[d] ? lvl : (int64_t)env) * p.bits_bstride[d];
      unsigned b = bits16(bits + (int64_t)(cr + r) * p.row_words[d], cc + c0) &
                   ((1u << ncols) - 1u);
      if (p.stale_slot[d]) {
        const int sr = drec[PCL_D_AUX0], sc = drec[PCL_D_AUX1];
        if (r == sr && (unsigned)(sc - c0) < 16u) b |= 1u << (sc - c0);
      }
      paint_bits(px, b, 1);
    } else {
      const uint4 bd = *reinterpret_cast<const uint4*>(backdrop + (int64_t)r * p.pitch + c0);
      const uint32_t ch4 = p.chars[k] * 0x01010101u;
      px.x = __vcmpeq4(bd.x, ch4) & 0x01010101u; px.y = __vcmpeq4(bd.y, ch4) & 0x01010101u;
      px.z = __vcmpeq4(bd.z, ch4) & 0x01010101u; px.w = __vcmpeq4(bd.w, ch4) & 0x01010101u;
      const int sidx = p.sprite_of[k];
      if (sidx >= 0) {
        const int32_t* rec = p.sprites + ((int64_t)env * p.S + sidx) * PCL_SPRITE_WORDS;
        int sr = rec[PCL_S_ROW], sc = rec[PCL_S_COL];      // wrapped as render_kernel does
        sr += sr < 0 ? p.H : 0;
        sc += sc < 0 ? p.W : 0;
        const int dc = sc - c0;
        if ((rec[PCL_S_FLAGS] & 1) && sr == r && (unsigned)sc < (unsigned)p.W && (unsigned)dc < 16u) {
          uint32_t* w = dc < 4 ? &px.x : dc < 8 ? &px.y : dc < 12 ? &px.z : &px.w;
          *w |= 1u << ((dc & 3) * 8);
        }
      }
    }
    *reinterpret_cast<uint4*>(out + ((int64_t)k * p.H + r) * p.pitch + c0) = px;
  }
}

__global__ void __launch_bounds__(128) crop_kernel(const CropParams p) {
  __shared__ int s_hist[4][256];
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x * 4 + (threadIdx.x >> 5);
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");     // the step kernel's board and records
  if (env >= p.B) return;
  int wr, wc;
  crop_corner(p, env, lane, s_hist[threadIdx.x >> 5], &wr, &wc);
  // _do_crop :118-227: pad fill + window copy, 4 cells per lane per round; word
  // stores wherever the env's output row is word aligned (cells % 4 == 0 or env
  // aligned), bytes for the ragged rest.
  const uint8_t* board = p.board + (int64_t)env * p.H * p.pitch;
  const int cells = p.crop.rows * p.crop.cols;
  uint8_t* out = p.out + (int64_t)env * cells;
  const int mis = (int)(reinterpret_cast<uintptr_t>(out) & 3);     // bytes before the first aligned word
  const int head = mis ? 4 - mis : 0;
  if (lane < head && lane < cells) {
    const uint32_t v = crop_word(p, board, wr, wc, lane, cells);
    out[lane] = (uint8_t)v;
  }
  for (int i = head + lane * 4; i < cells; i += 128) {
    const uint32_t v = crop_word(p, board, wr, wc, i, cells);
    if (i + 4 <= cells) {
      *reinterpret_cast<uint32_t*>(out + i) = v;
    } else {
      for (int k = 0; i + k < cells; ++k) out[i + k] = (uint8_t)(v >> (8 * k));
    }
  }
}

// ---- crop + pack + all-gather + signal in ONE kernel (SURVEY 8e) -------------
// One warp per env: window corner (as crop_kernel), the crop gathered straight into
// the env's hand-off record (view bytes, reward, discount, done | has_reward << 8),
// the record stored with 16-byte stores into row first_row + env of EVERY rank's
// gather buffer over NVLink (or once through the NVLS multicast address).  The last
// block to finish publishes this rank's step number in every peer's flag word and
// then waits until every peer has published the same step here, so when the kernel
// retires the local gather buffer holds all ranks' records: no collective call, no
// separate barrier kernel.  The parts of the gather buffer alternate by step; the step
// counter lives in device memory, so the launch is CUDA-graph capturable.  With lag 1
// (split phase, >= 3 parts) the kernel signals this step but waits only for the previous
// one, which by then has long arrived: the cross-GPU wait leaves the critical path and
// consumers read one step behind.
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_v4(void* mc, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
               :: "l"(mc), "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)),
                  "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w)) : "memory");
}

__global__ void __launch_bounds__(128) crop_handoff_kernel(const CropParams p,
                                                           const HandoffParams x) {
  __shared__ int s_hist[4][256];
  __shared__ __align__(16) uint32_t s_rec[4][64];          // record words of this block's envs
  __shared__ int s_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int env = blockIdx.x * 4 + warp;
  // Programmatic dependent launch: resident while the step kernel drains, reads
  // nothing before it (and the previous hand-off, which bumps the counter) is done.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const uint32_t step = x.local[0];                        // steps completed so far
  const int64_t half = (int64_t)(step % (uint32_t)x.n_bufs) * x.rows * x.record_bytes;   // this step's part
  if (env < p.B) {
    int wr, wc;
    crop_corner(p, env, lane, s_hist[warp], &wr, &wc);
    const uint8_t* board = p.board + (int64_t)env * p.H * p.pitch;
    const int cells = p.crop.rows * p.crop.cols;
    const int view_words = (cells + 3) >> 2, words = x.record_bytes >> 2;
    for (int w = lane; w < words; w += 32) {
      uint32_t v = 0;                                      // padding up to record_bytes
      if (w < view_words) v = crop_word(p, board, wr, wc, w * 4, cells);
      else if (w == view_words) v = (uint32_t)x.out.d_reward[env];
      else if (w == view_words + 1) v = __float_as_uint(x.out.d_discount[env]);
      else if (w == view_words + 2)
        v = (uint32_t)x.out.d_done[env] | ((uint32_t)x.out.d_has_reward[env] << 8);
      s_rec[warp][w] = v;
    }
    __syncwarp();
    const int64_t row_off = half + (x.first_row + env) * x.record_bytes;
    const int vecs = x.record_bytes >> 4;                  // record_bytes is a multiple of 16 here
    if (x.multicast) {
      for (int q = lane; q < vecs; q += 32)
        multimem_st_v4(x.multicast + row_off + q * 16,
                       *reinterpret_cast<const uint4*>(&s_rec[warp][q * 4]));
    } else {
      for (int q = lane; q < vecs * x.n_peers; q += 32) {
        const int d = q / vecs, k = q - d * vecs;
        *reinterpret_cast<uint4*>(x.peer_base[d] + row_off + k * 16) =
            *reinterpret_cast<const uint4*>(&s_rec[warp][k * 4]);
      }
    }
  }
  // ---- publish: every block fences its peer stores, the last one signals --------
  if (x.signal_kernel) return;         // handoff_signal_kernel, launched behind this one, does it
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(&x.local[1], 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence_system();
  if (threadIdx.x < x.n_peers)                             // my step has landed on peer d
    st_release_sys(x.peer_flags[threadIdx.x] + x.rank, step + 1);
  if (threadIdx.x < x.n_peers) {       // wait for every peer's records: of this step, or
    const uint32_t* mine = x.peer_flags[x.rank] + threadIdx.x;          // (lag 1) of the previous one
    const uint32_t want = step + 1u - (uint32_t)x.lag;
    while ((int32_t)(ld_acquire_sys(mine) - want) < 0) { __nanosleep(20); }
  }
  __syncthreads();
  if (threadIdx.x == 0) { x.local[1] = 0; x.local[0] = step + 1; __threadfence(); }
}

// The publish step as its own one-warp kernel, stream-ordered behind crop_handoff_kernel
// (PCL_HANDOFF_SIGNAL_KERNEL).  That kernel has RETIRED when this one starts, so its peer
// stores are complete (a grid's memory operations are performed before a dependent grid
// begins); what is left is one release store per peer and the acquire poll.  Timing probes
// at N = 2 (tools/handoff_probe.py) on the project's earlier target GPU found the per-block
// system fences and the last block's signalling inside the big kernel slower than this
// kernel; not repeated on H100.
__global__ void __launch_bounds__(32) handoff_signal_kernel(const HandoffParams x) {
  const uint32_t step = x.local[0];
  if (threadIdx.x < x.n_peers) {
    __threadfence_system();
    st_release_sys(x.peer_flags[threadIdx.x] + x.rank, step + 1);
    const uint32_t* mine = x.peer_flags[x.rank] + threadIdx.x;
    const uint32_t want = step + 1u - (uint32_t)x.lag;
    while ((int32_t)(ld_acquire_sys(mine) - want) < 0) { __nanosleep(20); }
  }
  __syncwarp();
  if (threadIdx.x == 0) { x.local[0] = step + 1; __threadfence(); }
}

}  // namespace

cudaError_t launch_render(const RenderParams& p, cudaStream_t s) {
  // Loop bounds are compile-time so the per-segment code stays small.  One CTA per env
  // won an A/B on the project's earlier target GPU against persistent warps, a 2-stage
  // cp.async CTA pipeline, and balanced flat chunks with register staging or a per-thread
  // cp.async ring (those variants are deleted; not repeated on H100).
  if (p.D <= 2 && p.S <= 4) render_kernel<2, 4><<<p.B, kRenderThreads, 0, s>>>(p);
  else if (p.D <= 2 && p.S <= 8) render_kernel<2, 8><<<p.B, kRenderThreads, 0, s>>>(p);
  else if (p.D <= 2) render_kernel<2, 16><<<p.B, kRenderThreads, 0, s>>>(p);
  else if (p.S <= 4) render_kernel<8, 4><<<p.B, kRenderThreads, 0, s>>>(p);
  else render_kernel<8, 16><<<p.B, kRenderThreads, 0, s>>>(p);
  return cudaGetLastError();
}
cudaError_t launch_layers(const LayersParams& p, cudaStream_t s) {
  layers_kernel<<<p.B, 256, 0, s>>>(p);
  return cudaGetLastError();
}
cudaError_t launch_crop(const CropParams& p, cudaStream_t s) {
  if (p.crop.cols < 1 || (int64_t)p.crop.rows * p.crop.cols > PCL_MAX_CROP_CELLS) return cudaErrorInvalidValue;
  return launch_pdl(crop_kernel, (p.B + 3) / 4, 128, 0, s, p);
}
cudaError_t launch_crop_handoff(const CropParams& p, const HandoffParams& x, cudaStream_t s) {
  if (p.crop.cols < 1 || (int64_t)p.crop.rows * p.crop.cols > PCL_MAX_CROP_CELLS) return cudaErrorInvalidValue;
  cudaError_t e = launch_pdl(crop_handoff_kernel, (p.B + 3) / 4, 128, 0, s, p, x);
  if (e != cudaSuccess || !x.signal_kernel) return e;
  handoff_signal_kernel<<<1, 32, 0, s>>>(x);          // plain stream order: after the grid above retires
  return cudaGetLastError();
}

}  // namespace pcl
