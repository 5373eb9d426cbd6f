// pcl_board.cuh — the board-keeping step programs' shared machinery: a real board in
// shared memory, rendered after every update group (engine.py:725-735), and the per-warp
// copies of the env's records it is rendered from.  Used by fixture.cu and compiled.cu.
#pragma once

#include "pcl_device.cuh"
#include "pcl_kernels.cuh"

namespace pcl {
namespace board {

constexpr int kMaxEnt = PCL_MAX_SPRITES + PCL_MAX_DRAPES;

struct WarpState {                   // lives in shared memory, one per warp
  int32_t sprites[PCL_MAX_SPRITES][PCL_SPRITE_WORDS];
  int32_t drapes[PCL_MAX_DRAPES][PCL_DRAPE_WORDS];
  int32_t plot[PCL_PLOT_WORDS];
  uint32_t impassable[PCL_MAX_SPRITES][4];
  // One record per scrolling group (protocols/scrolling.py:198-241): the group an
  // entity belongs to is swapped into the `Plot` registers around its update.
  int32_t groups[PCL_MAX_SCROLL_GROUPS][PCL_GROUP_WORDS];
  uint8_t z[kMaxEnt + 8];
};

// Bytes of the smem board of one warp: H * pitch, rounded up to 16.
__host__ __device__ __forceinline__ size_t board_bytes(int H, int pitch) {
  return ((size_t)H * pitch + 15) & ~(size_t)15;
}

struct Ctx {
  const StepParams* p;
  WarpState* st;
  uint8_t* board;                    // smem, H * pitch
  const uint8_t* backdrop;
  int env, lane;
  int64_t lvl;                       // index of static level data
  uint32_t kept;                     // bit d: Scrolly d's curtain is kept in d_bits, not read
                                     // from its pattern (compiled.cu: patterns it writes)
};

// Row r of drape d's curtain bits (d_bits) in env c.env.
__device__ __forceinline__ uint32_t* bits_row(const Ctx& c, int d, int r) {
  const StepParams& p = *c.p;
  return p.st.d_bits[d] + (int64_t)c.env * p.st.bits_bstride[d] + (int64_t)r * p.BW;
}

__device__ __forceinline__ bool drape_bit(const Ctx& c, int d, int r, int col) {
  const StepParams& p = *c.p;
  if (p.drape_kind[d] && !((c.kept >> d) & 1)) {   // Scrolly: window of the pattern (drapes.py:689-695)
    const uint32_t* pat = p.st.d_pattern[d] + c.lvl * p.st.pattern_bstride[d];
    const int pr = c.st->drapes[d][PCL_D_CORNER_R] + r, pc = c.st->drapes[d][PCL_D_CORNER_C] + col;
    return bit_at(pat + (int64_t)pr * p.PWW, pc);
  }
  return bit_at(bits_row(c, d, r), col);
}

// engine.py:737-759 + rendering.py:98-160 into the smem board.  kWrap: sprite positions
// may lie off the board (compiled.cu's plain Sprites), and a visible sprite paints at its
// NumPy-wrapped cell, `board[tuple(position)]` (rendering.py:139): a negative row or
// column counts from the end once, and a position no cell matches paints nothing.
template <bool kWrap = false>
__device__ inline void render(const Ctx& c) {
  const StepParams& p = *c.p;
  const int n = p.S + p.D, cells = p.H * p.W;
  for (int i = c.lane; i < cells; i += 32) {
    const int r = i / p.W, col = i - r * p.W;
    int code = c.backdrop[(int64_t)r * p.pitch + col];
    for (int k = 0; k < n; ++k) {
      const int ch = c.st->z[k];
      for (int s = 0; s < p.S; ++s) {
        if (p.sprite_char[s] == ch) {
          const int32_t* rec = c.st->sprites[s];
          if (kWrap) {
            int sr = rec[PCL_S_ROW], sc = rec[PCL_S_COL];
            sr += sr < 0 ? p.H : 0;
            sc += sc < 0 ? p.W : 0;
            if ((rec[PCL_S_FLAGS] & 1) && sr == r && sc == col) code = ch;
          } else if ((rec[PCL_S_FLAGS] & 1) && rec[PCL_S_ROW] == r && rec[PCL_S_COL] == col) {
            code = ch;
          }
        }
      }
      for (int d = 0; d < p.D; ++d)
        if (p.drape_char[d] == ch && drape_bit(c, d, r, col)) code = ch;
    }
    c.board[(int64_t)r * p.pitch + col] = (uint8_t)code;
  }
  __syncwarp();
}

// Write a sprite back to its record in the warp's state (one lane, between warp barriers).
__device__ __forceinline__ void warp_store_sprite(int32_t* r, const Sprite& s, int lane) {
  __syncwarp();
  if (lane == 0) store_sprite(r, s);
  __syncwarp();
}

// scrolling.py:437-482 over the sprites in shared memory.
__device__ inline bool is_possible(const Ctx& c, const Plot& plot, int motion) {
  bool ok = true;
  for (int i = 0; i < c.p->S; ++i) {
    if ((plot.ego_mask >> i) & 1) {
      const int32_t* r = c.st->sprites[i];
      ok = ok && (r[PCL_S_AUX1] == plot.frame) && ((r[PCL_S_AUX0] >> motion) & 1);
    }
  }
  return ok;
}

// drapes.py:487-659 for drape d (same logic as pcl::scrolly_move, dynamic S).
__device__ inline void scrolly_move_dyn(const Ctx& c, int d, int motion, Plot& plot) {
  const StepParams& p = *c.p;
  int32_t* rec = c.st->drapes[d];
  Drape dp = load_drape(rec);
  const ScrollyCfg cfg = scrolly_cfg(p.H, p.W, p.PH, p.PW, p.margin[d][0], p.margin[d][1]);
  if (dp.last_frame < plot.frame) {
    dp.last_frame = plot.frame; dp.pre_r = dp.corner_r; dp.pre_c = dp.corner_c;
  }
  const int dr = motion_dr(motion), dc = motion_dc(motion);
  if (plot.order_frame == plot.frame) {
    if (dr != plot.order_r && dc != plot.order_c) plot.error |= PCL_ENV_ERR_ORDER_MISMATCH;
    dp.corner_r += plot.order_r; dp.corner_c += plot.order_c;
  } else if (motion != PCL_M_STAY) {
    if (!cfg.have_margins) {
      if (is_possible(c, plot, motion)) {
        const int nr = dp.corner_r + dr, nc = dp.corner_c + dc;
        const int orr = (0 <= nr && nr <= cfg.limit_r) ? dr : 0;
        const int occ = (0 <= nc && nc <= cfg.limit_c) ? dc : 0;
        dp.corner_r += orr; dp.corner_c += occ;
        plot.order_r = orr; plot.order_c = occ; plot.order_frame = plot.frame;
      }
    } else {
      bool want_v = false, want_h = false;
      for (int i = 0; i < p.S; ++i) {
        if ((plot.ego_mask >> i) & 1) {
          const int32_t* s = c.st->sprites[i];
          const int row = s[PCL_S_ROW], col = s[PCL_S_COL];
          const int nr = row + dr, nc = col + dc;
          want_v |= (row > nr && nr <= cfg.m_north) || (row < nr && nr >= cfg.m_south);
          want_h |= (col > nc && nc <= cfg.m_west) || (col < nc && nc >= cfg.m_east);
        }
      }
      if (want_v || want_h) {
        const int orr = want_v ? dr : 0, occ = want_h ? dc : 0;
        const int nr = dp.corner_r + orr, nc = dp.corner_c + occ;
        bool can = (0 <= nr && nr <= cfg.limit_r) && (0 <= nc && nc <= cfg.limit_c);
        can = can && is_possible(c, plot, motion);
        if (can) {
          dp.corner_r = nr; dp.corner_c = nc;
          plot.order_r = orr; plot.order_c = occ; plot.order_frame = plot.frame;
        }
      }
    }
  }
  __syncwarp();
  if (c.lane == 0) store_drape(rec, dp, PCL_D_AUX0);
  __syncwarp();
}

// Copy the env's sprite, drape and plot records and its z-order into the warp's state.
__device__ __forceinline__ void stage_records(WarpState* st, const int32_t* src_s,
                                              const int32_t* src_d, const int32_t* src_p,
                                              const uint8_t* src_z, int S, int D, int lane) {
  for (int i = lane; i < S * PCL_SPRITE_WORDS; i += 32) (&st->sprites[0][0])[i] = src_s[i];
  for (int i = lane; i < D * PCL_DRAPE_WORDS; i += 32) (&st->drapes[0][0])[i] = src_d[i];
  if (lane < PCL_PLOT_WORDS) st->plot[lane] = src_p[lane];
  if (lane < S + D) st->z[lane] = src_z[lane];
}

// The board every entity of the first update group reads: the pre-initial render
// (engine.py:572-578) at a restart, else last step's final board from `g_board`.
template <bool kWrap = false>
__device__ __forceinline__ void stage_board(const Ctx& c, bool restart, const uint8_t* g_board) {
  if (restart) {
    render<kWrap>(c);
  } else {
    const int n16 = (c.p->H * c.p->pitch) >> 4;
    for (int i = c.lane; i < n16; i += 32)
      reinterpret_cast<uint4*>(c.board)[i] = reinterpret_cast<const uint4*>(g_board)[i];
    __syncwarp();
  }
}

// Write the warp's records, z-order and board back to the env (after __syncwarp).
__device__ __forceinline__ void store_env(const Ctx& c, int32_t* g_sprites, int32_t* g_drapes,
                                         int32_t* g_plot, uint8_t* g_z, uint8_t* g_board) {
  const StepParams& p = *c.p;
  const WarpState* st = c.st;
  const int lane = c.lane, S = p.S, D = p.D;
  for (int i = lane; i < S * PCL_SPRITE_WORDS; i += 32) g_sprites[i] = (&st->sprites[0][0])[i];
  for (int i = lane; i < D * PCL_DRAPE_WORDS; i += 32) g_drapes[i] = (&st->drapes[0][0])[i];
  if (lane < PCL_PLOT_WORDS) g_plot[lane] = st->plot[lane];
  if (lane < S + D) g_z[lane] = st->z[lane];
  const int n16 = (p.H * p.pitch) >> 4;
  for (int i = lane; i < n16; i += 32)
    reinterpret_cast<uint4*>(g_board)[i] = reinterpret_cast<const uint4*>(c.board)[i];
}

}  // namespace board
}  // namespace pcl
