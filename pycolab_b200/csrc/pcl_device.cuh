// pcl_device.cuh — device building blocks shared by the fused step kernels.
//
// Execution model: ONE WARP PER ENV.  Entity registers (sprite / drape / plot
// records) are loaded once, held REDUNDANTLY in every lane's registers, and
// all game logic is warp-uniform scalar code (no divergence); the lanes split
// up only for (a) board look-ups around a sprite (one lane per neighbour cell,
// combined with __ballot_sync) and (b) the paint loop (one lane per 16-byte
// row segment).  Everything here restates reference semantics; the citations
// are to /root/reference/pycolab.
#pragma once

#include <stdint.h>
#include <stddef.h>
#include <limits.h>

#include "../../include/pcl.h"
#include "pcl_kernels.cuh"

#define PCL_FULL 0xffffffffu
#define PCL_NEVER INT_MIN          // "-inf" frame (drapes.py:371) / None frame

namespace pcl {

// ---------------------------------------------------------------- records --

struct Sprite {                     // things.py:339-391 + sprites.py:153-205
  int row, col, vrow, vcol, flags, aux0, aux1, aux2;
};
struct Drape {                      // drapes.py:293-376
  int corner_r, corner_c, pre_r, pre_c, last_frame, aux0, aux1, aux2;
};
struct Plot {                       // plot.py:69-104 + scrolling.py:198-241
  int frame, game_over, error, episodes;
  int order_r, order_c, order_frame, ego_mask;
  int aux0, aux1, aux2, aux3;
  int crop_r, crop_c, crop_init, reserved;
};

// The structs are the records' word layout (include/pcl.h), so the codec below is the
// one place that knows it.  It takes a plain int32 pointer: a global record or one
// staged in shared memory.
static_assert(sizeof(Sprite) == PCL_SPRITE_WORDS * 4 && offsetof(Sprite, row) == PCL_S_ROW * 4 &&
              offsetof(Sprite, col) == PCL_S_COL * 4 && offsetof(Sprite, vrow) == PCL_S_VROW * 4 &&
              offsetof(Sprite, vcol) == PCL_S_VCOL * 4 && offsetof(Sprite, flags) == PCL_S_FLAGS * 4 &&
              offsetof(Sprite, aux0) == PCL_S_AUX0 * 4 && offsetof(Sprite, aux1) == PCL_S_AUX1 * 4 &&
              offsetof(Sprite, aux2) == PCL_S_AUX2 * 4, "Sprite is not the sprite record");
static_assert(sizeof(Drape) == PCL_DRAPE_WORDS * 4 &&
              offsetof(Drape, corner_r) == PCL_D_CORNER_R * 4 &&
              offsetof(Drape, corner_c) == PCL_D_CORNER_C * 4 &&
              offsetof(Drape, pre_r) == PCL_D_PRE_R * 4 && offsetof(Drape, pre_c) == PCL_D_PRE_C * 4 &&
              offsetof(Drape, last_frame) == PCL_D_LAST_FRAME * 4 &&
              offsetof(Drape, aux0) == PCL_D_AUX0 * 4 && offsetof(Drape, aux1) == PCL_D_AUX1 * 4 &&
              offsetof(Drape, aux2) == PCL_D_AUX2 * 4, "Drape is not the drape record");
static_assert(sizeof(Plot) == PCL_PLOT_WORDS * 4 && offsetof(Plot, frame) == PCL_P_FRAME * 4 &&
              offsetof(Plot, game_over) == PCL_P_GAME_OVER * 4 &&
              offsetof(Plot, error) == PCL_P_ERROR * 4 && offsetof(Plot, episodes) == PCL_P_EPISODES * 4 &&
              offsetof(Plot, order_r) == PCL_P_ORDER_R * 4 && offsetof(Plot, order_c) == PCL_P_ORDER_C * 4 &&
              offsetof(Plot, order_frame) == PCL_P_ORDER_FRAME * 4 &&
              offsetof(Plot, ego_mask) == PCL_P_EGO_MASK * 4 && offsetof(Plot, aux0) == PCL_P_AUX0 * 4 &&
              offsetof(Plot, aux1) == PCL_P_AUX1 * 4 && offsetof(Plot, aux2) == PCL_P_AUX2 * 4 &&
              offsetof(Plot, aux3) == PCL_P_AUX3 * 4 && offsetof(Plot, crop_r) == PCL_P_CROP_R * 4 &&
              offsetof(Plot, crop_c) == PCL_P_CROP_C * 4 &&
              offsetof(Plot, crop_init) == PCL_P_CROP_INIT * 4 &&
              offsetof(Plot, reserved) == PCL_P_RESERVED * 4, "Plot is not the plot record");

__device__ __forceinline__ Sprite load_sprite(const int32_t* r) {
  Sprite s;
  s.row = r[PCL_S_ROW]; s.col = r[PCL_S_COL]; s.vrow = r[PCL_S_VROW]; s.vcol = r[PCL_S_VCOL];
  s.flags = r[PCL_S_FLAGS]; s.aux0 = r[PCL_S_AUX0]; s.aux1 = r[PCL_S_AUX1]; s.aux2 = r[PCL_S_AUX2];
  return s;
}
// The stores write the words before `end` (a PCL_S_* / PCL_D_* index), all eight by
// default.  A kernel that leaves a staged record's AUX words alone stores up to AUX0 and
// need not hold them in registers.
__device__ __forceinline__ void store_sprite(int32_t* r, const Sprite& s, int end = PCL_SPRITE_WORDS) {
  r[PCL_S_ROW] = s.row; r[PCL_S_COL] = s.col; r[PCL_S_VROW] = s.vrow; r[PCL_S_VCOL] = s.vcol;
  r[PCL_S_FLAGS] = s.flags;
  if (end > PCL_S_AUX0) r[PCL_S_AUX0] = s.aux0;
  if (end > PCL_S_AUX1) r[PCL_S_AUX1] = s.aux1;
  if (end > PCL_S_AUX2) r[PCL_S_AUX2] = s.aux2;
}
__device__ __forceinline__ Drape load_drape(const int32_t* r) {
  Drape d;
  d.corner_r = r[PCL_D_CORNER_R]; d.corner_c = r[PCL_D_CORNER_C];
  d.pre_r = r[PCL_D_PRE_R]; d.pre_c = r[PCL_D_PRE_C]; d.last_frame = r[PCL_D_LAST_FRAME];
  d.aux0 = r[PCL_D_AUX0]; d.aux1 = r[PCL_D_AUX1]; d.aux2 = r[PCL_D_AUX2];
  return d;
}
__device__ __forceinline__ void store_drape(int32_t* r, const Drape& d, int end = PCL_DRAPE_WORDS) {
  r[PCL_D_CORNER_R] = d.corner_r; r[PCL_D_CORNER_C] = d.corner_c;
  r[PCL_D_PRE_R] = d.pre_r; r[PCL_D_PRE_C] = d.pre_c; r[PCL_D_LAST_FRAME] = d.last_frame;
  if (end > PCL_D_AUX0) r[PCL_D_AUX0] = d.aux0;
  if (end > PCL_D_AUX1) r[PCL_D_AUX1] = d.aux1;
  if (end > PCL_D_AUX2) r[PCL_D_AUX2] = d.aux2;
}

// Engine directives accumulated during one step (plot.py:69-104).
struct Directives {
  int reward;
  int has_reward;
  int game_over;
  float discount;
};

__device__ __forceinline__ Directives fresh_directives() {
  Directives d;
  d.reward = 0; d.has_reward = 0; d.game_over = 0; d.discount = 1.0f;
  return d;
}
__device__ __forceinline__ void add_reward(Directives& d, int r) {  // plot.py:201
  d.reward += r; d.has_reward = 1;
}
__device__ __forceinline__ void terminate(Directives& d, float discount = 0.0f) {  // plot.py:176-199
  d.game_over = 1; d.discount = discount;
}
// plot.py:247-260.  Upstream rebuilds the directives (discount 1.0) after every
// step (plot.py:345-356, engine.py:845), so the "default" lasts for this step only.
__device__ __forceinline__ void change_default_discount(Directives& d, float discount) {
  d.discount = discount;
}

// ------------------------------------------------------------- MazeWalker --

__device__ __forceinline__ bool visible(const Sprite& s) { return s.flags & 1; }
__device__ __forceinline__ bool on_board(int r, int c, int H, int W) {
  return (unsigned)r < (unsigned)H && (unsigned)c < (unsigned)W;  // sprites.py:548
}

// sprites.py:315-352 (+ _on_board_exit/_on_board_enter :223-275).
__device__ __forceinline__ void walker_teleport(Sprite& s, int H, int W, int vr, int vc) {
  const bool was_on = on_board(s.vrow, s.vcol, H, W);
  const bool now_on = on_board(vr, vc, H, W);
  if (was_on && !now_on) {                     // exit: stash visibility, hide
    const int prior = (s.flags & 1) ? 2 : 1;
    s.flags = (prior << 1);                    // visible = 0
  }
  s.vrow = vr; s.vcol = vc;
  s.row = now_on ? vr : 0;
  s.col = now_on ? vc : 0;
  if (!was_on && now_on) {                     // enter: restore visibility
    const int prior = (s.flags >> 1) & 3;      // 0 None, 1 False, 2 True
    // `_visible = _prior_visible`; None is falsy for the renderer.
    s.flags = (s.flags & ~1) | (prior == 2 ? 1 : 0);
  }
}

// (drow, dcol) of a motion code, two bits per code packed in a constant:
// N NE E SE S SW W NW STAY -> drow+1 = 0 0 1 2 2 2 1 0 1, dcol+1 = 1 2 2 2 1 0 0 0 1.
__device__ __forceinline__ int motion_dr(int m) { return ((0x11A90 >> (2 * m)) & 3) - 1; }
__device__ __forceinline__ int motion_dc(int m) { return ((0x101A9 >> (2 * m)) & 3) - 1; }

// 3x3 neighbourhood "blocked" mask around the walker's VIRTUAL position: bit
// (dr+1)*3 + (dc+1).  Lane k < 9 evaluates one neighbour with `cell_blocked(r,
// c)` (the board of the last render vs the walker's impassable set,
// sprites.py:495-507); off-board neighbours are EDGE, which blocks only walkers
// confined to the board (sprites.py:503-506).
template <typename CellBlocked>
__device__ __forceinline__ unsigned neighbourhood(const Sprite& s, int H, int W,
                                                  bool confined, int lane,
                                                  CellBlocked cell_blocked) {
  const int k = lane < 9 ? lane : 4;
  const int r = s.vrow + k / 3 - 1;
  const int c = s.vcol + k % 3 - 1;
  bool blocked = false;
  if (lane < 9) {
    if (on_board(r, c, H, W)) blocked = cell_blocked(r, c);
    else blocked = confined;
  }
  return __ballot_sync(PCL_FULL, blocked) & 0x1ffu;
}

// sprites.py:479-546: is `motion` legal given the neighbourhood mask?
__device__ __forceinline__ bool motion_legal(unsigned blk, int motion) {
  const int dr = motion_dr(motion), dc = motion_dc(motion);
  if (dr == 0 && dc == 0) return true;
  const unsigned dest = (blk >> ((dr + 1) * 3 + (dc + 1))) & 1u;
  if (dr != 0 && dc != 0) {
    const unsigned f1 = (blk >> ((dr + 1) * 3 + 1)) & 1u;   // (dr, 0)
    const unsigned f2 = (blk >> (3 + (dc + 1))) & 1u;        // (0, dc)
    return !(dest || (f1 && f2));                            // sprites.py:539-543
  }
  return !dest;
}

// scrolling.py:437-482 over the single scrolling group '' the configured
// games use: every egocentric sprite must hold a permit for THIS frame that
// lists `motion`.  Permits live in the sprite record: aux0 = 9-bit motion mask,
// aux1 = frame the permit is valid at.
template <int S>
__device__ __forceinline__ bool scroll_is_possible(const Plot& plot, const Sprite (&sp)[S],
                                                   int motion) {
  bool ok = true;
#pragma unroll
  for (int i = 0; i < S; ++i) {
    if ((plot.ego_mask >> i) & 1) {
      ok = ok && (sp[i].aux1 == plot.frame) && ((sp[i].aux0 >> motion) & 1);
    }
  }
  return ok;
}

// sprites.py:356-389 `_move` for sprite `idx`.
template <typename CellBlocked>
__device__ __forceinline__ bool walker_move(Sprite& s, int idx, int motion, Plot& plot,
                                            int H, int W, bool confined, bool egocentric,
                                            int lane, CellBlocked cell_blocked) {
  const int dr = motion_dr(motion), dc = motion_dc(motion);
  // _obey_scrolling_order, sprites.py:413-454
  if (egocentric) plot.ego_mask |= (1 << idx);
  if (plot.order_frame == plot.frame) {
    walker_teleport(s, H, W, s.vrow - plot.order_r, s.vcol - plot.order_c);
    if (egocentric && plot.order_r != dr && plot.order_c != dc)
      plot.error |= PCL_ENV_ERR_ORDER_MISMATCH;
  }
  bool legal = true;
  unsigned blk = 0;
  if (motion != PCL_M_STAY || egocentric) {
    blk = neighbourhood(s, H, W, confined, lane, cell_blocked);
    legal = motion_legal(blk, motion);
  }
  if (legal && motion != PCL_M_STAY) {
    walker_teleport(s, H, W, s.vrow + dr, s.vcol + dc);      // _raw_move :391
    if (egocentric) blk = neighbourhood(s, H, W, confined, lane, cell_blocked);
  }
  if (egocentric) {                                          // :456-477 + scrolling.py:373-434
    int mask = 1 << PCL_M_STAY;
#pragma unroll
    for (int m = 0; m < 8; ++m) mask |= (motion_legal(blk, m) ? 1 : 0) << m;
    const int valid_at = plot.frame + 1;
    if (s.aux1 != valid_at) { s.aux1 = valid_at; s.aux0 = 0; }
    s.aux0 |= mask;
  }
  return legal;
}

// ---------------------------------------------------------------- Scrolly --

struct ScrollyCfg {               // drapes.py:338-364
  int limit_r, limit_c;           // _northwest_corner_limit
  int have_margins;
  int m_north, m_south, m_west, m_east;
};

__device__ __forceinline__ ScrollyCfg scrolly_cfg(int H, int W, int PH, int PW,
                                                  int margin_r, int margin_c) {
  ScrollyCfg c;
  c.limit_r = PH - H; c.limit_c = PW - W;
  c.have_margins = margin_r >= 0;
  c.m_north = margin_r - 1; c.m_south = H - margin_r;
  c.m_west = margin_c - 1;  c.m_east = W - margin_c;
  return c;
}

// drapes.py:378-411 pattern_position_prescroll: refresh the pre-scroll corner
// when this Scrolly has not moved yet in this frame.
__device__ __forceinline__ void scrolly_touch_prescroll(Drape& d, const Plot& plot) {
  if (d.last_frame < plot.frame) { d.pre_r = d.corner_r; d.pre_c = d.corner_c; }
}

// drapes.py:487-659 `_maybe_move`.  Returns true when the curtain must be
// re-derived from the pattern (always, upstream: every path ends in
// _update_curtain); the window itself is never materialised here.
template <int S>
__device__ __forceinline__ void scrolly_move(Drape& d, const ScrollyCfg& cfg, int motion,
                                             Plot& plot, const Sprite (&sp)[S]) {
  if (d.last_frame < plot.frame) {
    d.last_frame = plot.frame;
    d.pre_r = d.corner_r; d.pre_c = d.corner_c;
  }
  const int dr = motion_dr(motion), dc = motion_dc(motion);
  if (plot.order_frame == plot.frame) {          // obey an existing order :513-535
    if (dr != plot.order_r && dc != plot.order_c) plot.error |= PCL_ENV_ERR_ORDER_MISMATCH;
    d.corner_r += plot.order_r; d.corner_c += plot.order_c;
    return;
  }
  if (motion == PCL_M_STAY) return;
  if (!cfg.have_margins) {                       // :598-623
    if (scroll_is_possible(plot, sp, motion)) {
      const int nr = d.corner_r + dr, nc = d.corner_c + dc;
      const int orr = (0 <= nr && nr <= cfg.limit_r) ? dr : 0;
      const int occ = (0 <= nc && nc <= cfg.limit_c) ? dc : 0;
      d.corner_r += orr; d.corner_c += occ;
      plot.order_r = orr; plot.order_c = occ; plot.order_frame = plot.frame;
    }
    return;
  }
  bool want_v = false, want_h = false;           // :625-642 + :661-687
#pragma unroll
  for (int i = 0; i < S; ++i) {
    if ((plot.ego_mask >> i) & 1) {
      const int nr = sp[i].row + dr, nc = sp[i].col + dc;   // TRUE position
      want_v |= (sp[i].row > nr && nr <= cfg.m_north) || (sp[i].row < nr && nr >= cfg.m_south);
      want_h |= (sp[i].col > nc && nc <= cfg.m_west) || (sp[i].col < nc && nc >= cfg.m_east);
    }
  }
  if (!(want_v || want_h)) return;
  const int orr = want_v ? dr : 0, occ = want_h ? dc : 0;
  const int nr = d.corner_r + orr, nc = d.corner_c + occ;
  bool can = (0 <= nr && nr <= cfg.limit_r) && (0 <= nc && nc <= cfg.limit_c);
  can = can && scroll_is_possible(plot, sp, motion);   // full motion, :650-651
  if (can) {
    d.corner_r = nr; d.corner_c = nc;
    plot.order_r = orr; plot.order_c = occ; plot.order_frame = plot.frame;
  }
}

// ------------------------------------------------------------ bit helpers --

// 16 consecutive bits starting at bit `off` of a bit-packed row (rows carry one
// zero pad word so the second load never leaves the row).
__device__ __forceinline__ unsigned bits16(const uint32_t* row, int off) {
  const int w = off >> 5, sh = off & 31;
  const uint32_t lo = row[w];
  const uint32_t hi = row[w + 1];
  return __funnelshift_r(lo, hi, sh) & 0xffffu;
}
__device__ __forceinline__ bool bit_at(const uint32_t* row, int c) {
  return (row[c >> 5] >> (c & 31)) & 1u;
}
// 4 mask bits -> 4 mask bytes (0x00 / 0xff), cell j in byte j.
__device__ __forceinline__ uint32_t spread4(unsigned nib) {
  return ((nib * 0x00204081u) & 0x01010101u) * 0xffu;
}
// Paint `ch` into the 16-byte segment `seg` wherever `bits` is set.
__device__ __forceinline__ void paint_bits(uint4& seg, unsigned bits, uint32_t ch) {
  const uint32_t c4 = ch * 0x01010101u;
  uint32_t m;
  m = spread4(bits & 15u);         seg.x = (seg.x & ~m) | (c4 & m);
  m = spread4((bits >> 4) & 15u);  seg.y = (seg.y & ~m) | (c4 & m);
  m = spread4((bits >> 8) & 15u);  seg.z = (seg.z & ~m) | (c4 & m);
  m = spread4((bits >> 12) & 15u); seg.w = (seg.w & ~m) | (c4 & m);
}
// One-cell sprite paint (rendering.py:139): bit mask for the sprite inside the
// segment that starts at (r, c0), or 0.
__device__ __forceinline__ unsigned sprite_bit(const Sprite& s, int r, int c0) {
  const int dc = s.col - c0;
  return (visible(s) && s.row == r && (unsigned)dc < 16u) ? (1u << dc) : 0u;
}

// ------------------------------------------------- TMA (1-D bulk) tile moves --
// A board tile is a contiguous, 16-byte aligned run of H * pitch bytes, so it
// moves between HBM and shared memory as ONE bulk-copy instruction issued by
// one lane (SASS UBLKCP), completion tracked by an mbarrier (loads) or a bulk
// group (stores), instead of H * pitch / 512 vector load/store rounds per warp.

__device__ __forceinline__ uint32_t smem_addr(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_addr(bar)), "r"(arrivals));
  // Make the initialised barrier visible to the async proxy (the bulk copy
  // engine).  A CTA-scope proxy fence is enough for a barrier only this CTA
  // uses; the cluster-scope mbarrier_init fence would also flush L1 (CCTL.IVALL).
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// Global -> shared; `bytes` a multiple of 16.  Call from ONE thread.
__device__ __forceinline__ void tile_load_bulk(void* smem_dst, const void* gmem_src,
                                               uint32_t bytes, uint64_t* bar) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
               :: "r"(smem_addr(bar)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes "
               "[%0], [%1], %2, [%3];"
               :: "r"(smem_addr(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_addr(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" :: "r"(smem_addr(bar)), "r"(parity) : "memory");
}
// Shared -> global; make the generic-proxy writes to the tile visible to the
// async proxy first.  Call tile_store_bulk from ONE thread after a warp/block
// barrier; that thread must tile_store_wait() before the CTA can retire.
__device__ __forceinline__ void tile_store_fence() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void tile_store_bulk(void* gmem_dst, const void* smem_src,
                                                uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               :: "l"(gmem_dst), "r"(smem_addr(smem_src)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void tile_store_wait() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// ---------------------------------------------------- cp.async and char sets --

// Global -> shared, 16 bytes, bypassing L1.  Completion: cp_async_wait_all().
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::
               "r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem));
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;\n" ::: "memory");
}
// Is character `code` in a 128-bit character set (one bit per ASCII code)?
__device__ __forceinline__ bool in_set(const uint32_t* set, int code) {
  return (set[(code >> 5) & 3] >> (code & 31)) & 1u;
}

// ------------------------------------------------------------- env scoping --
// One launch steps (MODE_STEP) or resets (MODE_RESET) every env of the batch; an env
// is the batched stand-in for one Engine per episode (engine.py:520-581, 619-624).

enum { MODE_STEP = 0, MODE_RESET = 1 };
enum EnvRun { ENV_SKIP, ENV_STEP, ENV_RESTART };

// What env `env` does in this launch, given its plot's game_over word.  A reset
// restarts the envs the mask selects (all without a mask) and leaves the others
// alone.  A step restarts a finished env under auto_reset; without it the env stays
// frozen (the reference raises on play() after the episode ended).  A skipped env
// writes nothing, but its warp must still drain the async copies it issued.
__device__ __forceinline__ EnvRun env_run(const StepParams& p, int env, int was_over) {
  if (p.mode == MODE_RESET)
    return (p.env_mask == nullptr || p.env_mask[env] != 0) ? ENV_RESTART : ENV_SKIP;
  if (!was_over) return ENV_STEP;
  return p.auto_reset ? ENV_RESTART : ENV_SKIP;
}

// The env's action word; a reset and a restart play PCL_ACTION_NONE (its_showtime).
__device__ __forceinline__ int env_action(const StepParams& p, int env) {
  return p.mode == MODE_STEP ? p.actions[(int64_t)env * p.actions_per_env] : PCL_ACTION_NONE;
}

// What a restart keeps of the env's plot record: everything else comes from the
// *_init templates at the env's level, but the episode count goes up by one and the
// error word carries over.  Read it from the live plot record before the templates
// replace it; store_carry() puts it into the fresh record.
struct PlotCarry { int episodes, error; };
__device__ __forceinline__ PlotCarry plot_carry(const int32_t* plot, bool restart) {
  PlotCarry c;
  c.episodes = plot[PCL_P_EPISODES] + (restart ? 1 : 0);
  c.error = plot[PCL_P_ERROR];
  return c;
}
__device__ __forceinline__ void store_carry(int32_t* plot, const PlotCarry& c) {
  plot[PCL_P_EPISODES] = c.episodes; plot[PCL_P_ERROR] = c.error;
}

// The Plot a step starts from: the frame after the source record's (engine.py:716), the
// carried error word, and the source record's scrolling order (kOrder) or no order.  The
// AUX words are the program's to read.
template <bool kOrder = false>
__device__ __forceinline__ Plot step_plot(const int32_t* src, int error) {
  Plot q;
  q.frame = src[PCL_P_FRAME] + 1;
  q.error = error;
  if (kOrder) {
    q.order_r = src[PCL_P_ORDER_R]; q.order_c = src[PCL_P_ORDER_C];
    q.order_frame = src[PCL_P_ORDER_FRAME]; q.ego_mask = src[PCL_P_EGO_MASK];
  } else {
    q.order_r = q.order_c = 0; q.order_frame = PCL_NEVER; q.ego_mask = 0;
  }
  return q;
}

// Which scrolling-order words store_plot writes: none (the record keeps its own), only
// the order frame, back to PCL_NEVER (programs that never scroll), or all four.
enum PlotOrder { ORDER_KEEP, ORDER_CLEAR, ORDER_ALL };

// The engine's words of the plot record after a step: frame, game_over, the error word
// and the order words kOrder names.  The episode count is the carry's (store_carry); the
// AUX words are the program's to store, and the CROP words the cropper epilogue's.
template <PlotOrder kOrder>
__device__ __forceinline__ void store_plot(int32_t* rec, const Plot& q, const Directives& dir) {
  rec[PCL_P_FRAME] = q.frame; rec[PCL_P_GAME_OVER] = dir.game_over; rec[PCL_P_ERROR] = q.error;
  if (kOrder == ORDER_CLEAR) rec[PCL_P_ORDER_FRAME] = PCL_NEVER;
  if (kOrder == ORDER_ALL) {
    rec[PCL_P_ORDER_R] = q.order_r; rec[PCL_P_ORDER_C] = q.order_c;
    rec[PCL_P_ORDER_FRAME] = q.order_frame; rec[PCL_P_EGO_MASK] = q.ego_mask;
  }
}

// The step's outputs for env `env` (one lane stores them).
__device__ __forceinline__ void store_outputs(const pcl_outputs& out, int env, const Directives& dir) {
  out.d_reward[env] = dir.reward;
  out.d_has_reward[env] = (uint8_t)dir.has_reward;
  out.d_discount[env] = dir.discount;
  out.d_done[env] = (uint8_t)dir.game_over;
}
// The same for a program whose rewards are float64 (Program::float_reward): `reward` goes
// to d_reward_f64 and d_reward is not written.
__device__ __forceinline__ void store_outputs(const pcl_outputs& out, int env, const Directives& dir,
                                              double reward) {
  out.d_reward_f64[env] = reward;
  out.d_has_reward[env] = (uint8_t)dir.has_reward;
  out.d_discount[env] = dir.discount;
  out.d_done[env] = (uint8_t)dir.game_over;
}

}  // namespace pcl
