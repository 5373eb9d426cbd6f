// ordeal.cu — fused step kernel for the three sub-games of examples/ordeal.py
// (SURVEY.md §8f-4), the one real user of Plot.change_z_order (ordeal.py:182-185).
//
// p.program_arg[0] names the chapter (PCL_ORDEAL_*):
//   CASTLE  sprites P, D   one update group [P, D], z-order D P (dynamic)  (ordeal.py:79-82)
//   CAVERN  sprite P, drape S (bits)  group [P, S]                         (:85-89)
//   KANSAS  sprite P                                                       (:91-93)
// The Plot entries the reference keeps in Python dict slots ride in the plot
// record: AUX0 = has_sword, AUX1 = last_position (row << 16 | col, -1 = unset),
// AUX2 = next_chapter the player / the duck chose (PCL_ORDEAL_NEXT_*), AUX3 = the
// prior chapter (set by the host when Story builds the Engine, storytelling.py:453).
//
// Both entities of a group read the board of the LAST render (engine.py:725-735):
// `prev_char` rebuilds any of its cells from the start-of-step registers in z-order,
// so no previous board is carried between steps.  One warp per env; boards are small
// (<= 8 KiB, staged whole in shared memory like the classics).
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 4;
constexpr int kRecWords = 48;       // sprites 2 x 8, drape 8, pad 8, plot 16

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
ordeal_step(const StepParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int env = blockIdx.x * kWarpsPerBlock + warp;
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;
  const int H = p.H, W = p.W, pitch = p.pitch, S = p.S, D = p.D, BW = p.BW;
  const int chapter = p.program_arg[0];
  const int tile = H * pitch;
  uint8_t* my = smem_raw + warp * (kRecWords * 4 + tile);
  int32_t* rec = reinterpret_cast<int32_t*>(my);
  uint8_t* s_bd = my + kRecWords * 4;

  int32_t* g_sprites = p.st.d_sprites + (int64_t)env * S * PCL_SPRITE_WORDS;
  int32_t* g_drape = D ? p.st.d_drapes + (int64_t)env * PCL_DRAPE_WORDS : nullptr;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  uint8_t* g_z = p.st.d_z_order ? p.st.d_z_order + (int64_t)env * (S + D) : nullptr;
  uint32_t* sword = D ? p.st.d_bits[0] + (int64_t)env * p.st.bits_bstride[0] : nullptr;
  const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;
  for (int i = lane; i < (tile >> 4); i += 32) cp_async16(s_bd + i * 16, backdrop + i * 16);

  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) { cp_async_wait_all(); return; }
  const bool restart = run == ENV_RESTART;
  if (restart) {                                   // a fresh Engine (engine.py:520-581)
    const PlotCarry carry = plot_carry(g_plot, true);
    if (lane < S * 8) rec[lane] = __ldg(p.st.d_sprites_init + lvl * p.st.sprites_init_bstride + lane);
    if (D && lane >= 16 && lane < 24)
      rec[lane] = __ldg(p.st.d_drapes_init + lvl * p.st.drapes_init_bstride + lane - 16);
    if (lane < 16) rec[32 + lane] = __ldg(p.st.d_plot_init + lvl * p.st.plot_init_bstride + lane);
    if (D) {
      const uint32_t* src = p.st.d_bits_init[0] + lvl * p.st.bits_init_bstride[0];
      for (int i = lane; i < H * BW; i += 32) sword[i] = __ldg(src + i);
    }
    if (g_z && lane < S + D) g_z[lane] = p.st.d_z_order_init[lvl * p.st.z_order_init_bstride + lane];
    __syncwarp();
    if (lane == 0) store_carry(rec + 32, carry);
  } else {
    if (lane < S * 8) rec[lane] = g_sprites[lane];
    if (D && lane >= 16 && lane < 24) rec[lane] = g_drape[lane - 16];
    if (lane < 16) rec[32 + lane] = g_plot[lane];
  }
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  cp_async_wait_all();
  __syncwarp();

  Sprite pl = load_sprite(rec);
  Sprite dd = S > 1 ? load_sprite(rec + 8) : pl;
  Plot plot = step_plot(rec + 32, rec[32 + PCL_P_ERROR]);
  int has_sword = rec[32 + PCL_P_AUX0], last_pos = rec[32 + PCL_P_AUX1];
  int next_chapter = rec[32 + PCL_P_AUX2];
  const int prior = rec[32 + PCL_P_AUX3];
  Directives dir = fresh_directives();
  uint8_t z0 = p.sprite_char[0], z1 = 0;                     // z-order back to front
  if (S + D == 2) {
    z0 = g_z ? g_z[0] : (uint8_t)(D ? p.sprite_char[0] : p.sprite_char[1]);
    z1 = g_z ? g_z[1] : (uint8_t)(D ? p.drape_char[0] : p.sprite_char[0]);
  }

  // The board of the last render, cell by cell, from the start-of-step state.
  const Sprite pl0 = pl, dd0 = dd;
  auto entity_at = [&](uint8_t ch, int r, int c) -> bool {
    if (ch == p.sprite_char[0]) return visible(pl0) && pl0.row == r && pl0.col == c;
    if (S > 1 && ch == p.sprite_char[1]) return visible(dd0) && dd0.row == r && dd0.col == c;
    if (D && ch == p.drape_char[0]) return bit_at(sword + (int64_t)r * BW, c);
    return false;
  };
  auto prev_char = [&](int r, int c) -> int {
    int code = s_bd[r * pitch + c];
    if (entity_at(z0, r, c)) code = z0;
    if (z1 && entity_at(z1, r, c)) code = z1;
    return code;
  };

  // ---- PlayerSprite.update (ordeal.py:206-266) ------------------------------
  {
    const int limit_r = H - 1, limit_c = W - 1;              // self._limits :204
    auto blocked = [&](int r, int c) { return in_set(p.impassable[0], prev_char(r, c)); };
    auto leave = [&](int to) { next_chapter = to; terminate(dir); };
    int motion = PCL_M_NONE;
    if (action == 0) {
      if (chapter == PCL_ORDEAL_KANSAS && pl.row <= 0) leave(PCL_ORDEAL_CASTLE); else motion = PCL_M_N;
    } else if (action == 1) {
      if (chapter == PCL_ORDEAL_CASTLE && pl.row >= limit_r) leave(PCL_ORDEAL_KANSAS); else motion = PCL_M_S;
    } else if (action == 2) {
      if (chapter == PCL_ORDEAL_CAVERN && pl.col <= 0) leave(PCL_ORDEAL_KANSAS); else motion = PCL_M_W;
    } else if (action == 3) {
      if (chapter == PCL_ORDEAL_KANSAS && pl.col >= limit_c) leave(PCL_ORDEAL_CAVERN); else motion = PCL_M_E;
    } else if (action == 4) {
      leave(PCL_ORDEAL_NEXT_NONE);
    } else if (plot.frame == 0 && last_pos >= 0) {           // line up with the last game :248-264
      const int lr = last_pos >> 16, lc = last_pos & 0xffff;
      if (prior == PCL_ORDEAL_KANSAS && chapter == PCL_ORDEAL_CASTLE) walker_teleport(pl, H, W, limit_r, lc);
      else if (prior == PCL_ORDEAL_CASTLE && chapter == PCL_ORDEAL_KANSAS) walker_teleport(pl, H, W, 0, lc);
      else if (prior == PCL_ORDEAL_KANSAS && chapter == PCL_ORDEAL_CAVERN) walker_teleport(pl, H, W, lr, 0);
      else if (prior == PCL_ORDEAL_CAVERN && chapter == PCL_ORDEAL_KANSAS) walker_teleport(pl, H, W, lr, limit_c);
    }
    if (motion != PCL_M_NONE)
      walker_move(pl, 0, motion, plot, H, W, p.confined[0] != 0, false, lane, blocked);
    last_pos = (pl.row << 16) | pl.col;                      // :266
  }

  // ---- DragonduckSprite.update (:142-185) -----------------------------------
  bool z_changed = false;
  if (chapter == PCL_ORDEAL_CASTLE && S > 1 && plot.frame != 0) {
    auto blocked = [&](int r, int c) { return in_set(p.impassable[1], prev_char(r, c)); };
    const bool above = dd.row > pl.row, right = dd.col < pl.col, below = dd.row < pl.row,
               left = dd.col > pl.col;
    int motion = PCL_M_NONE;
    if (above && !right && !below && !left) motion = PCL_M_N;
    else if (above && right && !below && !left) motion = PCL_M_NE;
    else if (!above && right && !below && !left) motion = PCL_M_E;
    else if (!above && right && below && !left) motion = PCL_M_SE;
    else if (!above && !right && below && !left) motion = PCL_M_S;
    else if (!above && !right && below && left) motion = PCL_M_SW;
    else if (!above && !right && !below && left) motion = PCL_M_W;
    else if (above && !right && !below && left) motion = PCL_M_NW;
    if (motion != PCL_M_NONE)
      walker_move(dd, 1, motion, plot, H, W, p.confined[1] != 0, false, lane, blocked);
    // layers['P'][self.position] of the last render (occluded layers, rendering.py:177)
    if (prev_char(dd.row, dd.col) == p.sprite_char[0]) {
      next_chapter = PCL_ORDEAL_NEXT_NONE;
      terminate(dir);
      if (has_sword) {                       // change_z_order(move_this='D', in_front_of_that='P')
        add_reward(dir, 1);
        z0 = p.sprite_char[0]; z1 = p.sprite_char[1];
      } else {                               // change_z_order(move_this='P', in_front_of_that='D')
        add_reward(dir, -1);
        z0 = p.sprite_char[1]; z1 = p.sprite_char[0];
      }
      z_changed = true;
    }
  }

  // ---- SwordDrape.update (:120-124) -----------------------------------------
  if (chapter == PCL_ORDEAL_CAVERN && D) {
    if (bit_at(sword + (int64_t)pl.row * BW, pl.col)) { has_sword = 1; add_reward(dir, 1); }
    if (has_sword) {
      __syncwarp();
      for (int i = lane; i < H * BW; i += 32) sword[i] = 0;
      __syncwarp();
    }
  }

  // ---- _apply_and_clear_plot (engine.py:761-847) + records back
  __syncwarp();
  if (lane == 0) {
    store_sprite(rec, pl, PCL_S_AUX0);
    if (S > 1) store_sprite(rec + 8, dd, PCL_S_AUX0);
    store_plot<ORDER_KEEP>(rec + 32, plot, dir);
    rec[32 + PCL_P_AUX0] = has_sword; rec[32 + PCL_P_AUX1] = last_pos;
    rec[32 + PCL_P_AUX2] = next_chapter;
    store_outputs(p.out, env, dir);
    if (g_z && z_changed) { g_z[0] = z0; g_z[1] = z1; }
  }
  __syncwarp();
  if (lane < S * 8) g_sprites[lane] = rec[lane];
  if (D && lane >= 16 && lane < 24) g_drape[lane - 16] = rec[lane];
  if (lane < 16) g_plot[lane] = rec[32 + lane];

  // ---- final render in the (possibly new) z-order (engine.py:737-759)
  uint8_t* board = p.out.d_board + (int64_t)env * tile;
  const int segs_per_row = pitch >> 4;
  const int total = H * segs_per_row;
  for (int seg = lane; seg < total; seg += 32) {
    const int r = seg / segs_per_row;
    const int c0 = (seg - r * segs_per_row) << 4;
    uint4 px = *reinterpret_cast<const uint4*>(s_bd + r * pitch + c0);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const uint8_t ch = k == 0 ? z0 : z1;
      if (!ch) continue;
      unsigned m = 0;
      if (ch == p.sprite_char[0]) m = sprite_bit(pl, r, c0);
      else if (S > 1 && ch == p.sprite_char[1]) m = sprite_bit(dd, r, c0);
      else if (D && ch == p.drape_char[0] && c0 < W)    // a segment past the board is pad
        m = bits16(sword + (int64_t)r * BW, c0) & ((1u << min(16, W - c0)) - 1u);
      if (m) paint_bits(px, m, ch);
    }
    *reinterpret_cast<uint4*>(board + r * pitch + c0) = px;
  }
}

int check_spec(const pcl_spec& s) {
  const int chapter = s.program_arg[0];
  const int want_s = chapter == PCL_ORDEAL_CASTLE ? 2 : 1, want_d = chapter == PCL_ORDEAL_CAVERN ? 1 : 0;
  if (chapter != PCL_ORDEAL_CASTLE && chapter != PCL_ORDEAL_CAVERN && chapter != PCL_ORDEAL_KANSAS)
    return PCL_ERR_INVALID;
  if (s.n_sprites != want_s || s.n_drapes != want_d) return PCL_ERR_UNSUPPORTED;
  if (s.n_groups != 1 || s.group_len[0] != want_s + want_d) return PCL_ERR_UNSUPPORTED;
  if (s.group_chars[0] != s.sprite_char[0]) return PCL_ERR_UNSUPPORTED;     // the player moves first
  for (int i = 0; i < want_s; ++i) if (s.sprite_egocentric[i]) return PCL_ERR_UNSUPPORTED;
  if (s.rows >= 32768 || s.cols >= 32768 || s.rows * s.pitch > 8192) return PCL_ERR_UNSUPPORTED;
  if (want_d && !bit_rows_fit(s)) return PCL_ERR_INVALID;
  return PCL_OK;
}

int check_state(const pcl_spec& s, const pcl_state& st) {
  if (s.n_drapes && (!st.d_bits[0] || !st.d_bits_init[0] || st.bits_bstride[0] == 0))
    return PCL_ERR_INVALID;
  if (s.n_sprites + s.n_drapes == 2 && (!st.d_z_order || !st.d_z_order_init))
    return PCL_ERR_INVALID;                   // the kernel reads the z-order of two entities
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  const size_t smem = (kRecWords * 4 + (size_t)p.H * p.pitch) * kWarpsPerBlock;
  return launch_step(ordeal_step, p, kWarpsPerBlock, smem, s);
}

}  // namespace

const Program kOrdeal = {check_spec, check_state, curtain_bits, launch, nullptr,
                         /*float_reward=*/false, /*crop_epilogue=*/false,
                         /*scroll_groups=*/false};

}  // namespace pcl
