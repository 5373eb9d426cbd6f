// shockwave.cu — fused step kernel for examples/shockwave.py:91-197 (SURVEY.md §8f-4).
//
// One update group [' ', '^', 'P', '@'], z-order ' ' '^' '@' 'P' over a backdrop of '+'
// (what lies beneath everything) and '=' (walls).  Sprite 0 = the player, a MazeWalker
// confined to the board with impassable '='; drapes 0 = '@' (the shockwave), 1 = ' ' (the
// danger zone), 2 = '^' (the safe zone); ' ' and '^' never change (MinimalDrape), so
// their curtains are read from the per-level templates (pcl_state.d_bits_init[1..2]).
//
//   P: action 0 = _north, 1 = _west, 2 = _east, 3 = _stay, anything else: no call  (:98-109)
//   '@' (after P, same group, so every `layers[...]` it consults is the STALE board of
//   the previous render, engine.py:725):
//     curtain empty -> impact = np.random.randint(0, H * W) (MT19937, masked rejection),
//       distance = Euclidean distance to it, steps_since_impact = 0               (:129-140)
//     curtain = steps < distance <= steps + width, minus walls — compared on SQUARED
//       integer distances, exact because steps is an integer                       (:145-149)
//     P's position shows '^' on the stale board (safe-zone cell not covered by the OLD
//       curtain, nor by P itself one frame ago): reward +1, terminate              (:152-156)
//     P under the NEW curtain and in the danger zone: reward -1, terminate         (:158-163)
//     steps_since_impact += 1
// '=' is never covered on a rendered board (each art cell belongs to exactly one of the
// backdrop / a drape / the sprite, and the curtain excludes walls), so "stale board == '='"
// is "backdrop == '='", for the walker's impassable test as well.
// The shockwave's curtain lives bit-packed in pcl_state.d_bits[0] (one row per lane), its
// impact cell and step count in the drape record's AUX0 / AUX1; program_arg[0] = width.
// One warp per env; boards up to 32 rows x 64 columns.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"
#include "pcl_mt.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 4;
typedef unsigned long long u64;

__device__ __forceinline__ u64 row_bits(const uint32_t* base, int r, int BW) {
  const uint32_t* row = base + (int64_t)r * BW;
  return (u64)row[0] | (BW > 1 ? (u64)row[1] << 32 : 0ull);
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
shockwave_step(const StepParams p) {
  __shared__ u64 s_rows[kWarpsPerBlock][32];          // the new curtain, a row per lane, for the render
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;
  const int H = p.H, W = p.W, pitch = p.pitch, BW = p.BW;
  int32_t* g_sprite = p.st.d_sprites + (int64_t)env * PCL_SPRITE_WORDS;
  int32_t* g_drapes = p.st.d_drapes + (int64_t)env * 3 * PCL_DRAPE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;
  uint32_t* wave_bits = p.st.d_bits[0] + (int64_t)env * p.st.bits_bstride[0];
  const uint32_t* danger_bits = p.st.d_bits_init[1] + lvl * p.st.bits_init_bstride[1];
  const uint32_t* safe_bits = p.st.d_bits_init[2] + lvl * p.st.bits_init_bstride[2];

  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) return;
  const bool restart = run == ENV_RESTART;
  const int32_t* src_s = restart ? p.st.d_sprites_init + lvl * p.st.sprites_init_bstride : g_sprite;
  const int32_t* src_d = restart ? p.st.d_drapes_init + lvl * p.st.drapes_init_bstride : g_drapes;
  const int32_t* src_p = restart ? p.st.d_plot_init + lvl * p.st.plot_init_bstride : g_plot;
  Sprite pl = load_sprite(src_s);
  pl.aux0 = pl.aux1 = pl.aux2 = 0;                                    // stored as zeros
  int impact = src_d[PCL_D_AUX0], steps = src_d[PCL_D_AUX1];
  const PlotCarry carry = plot_carry(g_plot, restart);
  Plot plot = step_plot(src_p, carry.error);
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  Directives dir = fresh_directives();
  // Row `lane` of the curtain the LAST render showed (the art's '@' cells after a restart).
  const uint32_t* old_base = restart ? p.st.d_bits_init[0] + lvl * p.st.bits_init_bstride[0] : wave_bits;
  const u64 old_row = lane < H ? row_bits(old_base, lane, BW) : 0ull;
  const int old_row_p = pl.row, old_col_p = pl.col;
  const bool old_vis_p = visible(pl);

  // ---- PlayerSprite.update (:98-109)
  const int motion = action == 0 ? PCL_M_N : action == 1 ? PCL_M_W : action == 2 ? PCL_M_E
                   : action == 3 ? PCL_M_STAY : PCL_M_NONE;
  auto wall = [&](int r, int c) { return in_set(p.impassable[0], backdrop[r * pitch + c]); };
  if (motion != PCL_M_NONE)
    walker_move(pl, 0, motion, plot, H, W, p.confined[0] != 0, false, lane, wall);

  // ---- ShockwaveDrape.update (:126-165)
  if (!__any_sync(PCL_FULL, old_row != 0ull)) {                       // :129
    uint32_t* mt = p.st.d_rng + (int64_t)env * PCL_MT_WORDS;
    impact = (int)mt_below(mt, (uint32_t)(H * W), lane);              // np.random.randint(0, size)
    steps = 0;
  }
  const int ir = impact / W, ic = impact - ir * W;                    // np.unravel_index
  const int width = p.program_arg[0];
  const int lo2 = steps * steps, hi2 = (steps + width) * (steps + width);
  u64 new_row = 0ull;
  if (lane < H) {
    const int dr2 = (lane - ir) * (lane - ir);
    for (int c = 0; c < W; ++c) {
      const int d2 = dr2 + (c - ic) * (c - ic);
      if (d2 > lo2 && d2 <= hi2 && !wall(lane, c)) new_row |= 1ull << c;
    }
  }
  // The player's cell, as every lane needs it: rows of the old / new curtain and the
  // two static drapes at P's row.
  const int pr = pl.row, pc = pl.col;
  const u64 old_at = __shfl_sync(PCL_FULL, old_row, pr);
  const u64 new_at = __shfl_sync(PCL_FULL, new_row, pr);
  const bool safe_here = (row_bits(safe_bits, pr, BW) >> pc) & 1ull;
  const bool danger_here = (row_bits(danger_bits, pr, BW) >> pc) & 1ull;
  const bool stale_shows_safe = safe_here && !((old_at >> pc) & 1ull) &&
                                !(old_vis_p && old_row_p == pr && old_col_p == pc);
  if (stale_shows_safe) { add_reward(dir, 1); terminate(dir); }      // :152-156
  if (((new_at >> pc) & 1ull) && danger_here) { add_reward(dir, -1); terminate(dir); }
  steps += 1;

  s_rows[threadIdx.x >> 5][lane] = new_row;
  __syncwarp();
  if (lane < H) {
    uint32_t* row = wave_bits + (int64_t)lane * BW;
    row[0] = (uint32_t)new_row;
    if (BW > 1) row[1] = (uint32_t)(new_row >> 32);
  }
  if (lane == 0) {
    store_sprite(g_sprite, pl);
    g_drapes[PCL_D_AUX0] = impact; g_drapes[PCL_D_AUX1] = steps;
    g_drapes[PCL_D_LAST_FRAME] = PCL_NEVER;
    store_carry(g_plot, carry);
    store_plot<ORDER_CLEAR>(g_plot, plot, dir);
    store_outputs(p.out, env, dir);
  }

  // ---- render (engine.py:737-759): backdrop, ' ', '^', '@', P
  uint8_t* board = p.out.d_board + (int64_t)env * H * pitch;
  const int segs_per_row = pitch >> 4;
  const int total = H * segs_per_row;
  for (int seg = lane; seg < total; seg += 32) {
    const int r = seg / segs_per_row;
    const int c0 = (seg - r * segs_per_row) << 4;
    uint4 px = *reinterpret_cast<const uint4*>(backdrop + r * pitch + c0);
    const u64 wave_r = s_rows[threadIdx.x >> 5][r];
    paint_bits(px, (unsigned)((row_bits(danger_bits, r, BW) >> c0) & 0xffffull), p.drape_char[1]);
    paint_bits(px, (unsigned)((row_bits(safe_bits, r, BW) >> c0) & 0xffffull), p.drape_char[2]);
    paint_bits(px, (unsigned)((wave_r >> c0) & 0xffffull), p.drape_char[0]);
    const unsigned m = sprite_bit(pl, r, c0);
    if (m) paint_bits(px, m, p.sprite_char[0]);
    *reinterpret_cast<uint4*>(board + r * pitch + c0) = px;
  }
}

int check_spec(const pcl_spec& s) {
  if (s.n_sprites != 1 || s.n_drapes != 3) return PCL_ERR_UNSUPPORTED;
  // one update group [' ', '^', P, '@'] (the two static drapes may come in either
  // order), z-order ' ' '^' '@' P
  if (s.n_groups != 1 || s.group_len[0] != 4 || s.group_chars[2] != s.sprite_char[0] ||
      s.group_chars[3] != s.drape_char[0]) return PCL_ERR_UNSUPPORTED;
  if (s.z_order[0] != s.drape_char[1] || s.z_order[1] != s.drape_char[2] ||
      s.z_order[2] != s.drape_char[0] || s.z_order[3] != s.sprite_char[0]) return PCL_ERR_UNSUPPORTED;
  if (!s.sprite_confined[0] || s.sprite_egocentric[0]) return PCL_ERR_UNSUPPORTED;
  if (s.rows > 32 || s.cols > 64) return PCL_ERR_UNSUPPORTED;      // a curtain row per lane, 64-bit rows
  if (!bit_rows_fit(s)) return PCL_ERR_INVALID;
  if (s.program_arg[0] < 0 || s.program_arg[0] > 1024) return PCL_ERR_INVALID;
  return PCL_OK;
}

int check_state(const pcl_spec&, const pcl_state& st) {
  if (!st.d_bits[0] || st.bits_bstride[0] == 0 || !st.d_rng) return PCL_ERR_INVALID;
  for (int d = 0; d < 3; ++d) if (!st.d_bits_init[d]) return PCL_ERR_INVALID;
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  return launch_step(shockwave_step, p, kWarpsPerBlock, 0, s);
}

}  // namespace

const Program kShockwave = {check_spec, check_state, curtain_bits, launch, nullptr,
                            /*float_reward=*/false, /*crop_epilogue=*/false,
                            /*scroll_groups=*/false};

}  // namespace pcl
