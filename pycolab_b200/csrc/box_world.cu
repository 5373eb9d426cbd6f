// box_world.cu — fused step kernel for examples/research/box_world/box_world.py:127-271.
//
// One MazeWalker '.' (impassable '#', confined) and up to 41 object drapes — keys 'a'-'t',
// locks 'A'-'T' and the gem '*' — in ONE update group ['.', sorted objects], objects behind
// the player.  The reference never puts two objects on one cell (a held key sits at (0, 0),
// over the '#' wall), so the objects are one per-env byte grid instead of drapes of their
// own: d_bits[0] viewed as u8 [rows, pitch], 0 = no object, else the character, with bit 7
// set on a distractor lock cell (`distractors` is per cell upstream).  Its reset template,
// d_bits_init[0], is the level's.  The spec then has no drapes, so every level of one
// grid_size and max_num_steps shares one handle.
//
// One warp per env; lane r stages board row r of the grid in shared memory and paints board
// row r.  The game logic is warp-uniform scalar code against the board of the last render:
//   * actions 0-3 (N S W E) only; anything else does nothing — no reward, no step counted.
//   * A valid action pays 0 (so has_reward is set); the player enters a free cell, a lock if
//     board[0, 0] holds its key, a key or the gem if no lock stands at column + 1.
//   * The step counter (sprite AUX0) goes up; counter > program_arg[0] terminates.
//   * Whenever the target holds an object, the_plot['over_this'] = (char, player position
//     after the move): plot AUX0 = char, AUX1 = row << 16 | col.  It persists, so every
//     frame the drape of that char acts if its curtain holds that cell: the gem pays 10 and
//     terminates; a key moves to (0, 0), dropping the held one; a lock clears, consumes the
//     held key and pays +1, or -1 and terminates on a distractor cell.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 4;
constexpr int kMaxSide = 32;                     // one lane per board row, <= 32 bytes per row
constexpr int kDistractor = 0x80;

__device__ __forceinline__ bool is_key(int c) { return c >= 'a' && c <= 't'; }
__device__ __forceinline__ bool is_lock(int c) { return c >= 'A' && c <= 'T'; }

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
box_world_step(const StepParams p) {
  __shared__ __align__(16) uint8_t s_grid[kWarpsPerBlock][kMaxSide * kMaxSide];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int env = blockIdx.x * kWarpsPerBlock + warp;
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;
  const int H = p.H, pitch = p.pitch, segs = p.pitch >> 4;
  int32_t* g_sprite = p.st.d_sprites + (int64_t)env * PCL_SPRITE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  uint8_t* g_grid = reinterpret_cast<uint8_t*>(p.st.d_bits[0] + (int64_t)env * p.st.bits_bstride[0]);

  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) return;
  const bool restart = run == ENV_RESTART;
  const int32_t* src_s = restart ? p.st.d_sprites_init + lvl * p.st.sprites_init_bstride : g_sprite;
  const int32_t* src_p = restart ? p.st.d_plot_init + lvl * p.st.plot_init_bstride : g_plot;
  const uint8_t* src_g = restart
      ? reinterpret_cast<const uint8_t*>(p.st.d_bits_init[0] + lvl * p.st.bits_init_bstride[0])
      : g_grid;
  uint8_t* grid = s_grid[warp];
  if (lane < H)
    for (int q = 0; q < segs; ++q)
      reinterpret_cast<uint4*>(grid + lane * pitch)[q] =
          reinterpret_cast<const uint4*>(src_g + lane * pitch)[q];

  Sprite pl = load_sprite(src_s);
  pl.aux1 = pl.aux2 = 0;                           // stored as zeros
  int steps = pl.aux0;                             // PlayerSprite._step_counter
  const PlotCarry carry = plot_carry(g_plot, restart);
  Plot plot = step_plot(src_p, carry.error);
  int over_ch = src_p[PCL_P_AUX0];                 // the_plot['over_this']: 0 = unset
  int over_at = src_p[PCL_P_AUX1];
  const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;
  __syncwarp();

  // the board of the last render where the player is not: an object, else the backdrop
  auto board_at = [&](int r, int c) -> int {
    const int g = grid[r * pitch + c] & 0x7f;
    return g ? g : backdrop[r * pitch + c];
  };
  const int held = board_at(0, 0);                 // inventory_item
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  Directives dir = fresh_directives();

  // ---- PlayerSprite.update (:163-202)
  bool raised = false;                             // a look-up NumPy would refuse
  if (action >= 0 && action < 4) {
    add_reward(dir, 0);                            // REWARD_STEP
    const int tr = pl.row + (action == 0 ? -1 : action == 1 ? 1 : 0);
    const int tc = pl.col + (action == 2 ? -1 : action == 3 ? 1 : 0);
    // A level without its '#' ring: NumPy wraps index -1 and raises IndexError past the last
    // row or column, which latches PCL_ENV_ERR_INDEX and ends the update there (no step is
    // counted); the walker is confined, so it never steps off the board.
    raised = tr >= H || tc >= p.W;
    if (!raised) {
      const int row = (tr < 0 ? tr + H : tr) * pitch;
      const int at = row + (tc < 0 ? tc + p.W : tc);
      const bool on = tr >= 0 && tc >= 0;
      const int thing = grid[at] & 0x7f;
      bool move;
      if (!thing) {
        move = !in_set(p.impassable[0], backdrop[at]);
      } else {
        move = is_lock(thing) && held == thing + ('a' - 'A');
        if (move && on) { pl.row = pl.vrow = tr; pl.col = pl.vcol = tc; }
        raised = tc + 1 >= p.W;
        // BoxThing.is_locked_at: a lock at column + 1 (0 <= tc + 1; row -1 wraps)
        move = !raised && !is_lock(thing) && !is_lock(grid[row + tc + 1] & 0x7f);
      }
      if (move && on) { pl.row = pl.vrow = tr; pl.col = pl.vcol = tc; }
      if (thing && !raised) { over_ch = thing; over_at = (pl.row << 16) | pl.col; }
    }
    if (raised) plot.error |= PCL_ENV_ERR_INDEX;
    else if (++steps > p.program_arg[0]) terminate(dir);
  }

  // ---- the object drapes (:232-271), unless the player's update raised: only the one named
  // by over_this can act
  int changed = -1;                                // a grid row besides row 0 that changed
  if (over_ch && !raised) {
    const int oy = over_at >> 16, ox = over_at & 0xffff;
    const int cell = grid[oy * pitch + ox];
    if ((cell & 0x7f) == over_ch) {                // where_player_over_me
      if (over_ch == '*') {
        add_reward(dir, 10);
        terminate(dir);
      } else {
        changed = oy;
        __syncwarp();
        if (lane == 0) {
          grid[oy * pitch + ox] = 0;
          grid[0] = is_key(over_ch) ? over_ch : (is_key(held) ? 0 : grid[0]);
        }
        __syncwarp();
        if (!is_key(over_ch)) {
          if (cell & kDistractor) { add_reward(dir, -1); terminate(dir); }
          else add_reward(dir, 1);
        }
      }
    }
  }

  // ---- records, outputs and the grid rows that changed
  if (lane == 0) {
    pl.aux0 = steps;
    store_sprite(g_sprite, pl);
    store_carry(g_plot, carry);
    store_plot<ORDER_KEEP>(g_plot, plot, dir);
    g_plot[PCL_P_AUX0] = over_ch; g_plot[PCL_P_AUX1] = over_at;
    store_outputs(p.out, env, dir);
  }
  if (lane < H && (restart || (changed >= 0 && (lane == 0 || lane == changed))))
    for (int q = 0; q < segs; ++q)
      reinterpret_cast<uint4*>(g_grid + lane * pitch)[q] =
          reinterpret_cast<const uint4*>(grid + lane * pitch)[q];

  // ---- render (engine.py:737-759): backdrop, objects, then the player; lane r paints row r
  if (lane < H) {
    uint8_t* board = p.out.d_board + (int64_t)env * H * pitch + lane * pitch;
    const uint8_t* bd = backdrop + lane * pitch;
    for (int q = 0; q < segs; ++q) {
      const uint4 g4 = reinterpret_cast<const uint4*>(grid + lane * pitch)[q];
      const uint4 b4 = reinterpret_cast<const uint4*>(bd)[q];
      const uint32_t gw[4] = {g4.x, g4.y, g4.z, g4.w}, bw[4] = {b4.x, b4.y, b4.z, b4.w};
      uint32_t out[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t obj = gw[j] & 0x7f7f7f7fu;
        const uint32_t has = __vcmpne4(obj, 0u);   // 0xff in every byte holding an object
        out[j] = (obj & has) | (bw[j] & ~has);
      }
      const int c0 = q << 4;
      if (visible(pl) && pl.row == lane && pl.col >= c0 && pl.col < c0 + 16) {
        const int k = pl.col - c0;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if ((k >> 2) == j)
            out[j] = (out[j] & ~(0xffu << (8 * (k & 3)))) | ((uint32_t)p.sprite_char[0] << (8 * (k & 3)));
      }
      reinterpret_cast<uint4*>(board)[q] = make_uint4(out[0], out[1], out[2], out[3]);
    }
  }
}

int check_spec(const pcl_spec& s) {
  if (!chars_are(s.sprite_char, s.n_sprites, ".") || s.n_drapes != 0) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.z_order, 1, ".")) return PCL_ERR_UNSUPPORTED;
  const int lens[1] = {1};
  if (!groups_are(s, ".", lens, 1)) return PCL_ERR_UNSUPPORTED;
  if (!set_is(s.impassable[0], "#") || !s.sprite_confined[0] || s.sprite_egocentric[0])
    return PCL_ERR_UNSUPPORTED;
  // one lane per board row, and rows of at most 32 grid bytes
  if (s.rows > kMaxSide || s.pitch > kMaxSide) return PCL_ERR_UNSUPPORTED;
  if (s.rows < 3 || s.cols < 3) return PCL_ERR_INVALID;       // a walled board has an inside
  if (s.bits_words * 4 != s.pitch) return PCL_ERR_INVALID;    // the grid is u8 [rows, pitch]
  if (s.program_arg[0] < 0) return PCL_ERR_INVALID;           // max_num_steps
  return PCL_OK;
}

int check_state(const pcl_spec& s, const pcl_state& st) {
  if (!st.d_bits[0] || !st.d_bits_init[0]) return PCL_ERR_INVALID;
  if (st.bits_bstride[0] < (int64_t)s.rows * s.bits_words) return PCL_ERR_INVALID;
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  return launch_step(box_world_step, p, kWarpsPerBlock, 0, s);
}

}  // namespace

const Program kBoxWorld = {check_spec, check_state, nullptr, launch, nullptr,
                           /*float_reward=*/false, /*crop_epilogue=*/false,
                           /*scroll_groups=*/false};

}  // namespace pcl
