// hello.cu — fused step kernel for examples/hello_world.py:58-118 (SURVEY.md §8f-4).
//
// Plain Sprites (things.Sprite, not MazeWalkers) sliding diagonally with
// wrap-around and one Drape whose curtain is np.roll'ed one cell per action.  No
// entity reads the board, so a step is pure register arithmetic + the final render:
//   sprite s (aux0 = its direction set k): action a in 0..3 moves it by
//     (dy, dx) = (DY[k][a], DX[k][a]) modulo the board           (hello_world.py:113-118)
//   drape: the rolled curtain is the reset curtain shifted by (AUX0, AUX1) cells
//     along rows / columns, modulo H / W; +1 reward per roll, action 4 terminates (:77-87)
// The static curtain (d_bits_init, per level) is never copied: cell (r, c) of the
// live curtain is cell ((r - AUX0) mod H, (c - AUX1) mod W) of it.
// One warp per env; z-order comes from the spec ('12@34' upstream).
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 4;

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
hello_step(const StepParams p) {
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;
  const int H = p.H, W = p.W, pitch = p.pitch, S = p.S, BW = p.BW;
  int32_t* g_sprites = p.st.d_sprites + (int64_t)env * S * PCL_SPRITE_WORDS;
  int32_t* g_drape = p.st.d_drapes + (int64_t)env * PCL_DRAPE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;
  const uint32_t* base = p.st.d_bits_init[0] + lvl * p.st.bits_init_bstride[0];

  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) return;
  const bool restart = run == ENV_RESTART;
  const int32_t* src_s = restart ? p.st.d_sprites_init + lvl * p.st.sprites_init_bstride : g_sprites;
  const int32_t* src_d = restart ? p.st.d_drapes_init + lvl * p.st.drapes_init_bstride : g_drape;
  const int32_t* src_p = restart ? p.st.d_plot_init + lvl * p.st.plot_init_bstride : g_plot;
  // lane s < S owns sprite s; every lane knows the drape's roll counters
  Sprite sp = {};
  if (lane < S) sp = load_sprite(src_s + lane * PCL_SPRITE_WORDS);
  const int kset = sp.aux0;
  int roll_r = src_d[PCL_D_AUX0], roll_c = src_d[PCL_D_AUX1];
  const PlotCarry carry = plot_carry(g_plot, restart);
  const Plot plot = step_plot(src_p, carry.error);
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  Directives dir = fresh_directives();

  if (action >= 0 && action <= 3) {                                   // SlidingSprite.update
    if (lane < S) {
      // _DX / _DY (hello_world.py:96-97): sets 0,1 share DX, sets 2,3 negate it;
      // DY of set 0 = (-1, 1, 1, -1), set 1 and 2 negate it, set 3 equals set 0.
      const int dx0 = (action & 1) ? 1 : -1;
      const int dy0 = (action == 1 || action == 2) ? 1 : -1;
      const int dx = (kset >= 2) ? -dx0 : dx0;
      const int dy = (kset == 1 || kset == 2) ? -dy0 : dy0;
      sp.col = (sp.col + dx + W) % W;
      sp.row = (sp.row + dy + H) % H;
    }
    // RollingDrape.update: axes (0, 0, 1, 1), shifts (-1, 1, -1, 1)
    if (action < 2) roll_r = (roll_r + (action == 0 ? H - 1 : 1)) % H;
    else roll_c = (roll_c + (action == 2 ? W - 1 : 1)) % W;
    add_reward(dir, 1);
  } else if (action == 4) {
    terminate(dir);
  }

  __syncwarp();
  if (lane < S) {                                   // a plain Sprite: virtual = true position
    sp.vrow = sp.row; sp.vcol = sp.col;
    store_sprite(g_sprites + lane * PCL_SPRITE_WORDS, sp, PCL_S_AUX1);
  }
  if (lane == 0) {
    g_drape[PCL_D_AUX0] = roll_r; g_drape[PCL_D_AUX1] = roll_c;
    g_drape[PCL_D_LAST_FRAME] = src_d[PCL_D_LAST_FRAME];
    store_carry(g_plot, carry);
    store_plot<ORDER_CLEAR>(g_plot, plot, dir);
    store_outputs(p.out, env, dir);
  }

  // ---- render (engine.py:737-759): backdrop, then the z-order back to front.
  // Every lane learns all sprite cells first (S <= 4), then paints whole cells.
  int s_row[4], s_col[4], s_vis[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    s_row[k] = __shfl_sync(PCL_FULL, sp.row, k);
    s_col[k] = __shfl_sync(PCL_FULL, sp.col, k);
    s_vis[k] = k < S ? (__shfl_sync(PCL_FULL, sp.flags, k) & 1) : 0;
  }
  const int n = S + 1;
  uint8_t* board = p.out.d_board + (int64_t)env * H * pitch;
  for (int cell = lane; cell < H * pitch; cell += 32) {
    const int r = cell / pitch, c = cell - r * pitch;
    int code = 0;                                        // pitch padding stays 0
    if (c < W) {
      code = backdrop[r * pitch + c];
      for (int k = 0; k < n; ++k) {
        const int ch = p.program_arg[k];                 // z-order, back to front
        if (ch == p.drape_char[0]) {
          int sr = r - roll_r, sc = c - roll_c;
          if (sr < 0) sr += H;
          if (sc < 0) sc += W;
          if (bit_at(base + (int64_t)sr * BW, sc)) code = ch;
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (ch == p.sprite_char[q] && s_vis[q] && s_row[q] == r && s_col[q] == c) code = ch;
        }
      }
    }
    board[cell] = (uint8_t)code;
  }
}

int check_spec(const pcl_spec& s) {
  if (s.n_sprites < 1 || s.n_sprites > 4 || s.n_drapes != 1) return PCL_ERR_UNSUPPORTED;
  if (s.n_groups != 1 || s.group_len[0] != s.n_sprites + 1) return PCL_ERR_UNSUPPORTED;
  if (!bit_rows_fit(s)) return PCL_ERR_INVALID;
  for (int k = 0; k < s.n_sprites + 1; ++k)      // program_arg = the z-order
    if (s.program_arg[k] != s.z_order[k]) return PCL_ERR_INVALID;
  return PCL_OK;
}

int check_state(const pcl_spec&, const pcl_state& st) {
  return st.d_bits_init[0] ? PCL_OK : PCL_ERR_INVALID;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  return launch_step(hello_step, p, kWarpsPerBlock, 0, s);
}

}  // namespace

// The drape's curtain is held implicitly (the reset curtain rolled by AUX0 / AUX1).
const Program kHello = {check_spec, check_state, nullptr, launch, nullptr,
                        /*float_reward=*/false, /*crop_epilogue=*/false,
                        /*scroll_groups=*/false};

}  // namespace pcl
