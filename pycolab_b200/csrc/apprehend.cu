// apprehend.cu — fused step kernel for examples/apprehend.py:56-131 (SURVEY.md §8f-4).
//
// Two MazeWalkers over an empty backdrop, one update group ['b', 'P'], z-order 'bP'
// (ascii_art.py:184: the flat update schedule), neither has impassable characters, so no
// entity reads the board and a step is register arithmetic + the final render:
//   ball 'b' (sprite 1, not confined): _south every frame — frame 0 included, its
//     update() ignores `actions` — then x_accumulator += dx; below -0.5: _west and += 1.0,
//     above 0.5: _east and -= 1.0; virtual row >= H: reward -1 + terminate  (:109-131)
//   player 'P' (sprite 0, confined to the board): action 0 = _west, 1 = _east; on the
//     ball's virtual position: reward +1 + terminate                           (:76-87)
// The ball's slope dx = random.uniform(-2.499, 2.499) / (H - 1.0) is a float64 drawn from
// PYTHON's `random` when the sprite is built (:103), i.e. once per episode: with a per-env
// MT19937 state bound (pcl_state.d_rng, the words of random.Random(seed).getstate()) the
// kernel draws it at every (re)start exactly as random.uniform does — a + (b - a) *
// random(), random() = genrand_res53 — with correctly-rounded f64 operations only (no FMA
// contraction); without one (the single-env facade, whose Python sprite has already drawn)
// dx comes from the reset template.  dx lives in the ball's AUX0/AUX1 (f64 bits lo/hi), the
// accumulator in the plot's AUX0/AUX1.  One warp per env.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"
#include "pcl_mt.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 4;

__device__ __forceinline__ double f64_of(int lo, int hi) {
  return __hiloint2double(hi, lo);
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
apprehend_step(const StepParams p) {
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;
  const int H = p.H, W = p.W, pitch = p.pitch;
  int32_t* g_sprites = p.st.d_sprites + (int64_t)env * 2 * PCL_SPRITE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;

  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) return;
  const bool restart = run == ENV_RESTART;
  const int32_t* src_s = restart ? p.st.d_sprites_init + lvl * p.st.sprites_init_bstride : g_sprites;
  const int32_t* src_p = restart ? p.st.d_plot_init + lvl * p.st.plot_init_bstride : g_plot;
  Sprite pl = load_sprite(src_s), ball = load_sprite(src_s + PCL_SPRITE_WORDS);
  pl.aux0 = pl.aux1 = pl.aux2 = 0;                                    // stored as zeros
  ball.aux2 = 0;
  const PlotCarry carry = plot_carry(g_plot, restart);
  Plot plot = step_plot(src_p, carry.error);
  double dx = f64_of(ball.aux0, ball.aux1);
  double acc = f64_of(src_p[PCL_P_AUX0], src_p[PCL_P_AUX1]);
  if (restart && p.st.d_rng != nullptr) {                             // BallSprite.__init__ :103
    uint32_t* mt = reinterpret_cast<uint32_t*>(p.st.d_rng) + (int64_t)env * PCL_MT_WORDS;
    const double r53 = mt_random53(mt, lane);
    const double u = __dadd_rn(-2.499, __dmul_rn(__dsub_rn(2.499, -2.499), r53));   // random.uniform
    dx = __ddiv_rn(u, __dsub_rn((double)H, 1.0));
    acc = 0.0;                                                         // :107
  }
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  Directives dir = fresh_directives();
  auto never_blocked = [](int, int) { return false; };

  // ---- BallSprite.update (:109-131), first in the group
  walker_move(ball, 1, PCL_M_S, plot, H, W, false, false, lane, never_blocked);
  acc = __dadd_rn(acc, dx);
  if (acc < -0.5) {
    walker_move(ball, 1, PCL_M_W, plot, H, W, false, false, lane, never_blocked);
    acc = __dadd_rn(acc, 1.0);
  } else if (acc > 0.5) {
    walker_move(ball, 1, PCL_M_E, plot, H, W, false, false, lane, never_blocked);
    acc = __dsub_rn(acc, 1.0);
  }
  if (ball.vrow >= H) { add_reward(dir, -1); terminate(dir); }
  // ---- PlayerSprite.update (:76-87)
  if (action == 0) walker_move(pl, 0, PCL_M_W, plot, H, W, true, false, lane, never_blocked);
  else if (action == 1) walker_move(pl, 0, PCL_M_E, plot, H, W, true, false, lane, never_blocked);
  if (pl.vrow == ball.vrow && pl.vcol == ball.vcol) { add_reward(dir, 1); terminate(dir); }

  __syncwarp();
  if (lane == 0) {
    ball.aux0 = __double2loint(dx); ball.aux1 = __double2hiint(dx);
    store_sprite(g_sprites, pl);
    store_sprite(g_sprites + PCL_SPRITE_WORDS, ball);
    store_carry(g_plot, carry);
    store_plot<ORDER_CLEAR>(g_plot, plot, dir);
    g_plot[PCL_P_AUX0] = __double2loint(acc); g_plot[PCL_P_AUX1] = __double2hiint(acc);
    store_outputs(p.out, env, dir);
  }

  // ---- render (engine.py:737-759): backdrop, 'b', then 'P' on top
  uint8_t* board = p.out.d_board + (int64_t)env * H * pitch;
  const int segs_per_row = pitch >> 4;
  const int total = H * segs_per_row;
  for (int seg = lane; seg < total; seg += 32) {
    const int r = seg / segs_per_row;
    const int c0 = (seg - r * segs_per_row) << 4;
    uint4 px = *reinterpret_cast<const uint4*>(backdrop + r * pitch + c0);
    unsigned m = sprite_bit(ball, r, c0);
    if (m) paint_bits(px, m, p.sprite_char[1]);
    m = sprite_bit(pl, r, c0);
    if (m) paint_bits(px, m, p.sprite_char[0]);
    *reinterpret_cast<uint4*>(board + r * pitch + c0) = px;
  }
}

int check_spec(const pcl_spec& s) {
  if (s.n_sprites != 2 || s.n_drapes != 0) return PCL_ERR_UNSUPPORTED;
  // one update group: the ball, then the catcher; the catcher is drawn on top
  if (s.n_groups != 1 || s.group_len[0] != 2 || s.group_chars[0] != s.sprite_char[1] ||
      s.group_chars[1] != s.sprite_char[0]) return PCL_ERR_UNSUPPORTED;
  if (s.z_order[0] != s.sprite_char[1] || s.z_order[1] != s.sprite_char[0]) return PCL_ERR_UNSUPPORTED;
  if (!s.sprite_confined[0] || s.sprite_confined[1]) return PCL_ERR_UNSUPPORTED;
  for (int i = 0; i < 2; ++i) {
    if (s.sprite_egocentric[i]) return PCL_ERR_UNSUPPORTED;
    for (int w = 0; w < 4; ++w) if (s.impassable[i][w]) return PCL_ERR_UNSUPPORTED;
  }
  if (s.rows < 2) return PCL_ERR_INVALID;          // the slope divides by rows - 1
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  return launch_step(apprehend_step, p, kWarpsPerBlock, 0, s);
}

}  // namespace

const Program kApprehend = {check_spec, nullptr, nullptr, launch, nullptr,
                            /*float_reward=*/false, /*crop_epilogue=*/false,
                            /*scroll_groups=*/false};

}  // namespace pcl
