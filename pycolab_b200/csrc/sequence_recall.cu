// sequence_recall.cu — fused step kernel for examples/research/lp-rnn/sequence_recall.py:107-317.
//
// MazeWalker 'P' (impassable '#', confined), the mask drape 'M' over the four light pads
// '1'-'4' of the backdrop and the start-box drape '%'; one update group P M %, z-order MP%.
// One warp per env: the state machine is warp-uniform scalar code, lane r paints row r.
//
// the_plot['program'] is always the list _make_program built, less the states already
// popped, so the device keeps a program counter over its fixed shape (plot AUX0): for a
// sequence of L lights, pc 2k / 2k+1 (k < L) are (OFF, off frames) / (ON, on frames, light
// k), pc 2L is (OFF, max(1, pause_frames)), pc 2L+1+2k / 2L+2+2k are (SEEK, light k) /
// (EXIT,), and pc 4L is the QUIT that replaced the last EXIT.  Plot AUX1 = frames_in_state,
// AUX2 = timeout_frames (PCL_SEQUENCE_RECALL_NO_TIMEOUT = inf), AUX3 = the sequence, light
// k in bits 2k..2k+1 as 0-3 for '1'-'4'.
//
// What the reference does that a straight restatement could get wrong:
//   * OFF and ON test `frames_in_state == 1` before `>= duration` (:234-245), so a state of
//     duration 1 or 2 lasts two frames.
//   * '%' clears when, after M's update, frames_in_state == 1 and the state is SEEK (:268-271):
//     a SEEK that M leaves in its first frame does not clear it.
//   * Rewards are float64 sums in update order: P's -0.005 (frames after the first), then a
//     SEEK's 1.0 or 0.0 (:251-253, :316).
//   * M's `curtain -= mask` is NumPy-1 boolean subtraction; every time it runs the light is
//     covered (an OFF or a left pad covered every light before), so it is and-not here.
// M's curtain is a 4-bit covered set (drape record AUX0) over the level's static light planes
// (the backdrop); its bit rows in d_bits[0] are rewritten only when the set changes, for the
// curtain export.  '%' is its art mask (d_bits_init[1]) and a cleared bit (record AUX0).
// At every (re)start with d_rng bound, the sequence is redrawn as sequence_length calls to
// random.choice('1234'), i.e. _randbelow(4) (:165).
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"
#include "pcl_mt.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 4;
enum { DM = 0, DPCT = 1 };
enum { kOff, kOn, kSeek, kExit, kQuit };

__global__ void __launch_bounds__(kWarpsPerBlock * 32, 4)
sequence_recall_step(const StepParams p) {
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;
  const int H = p.H, W = p.W, BW = p.BW, pitch = p.pitch;
  int32_t* g_sprite = p.st.d_sprites + (int64_t)env * PCL_SPRITE_WORDS;
  int32_t* g_drapes = p.st.d_drapes + (int64_t)env * 2 * PCL_DRAPE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;

  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) return;
  const bool restart = run == ENV_RESTART;
  const int32_t* src_s = restart ? p.st.d_sprites_init + lvl * p.st.sprites_init_bstride : g_sprite;
  const int32_t* src_d = restart ? p.st.d_drapes_init + lvl * p.st.drapes_init_bstride : g_drapes;
  const int32_t* src_p = restart ? p.st.d_plot_init + lvl * p.st.plot_init_bstride : g_plot;

  Sprite pl = load_sprite(src_s);
  pl.aux0 = pl.aux1 = pl.aux2 = 0;                                    // stored as zeros
  const int covered0 = src_d[PCL_D_AUX0];
  int covered = covered0;
  int cleared = src_d[PCL_DRAPE_WORDS + PCL_D_AUX0];
  const PlotCarry carry = plot_carry(g_plot, restart);
  Plot plot = step_plot(src_p, carry.error);
  int pc = src_p[PCL_P_AUX0], fis = src_p[PCL_P_AUX1], timeout = src_p[PCL_P_AUX2];
  uint32_t seq = (uint32_t)src_p[PCL_P_AUX3];
  const int L = p.program_arg[0];
  if (restart && p.st.d_rng != nullptr) {         // _make_program :165
    uint32_t* mt = reinterpret_cast<uint32_t*>(p.st.d_rng) + (int64_t)env * PCL_MT_WORDS;
    seq = 0;
#pragma unroll 1
    for (int k = 0; k < L; ++k) seq |= (uint32_t)mt_draw(mt, kMtPythonBelow, 4, lane) << (2 * k);
  }
  // The state at pc, its duration and its light (0-3).
  auto state_of = [&](int at, int& arg, int& light) {
    light = 0; arg = 0;
    if (at < 2 * L) {
      light = (seq >> (at & ~1)) & 3u;
      arg = (at & 1) ? p.program_arg[1] : p.program_arg[2];
      return (at & 1) ? (int)kOn : (int)kOff;
    }
    if (at == 2 * L) { arg = p.program_arg[3]; return (int)kOff; }
    if (at >= 4 * L) return (int)kQuit;
    const int k = at - 2 * L - 1;
    light = (seq >> (k & ~1)) & 3u;
    return (k & 1) ? (int)kExit : (int)kSeek;
  };
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  Directives dir = fresh_directives();
  double reward = 0.0;
  auto pay = [&](double r) {                       // plot.py:201-214, a float sum
    reward = dir.has_reward ? __dadd_rn(reward, r) : r;
    dir.has_reward = 1;
  };
  const int f = plot.frame;
  int arg, light;
  int state = state_of(pc, arg, light);

  // ---- PlayerSprite.update (:288-317) against the last board: '#' is only ever the backdrop's
  if (action == 0 || action == 6) {
    timeout = 1;
  } else if ((state == kSeek || state == kExit) && action >= 1 && action <= 4) {
    const int motion = action == 1 ? PCL_M_N : action == 2 ? PCL_M_S : action == 3 ? PCL_M_W
                                                                                  : PCL_M_E;
    walker_move(pl, 0, motion, plot, H, W, true, false, lane,
                [&](int r, int c) { return backdrop[r * pitch + c] == '#'; });
  }
  if (timeout <= 0) {
    terminate(dir);
  } else {
    if (f > 1) pay(-0.005);
    if (timeout != PCL_SEQUENCE_RECALL_NO_TIMEOUT) timeout -= 1;
  }

  // ---- MaskDrape.update (:213-262)
  fis += 1;
  const int above = backdrop[pl.row * pitch + pl.col];
  if (state == kQuit) {
    if (fis == 1) timeout = 1;
  } else if (state == kOff || state == kOn) {
    if (fis == 1) covered = state == kOff ? 0xf : covered & ~(1 << light);
    else if (fis >= arg) { ++pc; fis = 0; }
  } else if (state == kSeek) {
    if (above != ' ') {
      covered &= ~(1 << (above - '1'));
      pay(above - '1' == light ? 1.0 : 0.0);
      ++pc; fis = 0;
    }
  } else if (above == ' ') {                       // EXIT
    covered = 0xf;
    ++pc; fis = 0;
  }
  state = state_of(pc, arg, light);

  // ---- WaitForSeekDrape.update (:268-271)
  const bool clear_now = !cleared && fis == 1 && state == kSeek;
  if (clear_now) cleared = 1;

  // ---- curtains: M's bit rows when its set changed, '%' at a restart and when it clears
  if (lane < H && (restart || covered != covered0 || clear_now)) {
    const uint32_t* pct_init = p.st.d_bits_init[DPCT] + lvl * p.st.bits_init_bstride[DPCT] + lane * BW;
    uint32_t* m_live = p.st.d_bits[DM] + (int64_t)env * p.st.bits_bstride[DM] + lane * BW;
    uint32_t* pct_live = p.st.d_bits[DPCT] + (int64_t)env * p.st.bits_bstride[DPCT] + lane * BW;
    for (int w = 0; w < BW; ++w) {
      uint32_t bits = 0;
      for (int c = 32 * w; c < min(32 * w + 32, W); ++c) {
        const int ch = backdrop[lane * pitch + c] - '1';
        if (ch >= 0 && ch < 4 && ((covered >> ch) & 1)) bits |= 1u << (c & 31);
      }
      m_live[w] = bits;
      pct_live[w] = cleared ? 0u : pct_init[w];
    }
  }

  if (lane == 0) {
    store_sprite(g_sprite, pl);
    const int32_t* init_d = p.st.d_drapes_init + lvl * p.st.drapes_init_bstride;
#pragma unroll
    for (int d = 0; d < 2; ++d) {
      int32_t* r = g_drapes + d * PCL_DRAPE_WORDS;
      const int32_t* r0 = init_d + d * PCL_DRAPE_WORDS;
      for (int w = 0; w < PCL_DRAPE_WORDS; ++w) r[w] = r0[w];
      r[PCL_D_AUX0] = d == DM ? covered : cleared;
    }
    store_carry(g_plot, carry);
    store_plot<ORDER_CLEAR>(g_plot, plot, dir);
    g_plot[PCL_P_AUX0] = pc; g_plot[PCL_P_AUX1] = fis;
    g_plot[PCL_P_AUX2] = timeout; g_plot[PCL_P_AUX3] = (int)seq;
    store_outputs(p.out, env, dir, dir.has_reward ? reward : 0.0);
  }

  // ---- render (engine.py:737-759): backdrop, M over the covered lights, P, '%'
  if (lane < H) {
    const uint32_t* pct = p.st.d_bits_init[DPCT] + lvl * p.st.bits_init_bstride[DPCT] + lane * BW;
    const uint8_t* brow = backdrop + lane * pitch;
    uint8_t* board = p.out.d_board + (int64_t)env * H * pitch + lane * pitch;
    for (int c0 = 0; c0 < pitch; c0 += 16) {
      uint4 px = *reinterpret_cast<const uint4*>(brow + c0);
      unsigned m = 0;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int ch = brow[c0 + j] - '1';
        if (ch >= 0 && ch < 4 && ((covered >> ch) & 1)) m |= 1u << j;
      }
      if (m) paint_bits(px, m, p.drape_char[DM]);
      m = sprite_bit(pl, lane, c0);
      if (m) paint_bits(px, m, p.sprite_char[0]);
      m = cleared || c0 >= W ? 0u : bits16(pct, c0);
      if (m) paint_bits(px, m, p.drape_char[DPCT]);
      *reinterpret_cast<uint4*>(board + c0) = px;
    }
  }
}

int check_spec(const pcl_spec& s) {
  if (!chars_are(s.sprite_char, s.n_sprites, "P")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.drape_char, s.n_drapes, "M%")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.z_order, 3, "MP%")) return PCL_ERR_UNSUPPORTED;
  const int lens[1] = {3};
  if (!groups_are(s, "PM%", lens, 1)) return PCL_ERR_UNSUPPORTED;
  if (!set_is(s.impassable[0], "#") || !s.sprite_confined[0] || s.sprite_egocentric[0])
    return PCL_ERR_UNSUPPORTED;
  // one board row per lane
  if (s.rows > 32 || s.cols > 64) return PCL_ERR_UNSUPPORTED;
  if (!bit_rows_fit(s)) return PCL_ERR_INVALID;
  // the sequence is one 32-bit plot word, two bits per light
  if (s.program_arg[0] < 1 || s.program_arg[0] > 16) return PCL_ERR_UNSUPPORTED;
  if (s.program_arg[3] < 1) return PCL_ERR_INVALID;          // max(1, pause_frames)
  return PCL_OK;
}

int check_state(const pcl_spec&, const pcl_state& st) {
  for (int d = 0; d < 2; ++d)
    if (!st.d_bits[d] || !st.d_bits_init[d] || st.bits_bstride[d] == 0) return PCL_ERR_INVALID;
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  return launch_step(sequence_recall_step, p, kWarpsPerBlock, 0, s);
}

}  // namespace

const Program kSequenceRecall = {check_spec, check_state, curtain_bits, launch, nullptr,
                                 /*float_reward=*/true, /*crop_epilogue=*/false,
                                 /*scroll_groups=*/false};

}  // namespace pcl
