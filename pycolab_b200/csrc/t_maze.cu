// t_maze.cu — fused step kernel for examples/research/lp-rnn/t_maze.py:180-505.
//
// One egocentric MazeWalker 'P' (impassable '#') on a 7 x 11 board, a plain cue drape 'Q'
// and five PseudoTeleportingScrollys with margins None over one world pattern: walls '#',
// speckle '*', goals 'l' / 'r' and the teleporter 't'.  Update groups [Q # *] [P] [l t r],
// z-order *#ltrQP (back to front).  One warp per env; game logic is warp-uniform scalar
// code, the lanes split up for the walker's neighbourhood, the paint and the speckle draw.
//
// What the reference does that a straight restatement could get wrong:
//   * Teleporting is np.roll of every Scrolly's OWN pattern at the start of its own update
//     in the frame an order names (:315-320).  Each Scrolly keeps its cumulative roll
//     (record AUX0 = rows << 16 | cols): '#' and '*' roll in group 0, 'l' 't' 'r' in group 2,
//     and 'r' misses a roll when 't' places the next order in the very frame the last one
//     is obeyed (limbo_time 2, or a second teleport) — reproduced, not repaired.
//   * The walker's legality check and permits read the board rendered after group 0
//     (engine.py:725-735): '#' and '*' already scrolled and rolled, 'l' 't' 'r' still at
//     their old corners and rolls, 'Q' (after its update) drawn above '#', 'P' at its old
//     cell.
//   * Rewards are float64: Q pays -0.001 when frame > 1 (:282-283), a goal later in the same
//     frame adds +-1.0 (:489-492), so the step's reward is __dadd_rn(-0.001, +-1.0).  They go
//     to pcl_outputs.d_reward_f64; Directives carries only has_reward / discount / done.
//   * A goal sets timeout_frames = frame + 1: the episode ends in Q at the NEXT frame with no
//     reward (:280-281); quitting (actions 0 / 6) does the same (:244-245).
//   * With cue_after_teleport False, Q deletes yo_we_have_teleported on the frame after a
//     teleport (:273-275); from then on the teleporter tests the player every frame again.
//   * The teleporter is empty for teleport_delay updates, its_showtime's included, then the
//     saved (never rolled: a teleport needs a visible teleporter) pattern is back (:397-428).
// At every (re)start with d_rng bound, the cue side is random.random() < 0.5 from slot 0
// (Python's `random`, :262) and the speckle is np.random.rand(PH, PW) < 0.4 from slot 1
// (NumPy's RandomState, :365), drawn warp-parallel: the generator is staged in shared memory,
// each twist is followed by lanes tempering word pairs side by side and balloting the
// "clear" bits into a per-warp bit stream in C order, from which the env's '*' pattern is
// written word by word.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"
#include "pcl_mt.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 4;
enum { DQ = 0, DWALL = 1, DDIRT = 2, DLEFT = 3, DTELE = 4, DRIGHT = 5, ND = 6 };
constexpr int kLimboRow = 4, kLimboCol = 140, kLimboDx = -46;   // TeleporterDrape :408-415
// The speckle redraw writes a per-warp bit stream of this many words (one bit per pattern
// cell); check_spec refuses larger patterns.
constexpr int kMaxStreamWords = 480;

struct WarpScratch {
  uint32_t mt[PCL_MT_WORDS + 3];
  uint32_t stream[kMaxStreamWords + 2];
};

__device__ __forceinline__ uint32_t temper(uint32_t y) {
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}
// random_sample() < 0.4 for the double made of outputs a, b (NumPy's legacy random_sample and
// Python's genrand_res53 are both (a >> 5) * 2^26 + (b >> 6) scaled by 2^-53, exactly): the
// double 0.4 is 3602879701896397 * 2^-53, so the test is one integer compare.
__device__ __forceinline__ bool below_0_4(uint32_t a, uint32_t b) {
  const uint64_t n = ((uint64_t)(a >> 5) << 26) | (uint64_t)(b >> 6);
  return n < 3602879701896397ull;
}

// Cell (r, c) of a pattern rolled by `roll` (np.roll by -rows, -cols: cell (r, c) shows base
// cell (r + rows, c + cols), wrapped).  0 <= r < PH, 0 <= c < PW.
__device__ __forceinline__ bool rolled_bit(const uint32_t* base, int PWW, int PH, int PW, int roll,
                                           int r, int c) {
  int rr = r + (roll >> 16);
  if (rr >= PH) rr -= PH;
  int cc = c + (roll & 0xffff);
  if (cc >= PW) cc -= PW;
  return (base[rr * PWW + (cc >> 5)] >> (cc & 31)) & 1u;
}
__device__ __forceinline__ int roll_by(int roll, int rows, int cols, int PH, int PW) {
  int r = ((roll >> 16) + rows) % PH;
  if (r < 0) r += PH;
  int c = ((roll & 0xffff) + cols) % PW;
  if (c < 0) c += PW;
  return (r << 16) | c;
}

// np.random.rand(PH, PW) < 0.4 from the staged generator: bit k of `stream` is set when draw
// k (C order) is below 0.4.  Consumes exactly 2 * PH * PW outputs.
__device__ void speckle_stream(uint32_t* mt, uint32_t* stream, int total, int lane) {
  int pos = (int)mt[624];
  int d = 0;
  uint32_t carry = 0;
  bool have_carry = false;
  while (d < total) {
    if (pos >= 624) { mt_twist(mt, lane); pos = 0; }
    if (have_carry) {                                 // a pair split by the twist
      if (lane == 0 && below_0_4(carry, temper(mt[0]))) stream[d >> 5] |= 1u << (d & 31);
      __syncwarp();
      ++d; pos = 1; have_carry = false;
      continue;
    }
    const int npairs = min((624 - pos) >> 1, total - d);
    for (int base = 0; base < npairs; base += 32) {
      const int i = base + lane;
      bool clear = false;
      if (i < npairs) clear = below_0_4(temper(mt[pos + 2 * i]), temper(mt[pos + 2 * i + 1]));
      const unsigned m = __ballot_sync(PCL_FULL, clear);
      if (lane == 0 && m) {
        const int c0 = d + base, w = c0 >> 5, sh = c0 & 31;
        stream[w] |= m << sh;
        if (sh) stream[w + 1] |= m >> (32 - sh);
      }
    }
    __syncwarp();
    d += npairs; pos += 2 * npairs;
    if (d < total && pos == 623) { carry = temper(mt[623]); have_carry = true; pos = 624; }
  }
  __syncwarp();
  if (lane == 0) mt[624] = (uint32_t)pos;
  __syncwarp();
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
t_maze_step(const StepParams p) {
  __shared__ WarpScratch scratch[kWarpsPerBlock];
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;
  const int H = p.H, W = p.W, PH = p.PH, PW = p.PW, PWW = p.PWW, BW = p.BW;
  int32_t* g_sprite = p.st.d_sprites + (int64_t)env * PCL_SPRITE_WORDS;
  int32_t* g_drapes = p.st.d_drapes + (int64_t)env * ND * PCL_DRAPE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;

  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) return;
  const bool restart = run == ENV_RESTART;
  const int32_t* src_s = restart ? p.st.d_sprites_init + lvl * p.st.sprites_init_bstride : g_sprite;
  const int32_t* src_d = restart ? p.st.d_drapes_init + lvl * p.st.drapes_init_bstride : g_drapes;
  const int32_t* src_p = restart ? p.st.d_plot_init + lvl * p.st.plot_init_bstride : g_plot;

  Sprite pl[1] = {load_sprite(src_s)};
  pl[0].aux2 = 0;                                                     // stored as zero
  Drape dr[ND];
#pragma unroll
  for (int d = 0; d < ND; ++d) dr[d] = load_drape(src_d + d * PCL_DRAPE_WORDS);
  const PlotCarry carry = plot_carry(g_plot, restart);
  Plot plot = step_plot</*kOrder=*/true>(src_p, carry.error);
  int timeout = src_p[PCL_P_AUX0];                 // the_plot['timeout_frames']
  int tele_frame = src_p[PCL_P_AUX1];              // the_plot.get('teleportation_order_frame', -1)
  int tele_r = src_p[PCL_P_AUX2], tele_c = src_p[PCL_P_AUX3];   // the_plot['teleportation_order']

  const uint32_t* pattern[ND];
#pragma unroll
  for (int d = 1; d < ND; ++d)
    pattern[d] = p.st.d_pattern[d] + (d == DDIRT ? (int64_t)env : lvl) * p.st.pattern_bstride[d];
  uint32_t* dirt = p.st.d_pattern[DDIRT] + (int64_t)env * p.st.pattern_bstride[DDIRT];
  uint32_t* q_bits = p.st.d_bits[DQ] + (int64_t)env * p.st.bits_bstride[DQ];

  // ---- (re)start: the constructors' draws (CueDrape :262-266, SpeckleDrape :365)
  int which_goal = dr[DQ].aux0;                    // 0 'left', 1 'right'
  if (restart) {
    const bool draw = p.st.d_rng != nullptr;
    uint32_t* g_mt = p.st.d_rng + (int64_t)env * 2 * PCL_MT_WORDS;
    if (draw) which_goal = mt_random53(g_mt, lane) < 0.5 ? 0 : 1;
    // 'left' blanks columns 6 and up, 'right' columns 0-5 (:263-266)
    const uint32_t keep = which_goal == 0 ? 0x3fu : ~0x3fu;
    const uint32_t* q_init = p.st.d_bits_init[DQ] + lvl * p.st.bits_init_bstride[DQ];
    for (int i = lane; i < H * BW; i += 32) q_bits[i] = (i % BW == 0) ? (q_init[i] & keep) : 0u;
    uint32_t* stream = scratch[threadIdx.x >> 5].stream;
    const int total = PH * PW;
    if (draw) {
      uint32_t* mt = scratch[threadIdx.x >> 5].mt;
      const uint32_t* g_mt1 = g_mt + PCL_MT_WORDS;
      for (int i = lane; i < PCL_MT_WORDS; i += 32) mt[i] = g_mt1[i];
      for (int i = lane; i < (total >> 5) + 2; i += 32) stream[i] = 0u;
      __syncwarp();
      speckle_stream(mt, stream, total, lane);
      for (int i = lane; i < PCL_MT_WORDS; i += 32) g_mt[PCL_MT_WORDS + i] = mt[i];
    }
    const uint32_t* dirt_init = p.st.d_pattern_init[DDIRT] + lvl * p.st.pattern_init_bstride[DDIRT];
    for (int i = lane; i < PH * PWW; i += 32) {
      const int r = i / PWW, w = i - r * PWW;
      uint32_t v = dirt_init[i];
      if (draw && 32 * w < PW) {
        const int off = r * PW + 32 * w, k = off >> 5;
        uint32_t bits = __funnelshift_r(stream[k], stream[k + 1], off & 31);
        if (32 * w + 32 > PW) bits &= (1u << (PW - 32 * w)) - 1u;
        v &= ~bits;
      }
      dirt[i] = v;
    }
    __syncwarp();
  }
  bool yo = dr[DQ].aux1 != 0, in_limbo = dr[DQ].aux2 != 0;
  int delay = dr[DTELE].aux1, countdown = dr[DTELE].aux2;

  const int f = plot.frame;
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  const int level = p.program_arg[0];
  const bool cue_after_teleport = p.program_arg[1] != 0;
  // 0 <= frame - teleportation_order_frame <= 1: everybody _stays (:232, :345 ...)
  auto staying = [&]() { const int d = f - tele_frame; return 0 <= d && d <= 1; };
  // motion of '#', '*', 'l', 'r' (:345-356): PCL_M_NONE = no motion helper called
  const int dir_motion = action == 1 ? PCL_M_N : action == 2 ? PCL_M_S : action == 3 ? PCL_M_W
                         : action == 4 ? PCL_M_E : action == 5 ? PCL_M_STAY : PCL_M_NONE;
  const ScrollyCfg cfg = scrolly_cfg(H, W, PH, PW, -1, -1);
  Directives dir = fresh_directives();
  double reward = 0.0;
  auto pay = [&](double r) {                       // plot.py:201-214, a float sum
    reward = dir.has_reward ? __dadd_rn(reward, r) : r;
    dir.has_reward = 1;
  };
  auto roll_if_ordered = [&](int d) {              // PseudoTeleportingScrolly.update :315-320
    if (tele_frame == f) dr[d].aux0 = roll_by(dr[d].aux0, tele_r, tele_c, PH, PW);
  };
  auto place_order = [&](int rows, int cols) {     // :322-331
    tele_frame = f + 1; tele_r = rows; tele_c = cols;
  };

  // ---- group 0: CueDrape (:271-283), MazeDrape, SpeckleDrape (:341-382)
  bool q_clear = false;
  if (!cue_after_teleport && yo) { yo = false; q_clear = true; }
  if (f >= timeout) terminate(dir);
  else if (f > 1) pay(-0.001);
  const int scroll_motion = staying() ? PCL_M_STAY : dir_motion;
  roll_if_ordered(DWALL);
  if (scroll_motion != PCL_M_NONE) scrolly_move(dr[DWALL], cfg, scroll_motion, plot, pl);
  roll_if_ordered(DDIRT);
  if (scroll_motion != PCL_M_NONE) scrolly_move(dr[DDIRT], cfg, scroll_motion, plot, pl);
  if (q_clear) {
    for (int i = lane; i < H * BW; i += 32) q_bits[i] = 0u;
    __syncwarp();
  }

  // ---- group 1: PlayerSprite (:229-245) against the board rendered after group 0
  {
    const int pr0 = pl[0].row, pc0 = pl[0].col;
    const bool pvis0 = visible(pl[0]);
    auto wall_on_board = [&](int r, int c) {
      if (pvis0 && r == pr0 && c == pc0) return false;                      // 'P' on top
      if (!q_clear && ((q_bits[r * BW] >> c) & 1u)) return false;          // 'Q' above '#'
      if (rolled_bit(pattern[DRIGHT], PWW, PH, PW, dr[DRIGHT].aux0, r + dr[DRIGHT].corner_r,
                     c + dr[DRIGHT].corner_c)) return false;
      if (delay <= 0 && rolled_bit(pattern[DTELE], PWW, PH, PW, dr[DTELE].aux0,
                                   r + dr[DTELE].corner_r, c + dr[DTELE].corner_c)) return false;
      if (rolled_bit(pattern[DLEFT], PWW, PH, PW, dr[DLEFT].aux0, r + dr[DLEFT].corner_r,
                     c + dr[DLEFT].corner_c)) return false;
      return rolled_bit(pattern[DWALL], PWW, PH, PW, dr[DWALL].aux0, r + dr[DWALL].corner_r,
                        c + dr[DWALL].corner_c);
    };
    int motion = dir_motion;
    if (staying()) motion = PCL_M_STAY;
    else if (action == 0 || action == 6) timeout = f + 1;
    if (motion != PCL_M_NONE)
      walker_move(pl[0], 0, motion, plot, H, W, false, true, lane, wall_on_board);
  }

  // ---- group 2: GoalDrape 'l' (:480-505), TeleporterDrape (:419-468), GoalDrape 'r'
  auto goal = [&](int d, int name) {
    roll_if_ordered(d);
    scrolly_touch_prescroll(dr[d], plot);           // pattern_position_prescroll
    if (rolled_bit(pattern[d], PWW, PH, PW, dr[d].aux0, pl[0].row + dr[d].pre_r,
                   pl[0].col + dr[d].pre_c) && f < timeout) {
      pay(name == which_goal ? 1.0 : -1.0);
      timeout = f + 1;
    }
    const int m = staying() ? PCL_M_STAY : dir_motion;
    if (m != PCL_M_NONE) scrolly_move(dr[d], cfg, m, plot, pl);
  };
  goal(DLEFT, 0);
  {
    roll_if_ordered(DTELE);
    if (delay > 0) --delay;                         // visible once the delay is spent (:425-428)
    const int m = staying() ? PCL_M_STAY : dir_motion;
    scrolly_move(dr[DTELE], cfg, m == PCL_M_NONE ? PCL_M_STAY : m, plot, pl);
    if (!yo) {
      const int ppr = pl[0].row + dr[DTELE].corner_r, ppc = pl[0].col + dr[DTELE].corner_c;
      if (delay <= 0 && rolled_bit(pattern[DTELE], PWW, PH, PW, dr[DTELE].aux0, ppr, ppc)) {
        yo = true;
        if (countdown <= 0) {
          place_order(11 * level + 9, 0);
        } else {
          in_limbo = true;
          place_order(kLimboRow - ppr, kLimboCol - ppc);
        }
      }
    }
    if (in_limbo) {
      countdown -= 1;
      if (countdown == 0) { in_limbo = false; place_order(11 * level + 9, kLimboDx); }
    }
  }
  goal(DRIGHT, 1);

  __syncwarp();
  if (lane == 0) {
    store_sprite(g_sprite, pl[0]);
    dr[DQ].aux0 = which_goal; dr[DQ].aux1 = yo ? 1 : 0; dr[DQ].aux2 = in_limbo ? 1 : 0;
    dr[DTELE].aux1 = delay; dr[DTELE].aux2 = countdown;
#pragma unroll
    for (int d = 0; d < ND; ++d) store_drape(g_drapes + d * PCL_DRAPE_WORDS, dr[d]);
    store_carry(g_plot, carry);
    store_plot<ORDER_ALL>(g_plot, plot, dir);
    g_plot[PCL_P_AUX0] = timeout; g_plot[PCL_P_AUX1] = tele_frame;
    g_plot[PCL_P_AUX2] = tele_r; g_plot[PCL_P_AUX3] = tele_c;
    store_outputs(p.out, env, dir, dir.has_reward ? reward : 0.0);
  }

  // ---- render (engine.py:737-759): backdrop, then * # l t r Q P; lane k paints four cells
  uint8_t* board = p.out.d_board + (int64_t)env * H * 16;
  const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;
  for (int k = lane; k < H * 4; k += 32) {
    const int r = k >> 2, c0 = (k & 3) << 2;
    uint32_t word = 0;
    const uint32_t qrow = q_clear ? 0u : q_bits[r * BW];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + j;
      uint32_t ch = 0;
      if (c < W) {
        ch = backdrop[r * 16 + c];
        if (visible(pl[0]) && pl[0].row == r && pl[0].col == c) ch = p.sprite_char[0];
        else if ((qrow >> c) & 1u) ch = p.drape_char[DQ];
        else {
          const int order[5] = {DRIGHT, DTELE, DLEFT, DWALL, DDIRT};
#pragma unroll
          for (int k = 0; k < 5; ++k) {
            const int d = order[k];
            if (d == DTELE && delay > 0) continue;
            if (rolled_bit(pattern[d], PWW, PH, PW, dr[d].aux0, r + dr[d].corner_r,
                           c + dr[d].corner_c)) { ch = p.drape_char[d]; break; }
          }
        }
      }
      word |= ch << (8 * j);
    }
    reinterpret_cast<uint32_t*>(board + r * 16)[k & 3] = word;
  }
}

int check_spec(const pcl_spec& s) {
  if (!chars_are(s.sprite_char, s.n_sprites, "P")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.drape_char, s.n_drapes, "Q#*ltr")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.z_order, 7, "*#ltrQP")) return PCL_ERR_UNSUPPORTED;
  const int lens[3] = {3, 1, 3};
  if (!groups_are(s, "Q#*Pltr", lens, 3)) return PCL_ERR_UNSUPPORTED;
  if (!set_is(s.impassable[0], "#") || s.sprite_confined[0] || !s.sprite_egocentric[0])
    return PCL_ERR_UNSUPPORTED;
  for (int d = 1; d < 6; ++d) if (s.margins[d][0] >= 0) return PCL_ERR_UNSUPPORTED;
  // one board row per lane; the kernel paints 16-byte rows
  if (s.rows > 32 || s.pitch != 16) return PCL_ERR_UNSUPPORTED;
  if (s.pattern_rows < s.rows || s.pattern_cols < s.cols || s.pattern_rows >= 32768 ||
      s.pattern_cols >= 32768) return PCL_ERR_INVALID;
  if (s.pattern_words < (s.pattern_cols + 31) / 32 + 1) return PCL_ERR_INVALID;
  // the speckle redraw stages the generator and one bit per pattern cell per warp
  if (s.pattern_rows * s.pattern_cols > 32 * kMaxStreamWords) return PCL_ERR_UNSUPPORTED;
  if (!bit_rows_fit(s)) return PCL_ERR_INVALID;
  const int level = s.program_arg[0];
  // TeleporterDrape.__init__ (t_maze.py:415-417): the level's hallway lies inside the pattern
  if (level < 0 || 11 * level + 9 + 5 > s.pattern_rows) return PCL_ERR_INVALID;
  if (s.program_arg[1] != 0 && s.program_arg[1] != 1) return PCL_ERR_INVALID;
  return PCL_OK;
}

int check_state(const pcl_spec&, const pcl_state& st) {
  if (!st.d_bits[0] || !st.d_bits_init[0] || st.bits_bstride[0] == 0) return PCL_ERR_INVALID;
  for (int d = 1; d < 6; ++d) if (!st.d_pattern[d]) return PCL_ERR_INVALID;
  if (!st.d_pattern_init[2] || st.pattern_bstride[2] == 0) return PCL_ERR_INVALID;
  return PCL_OK;
}

// 'Q' is a plain drape; the Scrollys' patterns are rolled, which the layers kernel does
// not follow.
CurtainAt curtain(const pcl_spec&, int d) {
  return d == DQ ? CurtainAt::kBits : CurtainAt::kNone;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  return launch_step(t_maze_step, p, kWarpsPerBlock, 0, s);
}

}  // namespace

const Program kTMaze = {check_spec, check_state, curtain, launch, nullptr,
                        /*float_reward=*/true, /*crop_epilogue=*/false,
                        /*scroll_groups=*/false};

}  // namespace pcl
