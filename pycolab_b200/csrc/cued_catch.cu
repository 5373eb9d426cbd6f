// cued_catch.cu — fused step kernel for examples/research/lp-rnn/cued_catch.py:96-317.
//
// MazeWalker 'P' (impassable '', confined), plain Sprites 'a' and 'b' (the balls), the cue
// drape 'Q'; one update group P a b Q, z-order PabQ.  One warp per env: the game logic is
// warp-uniform scalar code, lane r holds board row r of Q's curtain and paints that row.
//
// What the reference does that a straight restatement could get wrong:
//   * Every frame pays: P adds int(caught) (sigma 0), or, with reward_sigma set, float(caught)
//     + random.normalvariate(0, sigma) when P stands in the correct ball's column and the
//     reward-free trials are spent, else the int 0 (:147-162).  The Python type of each
//     frame's reward goes to plot word AUX3 (1 = float), so the facade returns int 0 / float.
//   * The balls only move once the_plot['programming_complete'] is set, which Q does at the
//     end of its update, so they first move one frame after the programming phase (:183).
//   * _second_phase_reset draws random.randrange(4) BEFORE it tests for the last trial, so
//     the terminating reset consumes a draw too (:286-293).
//   * Q rewrites three row bands every frame (1:3, 3:5, -2:, Python slices at any height, so
//     they overlap on boards under 7 rows): the ball symbol before the cue, except in a trial
//     with always_show_ball_symbol, which shows it after (:277-279).  Every other row of its
//     curtain keeps the art's 'Q' cells forever, so the render reads those from the template.
//   * Upstream compares None with ints in Python 2 style (None < everything): an unset
//     'last_ball_reset' never exceeds the last reset frame, and _show_cue(None) shows nothing.
// At every (re)start with the facade flag (program_arg[3] bit 1) clear, the four cue->ball
// pairings are drawn as CPython 3.12's random.sample(['top'] * 2 + ['bottom'] * 2, 4) does
// (the pool method: _randbelow(4), (3), (2), (1)); with it set they come from the template
// (the Python CueDrape drew them) and only update()'s draws come from d_rng.  normalvariate
// is Lib/random.py's Kinderman-Monahan loop with correctly rounded f64 operations (no FMA
// contraction).  Its accept test zz <= -log(u2) takes the device's double log (within 1 ulp)
// unless zz lies within a few ulps of it; there it compares with the correctly rounded
// -log(u2), as CPython's (glibc's) log gives it, from a double-double log.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"
#include "pcl_mt.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 4;
enum { SP = 0, SA = 1, SB = 2 };
enum { kWhichUnset = 0, kWhichTop = 1, kWhichBottom = 2 };

// Cells [lo, hi) of a 64-cell row as bits.
__device__ __forceinline__ uint64_t cols_bits(int lo, int hi) {
  if (hi <= lo) return 0ull;
  const uint64_t upto = hi >= 64 ? ~0ull : (1ull << hi) - 1ull;
  return upto & ~((1ull << lo) - 1ull);
}

// Double-double arithmetic (Dekker / Knuth error-free transformations) for minus_log_rn.
struct DD { double hi, lo; };
__device__ __forceinline__ DD two_sum(double a, double b) {
  const double s = __dadd_rn(a, b), bb = __dsub_rn(s, a);
  return {s, __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb))};
}
__device__ __forceinline__ DD fast_two_sum(double a, double b) {
  const double s = __dadd_rn(a, b);
  return {s, __dsub_rn(b, __dsub_rn(s, a))};
}
__device__ __forceinline__ DD dd_add(DD x, DD y) {
  const DD s = two_sum(x.hi, y.hi);
  return fast_two_sum(s.hi, __dadd_rn(s.lo, __dadd_rn(x.lo, y.lo)));
}
__device__ __forceinline__ DD dd_mul(DD x, DD y) {
  const double p = __dmul_rn(x.hi, y.hi);
  const double e = __fma_rn(x.hi, y.hi, -p);
  return fast_two_sum(p, __dadd_rn(e, __dadd_rn(__dmul_rn(x.hi, y.lo), __dmul_rn(x.lo, y.hi))));
}
__device__ __forceinline__ DD dd_div(DD x, DD y) {
  const double q1 = __ddiv_rn(x.hi, y.hi);
  DD r = dd_add(x, dd_mul({-q1, 0.0}, y));
  const double q2 = __ddiv_rn(r.hi, y.hi);
  r = dd_add(r, dd_mul({-q2, 0.0}, y));
  return dd_add(fast_two_sum(q1, q2), {__ddiv_rn(r.hi, y.hi), 0.0});
}
// 1 / (2j + 1), j = 0..22, as double-doubles.
__constant__ DD kOddRecip[23] = {
    {1.0, 0.0}, {0.3333333333333333, 1.850371707708594e-17},
    {0.2, -1.1102230246251566e-17}, {0.14285714285714285, 7.93016446160826e-18},
    {0.1111111111111111, 6.1679056923619804e-18}, {0.09090909090909091, -2.523234146875356e-18},
    {0.07692307692307693, -4.270088556250602e-18}, {0.06666666666666667, 9.251858538542971e-19},
    {0.058823529411764705, 8.163404592832033e-19}, {0.05263157894736842, 2.921639538487254e-18},
    {0.047619047619047616, 2.64338815386942e-18}, {0.043478260869565216, 1.206764157201257e-18},
    {0.04, -8.326672684688674e-19}, {0.037037037037037035, 2.05596856412066e-18},
    {0.034482758620689655, 4.785444071660157e-19}, {0.03225806451612903, 8.953411488912552e-19},
    {0.030303030303030304, -8.410780489584519e-19}, {0.02857142857142857, 8.921435019309293e-19},
    {0.02702702702702703, -1.50030138462859e-18}, {0.02564102564102564, 8.896017825522087e-19},
    {0.024390243902439025, -8.46206573647223e-19}, {0.023255813953488372, 3.2273925134452225e-19},
    {0.022222222222222223, -8.480870326997723e-19}};
// -log(u2) correctly rounded, 0 < u2 <= 1: log to about 100 bits as k ln 2 + 2 atanh(s),
// u2 = 2^k m, m in [sqrt(1/2), sqrt(2)), s = (m - 1) / (m + 1), |s| < 0.172, summed to s^45.
// Called only when zz lies within 2^-50 relative of the device's -log(u2), so kept out of line.
__device__ __noinline__ double minus_log_rn(double u2) {
  int k;
  double m = frexp(u2, &k);
  if (m < 0.70710678118654752) { m = __dmul_rn(m, 2.0); k -= 1; }
  const DD s = dd_div({__dsub_rn(m, 1.0), 0.0}, two_sum(m, 1.0));
  const DD s2 = dd_mul(s, s);
  DD p = kOddRecip[22];
#pragma unroll 1
  for (int j = 21; j >= 0; --j) p = dd_add(dd_mul(p, s2), kOddRecip[j]);
  const DD ln2 = {0.6931471805599452862, 2.3190468138462996154e-17};
  const DD lg = dd_add(dd_mul(ln2, {(double)k, 0.0}), dd_mul(dd_mul(s, p), {2.0, 0.0}));
  return -__dadd_rn(lg.hi, lg.lo);
}

// The minimum-blocks bound lets ptxas take the registers it needs (72, 87 with kNoisy): with
// the block size alone it aims lower and spills around the draw loop.  kNoisy (reward_sigma
// set) compiles the normal draws in; the noiseless kernel leaves them, and the registers of
// their exact accept test, out.
template <bool kNoisy>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, 4)
cued_catch_step(const StepParams p) {
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (env >= p.B) return;
  const EnvAt e = env_at(p, env, 3, 1);
  const int H = p.H, W = p.W, BW = p.BW, pitch = p.pitch;

  const EnvRun run = env_run(p, env, e.plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) return;
  const bool restart = run == ENV_RESTART;
  const int32_t* src_s = e.start(restart, p.st.d_sprites_init, p.st.sprites_init_bstride, e.sprites);
  const int32_t* src_q = e.start(restart, p.st.d_drapes_init, p.st.drapes_init_bstride, e.drapes);
  const int32_t* src_p = e.start(restart, p.st.d_plot_init, p.st.plot_init_bstride, e.plot);

  Sprite sp[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    sp[i] = load_sprite(src_s + i * PCL_SPRITE_WORDS);
    sp[i].aux1 = sp[i].aux2 = 0;                                       // stored as zeros
  }
  // CueDrape (:229-245): phase, ticks, trial choice, last reset, trials left, pairings
  int phase = src_q[PCL_D_CORNER_R], tick1 = src_q[PCL_D_CORNER_C];
  int choice = src_q[PCL_D_PRE_R], tick2 = src_q[PCL_D_PRE_C];
  int last_reset = src_q[PCL_D_LAST_FRAME], trials = src_q[PCL_D_AUX0];
  int pairs = src_q[PCL_D_AUX1];
  const PlotCarry carry = plot_carry(e.plot, restart);
  const Plot plot = step_plot(src_p, carry.error);
  const int f = plot.frame;
  int programmed = src_p[PCL_P_AUX0], which = src_p[PCL_P_AUX1], ball_reset = src_p[PCL_P_AUX2];
  int ttr = sp[SP].aux0;                           // PlayerSprite._trials_till_reward

  uint32_t* mt = reinterpret_cast<uint32_t*>(p.st.d_rng) + (int64_t)env * PCL_MT_WORDS;
  const bool noisy = kNoisy;                       // program_arg[0] != 0
  const int icd = p.program_arg[1], cd = p.program_arg[2];
  const bool always_show = p.program_arg[3] & 1;
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  Directives dir = fresh_directives();

  // ---- PlayerSprite.update (:136-167), its motion; nothing is impassable, so no board look-up
  if (action == 1 && sp[SP].vrow > 1) {
    sp[SP].vrow -= 1; sp[SP].row = sp[SP].vrow;
  } else if (action == 2 && sp[SP].vrow < 2) {
    if (sp[SP].vrow + 1 < H) { sp[SP].vrow += 1; sp[SP].row = sp[SP].vrow; }   // confined
  } else if (action == 0 || action == 4) {
    terminate(dir);
  }
  const bool top = which == kWhichTop;             // 'a' if which_ball == 'top' else 'b'
  const bool same_col = sp[SP].col == (top ? sp[SA].col : sp[SB].col);
  const bool caught = same_col && sp[SP].row == (top ? sp[SA].row : sp[SB].row);
  const bool noisy_pay = noisy && same_col && ttr <= 0;

  // ---- BallSprite.update (:181-194), 'a' then 'b'
  if (programmed) {
#pragma unroll
    for (int i = SA; i <= SB; ++i) {
      sp[i].flags |= 1;
      if (sp[i].col < sp[SP].col) {
        sp[i].row = sp[i].vrow; sp[i].col = sp[i].vcol;                // _start_position
        ball_reset = f;
      } else {
        sp[i].col -= 1;
      }
    }
  }
  // Does CueDrape.update call _second_phase_reset (:265-274)?
  const bool trial_reset = phase == 0 ? tick1 - 1 <= 0 : ball_reset > last_reset;

  // ---- The step's draws, in stream order, through one mt_draw site (every inlined copy of
  // the twist costs registers): stages 0-3 the pairings at a (re)start (random.sample's
  // _randbelow(4), (3), (2), (1)), 4-5 normalvariate's u1 and 1 - u2 until it accepts, 6
  // the trial's randrange(4).
  enum { kPool = 0, kU1 = 4, kU2 = 5, kTrial = 6, kDone = 7 };
  const bool draw_pairs = restart && !(p.program_arg[3] & 2);
  int stage = draw_pairs ? kPool : noisy_pay ? kU1 : trial_reset ? kTrial : kDone;
  uint32_t pool = 0x3u;                            // bit k: pool[k] == 'top'
  if (draw_pairs) pairs = 0;
  double u1 = 0.0, z = 0.0;
  const double magic = __hiloint2double(p.program_arg[7], p.program_arg[6]);
#pragma unroll 1
  while (stage != kDone) {
    const MtRule rule = (stage == kU1 || stage == kU2) ? kMtRandom53 : kMtPythonBelow;
    const uint64_t r = mt_draw(mt, rule, stage < kU1 ? (uint64_t)(4 - stage) : 4ull, lane);
    if (stage < kU1) {                             // Lib/random.py sample(), the pool method
      const int j = (int)r, i = stage;
      pairs |= (int)((pool >> j) & 1u) << i;
      pool = (pool & ~(1u << j)) | (((pool >> (3 - i)) & 1u) << j);
      stage = i < 3 ? i + 1 : noisy_pay ? kU1 : trial_reset ? kTrial : kDone;
    } else if (kNoisy && stage == kU1) {
      u1 = __dmul_rn((double)r, 1.0 / 9007199254740992.0);
      stage = kU2;
    } else if (kNoisy && stage == kU2) {           // Lib/random.py normalvariate()
      const double u2 = __dsub_rn(1.0, __dmul_rn((double)r, 1.0 / 9007199254740992.0));
      z = __ddiv_rn(__dmul_rn(magic, __dsub_rn(u1, 0.5)), u2);
      const double zz = __dmul_rn(__dmul_rn(z, z), 0.25);   // z * z / 4.0, exactly
      double bound = -log(u2);
      if (fabs(__dsub_rn(zz, bound)) <= __dmul_rn(bound, 0x1p-50)) bound = minus_log_rn(u2);
      stage = zz <= bound ? (trial_reset ? kTrial : kDone) : kU1;
    } else {
      choice = (int)r;
      stage = kDone;
    }
  }

  // ---- PlayerSprite.update, its reward
  double reward_f64 = 0.0;
  if (noisy_pay) {                                 // float(caught) + (0 + z * sigma)
    const double sigma = __hiloint2double(p.program_arg[5], p.program_arg[4]);
    reward_f64 = __dadd_rn(caught ? 1.0 : 0.0, __dadd_rn(0.0, __dmul_rn(z, sigma)));
  }
  add_reward(dir, (!noisy && caught && ttr <= 0) ? 1 : 0);
  if (same_col && ttr > 0) --ttr;

  // ---- CueDrape.update (:247-317): what the three bands show after it
  const bool show_phase = phase == 0;
  int symbol = kWhichUnset, cue = -1;
  bool symbol_last = false;                        // shown after the cue (:277-279)
  if (phase == 0) {
    tick1 -= 1;
    cue = tick1 / icd;
    symbol = ((pairs >> cue) & 1) ? kWhichTop : kWhichBottom;
    if (tick1 <= 0) {
      phase = 1;
      programmed = 1;
    }
  }
  if (trial_reset) {                               // _second_phase_reset (:286-293)
    which = ((pairs >> choice) & 1) ? kWhichTop : kWhichBottom;
    tick2 = cd;
    last_reset = f;
    if (trials <= 0) terminate(dir);
    trials -= 1;
  }
  if (!show_phase) {
    if (tick2 > 0) {
      cue = choice;
      if (always_show) {
        symbol = ((pairs >> choice) & 1) ? kWhichTop : kWhichBottom;
        symbol_last = true;
      }
    }
    tick2 -= 1;
  }

  // ---- Q's curtain, row `lane`: the template outside the bands, the bands as shown, in the
  // order update() wrote them (they overlap on boards under 7 rows)
  uint64_t qrow = 0;
  bool banded = false;
  if (lane < H) {
    const uint32_t* init = e.level(p.st.d_bits_init[0], p.st.bits_init_bstride[0]) + lane * BW;
    qrow = (uint64_t)init[0] | (W > 32 ? (uint64_t)init[1] << 32 : 0ull);
    const bool in_symbol = lane >= 3 && lane < 5;
    const uint64_t symbol_row = symbol == kWhichTop ? cols_bits(0, min(6, W))
                                : symbol == kWhichBottom ? cols_bits(max(W - 6, 0), W) : 0ull;
    if (lane >= 1 && lane < 3) {                   // _show_phase_cue
      qrow = show_phase ? cols_bits(0, min(2, W)) | cols_bits(max(W - 2, 0), W) : 0ull;
      banded = true;
    }
    if (in_symbol && !symbol_last) {               // _show_ball_symbol
      qrow = symbol_row;
      banded = true;
    }
    if (lane >= H - 2) {                           // _show_cue
      const int width = W / 4;
      qrow = (cue >= 0 && cue < 4) ? cols_bits(cue * width, cue * width + width) : 0ull;
      banded = true;
    }
    if (in_symbol && symbol_last) {
      qrow = symbol_row;
      banded = true;
    }
    if (banded || restart) {
      uint32_t* live = p.st.d_bits[0] + (int64_t)env * p.st.bits_bstride[0] + lane * BW;
      live[0] = (uint32_t)qrow;
      live[1] = (uint32_t)(qrow >> 32);
      for (int w = 2; w < BW; ++w) live[w] = 0u;
    }
  }

  if (lane == 0) {
    const double ep_so_far = load_episode(p, env);   // overlaps the stores below
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      sp[i].aux0 = i == SP ? ttr : 0;
      store_sprite(e.sprites + i * PCL_SPRITE_WORDS, sp[i]);
    }
    store_drape(e.drapes, {phase, tick1, choice, tick2, last_reset, trials, pairs, 0});
    store_carry(e.plot, carry);
    apply_time_limit(p, plot, dir);
    store_episode(p, env, plot.frame, ep_so_far, noisy && noisy_pay ? reward_f64 : (double)dir.reward);
    store_plot<ORDER_CLEAR>(e.plot, plot, dir);
    e.plot[PCL_P_AUX0] = programmed; e.plot[PCL_P_AUX1] = which;
    e.plot[PCL_P_AUX2] = ball_reset; e.plot[PCL_P_AUX3] = noisy_pay ? 1 : 0;
    // has_reward is 1: PlayerSprite.update pays (possibly 0) at every step
    if (noisy) store_outputs(p.out, env, dir, noisy_pay ? reward_f64 : (double)dir.reward);
    else store_outputs(p.out, env, dir);
  }

  // ---- render (engine.py:737-759): backdrop, P, a, b, Q; lane r paints row r.  A ball
  // one column left of column 0 is drawn in the last column, as NumPy indexes.
  if (lane < H) {
    Sprite shown[3] = {sp[SP], sp[SA], sp[SB]};
#pragma unroll
    for (int i = 1; i < 3; ++i) if (shown[i].col < 0) shown[i].col += W;
    uint8_t* board = p.out.d_board + (int64_t)env * H * pitch + lane * pitch;
    for (int c0 = 0; c0 < pitch; c0 += 16) {
      uint4 px = *reinterpret_cast<const uint4*>(e.backdrop + lane * pitch + c0);
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const unsigned m = sprite_bit(shown[i], lane, c0);
        if (m) paint_bits(px, m, p.sprite_char[i]);
      }
      const unsigned q = c0 < 64 ? (unsigned)(qrow >> c0) & 0xffffu : 0u;
      if (q) paint_bits(px, q, p.drape_char[0]);
      *reinterpret_cast<uint4*>(board + c0) = px;
    }
  }
}

int check_spec(const pcl_spec& s) {
  if (!chars_are(s.sprite_char, s.n_sprites, "Pab")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.drape_char, s.n_drapes, "Q")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.z_order, 4, "PabQ")) return PCL_ERR_UNSUPPORTED;
  const int lens[1] = {4};
  if (!groups_are(s, "PabQ", lens, 1)) return PCL_ERR_UNSUPPORTED;
  if (!set_is(s.impassable[0], "") || !s.sprite_confined[0]) return PCL_ERR_UNSUPPORTED;
  for (int i = 0; i < 3; ++i) if (s.sprite_egocentric[i]) return PCL_ERR_UNSUPPORTED;
  // one board row per lane; a row of Q's curtain is one 64-bit word
  if (s.rows > 32 || s.cols > 64) return PCL_ERR_UNSUPPORTED;
  if (!bit_rows_fit(s)) return PCL_ERR_INVALID;
  const int64_t sigma = (int64_t)(uint32_t)s.program_arg[4] | (int64_t)s.program_arg[5] << 32;
  if (s.program_arg[0] != ((sigma << 1) != 0 ? 1 : 0)) return PCL_ERR_INVALID;   // -0.0 is 0
  // the first phase lasts 4 * initial_cue_duration frames (:241, :261)
  if (s.program_arg[1] < 1 || s.program_arg[1] > (1 << 28)) return PCL_ERR_INVALID;
  if (s.program_arg[3] & ~3) return PCL_ERR_INVALID;
  return PCL_OK;
}

int check_state(const pcl_spec&, const pcl_state& st) {
  // update() draws (randrange, normalvariate) at every trial: a generator is required
  if (!st.d_rng || !st.d_bits[0] || !st.d_bits_init[0] || st.bits_bstride[0] == 0)
    return PCL_ERR_INVALID;
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  return launch_step(p.program_arg[0] ? cued_catch_step<true> : cued_catch_step<false>, p,
                     kWarpsPerBlock, 0, s);
}

}  // namespace

const Program kCuedCatch = {check_spec, check_state, curtain_bits, launch, nullptr,
                            /*float_reward=*/false, /*crop_epilogue=*/false,
                            /*scroll_groups=*/false, nullptr, /*float_reward_arg0=*/true,
                            /*derive=*/nullptr, /*block_chaining=*/false, one_rng_slot};

}  // namespace pcl
