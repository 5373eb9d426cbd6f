// fixture.cu — the general step program: any mix of MazeWalkers, Scrollys and
// plain drapes, any update schedule, per-env dynamic z-order.
//
// This is the device counterpart of the reference's own test fixtures
// (tests/test_things.py: TestMazeWalker :203-250, TestScrolly :253-295,
// TestDrape :178-200): every entity performs the motion its action slot names
// (walkers/Scrollys call the matching motion helper, `_stay` by default), and
// Plot directives (add_reward, terminate_episode, change_z_order — injected
// upstream with test_things.post_update) arrive as extra action words.  It
// exists so that the prefab semantics (sprites.py, drapes.py, scrolling.py) and
// the engine's staging/z-order rules (engine.py:698-847) are exercised on the
// GPU in their full generality — diagonal moves, EDGE, confined walkers,
// arbitrary impassable sets, several egocentric walkers, margin-less
// scrolling — not only in the shapes the three example games use.
//
// Unlike the game kernels it keeps a real board: the render after every update
// group (engine.py:735) is materialised in shared memory, because an arbitrary
// walker may test any character.  One warp per env; speed is not the point.
//
// Action row (i32 [n_entities + 2 * PCL_FIXTURE_DIRECTIVES]): motion code per entity
// in UPDATE order, then up to PCL_FIXTURE_DIRECTIVES (opcode, argument) pairs applied
// in order, i.e. in the order the entities issued them (include/pcl.h PCL_DIR_*):
// add_reward(int), terminate_episode(f32 discount), change_default_discount(f32),
// change_z_order(move_this | in_front_of << 8).
#include "pcl_board.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 2;
using board::kMaxEnt;
using board::WarpState;
using board::Ctx;
using board::render;
using board::warp_store_sprite;
using board::scrolly_move_dyn;

// The order / egocentric-set registers of scrolling group g <-> `plot`.
__device__ __forceinline__ void group_in(Plot& plot, const WarpState* st, int g) {
  plot.order_r = st->groups[g][PCL_G_ORDER_R]; plot.order_c = st->groups[g][PCL_G_ORDER_C];
  plot.order_frame = st->groups[g][PCL_G_ORDER_FRAME];
  plot.ego_mask = st->groups[g][PCL_G_EGO_MASK];
}
__device__ __forceinline__ void group_out(const Plot& plot, WarpState* st, int g, int lane) {
  __syncwarp();
  if (lane == 0) {
    st->groups[g][PCL_G_ORDER_R] = plot.order_r; st->groups[g][PCL_G_ORDER_C] = plot.order_c;
    st->groups[g][PCL_G_ORDER_FRAME] = plot.order_frame;
    st->groups[g][PCL_G_EGO_MASK] = plot.ego_mask;
  }
  __syncwarp();
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
fixture_step(const StepParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int env = blockIdx.x * kWarpsPerBlock + warp;
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;   // index of static level data
  const int H = p.H, W = p.W, S = p.S, D = p.D, n = S + D;
  const size_t board_bytes = board::board_bytes(H, p.pitch);
  uint8_t* my = smem_raw + warp * (sizeof(WarpState) + board_bytes);
  WarpState* st = reinterpret_cast<WarpState*>(my);
  Ctx c;
  c.p = &p; c.st = st; c.board = my + sizeof(WarpState);
  c.backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;
  c.env = env; c.lane = lane; c.lvl = lvl; c.kept = 0;

  int32_t* g_sprites = p.st.d_sprites + (int64_t)env * S * PCL_SPRITE_WORDS;
  int32_t* g_drapes = p.st.d_drapes + (int64_t)env * D * PCL_DRAPE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  uint8_t* g_z = p.st.d_z_order + (int64_t)env * n;
  uint8_t* g_board = p.out.d_board + (int64_t)env * H * p.pitch;

  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) return;
  const bool restart = run == ENV_RESTART;
  const int32_t* src_s = restart ? p.st.d_sprites_init + lvl * p.st.sprites_init_bstride
                                 : g_sprites;
  const int32_t* src_d = restart ? p.st.d_drapes_init + lvl * p.st.drapes_init_bstride
                                 : g_drapes;
  const int32_t* src_p = restart ? p.st.d_plot_init + lvl * p.st.plot_init_bstride
                                 : g_plot;
  const uint8_t* src_z = restart ? p.st.d_z_order_init + lvl * p.st.z_order_init_bstride
                                 : g_z;
  const PlotCarry carry = plot_carry(g_plot, restart);
  board::stage_records(st, src_s, src_d, src_p, src_z, S, D, lane);
  for (int i = lane; i < S * 4; i += 32) (&st->impassable[0][0])[i] = p.impassable[i >> 2][i & 3];
  for (int i = lane; i < (int)board_bytes; i += 32) c.board[i] = 0;
  __syncwarp();
  // Scrolling groups: group 0 is the plot record's own order / egocentric words,
  // the others come from (or are restored into) pcl_state.d_groups.
  const int n_sg = p.n_scroll_groups;
  int32_t* g_groups = p.st.d_groups
      ? p.st.d_groups + (int64_t)env * PCL_MAX_SCROLL_GROUPS * PCL_GROUP_WORDS : nullptr;
  if (lane < PCL_GROUP_WORDS) st->groups[0][lane] = st->plot[PCL_P_ORDER_R + lane];
  if (g_groups && n_sg > 1) {
    const int32_t* src_g = restart ? p.st.d_groups_init + lvl * p.st.groups_init_bstride : g_groups;
    if (lane >= PCL_GROUP_WORDS && lane < n_sg * PCL_GROUP_WORDS)
      (&st->groups[0][0])[lane] = src_g[lane];
  }
  __syncwarp();
  if (restart) {
    if (lane == 0) store_carry(st->plot, carry);
    __syncwarp();
  }
  board::stage_board(c, restart, g_board);

  Plot plot = step_plot(st->plot, carry.error);
  group_in(plot, st, 0);
  Directives dir = fresh_directives();
  const int32_t* act = restart ? nullptr : p.actions + (int64_t)env * p.actions_per_env;

  // ---- update groups (engine.py:725-735)
  int k = 0;
  for (int g = 0; g < p.n_groups; ++g) {
    for (int e = 0; e < p.group_len[g]; ++e, ++k) {
      const int ch = p.group_chars[k];
      int motion = act ? act[k] : PCL_M_STAY;
      if (motion < 0 || motion > PCL_M_STAY) motion = PCL_M_STAY;   // test_things.py:247
      for (int s = 0; s < S; ++s) {
        if (p.sprite_char[s] != ch) continue;
        Sprite sp = load_sprite(st->sprites[s]);
        const uint32_t* imp = st->impassable[s];
        const uint8_t* board = c.board;
        const int pitch = p.pitch;
        group_in(plot, st, p.sprite_group[s]);
        walker_move(sp, s, motion, plot, H, W, p.confined[s] != 0, p.egocentric[s] != 0, lane,
                    [&](int r, int col) { return in_set(imp, board[r * pitch + col]); });
        group_out(plot, st, p.sprite_group[s], lane);
        warp_store_sprite(st->sprites[s], sp, lane);
      }
      for (int d = 0; d < D; ++d) {
        if (p.drape_char[d] == ch && p.drape_kind[d]) {
          group_in(plot, st, p.drape_group[d]);
          scrolly_move_dyn(c, d, motion, plot);
          group_out(plot, st, p.drape_group[d], lane);
        }
      }
    }
    render(c);
  }

  // ---- Plot directives (plot.py:136-260) + _apply_and_clear_plot (engine.py:761-847)
  if (act) {
    bool z_changed = false;
    for (int i = 0; i < PCL_FIXTURE_DIRECTIVES; ++i) {
      const int op = act[n + 2 * i], arg = act[n + 2 * i + 1];
      if (op == PCL_DIR_ADD_REWARD) {
        add_reward(dir, arg);                                    // plot.py:201-214
      } else if (op == PCL_DIR_TERMINATE) {
        terminate(dir, __int_as_float(arg));                     // plot.py:176-199
      } else if (op == PCL_DIR_DEFAULT_DISCOUNT) {
        change_default_discount(dir, __int_as_float(arg));       // plot.py:247-260
      } else if (op == PCL_DIR_Z_ORDER) {                        // plot.py:136-174
        const int z_this = arg & 0xff, z_that = (arg >> 8) & 0xff;   // 0 = None (rearmost)
        bool have_this = false, have_that = (z_that == 0);
        for (int k2 = 0; k2 < n; ++k2) {
          have_this |= st->z[k2] == z_this;
          have_that |= st->z[k2] == z_that;
        }
        // Moving an entity in front of itself makes upstream DROP it from the
        // catalogue (engine.py:826-832 skips it and never re-inserts it); that is
        // reported as a bad directive here instead of corrupting the z-order.
        if (!have_this || !have_that || z_this == z_that) {
          plot.error |= PCL_ENV_ERR_BAD_Z;   // engine.py:802-812 raises RuntimeError
        } else {
          __syncwarp();
          if (lane == 0) {
            uint8_t fresh[kMaxEnt];
            int m = 0;
            if (z_that == 0) fresh[m++] = (uint8_t)z_this;
            for (int k2 = 0; k2 < n; ++k2) {
              const uint8_t chz = st->z[k2];
              if (chz == z_this) continue;
              fresh[m++] = chz;
              if (chz == z_that) fresh[m++] = (uint8_t)z_this;
            }
            for (int k2 = 0; k2 < n; ++k2) st->z[k2] = fresh[k2];
          }
          __syncwarp();
          z_changed = true;
        }
      }
    }
    if (z_changed) render(c);                // should_rerender, engine.py:636
  }

  __syncwarp();
  if (lane == 0) {
    group_in(plot, st, 0);
    store_plot<ORDER_ALL>(st->plot, plot, dir);
    store_outputs(p.out, env, dir);
  }
  __syncwarp();
  board::store_env(c, g_sprites, g_drapes, g_plot, g_z, g_board);
  if (g_groups && n_sg > 1 && lane >= PCL_GROUP_WORDS && lane < n_sg * PCL_GROUP_WORDS)
    g_groups[lane] = (&st->groups[0][0])[lane];
}

// Any MazeWalker / Scrolly / plain-drape mix; entities and z-order must be consistent
// permutations of each other.
int check_spec(const pcl_spec& s) {
  const int n = s.n_sprites + s.n_drapes;
  if (n < 1) return PCL_ERR_INVALID;
  if (s.n_groups < 1 || s.n_groups > kMaxEnt) return PCL_ERR_INVALID;
  int total = 0;
  for (int g = 0; g < s.n_groups; ++g) total += s.group_len[g];
  if (total != n) return PCL_ERR_INVALID;
  for (int i = 0; i < n; ++i) {
    int in_z = 0, in_groups = 0;
    const uint8_t ch = i < s.n_sprites ? s.sprite_char[i] : s.drape_char[i - s.n_sprites];
    for (int k = 0; k < n; ++k) {
      in_z += s.z_order[k] == ch;
      in_groups += s.group_chars[k] == ch;
    }
    if (in_z != 1 || in_groups != 1 || ch == 0 || ch > 127) return PCL_ERR_INVALID;
  }
  for (int d = 0; d < s.n_drapes; ++d) {
    if (!s.drape_kind[d]) continue;
    if (s.pattern_rows < s.rows || s.pattern_cols < s.cols) return PCL_ERR_INVALID;
    if (s.pattern_words < (s.pattern_cols + 31) / 32 + 2) return PCL_ERR_INVALID;
    if (!margins_fit(s, d)) return PCL_ERR_INVALID;
  }
  if (!bit_rows_fit(s)) return PCL_ERR_INVALID;
  return PCL_OK;
}

int check_state(const pcl_spec& s, const pcl_state& st) {
  if (!st.d_z_order || !st.d_z_order_init) return PCL_ERR_INVALID;
  for (int d = 0; d < s.n_drapes; ++d) {
    if (s.drape_kind[d] ? !st.d_pattern[d] : !st.d_bits[d]) return PCL_ERR_INVALID;
  }
  return PCL_OK;
}

CurtainAt curtain(const pcl_spec& s, int d) {
  return s.drape_kind[d] ? CurtainAt::kPatternWindow : CurtainAt::kBits;
}

// A motion code per entity, then the Plot directives.
int actions_per_env(const pcl_spec& s) {
  return s.n_sprites + s.n_drapes + 2 * PCL_FIXTURE_DIRECTIVES;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  const size_t board_bytes = board::board_bytes(p.H, p.pitch);
  const size_t smem = (sizeof(WarpState) + board_bytes) * kWarpsPerBlock;
  return launch_step(fixture_step, p, kWarpsPerBlock, smem, s);
}

}  // namespace

const Program kFixture = {check_spec, check_state, curtain, launch, actions_per_env,
                          /*float_reward=*/false, /*crop_epilogue=*/false,
                          /*scroll_groups=*/true};

}  // namespace pcl
