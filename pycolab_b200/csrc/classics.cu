// classics.cu — fused step kernel for the single-walker games: examples/classics/
// {four_rooms,cliff_walk,chain_walk}.py and examples/fluvial_natation.py
// (SURVEY.md §8f-4).
//
// Each game is one MazeWalker 'P' over a static backdrop: one update group
// ['P'], z-order 'P', no drapes.  The only board cells the walker ever reads
// are the backdrop cells next to it (its own cell is never consulted), so the
// stale board IS the staged backdrop tile.  p.program_arg[0] picks the rule set:
//
//   PCL_CLASSIC_FOUR_ROOMS  actions 0-3 = N S W E; at (arg[1], arg[2]) = (4, 3):
//                           reward 1.0 + terminate          (four_rooms.py:68-80)
//   PCL_CLASSIC_CLIFF_WALK  actions 0-3 = N S W E, others return early; bottom
//                           row, 0 < col < W-2: -100.0 else -1.0; bottom row,
//                           0 < col: terminate              (cliff_walk.py:62-86)
//   PCL_CLASSIC_CHAIN_WALK  actions 0, 1 = W E; col 0: 1.0 + terminate; col W-1:
//                           100.0 + terminate               (chain_walk.py:60-73)
//
//   PCL_CLASSIC_FLUVIAL     examples/fluvial_natation.py:61-110: on even frames the
//                           backdrop rows [arg[1], arg[2]) rotate one cell west
//                           (RiverBackdrop.update; the rotation count lives in
//                           plot aux0, the backdrop array itself stays static)
//                           and the swimmer drifts west; actions 0, 1 = W E;
//                           virtual col < 0: -1 + terminate, >= W: +1 + terminate.
//
// classics rewards are float in the reference; d_reward carries the equal
// integer and the host facade converts back (engine.py).
//
// One warp per env like the other programs; the records travel through shared
// memory with coalesced loads, the tile with cp.async.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 4;
constexpr int kRecWords = 32;       // sprite 8, pad 8, plot 16

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
classics_step(const StepParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int env = blockIdx.x * kWarpsPerBlock + warp;
  if (env >= p.B) return;
  const EnvAt e = env_at(p, env, 1, 0);
  const int H = p.H, W = p.W, pitch = p.pitch;
  const int tile = H * pitch;
  uint8_t* my = smem_raw + warp * (kRecWords * 4 + tile);
  int32_t* rec = reinterpret_cast<int32_t*>(my);
  uint8_t* s_bd = my + kRecWords * 4;

  for (int i = lane; i < (tile >> 4); i += 32) cp_async16(s_bd + i * 16, e.backdrop + i * 16);

  const EnvRun run = env_run(p, env, e.plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) { cp_async_wait_all(); return; }
  const bool restart = run == ENV_RESTART;
  if (restart) {                                   // a fresh Engine (engine.py:520-581)
    const PlotCarry carry = plot_carry(e.plot, true);
    if (lane < 8) rec[lane] = __ldg(e.level(p.st.d_sprites_init, p.st.sprites_init_bstride) + lane);
    if (lane >= 16) rec[lane] = __ldg(e.level(p.st.d_plot_init, p.st.plot_init_bstride) + lane - 16);
    __syncwarp();
    if (lane == 0) store_carry(rec + 16, carry);
  } else {
    if (lane < 8) rec[lane] = e.sprites[lane];
    if (lane >= 16) rec[lane] = e.plot[lane - 16];
  }
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  cp_async_wait_all();
  __syncwarp();

  Sprite sp = load_sprite(rec);
  Plot plot = step_plot(rec + 16, rec[16 + PCL_P_ERROR]);
  plot.aux0 = rec[16 + PCL_P_AUX0];                          // river rotation count
  Directives dir = fresh_directives();

  const int rule = p.program_arg[0];
  auto blocked = [&](int r, int c) { return in_set(p.impassable[0], s_bd[r * pitch + c]); };
  int motion = PCL_M_NONE;
  if (rule == PCL_CLASSIC_FLUVIAL) {
    const bool even = (plot.frame & 1) == 0;
    // Backdrop.update runs first (engine.py:718-721); the swimmer's set of
    // impassable characters is empty (checked in pcl_create), so nobody reads the
    // stale board and the band can be re-staged for the final render right away.
    if (even) plot.aux0 = plot.aux0 + 1 == W ? 0 : plot.aux0 + 1;
    const int r0 = min(p.program_arg[1], H), r1 = min(p.program_arg[2], H);
    const int k = plot.aux0;
    for (int i = lane; i < (r1 - r0) * W; i += 32) {
      const int r = r0 + i / W, c = i - (r - r0) * W;
      int src = c + k;
      if (src >= W) src -= W;
      s_bd[r * pitch + c] = __ldg(e.backdrop + r * pitch + src);
    }
    __syncwarp();               // the walker's neighbourhood test reads cells other lanes wrote
    if (even) walker_move(sp, 0, PCL_M_W, plot, H, W, p.confined[0] != 0, false, lane, blocked);
    motion = action == 0 ? PCL_M_W : action == 1 ? PCL_M_E : PCL_M_NONE;
  } else if (rule == PCL_CLASSIC_CHAIN_WALK) {
    motion = action == 0 ? PCL_M_W : action == 1 ? PCL_M_E : PCL_M_NONE;
  } else {
    motion = action == 0 ? PCL_M_N : action == 1 ? PCL_M_S : action == 2 ? PCL_M_W
           : action == 3 ? PCL_M_E : PCL_M_NONE;
  }
  if (motion != PCL_M_NONE)
    walker_move(sp, 0, motion, plot, H, W, p.confined[0] != 0, false, lane, blocked);
  if (rule == PCL_CLASSIC_FLUVIAL) {
    if (sp.vcol < 0) { add_reward(dir, -1); terminate(dir); }
    else if (sp.vcol >= W) { add_reward(dir, 1); terminate(dir); }
  } else if (rule == PCL_CLASSIC_FOUR_ROOMS) {
    if (sp.row == p.program_arg[1] && sp.col == p.program_arg[2]) { add_reward(dir, 1); terminate(dir); }
  } else if (rule == PCL_CLASSIC_CLIFF_WALK) {
    if (motion != PCL_M_NONE) {
      const bool bottom = sp.row == H - 1;
      add_reward(dir, (bottom && 0 < sp.col && sp.col < W - 2) ? -100 : -1);
      if (bottom && 0 < sp.col) terminate(dir);
    }
  } else {
    if (sp.col == 0) { add_reward(dir, 1); terminate(dir); }
    else if (sp.col == W - 1) { add_reward(dir, 100); terminate(dir); }
  }

  // ---- _apply_and_clear_plot (engine.py:761-847) + records back
  __syncwarp();                 // every lane has read the staged records (racecheck: WAR)
  if (lane == 0) {
    const double ep_so_far = load_episode(p, env);   // overlaps the stores below
    store_sprite(rec, sp, PCL_S_AUX0);
    apply_time_limit(p, plot, dir);
    store_episode(p, env, plot.frame, ep_so_far, (double)dir.reward);
    store_plot<ORDER_KEEP>(rec + 16, plot, dir);
    rec[16 + PCL_P_AUX0] = plot.aux0;
    store_outputs(p.out, env, dir);
  }
  __syncwarp();
  if (lane < 8) e.sprites[lane] = rec[lane];
  if (lane >= 16) e.plot[lane - 16] = rec[lane];

  // ---- final render: backdrop + P (engine.py:737-759)
  uint8_t* board = p.out.d_board + (int64_t)env * tile;
  const int segs_per_row = pitch >> 4;
  const int total = H * segs_per_row;
  for (int seg = lane; seg < total; seg += 32) {
    const int r = seg / segs_per_row;
    const int c0 = (seg - r * segs_per_row) << 4;
    uint4 px = *reinterpret_cast<const uint4*>(s_bd + r * pitch + c0);
    const unsigned m = sprite_bit(sp, r, c0);
    if (m) paint_bits(px, m, p.sprite_char[0]);
    *reinterpret_cast<uint4*>(board + r * pitch + c0) = px;
  }
}

int check_spec(const pcl_spec& s) {
  if (!chars_are(s.sprite_char, s.n_sprites, "P") || s.n_drapes != 0) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.z_order, 1, "P")) return PCL_ERR_UNSUPPORTED;
  const int lens[1] = {1};
  if (!groups_are(s, "P", lens, 1)) return PCL_ERR_UNSUPPORTED;
  if (s.sprite_egocentric[0]) return PCL_ERR_UNSUPPORTED;
  const int rule = s.program_arg[0];
  if (rule != PCL_CLASSIC_FOUR_ROOMS && rule != PCL_CLASSIC_CLIFF_WALK &&
      rule != PCL_CLASSIC_CHAIN_WALK && rule != PCL_CLASSIC_FLUVIAL) return PCL_ERR_INVALID;
  if (rule == PCL_CLASSIC_FLUVIAL) {
    // The kernel re-stages the flowing rows before the swimmer moves, which is
    // only equivalent when the swimmer never looks at the board.
    if (!set_is(s.impassable[0], "")) return PCL_ERR_UNSUPPORTED;
    if (s.program_arg[1] < 0 || s.program_arg[2] < s.program_arg[1]) return PCL_ERR_INVALID;
  }
  if (s.rows * s.pitch > 8192) return PCL_ERR_UNSUPPORTED;   // the tile is staged per env in smem
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  const size_t smem = (kRecWords * 4 + (size_t)p.H * p.pitch) * kWarpsPerBlock;
  return launch_step(classics_step, p, kWarpsPerBlock, smem, s);
}

}  // namespace

const Program kClassics = {check_spec, nullptr, nullptr, launch, nullptr,
                           /*float_reward=*/false, /*crop_epilogue=*/false,
                           /*scroll_groups=*/false};

}  // namespace pcl
