// warehouse.cu — fused step kernel for examples/warehouse_manager.py.
//
// Update groups [[boxes...], ['X'], ['P']] (warehouse_manager.py:168-170),
// z-order = the same sequence flattened (:176-178): boxes, then the JudgeDrape
// 'X' over boxes that sit on goals, then the player on top.
//
// Sprite order: boxes in update order, then P (index n_boxes).  Drape 0 = 'X';
// its curtain is never stored: after every JudgeDrape.update it is exactly
// {box cells} & (backdrop == '_') (:247-254), so one bit per box ("this box
// is drawn as X") carries it: box aux0.  Drape aux0 = _last_num_boxes_on_goals.
//
// Boards the entities read (engine.py:698-735): the boxes see the PREVIOUS
// step's final board (nothing has been re-rendered yet), the player sees the
// render after the judge ran.  Both are evaluated per cell on demand from the
// records + the backdrop tile.
//
// Memory schedule (one warp per env): records -> smem with coalesced loads; the
// whole backdrop tile -> smem with cp.async (it is both the board's base layer
// and the only thing the look-ups need); all game logic then runs out of
// shared memory with one lane per box; the board is the staged tile streamed
// back out with uint4 stores plus <= 11 single-byte patches for the sprites.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"

namespace pcl {

namespace {

constexpr int kMaxS = 11;           // up to ten boxes + P
constexpr int kWarpsPerBlock = 4;
constexpr int kRecWords = 128;      // 11 * 8 sprite words + 8 drape + 16 plot, padded

__device__ __forceinline__ int motion_of_action(int a) {    // :214-226, :288-295
  return a == 0 ? PCL_M_N : a == 1 ? PCL_M_S : a == 2 ? PCL_M_W : PCL_M_E;
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32, 8)
warehouse_step(const StepParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int env = blockIdx.x * kWarpsPerBlock + warp;
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;   // index of static level data
  const int H = p.H, W = p.W, S = p.S, NB = p.S - 1, pitch = p.pitch;
  const size_t tile = (size_t)H * pitch;
  uint8_t* my = smem_raw + warp * (kRecWords * 4 + tile);
  int32_t* rec = reinterpret_cast<int32_t*>(my);          // [0, 88) sprites, [96, 104) drape, [112, 128) plot
  uint8_t* s_bd = my + kRecWords * 4;
  int32_t* r_judge = rec + 96;
  int32_t* r_plot = rec + 112;

  int32_t* g_sprites = p.st.d_sprites + (int64_t)env * S * PCL_SPRITE_WORDS;
  int32_t* g_drapes = p.st.d_drapes + (int64_t)env * PCL_DRAPE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;

  // ---- the backdrop tile does not depend on anything: start it first, as one
  // TMA bulk copy tracked by this warp's mbarrier (rec words 104..105 are padding).
  uint64_t* bar = reinterpret_cast<uint64_t*>(rec + 104);
  if (lane == 0) mbar_init(bar, 1);
  __syncwarp();
  if (lane == 0) tile_load_bulk(s_bd, backdrop, (uint32_t)tile, bar);
  // ---- records -> smem: the live state first, unconditionally, in one round
  // trip; whether the env restarts is decided from the staged plot record.
  for (int i = lane; i < S * PCL_SPRITE_WORDS; i += 32) rec[i] = g_sprites[i];
  if (lane < PCL_DRAPE_WORDS) r_judge[lane] = g_drapes[lane];
  if (lane >= 16) r_plot[lane - 16] = g_plot[lane - 16];
  int action = env_action(p, env);
  __syncwarp();
  const EnvRun run = env_run(p, env, r_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) { mbar_wait(bar, 0); return; }
  if (run == ENV_RESTART) {                    // a fresh Engine: templates over the live state
    const PlotCarry carry = plot_carry(r_plot, true);
    __syncwarp();
    const int32_t* ss = p.st.d_sprites_init + lvl * p.st.sprites_init_bstride;
    const int32_t* sd = p.st.d_drapes_init + lvl * p.st.drapes_init_bstride;
    const int32_t* sp = p.st.d_plot_init + lvl * p.st.plot_init_bstride;
    for (int i = lane; i < S * PCL_SPRITE_WORDS; i += 32) rec[i] = ss[i];
    if (lane < PCL_DRAPE_WORDS) r_judge[lane] = sd[lane];
    if (lane >= 16) r_plot[lane - 16] = sp[lane - 16];
    action = PCL_ACTION_NONE;
    __syncwarp();
    if (lane == 0) store_carry(r_plot, carry);
  }
  mbar_wait(bar, 0);
  __syncwarp();

  Plot plot = step_plot(r_plot, r_plot[PCL_P_ERROR]);
  Directives dir = fresh_directives();

  // Player as of the previous render; box i's record sits in lane i.
  Sprite player = load_sprite(rec + NB * PCL_SPRITE_WORDS);
  const bool pl_vis = visible(player);
  const int pl_row = player.row, pl_col = player.col;
  // Sprite characters -> smem (rec words 88..95 are padding); static indices only,
  // so the parameter block is never copied to local memory.
  uint8_t* s_chars = reinterpret_cast<uint8_t*>(rec + 88);
  {
    int ch = 0;
#pragma unroll
    for (int i = 0; i < kMaxS; ++i) if (i == lane) ch = p.sprite_char[i];
    if (lane < kMaxS) s_chars[lane] = (uint8_t)ch;
    __syncwarp();
  }
  const int P_CHAR = s_chars[NB];
  const bool is_box = lane < NB;
  const int32_t* mine = rec + (is_box ? lane : 0) * PCL_SPRITE_WORDS;
  int b_row = mine[PCL_S_ROW], b_col = mine[PCL_S_COL];

  // Character of the stale board (= previous final render) at (r, c): P on top,
  // then 'X' where the judge marked a box, else the last visible box there, else
  // the backdrop.  A box off the board sits at (0, 0) and the judge marks it there
  // too, but only a visible box paints its own character.  The judge's mark is a
  // property of the cell, so every box at (r, c) carries the same AUX0.
  // Box positions are still the old ones in `rec` while this is used.
  auto stale_cell = [&](int r, int c) -> int {
    if (pl_vis && r == pl_row && c == pl_col) return P_CHAR;
    int code = s_bd[r * pitch + c];
    for (int i = 0; i < NB; ++i) {
      const int32_t* b = rec + i * PCL_SPRITE_WORDS;
      if (b[PCL_S_ROW] == r && b[PCL_S_COL] == c) {
        if (b[PCL_S_AUX0]) code = 'X';
        else if (b[PCL_S_FLAGS] & 1) code = s_chars[i];
      }
    }
    return code;
  };

  // ---- group 0: boxes (BoxSprite.update, warehouse_manager.py:208-226)
  if (action >= 0 && action <= 3) {
    // layers['P'][rows +- 1, cols +- 1] with NumPy index rules: -1 wraps, >= size raises.
    const int dr = action == 0 ? 1 : action == 1 ? -1 : 0;
    const int dc = action == 2 ? 1 : action == 3 ? -1 : 0;
    int rr = b_row + dr, cc = b_col + dc;
    if (rr < 0) rr += H;
    if (cc < 0) cc += W;
    const bool oob = is_box && (rr >= H || cc >= W);
    const bool pushed = is_box && !oob && pl_vis && rr == pl_row && cc == pl_col;
    if (__any_sync(PCL_FULL, oob)) plot.error |= PCL_ENV_ERR_INDEX;
    const unsigned who = __ballot_sync(PCL_FULL, pushed);
    // One box on the board can be next to P, but every box off the board sits at
    // (0, 0), so several can be pushed at once.  Each moves against the stale board:
    // its lane keeps the new record in registers until all of them have moved.
    Sprite moved = {};
    for (unsigned left = who; left; left &= left - 1) {
      const int j = __ffs(left) - 1;
      Sprite box = load_sprite(rec + j * PCL_SPRITE_WORDS);
      uint32_t imp[4];
#pragma unroll
      for (int w = 0; w < 4; ++w) imp[w] = p.impassable[0][w];
#pragma unroll
      for (int i = 1; i < kMaxS - 1; ++i)
        if (i == j) {
#pragma unroll
          for (int w = 0; w < 4; ++w) imp[w] = p.impassable[i][w];
        }
      walker_move(box, j, motion_of_action(action), plot, H, W, false, false, lane,
                  [&](int r2, int c2) { return in_set(imp, stale_cell(r2, c2)); });
      if (lane == j) moved = box;
    }
    if (who) {
      __syncwarp();
      if (pushed) {
        store_sprite(rec + lane * PCL_SPRITE_WORDS, moved, PCL_S_AUX0);
        b_row = moved.row; b_col = moved.col;
      }
      __syncwarp();
    }
  }

  // ---- group 1: JudgeDrape.update (:245-266), one lane per box.  The curtain counts a
  // cell once: the last box in it counts.  Boxes share a cell while off the board (at
  // (0, 0)), or after two of them came back onto it from one virtual cell; `covered`:
  // a later box (higher in z-order) is visible in this box's cell.
  bool last = is_box, covered = false, goal = false;
  if (is_box) {
    for (int i = lane + 1; i < NB; ++i) {
      const int32_t* b = rec + i * PCL_SPRITE_WORDS;
      if (b[PCL_S_ROW] == b_row && b[PCL_S_COL] == b_col) {
        last = false;
        covered |= b[PCL_S_FLAGS] & 1;
      }
    }
    goal = s_bd[b_row * pitch + b_col] == '_';
  }
  const int num_boxes = __popc(__ballot_sync(PCL_FULL, last));
  const int on_goals = __popc(__ballot_sync(PCL_FULL, last && goal));
  if (is_box) rec[lane * PCL_SPRITE_WORDS + PCL_S_AUX0] = goal ? 1 : 0;
  add_reward(dir, on_goals - r_judge[PCL_D_AUX0]);
  if (action == 5 || on_goals == num_boxes) terminate(dir);
  __syncwarp();

  // ---- group 2: PlayerSprite.update (:284-295); board = boxes moved, X redrawn
  if (action >= 0 && action <= 3) {
    uint32_t imp[4];
#pragma unroll
    for (int w = 0; w < 4; ++w) imp[w] = p.impassable[kMaxS - 1][w];
#pragma unroll
    for (int i = 1; i < kMaxS - 1; ++i)
      if (i == NB) {
#pragma unroll
        for (int w = 0; w < 4; ++w) imp[w] = p.impassable[i][w];
      }
    walker_move(player, NB, motion_of_action(action), plot, H, W, false, false, lane,
                [&](int r2, int c2) { return in_set(imp, stale_cell(r2, c2)); });
  }

  // ---- _apply_and_clear_plot + records back
  __syncwarp();
  if (lane == 0) {
    const double ep_so_far = load_episode(p, env);   // overlaps the stores below
    store_sprite(rec + NB * PCL_SPRITE_WORDS, player, PCL_S_AUX0);
    r_judge[PCL_D_AUX0] = on_goals;
    apply_time_limit(p, plot, dir);
    store_episode(p, env, plot.frame, ep_so_far, (double)dir.reward);
    store_plot<ORDER_KEEP>(r_plot, plot, dir);
    store_outputs(p.out, env, dir);
  }
  __syncwarp();
  for (int i = lane; i < S * PCL_SPRITE_WORDS; i += 32) g_sprites[i] = rec[i];
  if (lane < PCL_DRAPE_WORDS) g_drapes[lane] = r_judge[lane];
  if (lane >= 16) g_plot[lane - 16] = r_plot[lane - 16];

  // ---- final render: patch the sprite cells into the staged tile, stream it out.
  // The judge marks every box's position, (0, 0) for a box off the board, so a
  // marked box paints 'X' whether it is visible or not.  An unmarked box paints
  // its own character if it is visible and not covered.  P goes last, on top.
  if (is_box && (goal || ((mine[PCL_S_FLAGS] & 1) && !covered)))
    s_bd[b_row * pitch + b_col] = goal ? 'X' : s_chars[lane];
  __syncwarp();
  if (lane == 0 && visible(player)) s_bd[player.row * pitch + player.col] = (uint8_t)P_CHAR;
  __syncwarp();
  uint8_t* board = p.out.d_board + (int64_t)env * tile;
  tile_store_fence();
  __syncwarp();
  if (lane == 0) {
    tile_store_bulk(board, s_bd, (uint32_t)tile);
    tile_store_wait();                       // the tile must outlive the copy's reads
  }
}

// Dynamic shared memory of one block (kWarpsPerBlock envs): each warp stages its
// records and its whole backdrop tile.
size_t block_smem(int H, int pitch) {
  return (kRecWords * 4 + (size_t)H * pitch) * kWarpsPerBlock;
}

int check_spec(const pcl_spec& s) {
  const int nb = s.n_sprites - 1;
  if (nb < 1 || nb > 10) return PCL_ERR_UNSUPPORTED;
  if (block_smem(s.rows, s.pitch) > kMaxBlockSmem) return PCL_ERR_UNSUPPORTED;
  if (s.sprite_char[nb] != 'P') return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.drape_char, s.n_drapes, "X")) return PCL_ERR_UNSUPPORTED;
  const char* order = "1234567890";
  int k = 0;
  for (int i = 0; i < nb; ++i) {
    while (order[k] && order[k] != (char)s.sprite_char[i]) ++k;
    if (!order[k]) return PCL_ERR_UNSUPPORTED;
    ++k;
    if (s.z_order[i] != s.sprite_char[i]) return PCL_ERR_UNSUPPORTED;
    if (s.sprite_confined[i] || s.sprite_egocentric[i]) return PCL_ERR_UNSUPPORTED;
  }
  if (s.z_order[nb] != 'X' || s.z_order[nb + 1] != 'P') return PCL_ERR_UNSUPPORTED;
  if (s.n_groups != 3 || s.group_len[0] != nb || s.group_len[1] != 1 || s.group_len[2] != 1)
    return PCL_ERR_UNSUPPORTED;
  for (int i = 0; i < nb; ++i)
    if (s.group_chars[i] != s.sprite_char[i]) return PCL_ERR_UNSUPPORTED;
  if (s.group_chars[nb] != 'X' || s.group_chars[nb + 1] != 'P') return PCL_ERR_UNSUPPORTED;
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  return launch_step(warehouse_step, p, kWarpsPerBlock, block_smem(p.H, p.pitch), s);
}

}  // namespace

// 'X' is held implicitly by the boxes: no curtain to resolve.
const Program kWarehouse = {check_spec, nullptr, nullptr, launch, nullptr,
                            /*float_reward=*/false, /*crop_epilogue=*/false,
                            /*scroll_groups=*/false};

}  // namespace pcl
