// better_scrolly.cu — fused step kernel for examples/better_scrolly_maze.py
// (SURVEY.md §8f-1: the cropper-based maze).
//
// One update group ['a','b','c','P','@'] and z-order 'abc@P'
// (better_scrolly_maze.py:209-221): the walls live in the backdrop, the whole
// world is the board, and the "scrolling" is done after the step by croppers
// (pcl_crop).  With a single group every entity reads the PREVIOUS step's final
// board (engine.py:729-735), so the kernel keeps the previous sprite cells as a
// snapshot and evaluates stale cells on demand from the staged backdrop tile,
// the staged coin bits and that snapshot.
//
// Sprite order P,a,b,c (0..3); drape 0 = '@' whose curtain (bit-packed,
// board-sized) is primary, mutable state.  Registers: patroller aux0 =
// _moving_east (:286); plot aux0 = coins left.
//
// Memory schedule as in scrolly_maze.cu: records -> smem (coalesced), backdrop
// tile + coin rows -> smem with cp.async, logic on registers/ballots, board
// composed from smem and streamed out with uint4 stores.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"

namespace pcl {

namespace {

constexpr int kS = 4;
constexpr int kWarpsPerBlock = 4;
constexpr int kRecWords = 64;       // 4 sprites * 8, drape 8, pad 8, plot 16

__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::
               "r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem));
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32, 7)
better_scrolly_step(const StepParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int env = blockIdx.x * kWarpsPerBlock + warp;
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;   // index of static level data
  const int H = p.H, W = p.W, pitch = p.pitch, BW = p.BW;
  const size_t tile = (size_t)H * pitch;
  const size_t bits_bytes = (((size_t)H * BW * 4) + 15) & ~(size_t)15;
  uint8_t* my = smem_raw + warp * (kRecWords * 4 + tile + bits_bytes);
  int32_t* rec = reinterpret_cast<int32_t*>(my);
  uint8_t* s_bd = my + kRecWords * 4;
  uint32_t* s_coin = reinterpret_cast<uint32_t*>(s_bd + tile);

  int32_t* g_sprites = p.st.d_sprites + (int64_t)env * kS * PCL_SPRITE_WORDS;
  int32_t* g_drapes = p.st.d_drapes + (int64_t)env * PCL_DRAPE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  uint32_t* g_coin = p.st.d_bits[0] + (int64_t)env * p.st.bits_bstride[0];
  const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;

  {
    const int n16 = (int)(tile >> 4);
    for (int i = lane; i < n16; i += 32) cp_async16(s_bd + i * 16, backdrop + i * 16);
  }
  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) { cp_async_wait_all(); return; }
  const bool restart = run == ENV_RESTART;
  const int nbits = H * BW;
  if (restart) {
    const PlotCarry carry = plot_carry(g_plot, true);
    rec[lane] = __ldg(p.st.d_sprites_init + lvl * p.st.sprites_init_bstride + lane);
    if (lane < 8) rec[32 + lane] = __ldg(p.st.d_drapes_init +
                                         lvl * p.st.drapes_init_bstride + lane);
    if (lane >= 16) rec[32 + lane] = __ldg(p.st.d_plot_init +
                                           lvl * p.st.plot_init_bstride + lane - 16);
    // Fresh coins (one Engine per episode): template -> live curtain and smem.
    const uint32_t* src = p.st.d_bits_init[0] + lvl * p.st.bits_init_bstride[0];
    for (int i = lane; i < nbits; i += 32) { const uint32_t w = __ldg(src + i); g_coin[i] = w; s_coin[i] = w; }
    __syncwarp();
    if (lane == 0) store_carry(rec + 48, carry);
  } else {
    rec[lane] = g_sprites[lane];
    if (lane < 8) rec[32 + lane] = g_drapes[lane];
    if (lane >= 16) rec[32 + lane] = g_plot[lane - 16];
    for (int i = lane; i < nbits; i += 32) cp_async4(s_coin + i, g_coin + i);
  }
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  cp_async_wait_all();
  __syncwarp();

  Sprite sp[kS];
#pragma unroll
  for (int i = 0; i < kS; ++i) sp[i] = load_sprite(rec + i * PCL_SPRITE_WORDS);
  Plot plot = step_plot(rec + 48, rec[48 + PCL_P_ERROR]);
  plot.aux0 = rec[48 + PCL_P_AUX0];
  Directives dir = fresh_directives();

  // Snapshot of the previous render's sprites (z-order a b c @ P).
  int o_row[kS], o_col[kS];
  bool o_vis[kS];
#pragma unroll
  for (int i = 0; i < kS; ++i) { o_row[i] = sp[i].row; o_col[i] = sp[i].col; o_vis[i] = visible(sp[i]); }
  auto stale_cell = [&](int r, int c) -> int {
    if (o_vis[0] && r == o_row[0] && c == o_col[0]) return p.sprite_char[0];
    if (bit_at(s_coin + r * BW, c)) return '@';
    int code = s_bd[r * pitch + c];
#pragma unroll
    for (int i = 1; i < kS; ++i)
      if (o_vis[i] && r == o_row[i] && c == o_col[i]) code = p.sprite_char[i];
    return code;
  };

  // ---- patrollers a, b, c (PatrollerSprite.update :288-305)
#pragma unroll
  for (int i = 1; i < kS; ++i) {
    auto blocked = [&](int r, int c) { return in_set(p.impassable[i], stale_cell(r, c)); };
    if (plot.frame % 2) {
      walker_move(sp[i], i, PCL_M_STAY, plot, H, W, false, false, lane, blocked);
    } else {
      // layers['#'][row, col -+ 1] with NumPy index rules.
      const int row = sp[i].row;
      int cw = sp[i].col - 1, ce = sp[i].col + 1;
      if (cw < 0) cw += W;
      if (ce >= W) { plot.error |= PCL_ENV_ERR_INDEX; ce = W - 1; }
      if (stale_cell(row, cw) == '#') sp[i].aux0 = 1;
      if (stale_cell(row, ce) == '#') sp[i].aux0 = 0;
      walker_move(sp[i], i, sp[i].aux0 ? PCL_M_E : PCL_M_W, plot, H, W, false, false, lane,
                  blocked);
      if (sp[i].row == sp[0].row && sp[i].col == sp[0].col) terminate(dir);
    }
  }
  // ---- P (PlayerSprite.update :263-276)
  {
    const int motion = action == 0 ? PCL_M_N : action == 1 ? PCL_M_S : action == 2 ? PCL_M_W
                     : action == 3 ? PCL_M_E : action == 4 ? PCL_M_STAY : PCL_M_NONE;
    if (motion != PCL_M_NONE)
      walker_move(sp[0], 0, motion, plot, H, W, false, false, lane,
                  [&](int r, int c) { return in_set(p.impassable[0], stale_cell(r, c)); });
    if (action == 5) terminate(dir);
  }
  // ---- '@' (CashDrape.update :314-324)
  {
    const int pr = sp[0].row, pc = sp[0].col;
    uint32_t* word = s_coin + pr * BW + (pc >> 5);
    if ((*word >> (pc & 31)) & 1u) {
      add_reward(dir, 100);
      __syncwarp();
      if (lane == 0) {
        *word &= ~(1u << (pc & 31));
        g_coin[pr * BW + (pc >> 5)] = *word;
      }
      __syncwarp();
      plot.aux0 -= 1;
      if (plot.aux0 == 0) terminate(dir);
    }
  }

  // ---- _apply_and_clear_plot + records back
  __syncwarp();
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < kS; ++i) store_sprite(rec + i * PCL_SPRITE_WORDS, sp[i], PCL_S_AUX1);
    store_plot<ORDER_KEEP>(rec + 48, plot, dir);
    rec[48 + PCL_P_AUX0] = plot.aux0;
    store_outputs(p.out, env, dir);
  }
  __syncwarp();
  g_sprites[lane] = rec[lane];
  if (lane < 8) g_drapes[lane] = rec[32 + lane];
  if (lane >= 16) g_plot[lane - 16] = rec[32 + lane];

  // ---- final render, z-order a b c @ P (engine.py:737-759).  a, b, c lie under
  // the coins: patch them into the staged tile up front; coins come from the
  // bit rows (segment sg of a row = its sg-th 16-bit half-word); P is the top
  // layer, patched into the one segment that holds it.
  __syncwarp();
  if (lane == 0) {
#pragma unroll
    for (int i = 1; i < kS; ++i)
      if (visible(sp[i])) s_bd[sp[i].row * pitch + sp[i].col] = p.sprite_char[i];
  }
  __syncwarp();
  const int spr = pitch >> 4;
  const int total = H * spr;
  const int p_seg = visible(sp[0]) ? sp[0].row * spr + (sp[0].col >> 4) : -1;
  const unsigned p_bit = 1u << (sp[0].col & 15);
  const uint4* src = reinterpret_cast<const uint4*>(s_bd);
  uint4* dst = reinterpret_cast<uint4*>(p.out.d_board + (int64_t)env * tile);
  int r = lane / spr, sg = lane - r * spr;     // this lane's (row, segment) and its stride
  const int dr = 32 / spr, dsg = 32 - dr * spr;
  for (int seg = lane; seg < total; seg += 32) {
    uint4 px = src[seg];
    const unsigned coin_bits = reinterpret_cast<const uint16_t*>(s_coin + r * BW)[sg];
    if (coin_bits) paint_bits(px, coin_bits, '@');
    if (seg == p_seg) paint_bits(px, p_bit, p.sprite_char[0]);
    dst[seg] = px;
    r += dr; sg += dsg;
    if (sg >= spr) { sg -= spr; ++r; }
  }
}

int check_spec(const pcl_spec& s) {
  if (!chars_are(s.sprite_char, s.n_sprites, "Pabc")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.drape_char, s.n_drapes, "@")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.z_order, 5, "abc@P")) return PCL_ERR_UNSUPPORTED;
  const int lens[1] = {5};
  if (!groups_are(s, "abcP@", lens, 1)) return PCL_ERR_UNSUPPORTED;
  for (int i = 0; i < 4; ++i)
    if (s.sprite_confined[i] || s.sprite_egocentric[i]) return PCL_ERR_UNSUPPORTED;
  if (!bit_rows_fit(s)) return PCL_ERR_INVALID;
  return PCL_OK;
}

int check_state(const pcl_spec&, const pcl_state& st) {
  if (!st.d_bits[0] || !st.d_bits_init[0] || st.bits_bstride[0] == 0) return PCL_ERR_INVALID;
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  const size_t bits_bytes = (((size_t)p.H * p.BW * 4) + 15) & ~(size_t)15;
  const size_t smem = (kRecWords * 4 + (size_t)p.H * p.pitch + bits_bytes) * kWarpsPerBlock;
  return launch_step(better_scrolly_step, p, kWarpsPerBlock, smem, s);
}

}  // namespace

const Program kBetterScrolly = {check_spec, check_state, curtain_bits, launch, nullptr,
                                /*float_reward=*/false, /*crop_epilogue=*/false,
                                /*scroll_groups=*/false};

}  // namespace pcl
