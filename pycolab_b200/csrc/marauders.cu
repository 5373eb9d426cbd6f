// marauders.cu — fused step kernel for examples/extraterrestrial_marauders.py.
//
// Single update group ['P','B','X','a','b','c','d','y','z'] which is also the
// z-order (extraterrestrial_marauders.py:91-101), so every entity reads the
// PREVIOUS step's board (engine.py:729-735).  Sprite order P,a,b,c,d,y,z
// (0..6); drapes 'B' (0) and 'X' (1) whose curtains are the primary state:
// bit-packed rows, row r lives in lane r's registers (rows <= 32, cols <= 64).
//
// Registers: X drape aux0 = _dx (:140); plot aux0 / aux1 = 'last_player_shot'
// / 'last_marauder_shot' frames (:214-215, :248-249).  The per-env MT19937
// stream reproduces numpy.random.choice (:253): legacy RandomState draws an
// index by masked rejection over tempered 32-bit outputs.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"
#include "pcl_mt.cuh"

namespace pcl {

namespace {

constexpr int kS = 7;
constexpr int kWarpsPerBlock = 4;
typedef unsigned long long u64;

__device__ __forceinline__ bool same_cell(const Sprite& a, const Sprite& b) {
  return a.row == b.row && a.col == b.col;
}

constexpr int kRecWords = 96;        // 7 sprites * 8 = 56, 2 drapes * 8 = 16, plot 16, pad

__global__ void __launch_bounds__(kWarpsPerBlock * 32, 7)
marauders_step(const StepParams p) {
  // Records are staged in shared memory with coalesced loads; only the fields
  // this game uses are pulled into registers (keeps the kernel at one wave).
  __shared__ int32_t s_rec[kWarpsPerBlock][kRecWords];
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (env >= p.B) return;
  const int H = p.H, W = p.W;
  int32_t* rec = s_rec[threadIdx.x >> 5];
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;   // index of static level data

  int32_t* g_sprites = p.st.d_sprites + (int64_t)env * kS * PCL_SPRITE_WORDS;
  int32_t* g_drapes = p.st.d_drapes + (int64_t)env * 2 * PCL_DRAPE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  uint32_t* g_bunk = p.st.d_bits[0] + (int64_t)env * p.st.bits_bstride[0];
  uint32_t* g_mara = p.st.d_bits[1] + (int64_t)env * p.st.bits_bstride[1];
  uint32_t* mt = p.st.d_rng + (int64_t)env * PCL_MT_WORDS;

  // The tile does not depend on anything: start it first (cp.async, no registers).
  extern __shared__ __align__(16) uint8_t s_tiles[];
  const int tile = H * p.pitch;
  uint8_t* s_bd = s_tiles + (threadIdx.x >> 5) * tile;
  {
    const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;
    for (int i = lane; i < (tile >> 4); i += 32) cp_async16(s_bd + i * 16, backdrop + i * 16);
  }
  // Live state first, unconditionally, in ONE round trip; whether the env restarts
  // is decided from the staged plot record (no load waits on another load).
  const int BW = p.BW;
  auto load_row = [&](const uint32_t* base) -> u64 {
    if (lane >= H) return 0;
    const uint32_t* row = base + lane * BW;
    return (u64)row[0] | ((u64)row[1] << 32);
  };
  rec[lane] = g_sprites[lane];
  if (lane < 24) rec[32 + lane] = g_sprites[32 + lane];
  rec[56 + lane] = lane < 16 ? g_drapes[lane] : g_plot[lane - 16];
  u64 brow = load_row(g_bunk), xrow = load_row(g_mara);   // lane r holds row r of B / X
  int action = env_action(p, env);
  __syncwarp();
  const EnvRun run = env_run(p, env, rec[72 + PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) { cp_async_wait_all(); return; }
  if (run == ENV_RESTART) {                    // a fresh Engine: templates over the live state
    const PlotCarry carry = plot_carry(rec + 72, true);
    __syncwarp();
    const int32_t* ss = p.st.d_sprites_init + lvl * p.st.sprites_init_bstride;
    rec[lane] = ss[lane];
    if (lane < 24) rec[32 + lane] = ss[32 + lane];
    rec[56 + lane] = lane < 16 ? (p.st.d_drapes_init + lvl * p.st.drapes_init_bstride)[lane]
                               : (p.st.d_plot_init + lvl * p.st.plot_init_bstride)[lane - 16];
    brow = load_row(p.st.d_bits_init[0] + lvl * p.st.bits_init_bstride[0]);
    xrow = load_row(p.st.d_bits_init[1] + lvl * p.st.bits_init_bstride[1]);
    action = PCL_ACTION_NONE;
    __syncwarp();
    if (lane == 0) store_carry(rec + 72, carry);
    __syncwarp();
  }
  Sprite sp[kS];
#pragma unroll
  for (int i = 0; i < kS; ++i) sp[i] = load_sprite(rec + i * PCL_SPRITE_WORDS);
  Drape marauders;
  marauders.aux0 = rec[56 + PCL_DRAPE_WORDS + PCL_D_AUX0];
  Plot plot = step_plot(rec + 72, rec[72 + PCL_P_ERROR]);
  plot.aux0 = rec[72 + PCL_P_AUX0]; plot.aux1 = rec[72 + PCL_P_AUX1];
  Directives dir = fresh_directives();

  // ---- the stale board, as far as anybody looks at it --------------------
  // top[i]: bolt i is the visible character of its cell (layers[c] = board==c,
  // rendering.py:177); a later bolt in z-order hides an earlier one.
  bool top[kS];
#pragma unroll
  for (int i = 1; i < kS; ++i) {
    top[i] = visible(sp[i]);
#pragma unroll
    for (int j = i + 1; j < kS; ++j)
      if (visible(sp[j]) && same_cell(sp[i], sp[j])) top[i] = false;
  }
  // layers['X'] of the stale board: marauders not hidden under a bolt.
  u64 seen = xrow;
#pragma unroll
  for (int i = 1; i < kS; ++i)
    if (visible(sp[i]) && sp[i].row == lane) seen &= ~(1ull << sp[i].col);
  // Old bolt cells (bolts only move in their own update, after B and X).
  auto never_blocked = [](int, int) { return false; };

  // ---- P (PlayerSprite.update :178-186)
  if (action == 0) walker_move(sp[0], 0, PCL_M_W, plot, H, W, true, false, lane, never_blocked);
  else if (action == 1) walker_move(sp[0], 0, PCL_M_E, plot, H, W, true, false, lane, never_blocked);
  else if (action == 4) terminate(dir);

  // ---- B (BunkerDrape.update :113-120)
  int bunker_hitters = 0, nb = 0;
#pragma unroll
  for (int i = 1; i < kS; ++i) {
    const bool mine = top[i] && sp[i].row == lane && ((brow >> sp[i].col) & 1ull);
    const bool hit = __any_sync(PCL_FULL, mine);
    if (mine) brow &= ~(1ull << sp[i].col);
    if (hit) { bunker_hitters |= 1 << i; nb += 1; }
  }
  add_reward(dir, -nb);

  // ---- X (MarauderDrape.update :142-163)
  int marauder_hitters = 0, nx = 0;
#pragma unroll
  for (int i = 1; i <= 4; ++i) {
    const bool mine = top[i] && sp[i].row == lane && ((xrow >> sp[i].col) & 1ull);
    const bool hit = __any_sync(PCL_FULL, mine);
    if (mine) xrow &= ~(1ull << sp[i].col);
    if (hit) { marauder_hitters |= 1 << i; nx += 1; }
  }
  add_reward(dir, nx * 10);
  {
    const bool none_left = !__any_sync(PCL_FULL, xrow != 0);
    const u64 row10 = __shfl_sync(PCL_FULL, xrow, 10);
    if (none_left || (H > 10 && row10 != 0)) {
      terminate(dir);
    } else {
      int count = __popcll(xrow);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) count += __shfl_xor_sync(PCL_FULL, count, o);
      // frame % max(1, count // 8.0000001): the float floor-division equals
      // (count - 1) / 8 for every 1 <= count <= 2^20.
      const int period = max(1, (count - 1) / 8);
      if (plot.frame % period == 0) {
        const u64 edge = (1ull) | (1ull << (W - 1));
        if (__any_sync(PCL_FULL, (xrow & edge) != 0)) {
          marauders.aux0 = -marauders.aux0;
          const u64 up = __shfl_sync(PCL_FULL, xrow, (lane + H - 1) % H);   // np.roll(+1, axis 0)
          xrow = lane < H ? up : 0;
        }
        const u64 full = (W == 64) ? ~0ull : ((1ull << W) - 1ull);
        if (marauders.aux0 > 0) xrow = ((xrow << 1) | (xrow >> (W - 1))) & full;
        else xrow = ((xrow >> 1) | ((xrow & 1ull) << (W - 1))) & full;
      }
    }
  }

  // ---- upward bolts a..d (UpwardLaserBoltSprite :198-220)
#pragma unroll
  for (int i = 1; i <= 4; ++i) {
    if (visible(sp[i])) {
      if (((bunker_hitters | marauder_hitters) >> i) & 1) walker_teleport(sp[i], H, W, -1, -1);
      else walker_move(sp[i], i, PCL_M_N, plot, H, W, false, false, lane, never_blocked);
    } else if (action == 2) {
      if (plot.aux0 != plot.frame) {
        plot.aux0 = plot.frame;
        walker_teleport(sp[i], H, W, sp[0].row - 1, sp[0].col);
      }
    }
  }
  // ---- downward bolts y, z (DownwardLaserBoltSprite :232-256)
#pragma unroll
  for (int i = 5; i < kS; ++i) {
    if (visible(sp[i])) {
      if ((bunker_hitters >> i) & 1) {
        walker_teleport(sp[i], H, W, -1, -1);
      } else {
        if (same_cell(sp[i], sp[0])) terminate(dir);
        walker_move(sp[i], i, PCL_M_S, plot, H, W, false, false, lane, never_blocked);
      }
    } else if (plot.aux1 != plot.frame) {
      plot.aux1 = plot.frame;
      // cols = nonzero(layers['X'].sum(axis=0)); col = choice(cols)
      u64 colmask = seen;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) colmask |= __shfl_xor_sync(PCL_FULL, colmask, o);
      const int n = __popcll(colmask);
      if (n == 0) {
        plot.error |= PCL_ENV_ERR_EMPTY_CHOICE;   // the reference raises ValueError here
      } else {
        int k = (int)mt_below(mt, (uint32_t)n, lane);
        u64 m = colmask;
        for (int t = 0; t < k; ++t) m &= m - 1;   // drop the k lowest set bits
        const int col = __ffsll((long long)m) - 1;
        const unsigned rows_with = __ballot_sync(PCL_FULL, (seen >> col) & 1ull);
        const int row = (31 - __clz((int)rows_with)) + 1;
        walker_teleport(sp[i], H, W, row, col);
      }
    }
  }

  // ---- _apply_and_clear_plot + state write-back
  if (lane < H) {
    uint32_t* rb = g_bunk + lane * BW;
    uint32_t* rx = g_mara + lane * BW;
    rb[0] = (uint32_t)brow; rb[1] = (uint32_t)(brow >> 32);
    rx[0] = (uint32_t)xrow; rx[1] = (uint32_t)(xrow >> 32);
  }
  __syncwarp();
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < kS; ++i) store_sprite(rec + i * PCL_SPRITE_WORDS, sp[i], PCL_S_AUX0);
    rec[56 + PCL_DRAPE_WORDS + PCL_D_AUX0] = marauders.aux0;
    apply_time_limit(p, plot, dir);
    store_plot<ORDER_KEEP>(rec + 72, plot, dir);
    rec[72 + PCL_P_AUX0] = plot.aux0; rec[72 + PCL_P_AUX1] = plot.aux1;
    store_outputs(p.out, env, dir);
    store_episode(p, env, plot.frame, load_episode(p, env), (double)dir.reward);
  }
  __syncwarp();
  g_sprites[lane] = rec[lane];
  if (lane < 24) g_sprites[32 + lane] = rec[32 + lane];
  if (lane < 16) g_drapes[lane] = rec[56 + lane]; else g_plot[lane - 16] = rec[56 + lane];

  // ---- final render, z-order P B X a b c d y z (engine.py:737-759): P lies under
  // both drapes, the bolts over them.  P is patched into the staged tile, the
  // drape bits are composed over it in place, the six bolt cells are patched on
  // top, and the tile streams out.
  cp_async_wait_all();
  __syncwarp();
  if (lane == 0 && visible(sp[0])) s_bd[sp[0].row * p.pitch + sp[0].col] = p.sprite_char[0];
  __syncwarp();
  const int spr = p.pitch >> 4;
  const int total = H * spr;
  uint4* tile4 = reinterpret_cast<uint4*>(s_bd);
  {
    int r = lane / spr, sg = lane - r * spr;   // this lane's (row, segment) and its stride
    const int dr = 32 / spr, dsg = 32 - dr * spr;
    for (int base = 0; base < total; base += 32) {
      const int seg = base + lane;
      const bool active = seg < total;
      const u64 b = __shfl_sync(PCL_FULL, brow, active ? r : 0);
      const u64 x = __shfl_sync(PCL_FULL, xrow, active ? r : 0);
      if (active) {
        uint4 px = tile4[seg];
        paint_bits(px, (unsigned)shr_u64(b, sg << 4) & 0xffffu, 'B');   // 0 past column 64
        paint_bits(px, (unsigned)shr_u64(x, sg << 4) & 0xffffu, 'X');
        tile4[seg] = px;
      }
      r += dr; sg += dsg;
      if (sg >= spr) { sg -= spr; ++r; }
    }
  }
  __syncwarp();
  if (lane == 0) {
#pragma unroll
    for (int i = 1; i < kS; ++i)
      if (visible(sp[i])) s_bd[sp[i].row * p.pitch + sp[i].col] = p.sprite_char[i];
  }
  __syncwarp();
  uint4* dst = reinterpret_cast<uint4*>(p.out.d_board + (int64_t)env * tile);
  for (int seg = lane; seg < total; seg += 32) dst[seg] = tile4[seg];
}

// Shared memory of one block (kWarpsPerBlock envs): the static records plus one staged
// H x pitch tile per warp.
size_t block_smem(int H, int pitch) {
  return sizeof(int32_t) * kWarpsPerBlock * kRecWords + (size_t)H * pitch * kWarpsPerBlock;
}

int check_spec(const pcl_spec& s) {
  if (!chars_are(s.sprite_char, s.n_sprites, "Pabcdyz")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.drape_char, s.n_drapes, "BX")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.z_order, 9, "PBXabcdyz")) return PCL_ERR_UNSUPPORTED;
  const int lens[1] = {9};
  if (!groups_are(s, "PBXabcdyz", lens, 1)) return PCL_ERR_UNSUPPORTED;
  if (s.rows > 32 || s.rows < 11 || s.cols > 64 || s.bits_words < 2)
    return PCL_ERR_UNSUPPORTED;
  if (block_smem(s.rows, s.pitch) > kMaxBlockSmem) return PCL_ERR_UNSUPPORTED;
  for (int i = 0; i < 7; ++i) {
    if (!set_is(s.impassable[i], "")) return PCL_ERR_UNSUPPORTED;
    if (s.sprite_confined[i] != (i == 0) || s.sprite_egocentric[i]) return PCL_ERR_UNSUPPORTED;
  }
  return PCL_OK;
}

int check_state(const pcl_spec&, const pcl_state& st) {
  for (int d = 0; d < 2; ++d)
    if (!st.d_bits[d] || !st.d_bits_init[d] || st.bits_bstride[d] == 0) return PCL_ERR_INVALID;
  if (!st.d_rng) return PCL_ERR_INVALID;
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  const size_t smem = (size_t)p.H * p.pitch * kWarpsPerBlock;   // one staged tile per warp
  return launch_step(marauders_step, p, kWarpsPerBlock, smem, s, /*pdl=*/true,
                     block_smem(p.H, p.pitch) - smem);
}

}  // namespace

const Program kMarauders = {check_spec, check_state, curtain_bits, launch, nullptr,
                            /*float_reward=*/false, /*crop_epilogue=*/false,
                            /*scroll_groups=*/false, /*check_code=*/nullptr,
                            /*float_reward_arg0=*/false, /*derive=*/nullptr, /*block_chaining=*/false,
                            one_rng_slot};

}  // namespace pcl
