// aperture.cu — fused step kernel for examples/aperture.py (SURVEY.md §8f-4).
//
// Entities: sprite 'A' (MazeWalker, impassable '#.@'), drape 'X' (ApertureDrape).
// Update groups [['A'], ['X']], z-order 'XA' (aperture.py:188-196).  The drape's
// whole state is its list of at most two aperture cells (`_apertures`, :161),
// kept in the drape record as AUX0 / AUX1 = row << 16 | col, or -1 for None; the
// curtain is those cells and is never stored.
//
//   group 0, PlayerSprite.update (:130-149): actions 0-3 walk N S W E (9 quits)
//     on the STALE board (previous final render: backdrop, apertures, A where it
//     was); then `layers['C'][position]` pays 1 and ends the episode, and
//     `layers['X'][position]` teleports to the first OTHER aperture.
//   group 1, ApertureDrape.update (:163-190): actions 5-8 fire the blaster up,
//     left, down, right from A's new position across the re-rendered board; the
//     ray stops at the board edge, a '#' or an aperture, and the first '@' it
//     meets becomes the newest aperture (the oldest of two is dropped).
//
// One warp per env; the ray is lane-parallel (lane k tests step k+1, a ballot
// finds the first cell that stops it).
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 4;
constexpr int kRecWords = 32;       // sprite 8, drape 8, plot 16

__device__ __forceinline__ int pack_cell(int r, int c) { return (r << 16) | c; }

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
aperture_step(const StepParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int env = blockIdx.x * kWarpsPerBlock + warp;
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;
  const int H = p.H, W = p.W, pitch = p.pitch;
  const int tile = H * pitch;
  uint8_t* my = smem_raw + warp * (kRecWords * 4 + tile);
  int32_t* rec = reinterpret_cast<int32_t*>(my);
  uint8_t* s_bd = my + kRecWords * 4;

  int32_t* g_sprite = p.st.d_sprites + (int64_t)env * PCL_SPRITE_WORDS;
  int32_t* g_drape = p.st.d_drapes + (int64_t)env * PCL_DRAPE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  const uint8_t* backdrop = p.st.d_backdrop + lvl * p.st.backdrop_bstride;
  for (int i = lane; i < (tile >> 4); i += 32) cp_async16(s_bd + i * 16, backdrop + i * 16);

  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) { cp_async_wait_all(); return; }
  const bool restart = run == ENV_RESTART;
  if (restart) {                                   // a fresh Engine (engine.py:520-581)
    const PlotCarry carry = plot_carry(g_plot, true);
    if (lane < 8) rec[lane] = __ldg(p.st.d_sprites_init + lvl * p.st.sprites_init_bstride + lane);
    else if (lane < 16) rec[lane] = __ldg(p.st.d_drapes_init + lvl * p.st.drapes_init_bstride + lane - 8);
    else rec[lane] = __ldg(p.st.d_plot_init + lvl * p.st.plot_init_bstride + lane - 16);
    __syncwarp();
    if (lane == 0) store_carry(rec + 16, carry);
  } else {
    rec[lane] = lane < 8 ? g_sprite[lane] : lane < 16 ? g_drape[lane - 8] : g_plot[lane - 16];
  }
  const int action = restart ? PCL_ACTION_NONE : env_action(p, env);
  cp_async_wait_all();
  __syncwarp();

  Sprite sp = load_sprite(rec);
  int ap0 = rec[8 + PCL_D_AUX0], ap1 = rec[8 + PCL_D_AUX1];    // _apertures[0], [1]
  Plot plot = step_plot(rec + 16, rec[16 + PCL_P_ERROR]);
  Directives dir = fresh_directives();

  // ---- group 0: PlayerSprite.update on the stale board -------------------
  const bool old_vis = visible(sp);
  const int old_cell = pack_cell(sp.row, sp.col);
  auto stale_cell = [&](int r, int c) -> int {
    const int cell = pack_cell(r, c);
    if (old_vis && cell == old_cell) return p.sprite_char[0];
    if (cell == ap0 || cell == ap1) return p.drape_char[0];
    return s_bd[r * pitch + c];
  };
  const int motion = action == 0 ? PCL_M_N : action == 1 ? PCL_M_S : action == 2 ? PCL_M_W
                   : action == 3 ? PCL_M_E : PCL_M_NONE;
  if (motion != PCL_M_NONE)
    walker_move(sp, 0, motion, plot, H, W, p.confined[0] != 0, false, lane,
                [&](int r, int c) { return in_set(p.impassable[0], stale_cell(r, c)); });
  else if (action == 9)
    terminate(dir);
  {
    const int here = stale_cell(sp.row, sp.col);
    if (here == 'C') { add_reward(dir, 1); terminate(dir); }
    if (here == p.drape_char[0]) {                  // destinations[0], :147-149
      const int me = pack_cell(sp.row, sp.col);
      const int dest = (ap0 >= 0 && ap0 != me) ? ap0 : (ap1 >= 0 && ap1 != me) ? ap1 : -1;
      if (dest >= 0) walker_teleport(sp, H, W, dest >> 16, dest & 0xffff);
    }
  }

  // ---- group 1: ApertureDrape.update on the re-rendered board ------------
  if (action >= 5 && action <= 8) {
    const int dy = action == 5 ? -1 : action == 7 ? 1 : 0;
    const int dx = action == 6 ? -1 : action == 8 ? 1 : 0;
    const int a_cell = visible(sp) ? pack_cell(sp.row, sp.col) : -1;
    const int reach = max(H, W);                    // xrange(1, max(height, width))
    for (int base = 1; base < reach; base += 32) {
      const int step = base + lane;
      const int cy = sp.row + dy * step, cx = sp.col + dx * step;
      bool stop = false, hit = false;
      if (step < reach) {
        if (!on_board(cy, cx, H, W)) {
          stop = true;
        } else {
          const int cell = pack_cell(cy, cx);
          const int ch = cell == a_cell ? (int)p.sprite_char[0]
                       : (cell == ap0 || cell == ap1) ? (int)p.drape_char[0]
                       : (int)s_bd[cy * pitch + cx];
          stop = ch == '#' || ch == p.drape_char[0];
          hit = ch == '@';
        }
      }
      const unsigned stops = __ballot_sync(PCL_FULL, stop);
      const unsigned hits = __ballot_sync(PCL_FULL, hit);
      if (stops | hits) {
        const int first = __ffs(stops | hits) - 1;
        if ((hits >> first) & 1u) {                 // self._apertures[1:] + [(y, x)]
          const int s2 = base + first;
          ap0 = ap1;
          ap1 = pack_cell(sp.row + dy * s2, sp.col + dx * s2);
        }
        break;
      }
    }
  }

  // ---- _apply_and_clear_plot (engine.py:761-847) + records back
  __syncwarp();                 // every lane has read the staged records (racecheck: WAR)
  if (lane == 0) {
    store_sprite(rec, sp, PCL_S_AUX0);
    rec[8 + PCL_D_AUX0] = ap0; rec[8 + PCL_D_AUX1] = ap1;
    store_plot<ORDER_KEEP>(rec + 16, plot, dir);
    store_outputs(p.out, env, dir);
    // final render, z-order X then A: patch the staged tile (engine.py:737-759)
    if (ap0 >= 0) s_bd[(ap0 >> 16) * pitch + (ap0 & 0xffff)] = p.drape_char[0];
    if (ap1 >= 0) s_bd[(ap1 >> 16) * pitch + (ap1 & 0xffff)] = p.drape_char[0];
    if (visible(sp)) s_bd[sp.row * pitch + sp.col] = p.sprite_char[0];
  }
  __syncwarp();
  if (lane < 8) g_sprite[lane] = rec[lane];
  else if (lane < 16) g_drape[lane - 8] = rec[lane];
  else g_plot[lane - 16] = rec[lane];

  const uint4* src = reinterpret_cast<const uint4*>(s_bd);
  uint4* dst = reinterpret_cast<uint4*>(p.out.d_board + (int64_t)env * tile);
  for (int seg = lane; seg < (tile >> 4); seg += 32) dst[seg] = src[seg];
}

int check_spec(const pcl_spec& s) {
  if (s.n_sprites != 1 || s.n_drapes != 1) return PCL_ERR_UNSUPPORTED;
  if (s.z_order[0] != s.drape_char[0] || s.z_order[1] != s.sprite_char[0]) return PCL_ERR_UNSUPPORTED;
  if (s.n_groups != 2 || s.group_len[0] != 1 || s.group_len[1] != 1 ||
      s.group_chars[0] != s.sprite_char[0] || s.group_chars[1] != s.drape_char[0])
    return PCL_ERR_UNSUPPORTED;
  if (s.sprite_egocentric[0]) return PCL_ERR_UNSUPPORTED;
  if (s.rows >= 32768 || s.cols >= 32768 || s.rows * s.pitch > 8192) return PCL_ERR_UNSUPPORTED;
  return PCL_OK;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  const size_t smem = (kRecWords * 4 + (size_t)p.H * p.pitch) * kWarpsPerBlock;
  return launch_step(aperture_step, p, kWarpsPerBlock, smem, s);
}

}  // namespace

// The drape's curtain is held implicitly (its record's AUX0 / AUX1): nothing to resolve.
const Program kAperture = {check_spec, nullptr, nullptr, launch, nullptr,
                           /*float_reward=*/false, /*crop_epilogue=*/false,
                           /*scroll_groups=*/false};

}  // namespace pcl
